"""GPU tests of gf_fm_window (csrc/fm_window.cu): the FeatureManager whose landmark table stays on the device, against the host
mirror feature_manager.FeatureManager driven with the same calls.  After every call the whole table and the call's return
values are compared: integers, ids, flags, list order and observation rows must be equal, and so must every depth, because
both sides run the same device functions (csrc/fm_device.cuh)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _cam():
    from ground_fusion_b200.synth import IDC_CAM
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    return cam, [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]


ROW_BYTES = 112       # sizeof(gf_ba_visual_factor)


def _bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


def mirror_table(fm):
    return [dict(feature_id=it.feature_id, start_frame=it.start_frame, n_obs=len(it.obs), estimated_depth=float(it.estimated_depth),
                 estimate_flag=it.estimate_flag, solve_flag=it.solve_flag, obs=np.asarray(it.obs, np.float64).reshape(-1, 9)) for it in fm.feature]


def assert_same_table(got, want, what=""):
    assert [r["feature_id"] for r in got] == [r["feature_id"] for r in want], what
    for g, w in zip(got, want):
        for k in ("start_frame", "n_obs", "estimate_flag", "solve_flag"):
            assert g[k] == w[k], (what, k, w["feature_id"], g[k], w[k])
        assert np.array_equal(_bits(g["estimated_depth"]), _bits(w["estimated_depth"])), (what, w["feature_id"], g["estimated_depth"], w["estimated_depth"])
        assert np.array_equal(_bits(g["obs"]), _bits(w["obs"])), (what, w["feature_id"])


def python_factor_arrays(fm):
    """What replay.WindowEstimator.optimization builds from a host manager."""
    from ground_fusion_b200.ba_problem import Problem
    feats = list(fm.iter_ba_features())
    pb = Problem(11, len(feats))
    rows = []
    for k, (start, obs, est_depth, flag) in enumerate(feats):
        pb.para_feature[k] = 1.0 / est_depth
        pb.feature_const[k] = 1 if flag == 1 else 0
        p0, v0, t0 = obs[0]
        for a in range(1, len(obs)):
            pj, vj, tj = obs[a]
            rows.append((start, start + a, k, p0, pj, v0, vj, t0, tj))
    pb.set_visual(rows)
    return pb, len(feats)


class Both:
    """A FeatureManager and a FeatureWindow behind one set of methods: every call goes to both, and the return values and the
    two tables are compared before it returns.  replay() drives it like any manager."""

    def __init__(self, **kw):
        from ground_fusion_b200.feature_manager import FeatureManager
        from ground_fusion_b200.feature_window import FeatureWindow
        mf = kw.pop("max_features", 2048)
        self.m, self.w = FeatureManager(**kw), FeatureWindow(max_features=mf, **kw)
        self.calls = {}
        self.log = []                   # (call, table size) and every return value, to compare two runs
        self.max_par_rel = 0.0
        self.seen = set()               # the cases the calls reached

    def check(self, what):
        self.calls[what] = self.calls.get(what, 0) + 1
        got, want = self.w.read(), mirror_table(self.m)
        assert_same_table(got, want, what)
        self.log.append((what, len(got)))
        return got

    def addFeatureCheckParallax(self, fc, image, td):
        before = {it.feature_id: it for it in self.m.feature}
        a, b = self.m.addFeatureCheckParallax(fc, image, td), self.w.addFeatureCheckParallax(fc, image, td)
        assert a == b, (fc, a, b)
        assert (self.m.last_track_num, self.m.new_feature_num, self.m.long_track_num) == (self.w.last_track_num, self.w.new_feature_num, self.w.long_track_num)
        pa, pb = self.m.last_average_parallax, self.w.last_average_parallax
        assert abs(pa - pb) <= 1e-13 * abs(pa), (pa, pb)
        if pa:
            self.max_par_rel = max(self.max_par_rel, abs(pa - pb) / abs(pa)); self.seen.add("parallax")
        if not image:
            self.seen.add("empty frame")
        elif not any(k in before for k in image):
            self.seen.add("only new ids")
        if any(k in before and before[k].start_frame + len(before[k].obs) - 1 < fc - 1 for k in image):
            self.seen.add("skipped a frame")
        if self.m.feature and any(x.feature_id > y.feature_id for x, y in zip(self.m.feature, self.m.feature[1:])):
            self.seen.add("list not sorted by id")
        self.log.append((b, self.w.last_track_num, self.w.new_feature_num, self.w.long_track_num, float(pb).hex()))
        self.check("add")
        return b

    def triangulateAll(self, *a):
        self.m.triangulateAll(*a); self.w.triangulateAll(*a)
        t = self.check("triangulate")
        self.seen |= {"flag %d" % r["estimate_flag"] for r in t}

    def fillProblem(self, pb):
        want, n = python_factor_arrays(self.m)
        got_n = self.w.fillProblem(pb)
        assert got_n == n and pb.n_visual == want.n_visual and pb.n_features == n
        assert bytes(pb.visual)[:pb.n_visual * ROW_BYTES] == bytes(want.visual)[:want.n_visual * ROW_BYTES]
        assert np.array_equal(_bits(pb.para_feature[:n]), _bits(want.para_feature[:n])) and np.array_equal(pb.feature_const[:n], want.feature_const[:n])
        assert np.array_equal(_bits(self.w.getDepthVector()), _bits(self.m.getDepthVector()))
        assert self.w.getFeatureCount() == self.m.getFeatureCount()
        if pb.n_visual:
            self.seen.add("factors")
        self.calls["fill"] = self.calls.get("fill", 0) + 1
        self.log.append(("fill", n, pb.n_visual, bytes(pb.visual)[:pb.n_visual * ROW_BYTES]))
        return n

    def setDepth(self, x):
        self.m.setDepth(x); self.w.setDepth(x)
        t = self.check("setDepth")
        if any(r["solve_flag"] == 2 for r in t):
            self.seen.add("solve_flag 2")

    def _set(self, name, *a):
        a_, b_ = getattr(self.m, name)(*a), getattr(self.w, name)(*a)
        assert a_ == b_, (name, sorted(a_), sorted(b_))
        order = [it.feature_id for it in self.m.feature if it.feature_id in a_]
        assert self.w.last_outlier_ids == order                                  # ids come back in list order
        if a_:
            self.seen.add(name)
        self.log.append((name, tuple(order)))
        return b_

    def outliersRejection(self, *a):
        return self._set("outliersRejection", *a)

    def movingConsistencyCheckW(self, *a):
        return self._set("movingConsistencyCheckW", *a)

    def predictPtsInNextFrame(self, *a):
        a_, b_ = self.m.predictPtsInNextFrame(*a), self.w.predictPtsInNextFrame(*a)
        assert list(a_) == list(b_)
        for k in a_:
            assert np.array_equal(_bits(a_[k]), _bits(b_[k])), k
        if a_:
            self.seen.add("prediction")
        self.log.append(("predict", tuple((k, v.tobytes()) for k, v in b_.items())))
        return b_

    def _removal(self, name, *a):
        n0 = len(self.m.feature)
        getattr(self.m, name)(*a); getattr(self.w, name)(*a)
        self.check(name)
        if len(self.m.feature) < n0:
            self.seen.add(name + " removed")

    def removeOutlier(self, ids):
        self._removal("removeOutlier", ids)

    def removeFailures(self):
        self._removal("removeFailures")

    def removeBackShiftDepth(self, *a):
        self._removal("removeBackShiftDepth", *a)

    def removeBack(self):
        self._removal("removeBack")

    def removeFront(self, fc):
        self._removal("removeFront", fc)

    def close(self):
        self.w.close()


def _replay(fm, n, **kw):
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import SyntheticStream
    _, p8 = _cam()
    dynamic = kw.pop("dynamic", False)
    tr, ba = FeatureTracker(640, 480, p8, 150, 30, 1, 1), BundleAdjuster(0)
    out = replay(SyntheticStream(seed=0, dynamic=dynamic), tr, fm, ba, n, **kw)
    tr.close(); ba.close()
    return out


@pytest.mark.parametrize("feedback,use_mcc", [(False, False), (False, True), (True, False), (True, True)])
def test_every_call_of_the_replayed_stream_matches_the_host_mirror(feedback, use_mcc):
    """The 48-frame synthetic stream of test_fm_gpu.py through tracker -> manager -> solver, the manager being both at once."""
    both = Both(depth_threshold=4.0)
    out = _replay(both, 48, feedback=feedback, use_mcc=use_mcc)
    both.close()
    assert out["n_margin_old"] > 5 and out["n_margin_second_new"] > 0 and out["ate_m"] < 5e-3
    need = {"parallax", "factors", "flag 1", "removeBackShiftDepth removed"}
    assert need <= both.seen, need - both.seen
    assert both.calls["add"] == 48 and both.calls["fill"] == 38 and both.calls["triangulate"] == 38
    if feedback:
        assert "prediction" in both.seen and out["n_predicted"] > 500
    assert both.max_par_rel <= 1e-13


def test_stream_with_boxes_skips_frames_like_the_host_mirror():
    """trackImagebox leaves the features inside a detection out of the frame: such a landmark misses a frame and comes back,
    and both managers append to its short list."""
    from ground_fusion_b200.synth import SyntheticStream
    st = SyntheticStream(seed=0, dynamic=True)
    n = 40
    boxes = [st.boxes(k) if k % 5 != 4 else np.zeros((0, 4), np.int64) for k in range(n)]
    both = Both(depth_threshold=4.0)
    out = _replay(both, n, boxes=boxes, dynamic=True)
    both.close()
    assert "skipped a frame" in both.seen and {"parallax", "factors"} <= both.seen
    assert out["n_margin_old"] > 0 and out["n_margin_second_new"] > 0


def test_two_runs_of_the_window_are_bit_identical():
    """The window alone (no solver, whose atomics are not ordered): every table, counter and the parallax, bit for bit."""
    from ground_fusion_b200.feature_window import FeatureWindow
    from test_fm_oracle import scene
    Ps, Rs, lms, frames = scene(seed=11, n_lm=700, noise=2e-4, depth_noise=0.01)
    tic, ric = np.array([0.02, -0.01, 0.03]), np.eye(3)
    runs = []
    for _ in range(2):
        w, log = FeatureWindow(depth_threshold=5.0, min_parallax_px=1.0), []
        for f in range(11):
            log.append((w.addFeatureCheckParallax(f, frames.get(f, {}), 0.0), w.last_track_num, w.long_track_num, float(w.last_average_parallax).hex()))
        w.triangulateAll(10, Ps, Rs, tic, ric)
        log.append(sorted(w.movingConsistencyCheckW(Ps, Rs, tic, ric)))
        log.append([(k, v.tobytes()) for k, v in w.predictPtsInNextFrame(10, Ps, Rs, tic, ric).items()])
        w.removeBackShiftDepth(Rs[0], Ps[0], Rs[1], Ps[1])
        log.append([(r["feature_id"], r["start_frame"], r["estimate_flag"], float(r["estimated_depth"]).hex(), r["obs"].tobytes()) for r in w.read()])
        w.close()
        runs.append(log)
    assert any(float.fromhex(x[3]) > 0 for x in runs[0][:11]), "the parallax sum was never reached"
    assert runs[0] == runs[1]


def _frame(ids, rng, depth=2.0):
    return {int(k): np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.3, 0.3), 1.0, rng.uniform(0, 640), rng.uniform(0, 480),
                              rng.normal(), rng.normal(), depth + rng.uniform(-0.5, 0.5)]) for k in ids}


def _poses(rng=None):
    Ps = np.array([[0.12 * k, 0.03 * np.sin(0.5 * k), 0.02 * k] for k in range(11)])
    Rs = np.array([[[np.cos(0.02 * k), 0, np.sin(0.02 * k)], [0, 1, 0], [-np.sin(0.02 * k), 0, np.cos(0.02 * k)]] for k in range(11)])
    return Ps, Rs, np.array([0.02, -0.01, 0.03]), np.eye(3)


def test_scripted_sequence_reaches_the_corner_cases():
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.ba_problem import Problem
    rng = np.random.default_rng(7)
    cap = 96
    both = Both(depth_threshold=3.0, max_features=cap)
    Ps, Rs, tic, ric = _poses()
    both.addFeatureCheckParallax(0, {}, 0.0)                                         # an empty frame on an empty table
    assert "empty frame" in both.seen and both.w.size() == 0
    both.addFeatureCheckParallax(0, _frame(range(10, 40), rng), 0.0)                 # only new ids
    assert "only new ids" in both.seen
    for fc in range(1, 5):
        both.addFeatureCheckParallax(fc, _frame(range(10, 40), rng), 0.01 * fc)
    both.triangulateAll(4, Ps, Rs, tic, ric)
    # a landmark removed while the tracker still tracks it comes back at the end of the list with a smaller id
    both.removeOutlier({12, 17, 999})
    assert "removeOutlier removed" in both.seen and len(both.m.feature) == 28
    both.addFeatureCheckParallax(5, _frame(list(range(10, 40)) + [50, 45], rng), 0.0)
    assert [it.feature_id for it in both.m.feature][-4:] == [12, 17, 45, 50] and "list not sorted by id" in both.seen
    # setDepth with negative inverse depths -> solve_flag 2 -> removeFailures
    n = both.fillProblem(Problem(11, 0))
    assert n == 28
    x = both.m.getDepthVector(); x[3] = -0.5; x[20] = -2.0
    both.setDepth(x)
    assert "solve_flag 2" in both.seen
    both.removeFailures()
    assert "removeFailures removed" in both.seen and len(both.m.feature) == 30
    both.outliersRejection(Ps, Rs, tic, ric); both.movingConsistencyCheckW(Ps, Rs, tic, ric)
    both.predictPtsInNextFrame(5, Ps, Rs, tic, ric)
    assert "prediction" in both.seen
    # fill the window, then removeFront on a full window: landmarks that start at frame_count move, the others lose row W - 1 - start
    for fc in range(6, 11):
        both.addFeatureCheckParallax(fc, _frame([10, 11, 13] + ([60, 61] if fc == 10 else []) + ([70] if fc >= 9 else []), rng), 0.0)
    assert any(it.start_frame == 10 for it in both.m.feature)
    both.removeFront(10)
    assert {it.feature_id: (it.start_frame, len(it.obs)) for it in both.m.feature}[60] == (9, 1)
    assert 70 in {it.feature_id for it in both.m.feature}
    both.addFeatureCheckParallax(10, _frame([10, 11, 70], rng), 0.0)
    both.removeFront(10)
    # the second removeFront takes 60 and 61 (one observation, in frame 9) out of the list
    assert not {60, 61} & {it.feature_id for it in both.m.feature} and "removeFront removed" in both.seen
    # removeBack leaving one observation, then leaving none
    for _ in range(4):
        both.removeBack()
    two = [it.feature_id for it in both.m.feature if it.start_frame == 0 and len(it.obs) == 2]
    assert two
    both.removeBack()
    assert all(len(it.obs) == 1 and it.start_frame == 0 for it in both.m.feature if it.feature_id in two)
    one = [it.feature_id for it in both.m.feature if it.start_frame == 0 and len(it.obs) == 1]
    assert set(two) <= set(one)
    both.removeBack()
    assert not set(one) & {it.feature_id for it in both.m.feature} and "removeBack removed" in both.seen
    both.removeBackShiftDepth(Rs[0], Ps[0], Rs[1], Ps[1])
    # fill the table exactly to max_features, then one landmark more
    room = cap - len(both.m.feature)
    both.addFeatureCheckParallax(3, _frame(range(1000, 1000 + room), rng), 0.0)
    assert both.w.size() == cap == len(both.m.feature)
    before = both.w.read()
    with pytest.raises(GfError, match="-4"):
        both.w.addFeatureCheckParallax(4, _frame([1000, 1001, 5000], rng), 0.0)
    assert_same_table(both.w.read(), before, "after GF_ERR_CAPACITY")
    # argument errors leave the table as it was, too
    bad = Ps.copy(); bad[3, 1] = np.nan
    for call in (lambda: both.w.triangulateAll(10, bad, Rs, tic, ric), lambda: both.w.outliersRejection(bad, Rs, tic, ric),
                 lambda: both.w.predictPtsInNextFrame(10, Ps, Rs * np.inf, tic, ric), lambda: both.w.addFeatureCheckParallax(11, _frame([1], rng), 0.0),
                 lambda: both.w.addFeatureCheckParallax(-1, _frame([1], rng), 0.0), lambda: both.w.removeFront(9), lambda: both.w.setDepth(np.ones(3))):
        with pytest.raises(GfError, match="-1"):
            call()
    assert_same_table(both.w.read(), before, "after GF_ERR_INVALID_ARG")
    # frame WINDOW_SIZE added twice without a slide: the landmark has a row per window frame already
    lone = FeatureWindow(depth_threshold=3.0, max_features=8)
    for fc in range(11):
        lone.addFeatureCheckParallax(fc, _frame([5], rng), 0.0)
    full = lone.read()
    assert full[0]["n_obs"] == 11 and full[0]["start_frame"] == 0
    with pytest.raises(GfError, match="-1"):
        lone.addFeatureCheckParallax(10, _frame([5, 6], rng), 0.0)
    assert_same_table(lone.read(), full, "after the twelfth observation was refused")
    lone.close()
    both.w.clearDepth()
    assert all(r["estimated_depth"] == -1.0 for r in both.w.read())
    both.w.clearState()
    assert both.w.size() == 0 and both.w.read() == []
    both.close()


@pytest.mark.parametrize("n_lm", [31, 32, 33, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025])
def test_table_sizes_around_the_warp_and_block_boundaries(n_lm):
    """Every operation once at landmark counts either side of 32, 64, 256 and 1024 (the kernels' warp, block and chunk sizes)."""
    from test_fm_oracle import scene
    Ps, Rs, lms, frames = scene(seed=n_lm, n_lm=n_lm, noise=2e-4, depth_noise=0.01)
    tic, ric = np.array([0.02, -0.01, 0.03]), np.eye(3)
    both = Both(depth_threshold=5.0)
    for f in range(11):
        both.addFeatureCheckParallax(f, frames.get(f, {}), 0.0)
    assert len(both.m.feature) == n_lm
    both.triangulateAll(10, Ps, Rs, tic, ric)
    from ground_fusion_b200.ba_problem import Problem
    n = both.fillProblem(Problem(11, 0))
    assert n > n_lm // 4
    x = both.m.getDepthVector(); x[::7] *= 0.4; x[5::13] = -1.0
    both.setDepth(x)
    assert both.outliersRejection(Ps, Rs, tic, ric) or n_lm < 40
    out = both.movingConsistencyCheckW(Ps, Rs, tic, ric)
    both.predictPtsInNextFrame(10, Ps, Rs, tic, ric)
    both.removeOutlier(out)
    both.removeFailures()
    both.removeBackShiftDepth(Rs[0] @ ric, Ps[0] + Rs[0] @ tic, Rs[1] @ ric, Ps[1] + Rs[1] @ tic)
    both.addFeatureCheckParallax(10, {k: v for k, v in frames.get(10, {}).items() if k in {it.feature_id for it in both.m.feature}}, 0.0)
    both.removeFront(10)
    both.removeBack()
    need = {"removeFailures removed", "prediction", "factors"} | ({"removeBackShiftDepth removed"} if n_lm > 200 else set())
    assert need <= both.seen, need - both.seen
    both.close()


def test_ingest_from_the_tracker_on_the_device():
    """addFrameFromTracker right after trackImage / trackImagebox leaves the table add_frame leaves with the observations the
    tracker returned, and the tracker carries on exactly like one that was never read this way."""
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.synth import SyntheticStream
    _, p8 = _cam()
    st = SyntheticStream(seed=0, dynamic=True)
    read, plain = FeatureTracker(640, 480, p8, 150, 30, 1, 1), FeatureTracker(640, 480, p8, 150, 30, 1, 1)
    from ground_fusion_b200.feature_manager import FeatureManager
    a, b, m = FeatureWindow(depth_threshold=4.0), FeatureWindow(depth_threshold=4.0), FeatureManager(depth_threshold=4.0)
    with pytest.raises(GfError, match="no frame"):
        b.addFrameFromTracker(read, 0, 0.0)
    left_out = boxed_known = 0
    for k in range(14):
        t, gray, depth = st.frame(k)
        fc = min(k, 10)
        if k % 3 == 1:
            obs, in_box = read.trackImageboxRaw(t, st.boxes(k), gray, depth)
            obs2, in_box2 = plain.trackImageboxRaw(t, st.boxes(k), gray, depth)
            assert np.array_equal(in_box, in_box2)
            left_out += int(in_box.sum())
            m_img = {int(o["id"]): o["v"].copy() for o in obs[~in_box]}
        else:
            obs, in_box = read.trackImageRaw(t, gray, depth), None
            obs2 = plain.trackImageRaw(t, gray, depth)
            m_img = {int(o["id"]): o["v"].copy() for o in obs}
        assert obs.tobytes() == obs2.tobytes() and len(obs) > 100, k
        ra = a.addFrame(fc, obs, in_box, 0.0)
        rb = b.addFrameFromTracker(read, fc, 0.0)
        assert ra == rb and (a.last_track_num, a.new_feature_num, a.long_track_num) == (b.last_track_num, b.new_feature_num, b.long_track_num)
        assert a.last_average_parallax == b.last_average_parallax
        assert_same_table(b.read(), a.read(), "frame %d" % k)
        # independently of the kernel's own bit test: the host mirror, given only the observations outside the boxes
        known = {it.feature_id for it in m.feature}
        if in_box is not None:
            boxed_known += sum(int(o["id"]) in known for o in obs[in_box])
        assert m.addFeatureCheckParallax(fc, m_img, 0.0) == rb
        assert_same_table(b.read(), mirror_table(m), "frame %d against the host mirror" % k)
        if k >= 10:
            a.removeBack(); b.removeBack(); m.removeBack()
    assert left_out > 0 and boxed_known > 0 and a.size() > 150
    for x in (read, plain, a, b):
        x.close()


def test_ingest_from_a_pipelined_tracker():
    """submit / wait with two frames in flight: the returned frame k is still on the device while frame k + 1 runs (ingested, equal to
    add_frame with what wait returned), and is refused once frame k + 2 has been submitted into its result slot."""
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.synth import SyntheticStream
    _, p8 = _cam()
    st = SyntheticStream(seed=0)
    tr = FeatureTracker(640, 480, p8, 150, 30, 1, 1)
    a, b = FeatureWindow(depth_threshold=4.0), FeatureWindow(depth_threshold=4.0)
    fr = [st.frame(k) for k in range(8)]
    fr = [(t, np.ascontiguousarray(g, np.uint8), np.ascontiguousarray(d, np.uint16)) for t, g, d in fr]
    later = [(fr[7][0] + 0.05 * j, fr[7 - j][1], fr[7 - j][2]) for j in range(1, 4)]      # frames 8, 9, 10
    tr.submit(*fr[0])
    for k in range(6):
        tr.submit(*fr[k + 1])                       # frame k + 1 in flight
        obs = tr.wait()                             # frame k returned
        assert len(obs) > 100
        assert a.addFrame(k, obs, None, 0.0) == b.addFrameFromTracker(tr, k, 0.0)
        assert_same_table(b.read(), a.read(), "pipelined frame %d" % k)
    # frame 6 is in flight: wait for it, then submit 7, which runs in the other result slot
    obs6 = tr.wait()
    tr.submit(*fr[7])
    assert b.addFrameFromTracker(tr, 6, 0.0) == a.addFrame(6, obs6, None, 0.0)      # 7 uses the other slot
    assert_same_table(b.read(), a.read(), "frame 6 with frame 7 in flight")
    before = b.read()
    tr.wait()                                       # 7 returned ...
    tr.submit(*later[0])
    tr.wait()                                       # ... then 8 returned, and 9 and 10 submitted
    tr.submit(*later[1])
    tr.submit(*later[2])
    # the tracker last returned frame 8 (slot 0); frame 10 was just submitted into slot 0
    with pytest.raises(GfError, match="no longer on the device"):
        b.addFrameFromTracker(tr, 7, 0.0)
    assert_same_table(b.read(), before, "after the refusal")
    tr.wait(); tr.wait()
    for x in (tr, a, b):
        x.close()


def test_a_tracker_on_another_device_is_refused():
    """The device check of add_frame_from_tracker; needs a second GPU to build the case."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: a tracker on another device cannot be built")
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.synth import SyntheticStream
    _, p8 = _cam()
    tr, w = FeatureTracker(640, 480, p8, 150, 30, 1, 1, device=1), FeatureWindow(device=0)
    t, gray, depth = SyntheticStream(seed=0).frame(0)
    tr.trackImage(t, gray, depth)
    with pytest.raises(GfError, match="another device"):
        w.addFrameFromTracker(tr, 0, 0.0)
    tr.close(); w.close()


def test_whole_loop_with_the_window_matches_the_host_manager(capsys):
    """replay() over the 64 frames of bench.py's `ate` configuration, FeatureWindow against FeatureManager and against the
    oracle pipeline.  The solve's atomics make two runs with one and the same manager differ in the last bits; that difference is
    measured here too and printed beside the one between the managers."""
    from ground_fusion_b200.feature_manager import FeatureManager
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.replay_adapters import oracle_components
    n = 64
    host1 = _replay(FeatureManager(depth_threshold=4.0), n)
    host2 = _replay(FeatureManager(depth_threshold=4.0), n)
    win = FeatureWindow(depth_threshold=4.0)
    got = _replay(win, n)
    win.close()
    cam, _ = _cam()
    tr, fm, ba = oracle_components(cam, depth_threshold=4.0)
    want = replay(SyntheticStream(seed=0), tr, fm, ba, n)
    assert got["iterations"] == host1["iterations"] == want["iterations"]
    assert (got["n_margin_old"], got["n_margin_second_new"]) == (host1["n_margin_old"], host1["n_margin_second_new"]) == (want["n_margin_old"], want["n_margin_second_new"])
    d_run = np.linalg.norm(host1["P_est"] - host2["P_est"], axis=1).max()
    d_win = np.linalg.norm(got["P_est"] - host1["P_est"], axis=1).max()
    d_orc = np.linalg.norm(got["P_est"] - want["P_est"], axis=1).max()
    with capsys.disabled():
        print("\n64-frame replay: window vs host manager %.3e m, host manager run to run %.3e m, window vs oracle pipeline %.3e m" % (d_win, d_run, d_orc))
    d_host = np.linalg.norm(host1["P_est"] - want["P_est"], axis=1).max()
    # Every call of the window is bit-equal to the host manager's (the tests above), so what separates the two trajectories is
    # the solve's unordered atomics, the same thing that separates two runs with one manager: 0.8e-9 and 2.0e-9 m measured
    # over these 64 frames, the window 0.5e-9 and 1.4e-9 m from the host manager on the same two occasions.  The bars are
    # therefore that noise as measured here, not a constant below it: the host manager misses a 1e-9 m bar against itself.
    noise = max(d_run, 1e-9)
    assert d_win <= 3 * noise and d_win < 1e-8, (d_win, d_run)
    # the oracle pipeline: where the host manager ends (3.9e-8 m), give or take the same noise
    assert abs(d_orc - d_host) <= 3 * noise and d_orc < 5e-8, (d_orc, d_host, d_run)
    assert abs(got["ate_m"] - want["ate_m"]) < 1e-4 and got["ate_m"] < 5e-3
