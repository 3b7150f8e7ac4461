"""GPU tests of gf_fm_window_group (FeatureWindowGroup): K FeatureWindows driven with one set of launches per call must give,
member by member and bit for bit, what K independent FeatureWindows give when fed the same calls: tables, keyframe flags,
counters, parallax, factor rows, para_feature / feature_const, outlier ids in list order and predictions."""
import ctypes

import numpy as np
import pytest

from test_fm_window_gpu import ROW_BYTES, _bits, assert_same_table

pytestmark = pytest.mark.gpu

W = 10
CAPS = [64, 256, 1024, 63, 257, 1025, 65, 255]      # around the 64 / 256 / 1024-thread boundaries of the kernels


def _rot(rng):
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    return q * np.sign(np.linalg.det(q))


def poses(rng):
    Ps = np.cumsum(rng.normal(0, 0.2, (W + 1, 3)), 0)
    Rs = np.stack([_rot(rng) * 0.02 + np.eye(3) * 0.98 for _ in range(W + 1)])
    Rs = np.stack([np.linalg.qr(R)[0] * np.sign(np.diag(np.linalg.qr(R)[1])) for R in Rs])   # near-identity rotations
    ric, tic = np.eye(3), np.array([0.05, 0.0, 0.02])
    return Ps, Rs.reshape(W + 1, 9), tic, ric.ravel()


class Stream:
    """One member's synthetic frames: ids carried over from the previous frame with probability 0.8, new ids after them, and
    normalised points / pixels / velocities / depths from a seeded generator.  Frame size stays far below the capacity."""

    def __init__(self, seed, cap, n=None):
        self.rng = np.random.default_rng(seed)
        self.n = n if n is not None else max(8, min(120, cap // 8))
        self.ids, self.next_id = [], 0

    def frame(self):
        keep = [i for i in self.ids if self.rng.random() < 0.8]
        new = list(range(self.next_id, self.next_id + self.n - len(keep)))
        self.next_id += len(new)
        self.ids = keep + new
        ids = np.array(self.ids, np.int32)
        self.rng.shuffle(ids)
        from ground_fusion_b200._lib import OBS_DTYPE
        o = np.zeros(len(ids), OBS_DTYPE)
        o["id"] = ids
        xy = self.rng.uniform(-0.5, 0.5, (len(ids), 2))
        d = self.rng.uniform(0.5, 4.0, len(ids))
        d[self.rng.random(len(ids)) < 0.3] = 0.0                      # no depth for some
        o["v"] = np.column_stack([xy, np.ones(len(ids)), 320 + 460 * xy[:, 0], 240 + 460 * xy[:, 1],
                                  self.rng.normal(0, 0.01, (len(ids), 2)), d])
        box = (self.rng.random(len(ids)) < 0.05).astype(np.uint8)
        return o, box


def make_windows(caps):
    from ground_fusion_b200.feature_window import FeatureWindow
    return [FeatureWindow(max_features=c) for c in caps]


def same_tables(group_members, singles, what):
    for k, (g, s) in enumerate(zip(group_members, singles)):
        assert_same_table(g.read(), s.read(), "%s, member %d" % (what, k))


def same_problem(a, b, what):
    assert a.n_features == b.n_features and a.n_visual == b.n_visual, what
    assert bytes(a.visual)[:a.n_visual * ROW_BYTES] == bytes(b.visual)[:b.n_visual * ROW_BYTES], what
    n = a.n_features
    assert np.array_equal(_bits(a.para_feature[:n]), _bits(b.para_feature[:n])) and np.array_equal(a.feature_const[:n], b.feature_const[:n]), what


def fc_of(m, step):
    return min(step + m % 4, W)          # members reach a full window at different steps


def remove_op(m, step, fc):
    from ground_fusion_b200 import _lib
    if fc < W:
        return _lib.FM_REMOVE_NONE
    return [_lib.FM_REMOVE_BACK_SHIFT_DEPTH, _lib.FM_REMOVE_FRONT, _lib.FM_REMOVE_BACK][(m + step) % 3]


def run_lockstep(K, steps, seed=0, compare_every_call=True, caps=None, sizes=None):
    """K members through the whole per-frame stage, as a group and as K single windows; everything compared.  caps / sizes:
    each member's capacity and observations per frame (default: CAPS cycled, frames far below the capacity)."""
    from ground_fusion_b200 import _lib
    from ground_fusion_b200.ba_problem import Problem
    from ground_fusion_b200.feature_window import FeatureWindowGroup
    caps = caps or [CAPS[k % len(CAPS)] for k in range(K)]
    gw, sw = make_windows(caps), make_windows(caps)
    grp = FeatureWindowGroup(gw)
    streams = [Stream(seed * 1000 + k, c, sizes[k] if sizes else None) for k, c in enumerate(caps)]
    prng = np.random.default_rng(seed + 77)
    seen = set()
    for step in range(steps):
        fcs = [fc_of(m, step) for m in range(K)]
        tds = [0.001 * m for m in range(K)]
        fr = [s.frame() for s in streams]
        got = grp.addFrames(fcs, [o for o, _ in fr], [b for _, b in fr], tds)
        for m in range(K):
            want = sw[m].addFrame(fcs[m], fr[m][0], fr[m][1], tds[m])
            assert got[m] == want, (step, m)
            a, b = gw[m], sw[m]
            assert (a.last_track_num, a.new_feature_num, a.long_track_num, a._n_upper) == (b.last_track_num, b.new_feature_num, b.long_track_num, b._n_upper)
            assert _bits(a.last_average_parallax) == _bits(b.last_average_parallax)
            seen.add("keyframe" if want else "non-keyframe")
        if compare_every_call:
            same_tables(gw, sw, "add %d" % step)
        ps = [poses(prng) for _ in range(K)]
        grp.triangulateAll(fcs, ps)
        for m in range(K):
            sw[m].triangulateAll(fcs[m], *ps[m])
        if compare_every_call:
            same_tables(gw, sw, "triangulate %d" % step)
        pg, pw = [Problem(11, 1) for _ in range(K)], [Problem(11, 1) for _ in range(K)]
        nf = grp.fillProblems(pg)
        for m in range(K):
            assert nf[m] == sw[m].fillProblem(pw[m])
            same_problem(pg[m], pw[m], "fill %d member %d" % (step, m))
            if pw[m].n_visual:
                seen.add("factors")
        xs = []
        for m in range(K):
            x = pw[m].para_feature[:pw[m].n_features] * 1.01
            x[3::7] *= -1                                             # solve_flag 2
            xs.append(x)
        grp.setDepths(xs)
        for m in range(K):
            sw[m].setDepth(xs[m])
        if compare_every_call:
            same_tables(gw, sw, "setDepth %d" % step)
        if step % 3 == 2:
            grp.removeFailures()
            for m in range(K):
                sw[m].removeFailures()
        mode = step % 2
        og = grp.movingConsistencyCheckW(ps) if mode else grp.outliersRejections(ps)
        for m in range(K):
            ow = sw[m].movingConsistencyCheckW(*ps[m]) if mode else sw[m].outliersRejection(*ps[m])
            assert og[m] == ow and gw[m].last_outlier_ids == sw[m].last_outlier_ids, (step, m)
            if ow:
                seen.add("outliers")
        pred_g = grp.predictPtsInNextFrame(fcs, ps)
        for m in range(K):
            pw_ = sw[m].predictPtsInNextFrame(fcs[m], *ps[m])
            assert list(pred_g[m]) == list(pw_), (step, m)
            for i in pw_:
                assert np.array_equal(_bits(pred_g[m][i]), _bits(pw_[i]))
            if pw_:
                seen.add("predictions")
        # every third member drops a few ids it tracks (removeOutlier), the others none
        drops = [set(int(i) for i in fr[m][0]["id"][:3]) if m % 3 == 0 else set() for m in range(K)]
        grp.removeOutliers(drops)
        for m in range(K):
            sw[m].removeOutlier(drops[m])
        ops = [remove_op(m, step, fcs[m]) for m in range(K)]
        shifts = []
        for m in range(K):
            R0, P0 = ps[m][1][0].reshape(3, 3), ps[m][0][0]
            R1, P1 = ps[m][1][1].reshape(3, 3), ps[m][0][1]
            shifts.append((R0, P0, R1, P1))
        grp.remove(ops, fcs, shifts)
        for m in range(K):
            op = ops[m]
            if op == _lib.FM_REMOVE_BACK_SHIFT_DEPTH:
                sw[m].removeBackShiftDepth(*shifts[m])
            elif op == _lib.FM_REMOVE_FRONT:
                sw[m].removeFront(W)
            elif op == _lib.FM_REMOVE_BACK:
                sw[m].removeBack()
        seen |= {"op %d" % o for o in ops}
        if step == steps - 2:
            grp.clearDepth()
            for m in range(K):
                sw[m].clearDepth()
        same_tables(gw, sw, "step %d" % step)
    assert grp.last_device_ms() >= 0
    grp.close()
    for w in gw + sw:
        w.close()
    return seen


@pytest.mark.parametrize("K", [1, 2, 3, 8, 64])
def test_group_matches_single_windows(K):
    seen = run_lockstep(K, 14 if K <= 8 else 12, seed=K, compare_every_call=K <= 8)
    assert {"keyframe", "factors", "predictions"} <= seen, seen
    if K >= 3:
        assert {"op 0", "op 1", "op 2", "op 3"} <= seen, seen     # in one step, members take different removals


def test_group_grids_with_tables_of_very_different_sizes():
    """One member's table grows past the 256- and 1024-thread boundaries of the single-CTA kernels (to about 1300 landmarks)
    while another holds a handful and a third a few hundred: the grids are sized by the largest member and every other
    member's surplus CTAs must exit against its own count."""
    seen = run_lockstep(3, 5, seed=11, caps=[2048, 64, 1025], sizes=[700, 8, 200])
    assert "factors" in seen or "keyframe" in seen


def test_remove_front_is_checked_per_member():
    from ground_fusion_b200 import _lib
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_window import FeatureWindowGroup
    gw = make_windows([256, 256])
    grp = FeatureWindowGroup(gw)
    st = [Stream(k, 256) for k in range(2)]
    for fc in range(W + 1):
        grp.addFrames([fc, fc], [s.frame()[0] for s in st], None, [0.0, 0.0])
    before = [w.read() for w in gw]
    with pytest.raises(GfError, match="member 1: remove_front takes frame_count == WINDOW_SIZE"):
        grp.remove([_lib.FM_REMOVE_BACK, _lib.FM_REMOVE_FRONT], [W, W - 1])
    for w, b in zip(gw, before):
        assert_same_table(w.read(), b)
    grp.remove([_lib.FM_REMOVE_FRONT, _lib.FM_REMOVE_NONE], [W, W - 1])
    assert grp.last_device_ms() >= 0
    grp.close()
    for w in gw:
        w.close()


def test_last_device_ms_before_any_call():
    from ground_fusion_b200.feature_window import FeatureWindowGroup
    gw = make_windows([64, 64])
    grp = FeatureWindowGroup(gw)
    assert 0.0 <= grp.last_device_ms() < 1.0                         # the two events recorded at creation
    grp.triangulateAll([0, 0], [poses(np.random.default_rng(0))] * 2)     # the next call reports no stale error
    grp.close()
    for w in gw:
        w.close()


def test_device_failures_are_per_member():
    """Member 1 gets more new landmarks than fit; member 2 a frame at WINDOW_SIZE twice without a slide (a twelfth observation
    row).  Both report in status with their tables unchanged; member 0 is applied as its single call would apply it."""
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_window import FeatureWindowGroup
    caps = [256, 64, 256]
    gw, sw = make_windows(caps), make_windows(caps)
    grp = FeatureWindowGroup(gw)
    st = [Stream(k, 256) for k in range(3)]
    # fill member 2 up to frame WINDOW_SIZE with the same ids every frame
    fixed = st[2].frame()
    for fc in range(W + 1):
        frs = [st[0].frame(), (fixed[0][:8], None), fixed]
        grp.addFrames([fc, fc, fc], [f[0] for f in frs], None, [0.0] * 3)
        for m in range(3):
            sw[m].addFrame(fc, frs[m][0], None, 0.0)
    same_tables(gw, sw, "before")
    before = [w.read() for w in gw]
    big = Stream(99, 2048)
    big.n, big.next_id = 200, 100000                                  # ids the table does not hold
    fresh = Stream(7, 256)
    fresh.next_id = 50000                                             # member 0: only new landmarks, so it fits and is applied
    frs = [fresh.frame(), big.frame(), fixed]
    with pytest.raises(GfError, match="member 1: .*max_features"):
        grp.addFrames([W, W, W], [f[0] for f in frs], None, [0.0] * 3)
    assert list(grp.last_status) == [0, -4, -1]
    sw[0].addFrame(W, frs[0][0], None, 0.0)
    for m, code in ((1, "max_features"), (2, "last window frame")):
        with pytest.raises(GfError, match=code):
            sw[m].addFrame(W, frs[m][0], None, 0.0)
    same_tables(gw, sw, "after")
    assert_same_table(gw[1].read(), before[1])
    assert_same_table(gw[2].read(), before[2])
    grp.close()
    for w in gw + sw:
        w.close()


def test_argument_errors_change_nothing():
    from ground_fusion_b200._lib import GfError, OBS_DTYPE
    from ground_fusion_b200.feature_window import FeatureWindow, FeatureWindowGroup
    import ground_fusion_b200._lib as L
    gw = make_windows([256, 256, 256])
    grp = FeatureWindowGroup(gw)
    st = [Stream(k, 256) for k in range(3)]
    for fc in range(4):
        grp.addFrames([fc] * 3, [s.frame()[0] for s in st], None, [0.0] * 3)
    before = [w.read() for w in gw]
    rng = np.random.default_rng(5)
    ps = [poses(rng) for _ in range(3)]
    bad = list(ps)
    Pbad = ps[2][0].copy(); Pbad[4, 1] = np.nan
    bad[2] = (Pbad,) + ps[2][1:]
    with pytest.raises(GfError, match="member 2: non-finite pose"):
        grp.triangulateAll([3, 3, 3], bad)
    with pytest.raises(GfError, match="member 1: frame_count out of range"):
        grp.triangulateAll([3, 11, 3], ps)
    frs = [s.frame()[0] for s in st]
    dup = frs[1].copy(); dup["id"][1] = dup["id"][0]
    with pytest.raises(GfError, match="member 1: feature id twice"):
        grp.addFrames([4, 4, 4], [frs[0], dup, frs[2]], None, [0.0] * 3)
    with pytest.raises(GfError, match="member 2: frame_count out of range"):
        grp.addFrames([4, 4, -1], frs, None, [0.0] * 3)
    with pytest.raises(GfError, match="member 0: bad argument"):
        lib = L.lib()
        n = np.zeros(3, np.int32)
        ids = (ctypes.c_void_p * 3)(None, gw[1]._ids.ctypes.data, gw[2]._ids.ctypes.data)
        P, R, t, r = [np.ascontiguousarray(np.stack([p[j] for p in ps]), np.float64) for j in range(4)]
        L.check(lib.gf_fm_window_group_outliers(grp._h, P.ctypes.data, R.ctypes.data, t.ctypes.data, r.ctypes.data, 0, ids, n.ctypes.data))
    with pytest.raises(GfError, match="member 0: set_depth takes"):
        grp.setDepths([np.zeros(0), np.ones(3), np.zeros(0)])
    for w, b in zip(gw, before):
        assert_same_table(w.read(), b)
    with pytest.raises(GfError, match="member 2: the window is listed twice"):
        FeatureWindowGroup([gw[0], gw[1], gw[0]])
    many = [FeatureWindow(max_features=16) for _ in range(L.FM_WINDOW_GROUP_MAX + 1)]
    with pytest.raises(GfError, match="member 64: "):
        FeatureWindowGroup(many)
    FeatureWindowGroup(many[:L.FM_WINDOW_GROUP_MAX]).close()
    for w in many:
        w.close()
    import torch
    if torch.cuda.device_count() > 1:
        other = FeatureWindow(max_features=16, device=1)
        with pytest.raises(GfError, match="member 1: bound to another device"):
            FeatureWindowGroup([gw[0], other])
        other.close()
    grp.close()
    for w in gw:
        w.close()


def test_direct_calls_between_group_calls():
    """Single calls on a member between group calls (and the group taking over again) give the tables of an all-single run."""
    from ground_fusion_b200.ba_problem import Problem
    from ground_fusion_b200.feature_window import FeatureWindowGroup
    caps = [256, 1024, 64]
    gw, sw = make_windows(caps), make_windows(caps)
    grp = FeatureWindowGroup(gw)
    st = [Stream(k + 10, c) for k, c in enumerate(caps)]
    rng = np.random.default_rng(3)
    for fc in range(W + 1):
        frs = [s.frame() for s in st]
        if fc % 2:
            grp.addFrames([fc] * 3, [f[0] for f in frs], [f[1] for f in frs], [0.0] * 3)
        else:
            for m in range(3):
                gw[m].addFrame(fc, frs[m][0], frs[m][1], 0.0)
        for m in range(3):
            sw[m].addFrame(fc, frs[m][0], frs[m][1], 0.0)
        ps = [poses(rng) for _ in range(3)]
        if fc % 3 == 0:
            gw[1].triangulateAll(fc, *ps[1])                         # one member directly, then the group for all
            grp.triangulateAll([fc] * 3, ps)
            sw[1].triangulateAll(fc, *ps[1])
            for m in range(3):
                sw[m].triangulateAll(fc, *ps[m])
        else:
            grp.triangulateAll([fc] * 3, ps)
            for m in range(3):
                sw[m].triangulateAll(fc, *ps[m])
        pg = [Problem(11, 1) for _ in range(3)]
        grp.fillProblems(pg)
        gw[2].setDepth(pg[2].para_feature[:pg[2].n_features] * 0.9)     # a member finishes the solve on its own
        for m in range(2):
            gw[m].setDepth(pg[m].para_feature[:pg[m].n_features] * 0.9)
        for m in range(3):
            pw = Problem(11, 1)
            sw[m].fillProblem(pw)
            sw[m].setDepth(pw.para_feature[:pw.n_features] * 0.9)
        same_tables(gw, sw, "frame %d" % fc)
    gw[0].removeBack()
    grp.removeFailures()
    sw[0].removeBack()
    for m in range(3):
        sw[m].removeFailures()
    same_tables(gw, sw, "end")
    grp.close()
    for w in gw + sw:
        w.close()


def _trackers(K):
    from ground_fusion_b200.feature_tracker import FeatureTracker, TrackerGroup
    from ground_fusion_b200.synth import idc_params8
    trs = [FeatureTracker(640, 480, idc_params8(), 150, 30, 1, 1, device=0) for _ in range(K)]
    return trs, TrackerGroup(trs)


def _frames(K, n):
    from ground_fusion_b200.synth import SyntheticStream
    out = []
    for k in range(K):
        s = SyntheticStream(seed=20 + k)
        out.append([tuple(np.ascontiguousarray(x) if isinstance(x, np.ndarray) else x for x in s.frame(f)) for f in range(n)])
    return out


def test_ingest_from_tracker_group():
    """Group ingest from a TrackerGroup's collected step equals single windows fed add_frame with the host results of that step,
    boxes included; pipelined (submit k + 1, wait k, ingest); each refusal leaves every table unchanged."""
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.feature_window import FeatureWindowGroup
    K, N = 3, 8
    fr = _frames(K, N + 2)
    trs, tg = _trackers(K)
    gw, sw = make_windows([1024] * K), make_windows([1024] * K)
    grp = FeatureWindowGroup(gw)
    with pytest.raises(GfError, match="collected no step"):
        grp.addFramesFromTrackerGroup(tg, [0] * K, [0.0] * K)
    boxes = [[np.array([[100 + 40 * k, 80, 260 + 40 * k, 240]]) for k in range(K)] for _ in range(N + 2)]

    def submit(f):
        tg.submit([fr[k][f][0] for k in range(K)], [fr[k][f][1].ctypes.data for k in range(K)],
                  [fr[k][f][2].ctypes.data for k in range(K)], boxes=boxes[f])
    submit(0)
    nbox = 0
    for f in range(N):
        if f + 1 < N:
            submit(f + 1)                                              # the next step runs while step f is ingested
        res = tg.wait()
        fc = min(f, W)
        got = grp.addFramesFromTrackerGroup(tg, [fc] * K, [0.0] * K)
        for k in range(K):
            obs, _, _, in_box = res[k]
            nbox += int(in_box.sum())
            assert got[k] == sw[k].addFrame(fc, obs, in_box.astype(np.uint8), 0.0)
        same_tables(gw, sw, "step %d" % f)
    assert nbox > 0
    before = [w.read() for w in gw]
    # the collected step's slot reused: two more steps submitted after it
    submit(N); submit(N + 1)
    with pytest.raises(GfError, match="no longer on the device"):
        grp.addFramesFromTrackerGroup(tg, [W] * K, [0.0] * K)
    tg.wait(); tg.wait()
    small = FeatureWindowGroup(gw[:K - 1])
    with pytest.raises(GfError, match="number of members"):
        small.addFramesFromTrackerGroup(tg, [W] * (K - 1), [0.0] * (K - 1))
    small.close()
    for w, b in zip(gw, before):
        assert_same_table(w.read(), b)
    grp.close(); tg.close()
    for x in gw + sw + trs:
        x.close()


def _p8():
    from ground_fusion_b200.synth import IDC_CAM
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    return [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]


def _independent(seed, n, feedback):
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import SyntheticStream
    tr, fm, ba = FeatureTracker(640, 480, _p8(), 150, 30, 1, 1), FeatureWindow(depth_threshold=4.0), BundleAdjuster(0)
    out = replay(SyntheticStream(seed=seed), tr, fm, ba, n, feedback=feedback)
    tr.close(); fm.close(); ba.close()
    return out


@pytest.mark.parametrize("feedback", [False, True])
def test_whole_loop_replay_group_matches_independent_replays(feedback, capsys):
    """replay_group over K = 4 streams (tracker group -> window group -> solve_multi -> marginalize_multi) against four
    independent replay() runs on FeatureWindow and single solves.  The solve's atomics are not ordered, so the trajectory bar
    is three times the run-to-run difference measured here (floor 1e-9 m, cap 1e-8 m)."""
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.replay import replay_group
    from ground_fusion_b200.synth import SyntheticStream
    K, n = 4, 40
    seeds = list(range(K))
    trs = [FeatureTracker(640, 480, _p8(), 150, 30, 1, 1) for _ in range(K)]
    wins = [FeatureWindow(depth_threshold=4.0) for _ in range(K)]
    bas = [BundleAdjuster(0) for _ in range(K)]
    got = replay_group([SyntheticStream(seed=s) for s in seeds], trs, wins, bas, n, feedback=feedback)
    for x in trs + wins + bas:
        x.close()
    d_run = d_grp = 0.0
    for s, g in zip(seeds, got):
        a, b, c = (_independent(s, n, feedback) for _ in range(3))
        # A solve that ends at its termination threshold can take one iteration more or less from run to run (the Hessian's
        # atomics are not ordered): where the independent runs agree the group must agree, elsewhere it must be one of theirs.
        for f, it in enumerate(g["iterations"]):
            ref = {a["iterations"][f], b["iterations"][f], c["iterations"][f]}
            assert it in ref, (s, f, it, ref)
        assert (g["n_margin_old"], g["n_margin_second_new"]) == (a["n_margin_old"], a["n_margin_second_new"]), s
        assert g["n_predicted"] == a["n_predicted"] and g["n_removed"] == a["n_removed"], s
        assert len(g["P_est"]) == len(a["P_est"]) > 0
        d_run = max(d_run, max(np.linalg.norm(x["P_est"] - y["P_est"], axis=1).max() for x, y in ((a, b), (a, c), (b, c))))
        d_grp = max(d_grp, min(np.linalg.norm(g["P_est"] - x["P_est"], axis=1).max() for x in (a, b, c)))
    if feedback:
        assert sum(g["n_predicted"] for g in got) > 0
    with capsys.disabled():
        print("\nreplay_group K=%d, %d frames, feedback=%s: group vs independent %.3e m, run to run %.3e m" % (K, n, feedback, d_grp, d_run))
    bar = min(max(3 * d_run, 1e-9), 1e-8)
    assert d_grp <= bar, (d_grp, d_run)
