"""GPU parity tests of the front end (run with -m gpu on an H100).

Every test calls the CUDA path through the C ABI (libgf_b200.so) and compares with the oracle:
cv2 4.13.0 for the three OpenCV calls the reference makes (feature_tracker.cpp:118-153,198) and
oracle/fe_oracle.py for FeatureTracker::trackImage as a whole.  Bar: bit-exact.
"""
import numpy as np
import pytest

from conftest import make_texture_image, warp_image

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("shape", [(640, 480), (1280, 720), (321, 243), (650, 490)])
def test_pyr_down_matches_cv2(gf, shape):
    img = make_texture_image(1, *shape)
    for _ in range(3):
        out = gf.pyr_down(img)
        assert np.array_equal(out, cv2.pyrDown(img))
        img = out


@pytest.mark.parametrize("seed,shape,contrast", [(0, (640, 480), 1.0), (1, (640, 480), 2.5), (2, (1280, 720), 1.5),
                                                   (3, (333, 207), 3.0), (4, (640, 480), 0.2)])
def test_min_eig_matches_cv2_bit_exact(gf, seed, shape, contrast):
    img = make_texture_image(seed, *shape, contrast=contrast)
    e, nfix = gf.corner_min_eigen_val(img)
    want = cv2.cornerMinEigenVal(img, 3, ksize=3)
    assert np.array_equal(bits(e), bits(want)), "%d px differ (fixups %d)" % ((bits(e) != bits(want)).sum(), nfix)


def test_min_eig_flat_and_saturated(gf):
    img = np.zeros((480, 640), np.uint8)
    img[100:200, 100:300] = 255
    img[300:, :] = 7
    e, _ = gf.corner_min_eigen_val(img)
    assert np.array_equal(bits(e), bits(cv2.cornerMinEigenVal(img, 3, ksize=3)))


@pytest.mark.parametrize("seed,contrast", [(0, 1.0), (1, 2.5), (2, 1.7)])
@pytest.mark.parametrize("max_level", [3, 1, 0])
def test_lk_matches_cv2_bit_exact(gf, seed, contrast, max_level):
    a = make_texture_image(seed, contrast=contrast)
    b = warp_image(a, 3.3 + seed, -2.1, 0.7)
    rng = np.random.default_rng(100 + seed)
    pts = np.stack([rng.uniform(-5, 645, 500), rng.uniform(-5, 485, 500)], 1).astype(np.float32)
    q_cv, st_cv, _ = cv2.calcOpticalFlowPyrLK(a, b, pts.reshape(-1, 1, 2), None, winSize=(21, 21), maxLevel=max_level)
    q, st = gf.calc_optical_flow_pyr_lk(a, b, pts, max_level)
    assert np.array_equal(st, st_cv.ravel())
    assert np.array_equal(bits(q), bits(q_cv.reshape(-1, 2)))


def test_lk_initial_flow_reverse_pass(gf):
    a = make_texture_image(5, contrast=1.5)
    b = warp_image(a, -2.6, 1.4, -0.4)
    rng = np.random.default_rng(7)
    pts = np.stack([rng.uniform(0, 640, 300), rng.uniform(0, 480, 300)], 1).astype(np.float32)
    fwd, _ = gf.calc_optical_flow_pyr_lk(a, b, pts, 3)
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
    r_cv, st_cv, _ = cv2.calcOpticalFlowPyrLK(b, a, fwd.reshape(-1, 1, 2), pts.reshape(-1, 1, 2).copy(), winSize=(21, 21),
                                              maxLevel=1, criteria=crit, flags=cv2.OPTFLOW_USE_INITIAL_FLOW)
    r, st = gf.calc_optical_flow_pyr_lk(b, a, fwd, 1, init=pts)
    assert np.array_equal(st, st_cv.ravel())
    assert np.array_equal(bits(r), bits(r_cv.reshape(-1, 2)))


def test_lk_empty_and_single(gf):
    a = make_texture_image(0)
    q, st = gf.calc_optical_flow_pyr_lk(a, a, np.zeros((0, 2), np.float32), 3)
    assert q.shape == (0, 2) and st.shape == (0,)
    q, st = gf.calc_optical_flow_pyr_lk(a, a, np.array([[320.5, 240.25]], np.float32), 3)
    q_cv, st_cv, _ = cv2.calcOpticalFlowPyrLK(a, a, np.array([[[320.5, 240.25]]], np.float32), None, winSize=(21, 21), maxLevel=3)
    assert np.array_equal(bits(q), bits(q_cv.reshape(-1, 2))) and st[0] == st_cv[0, 0]


def test_setmask_order_matches_std_sort(gf):
    from oracle.fe_oracle import setmask_order
    rng = np.random.default_rng(3)
    for n in (1, 2, 5, 16, 17, 18, 33, 64, 100, 150, 257, 300, 400, 511, 512, 513, 1000):
        for span in (1, 2, 6, 50, 1000):
            tc = np.sort(rng.integers(1, span + 1, n))[::-1].astype(np.int32)   # the tracker's input is non-increasing
            assert np.array_equal(gf.setmask_order(tc), setmask_order(tc))
            tc2 = rng.integers(1, span + 1, n).astype(np.int32)
            assert np.array_equal(gf.setmask_order(tc2), setmask_order(tc2))


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
@pytest.mark.parametrize("max_corners,min_dist,n_kept", [(150, 30, 0), (40, 30, 90), (500, 15, 120), (1000, 7, 0), (20, 30, 400)])
def test_gftt_matches_cv2(gf, seed, max_corners, min_dist, n_kept):
    img = make_texture_image(seed, contrast=1.0 + 0.5 * seed)
    rng = np.random.default_rng(seed)
    kept = np.stack([rng.uniform(1, 638, n_kept), rng.uniform(1, 478, n_kept)], 1).astype(np.float32)
    mask = np.full(img.shape, 255, np.uint8)
    for p in kept:
        cv2.circle(mask, (int(np.rint(p[0])), int(np.rint(p[1]))), min_dist, 0, -1)
    want = cv2.goodFeaturesToTrack(img, max_corners, 0.01, min_dist, mask=mask)
    want = np.zeros((0, 2), np.float32) if want is None else want.reshape(-1, 2)
    got, info = gf.good_features_to_track(img, max_corners, min_dist, kept)
    assert got.shape == want.shape and np.array_equal(got, want), info


def _run_sequence(gf, seed, n_frames, w=640, h=480, max_cnt=150, min_dist=30, noise=1.0):
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import IDC_CAM, FeatureTrackerOracle, PinholeCamera
    sc = w / 640.0
    cam = PinholeCamera(IDC_CAM["fx"] * sc, IDC_CAM["fy"] * sc, IDC_CAM["cx"] * sc, IDC_CAM["cy"] * sc,
                        IDC_CAM["k1"], IDC_CAM["k2"], IDC_CAM["p1"], IDC_CAM["p2"])
    stream = SyntheticStream(seed=seed, width=w, height=h, noise_sigma=noise)
    gpu = gf.FeatureTracker(w, h, cam.params8(), max_cnt, min_dist, 1, 1)
    ref = FeatureTrackerOracle(cam, max_cnt, min_dist, 1, 1)
    for k in range(n_frames):
        t, gray, depth = stream.frame(k)
        got = gpu.trackImageRaw(t, gray, depth)
        want = ref.trackImage(t, gray, depth)
        assert np.array_equal(gpu.last_status, ref.last_status), "frame %d: inlier mask differs" % k
        assert list(got["id"]) == list(ref.ids), "frame %d: feature ids / order differ" % k
        assert list(got["track_cnt"]) == list(ref.track_cnt), "frame %d" % k
        for o in got:
            assert np.array_equal(o["v"], want[int(o["id"])]), "frame %d id %d: %s vs %s" % (k, o["id"], o["v"], want[int(o["id"])])
        assert gpu.last_info["n_new"] == len(ref.last_n_pts)
    gpu.close()


def test_track_sequence_c2_bit_exact(gf):
    """BASELINE config C2: 640x480, 150 features, min_dist 30."""
    _run_sequence(gf, seed=0, n_frames=60)


def test_track_sequence_c3_300_features(gf):
    _run_sequence(gf, seed=1, n_frames=30, max_cnt=300, min_dist=20)


def test_track_sequence_c4_720p_500_features(gf):
    _run_sequence(gf, seed=2, n_frames=12, w=1280, h=720, max_cnt=500, min_dist=25)


def test_two_frames_in_flight_equals_blocking_calls(gf):
    """submit t+1 before collecting t (upload/pyramid/min-eig of t+1 overlap the tracking of t): same bits as trackImage,
    which is itself compared with the oracle above; frames with and without a depth image alternate to cover the
    rotated depth / parameter buffers."""
    from ground_fusion_b200.synth import SyntheticStream
    from ground_fusion_b200._lib import GfError
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    cam = PinholeCamera(**IDC_CAM)
    stream = SyntheticStream(seed=5)
    frames = [stream.frame(k) for k in range(25)]
    frames = [(t, g, (d if k % 7 != 3 else None)) for k, (t, g, d) in enumerate(frames)]
    a = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1)
    want = []
    for t, g, d in frames:
        obs = a.trackImageRaw(t, g, d).copy()
        want.append((obs, a.last_status.copy(), dict(a.last_info)))
    a.close()
    b = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1)
    got = []
    pending = 0
    for t, g, d in frames:
        b.submit(t, np.ascontiguousarray(g), None if d is None else np.ascontiguousarray(d))
        pending += 1
        if pending == 2:
            obs = b.wait().copy(); got.append((obs, b.last_status.copy(), dict(b.last_info))); pending -= 1
    with pytest.raises(GfError):
        b.removeOutliers({1})                      # state-changing calls need an empty pipeline
    while pending:
        obs = b.wait().copy(); got.append((obs, b.last_status.copy(), dict(b.last_info))); pending -= 1
    with pytest.raises(GfError):
        b.wait()
    assert len(got) == len(want)
    for k, ((o1, s1, i1), (o2, s2, i2)) in enumerate(zip(want, got)):
        assert i1 == i2, "frame %d: %s vs %s" % (k, i1, i2)
        assert np.array_equal(s1, s2), "frame %d" % k
        assert o1.tobytes() == o2.tobytes(), "frame %d" % k
    b.close()


@pytest.mark.parametrize("name", ["fe_c2_seed0", "fe_c3_seed1"])
def test_gpu_reproduces_golden_fixture(gf, name):
    """The committed fixtures (tests/golden/fe_*.npz, written by make_fe_golden.py from the cv2 oracle) replayed through the
    C ABI on the GPU: ids, inlier masks, new corners and observation vectors of every frame, bit for bit."""
    import os
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz"))
    seed, w, h, max_cnt, min_dist, frames = [int(v) for v in g["meta"]]
    params8 = [IDC_CAM[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]
    st = SyntheticStream(seed=seed, width=w, height=h)
    tr = gf.FeatureTracker(w, h, params8, max_cnt, min_dist, 1, 1)
    for k in range(frames):
        t, gray, depth = st.frame(k)
        got = tr.trackImageRaw(t, gray, depth)
        assert np.array_equal(got["id"], g["ids_%d" % k]), "frame %d: ids" % k
        assert np.array_equal(tr.last_status, g["status_%d" % k]), "frame %d: inlier mask" % k
        assert tr.last_info["n_new"] == len(g["npts_%d" % k]), "frame %d: new corners" % k
        assert np.array_equal(got["v"].reshape(-1, 8), g["obs_%d" % k]), "frame %d: observations" % k
    tr.close()


def test_missing_depth_frames_match_oracle(gf):
    """Frames whose depth image is missing (depth_cam = 1): the reference returns an EMPTY featureFrame
    (feature_tracker.cpp:342) but still advances its state; GPU and oracle are compared on every frame, the
    empty ones included."""
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import IDC_CAM, FeatureTrackerOracle, PinholeCamera
    cam = PinholeCamera(**IDC_CAM)
    stream = SyntheticStream(seed=6)
    gpu = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1)
    ref = FeatureTrackerOracle(cam, 150, 30, 1, 1)
    for k in range(16):
        t, gray, depth = stream.frame(k)
        if k % 5 == 2:
            depth = None
        got = gpu.trackImage(t, gray, depth)
        want = ref.trackImage(t, gray, depth)
        assert np.array_equal(gpu.last_status, ref.last_status), "frame %d" % k
        assert sorted(got) == sorted(want), "frame %d" % k
        if depth is None:
            assert len(got) == 0
        for fid in want:
            assert np.array_equal(got[fid], want[fid]), "frame %d id %d" % (k, fid)
    gpu.close()


def test_track_no_depth_image_quirk(gf):
    """depth_cam with an empty depth image yields an empty featureFrame (feature_tracker.cpp:342)."""
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    cam = PinholeCamera(**IDC_CAM)
    tr = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1)
    assert len(tr.trackImage(0.0, make_texture_image(0), None)) == 0
    tr.close()
    tr = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 0)   # mono: depth = -2.4
    out = tr.trackImage(0.0, make_texture_image(0), None)
    assert len(out) == 150 and all(v[7] == -2.4 for v in out.values())
    tr.close()


def test_prediction_and_remove_outliers(gf):
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import IDC_CAM, FeatureTrackerOracle, PinholeCamera
    cam = PinholeCamera(**IDC_CAM)
    stream = SyntheticStream(seed=4)
    gpu = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1)
    ref = FeatureTrackerOracle(cam, 150, 30, 1, 1)
    rng = np.random.default_rng(0)
    for k in range(10):
        t, gray, depth = stream.frame(k)
        got = gpu.trackImageRaw(t, gray, depth)
        want = ref.trackImage(t, gray, depth)
        assert list(got["id"]) == list(ref.ids), "frame %d" % k
        assert np.array_equal(gpu.last_status, ref.last_status), "frame %d" % k
        for o in got:
            assert np.array_equal(o["v"], want[int(o["id"])])
        if k in (3, 6):      # feed back "BA" predictions: true ray * depth, slightly perturbed, for 2/3 of the ids
            pred = {}
            for o in got[::3] if k == 3 else got[: len(got) * 2 // 3]:
                d = max(o["v"][7], 0.5)
                pred[int(o["id"])] = (o["v"][0] * d + rng.normal(0, 0.002), o["v"][1] * d + rng.normal(0, 0.002), d)
            gpu.setPrediction(pred); ref.setPrediction(pred)
        if k in (4, 7):
            rm = set(int(i) for i in got["id"][::7])
            gpu.removeOutliers(rm); ref.removeOutliers(rm)
        if k == 8:           # a prediction so bad that fewer than 10 succeed -> 3-level fallback path
            pred = {int(o["id"]): (5.0, 5.0, 1.0) for o in got}
            gpu.setPrediction(pred); ref.setPrediction(pred)
    gpu.close()


@pytest.fixture(params=["streams", "one-graph-per-frame"])
def batch_mode(request, monkeypatch):
    """gf_tracker_track_batch(_multi) has two orchestrations (DESIGN 1.3); the tracker reads GF_BATCH_PIPELINE when it is created."""
    if request.param == "one-graph-per-frame":
        monkeypatch.setenv("GF_BATCH_PIPELINE", "1")
    else:
        monkeypatch.delenv("GF_BATCH_PIPELINE", raising=False)
    return request.param


@pytest.mark.parametrize("on_device", [False, True])
def test_batch_pipeline_equals_blocking_calls(gf, on_device, batch_mode):
    """gf_tracker_track_batch runs one graph per frame ({track + select of frame f} || {intake + pyramid + min-eig of f+1});
    the frames must come out exactly as from trackImage: batches of 1, 2, 5, 7 and 10 frames back to back, frames without a
    depth image in between, a setPrediction before a batch (first frame takes the other path), a removeOutliers and a
    plain trackImage call between batches, host and device-resident frames."""
    import torch
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    cam = PinholeCamera(**IDC_CAM)
    stream = SyntheticStream(seed=9)
    frames = [stream.frame(k) for k in range(27)]
    frames = [(t, np.ascontiguousarray(g), (np.ascontiguousarray(d) if k % 6 != 4 else None)) for k, (t, g, d) in enumerate(frames)]
    splits = [1, 2, 5, 7, 10]                       # 25 frames in batches, then frame 25 alone, then a batch of one
    a = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1)
    b = gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1)
    keep = []

    def ptrs(fr):
        if not on_device:
            return [g.ctypes.data for _, g, _ in fr], [(d.ctypes.data if d is not None else 0) for _, _, d in fr]
        gs = [torch.from_numpy(g).cuda() for _, g, _ in fr]
        ds = [(torch.from_numpy(d.view(np.int16)).cuda() if d is not None else None) for _, _, d in fr]
        keep.append((gs, ds))
        torch.cuda.synchronize()
        return [x.data_ptr() for x in gs], [(x.data_ptr() if x is not None else 0) for x in ds]

    def plain(tr, fr):
        out = []
        for t, g, d in fr:
            obs = tr.trackImageRaw(t, g, d).copy()
            out.append((obs, tr.last_status.copy(), dict(tr.last_info)))
        return out

    def check(want, got, base):
        assert len(want) == len(got)
        for k, ((o1, s1, i1), (o2, s2, i2)) in enumerate(zip(want, got)):
            assert i1 == i2, "frame %d: %s vs %s" % (base + k, i1, i2)
            assert np.array_equal(s1, s2), "frame %d" % (base + k)
            assert o1.tobytes() == o2.tobytes(), "frame %d" % (base + k)

    pos = 0
    for n in splits:
        fr = frames[pos:pos + n]
        want = plain(a, fr)
        gp, dp = ptrs(fr)
        got = b.trackBatch([t for t, _, _ in fr], gp, dp, on_device=on_device)
        check(want, got, pos)
        pos += n
        last = want[-1][0]
        if n == 2:                                   # prediction pending when the next batch starts
            pred = {int(o["id"]): (o["v"][0] * 2.0, o["v"][1] * 2.0, 2.0) for o in last[::2]}
            a.setPrediction(pred); b.setPrediction(pred)
        if n == 5:
            rm = set(int(i) for i in last["id"][::5])
            a.removeOutliers(rm); b.removeOutliers(rm)
    check(plain(a, frames[25:26]), plain(b, frames[25:26]), 25)      # the per-frame path after batches ...
    fr = frames[26:27]
    gp, dp = ptrs(fr)
    check(plain(a, fr), b.trackBatch([fr[0][0]], gp, dp, on_device=on_device), 26)   # ... and a batch after it
    a.close(); b.close()


@pytest.mark.parametrize("on_device", [False, True])
def test_multi_stream_batch_equals_single_stream_batches(gf, on_device, batch_mode):
    """gf_tracker_track_batch_multi: three independent streams (different scenes, one without depth images, one with a pending
    prediction) fed by one host thread come out exactly as from three gf_tracker_track_batch calls."""
    import torch
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.synth import SyntheticStream
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    cam = PinholeCamera(**IDC_CAM)
    S, n = 3, 9
    frames = []
    for i in range(S):
        st = SyntheticStream(seed=20 + i)
        fr = [st.frame(k) for k in range(n + 2)]
        frames.append([(t, np.ascontiguousarray(g), (np.ascontiguousarray(d) if (i != 1 and k % 5 != 3) else None)) for k, (t, g, d) in enumerate(fr)])
    keep = []

    def ptrs(fr):
        if not on_device:
            return [g.ctypes.data for _, g, _ in fr], [(d.ctypes.data if d is not None else 0) for _, _, d in fr]
        gs = [torch.from_numpy(g).cuda() for _, g, _ in fr]
        ds = [(torch.from_numpy(d.view(np.int16)).cuda() if d is not None else None) for _, _, d in fr]
        keep.append((gs, ds)); torch.cuda.synchronize()
        return [x.data_ptr() for x in gs], [(x.data_ptr() if x is not None else 0) for x in ds]

    a = [gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1) for _ in range(S)]
    b = [gf.FeatureTracker(640, 480, cam.params8(), 150, 30, 1, 1) for _ in range(S)]
    for i in range(S):                          # two warm-up frames per stream, then a prediction on stream 2
        for t, g, d in frames[i][:2]:
            oa = a[i].trackImageRaw(t, g, d).copy(); b[i].trackImageRaw(t, g, d)
        if i == 2:
            pred = {int(o["id"]): (o["v"][0] * 2.0, o["v"][1] * 2.0, 2.0) for o in oa[::2]}
            a[i].setPrediction(pred); b[i].setPrediction(pred)
    want, gp, dp = [], [], []
    for i in range(S):
        g_, d_ = ptrs(frames[i][2:])
        gp.append(g_); dp.append(d_)
        want.append(a[i].trackBatch([t for t, _, _ in frames[i][2:]], g_, d_, on_device=on_device))
    got = FeatureTracker.trackBatchMulti(b, [[t for t, _, _ in frames[i][2:]] for i in range(S)], gp, dp, on_device=on_device)
    for i in range(S):
        assert len(got[i]) == n
        for k, ((o1, s1, i1), (o2, s2, i2)) in enumerate(zip(want[i], got[i])):
            assert i1 == i2, "stream %d frame %d" % (i, k)
            assert np.array_equal(s1, s2) and o1.tobytes() == o2.tobytes(), "stream %d frame %d" % (i, k)
    assert sum(len(o) for o, _, _ in got[1]) == 0 and sum(len(o) for o, _, _ in got[0]) > 500      # depth_cam without depth images: empty frames
    for tr in a + b:
        tr.close()
