"""GPU: the tracker's `equalize` option (gf_tracker_set_equalize / gf_stage_clahe).

The CLAHE kernels against cv2.createCLAHE(clip, grid).apply, bit for bit; and whole tracker sequences with equalisation on
against the cv2 oracle that equalises each frame before trackImage, as the reference does with `equalize` set -- through every
intake path (host / device frames, the two-frames-in-flight pipeline, batches, GF_NO_GRAPH, GF_LK_NO_TMA, profiling mode).  The sequences are dark and low-contrast, derived from the synthetic stream by a gamma and a contrast squeeze."""
import numpy as np
import pytest

from clahe_ref import cv2_clahe, dark_stream, make_equalizing_oracle, parity_image

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

SIZES = [(640, 480), (641, 480), (640, 481), (1280, 720), (1920, 1080), (377, 377), (424, 400), (752, 480)]
GRIDS = [(1, 1), (3, 11), (7, 5), (8, 8), (16, 16)]
CLIPS = [40.0, 3.0, 1.0, 0.5, 0.0]


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("grid", GRIDS)
def test_stage_clahe_matches_cv2_geometries(gf, w, h, grid):
    for kind, clip in (("random", 40.0), ("dark", 3.0), ("flat", 1.0), ("near_constant", 40.0)):
        img = parity_image(kind, w, h, seed=w + h)
        got, want = gf.clahe(img, clip, grid), cv2_clahe(img, clip, grid)
        assert np.array_equal(got, want), "%s clip %g: %d px differ" % (kind, clip, (got != want).sum())


@pytest.mark.parametrize("clip", CLIPS)
@pytest.mark.parametrize("kind", ["random", "dark", "flat", "near_constant", "constant"])
def test_stage_clahe_matches_cv2_clip_limits(gf, clip, kind):
    for (w, h), grid in (((640, 480), (8, 8)), ((641, 480), (8, 8)), ((424, 400), (7, 5)), ((640, 481), (16, 16)), ((1280, 720), (1, 1))):
        img = parity_image(kind, w, h, seed=3)
        assert np.array_equal(gf.clahe(img, clip, grid), cv2_clahe(img, clip, grid)), (w, h, grid)


def test_stage_clahe_row_pitch_and_limits(gf):
    from ground_fusion_b200._lib import GfError
    img = parity_image("dark", 643, 480, 1)
    buf = np.full((480, 700), 255, np.uint8)
    buf[:, :643] = img
    assert np.array_equal(gf.clahe(buf[:, :643]), cv2_clahe(img))
    for grid in ((0, 8), (8, 17), (17, 1)):
        with pytest.raises(GfError):
            gf.clahe(img, 40.0, grid)
    with pytest.raises(GfError):
        gf.clahe(np.zeros((200, 200), np.uint8))


def _cam(w):
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    sc = w / 640.0
    return PinholeCamera(IDC_CAM["fx"] * sc, IDC_CAM["fy"] * sc, IDC_CAM["cx"] * sc, IDC_CAM["cy"] * sc,
                         IDC_CAM["k1"], IDC_CAM["k2"], IDC_CAM["p1"], IDC_CAM["p2"])


def _oracle_results(frames, w, max_cnt=150, min_dist=30):
    """(ids, track_cnt, status, {id: v}, n_new) per frame from the equalising cv2 oracle."""
    ref = make_equalizing_oracle()(_cam(w), max_cnt, min_dist, 1, 1)
    out = []
    for t, g, d in frames:
        want = ref.trackImage(t, g, d)
        out.append((list(ref.ids), list(ref.track_cnt), ref.last_status.copy(), want, len(ref.last_n_pts)))
    return out


def _check(k, want, obs, status, info):
    ids, cnt, st, vmap, n_new = want
    assert np.array_equal(status, st), "frame %d: inlier mask differs" % k
    assert list(obs["id"]) == ids, "frame %d: feature ids / order differ" % k
    assert list(obs["track_cnt"]) == cnt, "frame %d" % k
    for o in obs:
        assert np.array_equal(o["v"], vmap[int(o["id"])]), "frame %d id %d" % (k, o["id"])
    assert info["n_new"] == n_new, "frame %d" % k


def _padded(a, pad):
    buf = np.full((a.shape[0], a.shape[1] + pad), np.iinfo(a.dtype).max, a.dtype)
    buf[:, :a.shape[1]] = a
    return buf[:, :a.shape[1]]


@pytest.mark.parametrize("w,h,n,pad", [(640, 480, 20, 0), (640, 481, 12, 0), (641, 481, 12, 13), (1280, 720, 8, 0)])
@pytest.mark.parametrize("on_device", [False, True])
def test_equalized_sequence_matches_oracle(gf, w, h, n, pad, on_device):
    import torch
    frames = dark_stream(seed=11, w=w, h=h, n=n)
    want = _oracle_results(frames, w)
    tr = gf.FeatureTracker(w, h, _cam(w).params8(), 150, 30, 1, 1, equalize=True)
    for k, (t, g, d) in enumerate(frames):
        if on_device:
            dg = torch.from_numpy(np.ascontiguousarray(g)).cuda()
            dd = torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda()
            torch.cuda.synchronize()
            obs = tr.trackDevice(t, dg.data_ptr(), dd.data_ptr())
        else:
            if pad:
                g, d = _padded(g, pad), _padded(d, pad)
                assert g.strides[0] > w
            obs = tr.trackImageRaw(t, g, d)
        _check(k, want[k], obs, tr.last_status, tr.last_info)
    tr.close()


def test_equalize_changes_the_outcome_and_off_is_unchanged(gf):
    """On the dark sequence equalisation changes what the tracker finds (so the parity above cannot pass by ignoring the option),
    and a tracker with it off still equals the plain oracle."""
    from oracle.fe_oracle import FeatureTrackerOracle
    w, h = 640, 480
    frames = dark_stream(seed=11, w=w, h=h, n=6)
    eq = _oracle_results(frames, w)
    ref = FeatureTrackerOracle(_cam(w), 150, 30, 1, 1)
    off = gf.FeatureTracker(w, h, _cam(w).params8(), 150, 30, 1, 1)
    differs = 0
    for k, (t, g, d) in enumerate(frames):
        want = ref.trackImage(t, g, d)
        obs = off.trackImageRaw(t, g, d)
        assert list(obs["id"]) == list(ref.ids) and np.array_equal(off.last_status, ref.last_status)
        for o in obs:
            assert np.array_equal(o["v"], want[int(o["id"])])
        eq_pts = {i: v[3:5].tobytes() for i, v in eq[k][3].items()}
        differs += sum(1 for o in obs if eq_pts.get(int(o["id"])) != o["v"][3:5].tobytes())
    assert differs > 100, differs
    off.close()


def test_set_equalize_only_before_the_first_frame(gf):
    from ground_fusion_b200._lib import GfError
    (t, g, d), = dark_stream(seed=11, w=640, h=480, n=1)
    tr = gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1)
    for grid in ((0, 8), (17, 8), (8, 17), (-1, 1)):
        if grid[0] == 0:
            tr.set_equalize(40.0, grid)            # 0 = off
        else:
            with pytest.raises(GfError):
                tr.set_equalize(40.0, grid)
    tr.set_equalize(40.0, (8, 8))
    tr.trackImageRaw(t, g, d)
    with pytest.raises(GfError):
        tr.set_equalize(40.0, (8, 8))
    with pytest.raises(GfError):
        tr.set_equalize(40.0, (0, 0))
    tr.close()


def test_kernels_per_frame(gf):
    """Equalisation adds exactly its two kernels per frame; with it off the tracker launches what it launched before the option
    existed: 3 pyrDown + 3 min-eig + k_track + k_compact_setmask + 2 GFTT selection kernels + k_select_finalize."""
    lib = gf._lib.lib()
    frames = dark_stream(seed=11, w=640, h=480, n=8)
    per_frame = {}
    for eq in (False, True):
        tr = gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1, equalize=eq)
        for t, g, d in frames[:2]:
            tr.trackImageRaw(t, g, d)               # graphs captured
        n0 = lib.gf_kernel_launch_count()
        for t, g, d in frames[2:]:
            tr.trackImageRaw(t, g, d)
        per_frame[eq] = (lib.gf_kernel_launch_count() - n0) / (len(frames) - 2)
        tr.close()
    assert per_frame[False] == 11 and per_frame[True] == 13, per_frame


def test_profiling_mode_counts_clahe_in_the_pyramid_stage(gf):
    frames = dark_stream(seed=11, w=640, h=480, n=6)
    want = _oracle_results(frames, 640)
    tr = gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1, equalize=True)
    tr.set_profiling(True)
    for k, (t, g, d) in enumerate(frames):
        obs = tr.trackImageRaw(t, g, d)
        _check(k, want[k], obs, tr.last_status, tr.last_info)
        assert tr.last_stage_ms()["pyramid"] > 0
    tr.close()


def _ptrs(frames, on_device, keep):
    import torch
    if not on_device:
        return [g.ctypes.data for _, g, _ in frames], [d.ctypes.data for _, _, d in frames]
    gs = [torch.from_numpy(g).cuda() for _, g, _ in frames]
    ds = [torch.from_numpy(d.view(np.int16)).cuda() for _, _, d in frames]
    keep.append((gs, ds))
    torch.cuda.synchronize()
    return [x.data_ptr() for x in gs], [x.data_ptr() for x in ds]


@pytest.fixture(params=["streams", "no-graph", "no-tma", "no-graph-no-tma"])
def orchestration(request, monkeypatch):
    """The five-stream pipeline with CUDA graphs, GF_NO_GRAPH, GF_LK_NO_TMA and both; the tracker reads them when it is created."""
    monkeypatch.delenv("GF_NO_GRAPH", raising=False)
    monkeypatch.delenv("GF_LK_NO_TMA", raising=False)
    if request.param in ("no-graph", "no-graph-no-tma"):
        monkeypatch.setenv("GF_NO_GRAPH", "1")
    if request.param in ("no-tma", "no-graph-no-tma"):
        monkeypatch.setenv("GF_LK_NO_TMA", "1")
    return request.param


@pytest.mark.parametrize("w,h", [(640, 480), (641, 481)])
@pytest.mark.parametrize("on_device", [False, True])
def test_equalized_batch_matches_oracle(gf, orchestration, on_device, w, h):
    if orchestration == "no-graph" and (on_device or w != 640):
        pytest.skip("GF_NO_GRAPH: once, host frames at 640x480")
    frames = [(t, np.ascontiguousarray(g), np.ascontiguousarray(d)) for t, g, d in dark_stream(seed=12, w=w, h=h, n=14)]
    want = _oracle_results(frames, w)
    tr = gf.FeatureTracker(w, h, _cam(w).params8(), 150, 30, 1, 1, equalize=True)
    keep = []
    pos = 0
    for n in (1, 5, 8):                                  # batches back to back: the pipeline state carries across calls
        fr = frames[pos:pos + n]
        gp, dp = _ptrs(fr, on_device, keep)
        got = tr.trackBatch([t for t, _, _ in fr], gp, dp, on_device=on_device)
        for k, (obs, st, info) in enumerate(got):
            _check(pos + k, want[pos + k], obs, st, info)
        pos += n
    tr.close()


@pytest.mark.parametrize("on_device", [False, True])
def test_equalized_batch_multi_matches_oracle(gf, orchestration, on_device):
    from ground_fusion_b200.feature_tracker import FeatureTracker
    if orchestration == "no-graph" and on_device:
        pytest.skip("GF_NO_GRAPH: once, host frames")
    S, n = 3, 8
    streams = [[(t, np.ascontiguousarray(g), np.ascontiguousarray(d)) for t, g, d in dark_stream(seed=30 + i, w=640, h=480, n=n)]
               for i in range(S)]
    want = [_oracle_results(fr, 640) for fr in streams]
    trs = [gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1, equalize=True) for _ in range(S)]
    keep = []
    ptrs = [_ptrs(fr, on_device, keep) for fr in streams]
    got = FeatureTracker.trackBatchMulti(trs, [[t for t, _, _ in fr] for fr in streams], [p[0] for p in ptrs], [p[1] for p in ptrs],
                                         on_device=on_device)
    for i in range(S):
        assert len(got[i]) == n
        for k, (obs, st, info) in enumerate(got[i]):
            _check(k, want[i][k], obs, st, info)
    for tr in trs:
        tr.close()
