"""GPU: trackImagebox (the `use_yolo` front end) against the cv2 oracle, bit for bit.

gf_stage_in_boxes against cv2.pointPolygonTest on the probe sets of box_ref; tracker sequences on the synthetic stream with a moving
object, fed its detections, 100-box lists with degenerate, inverted and out-of-image boxes, frames without boxes and a box over the
whole image -- through every intake path (host / device frames, two frames in flight, batches, GF_NO_GRAPH, GF_LK_NO_TMA,
profiling mode); the state invariant (boxes change in_box only); argument errors; the launch count; the C++ adaptor; and the
replay loop with USE_YOLO."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

from box_ref import FeatureTrackerOracleFastBox, closed_form, cv2_inside, probe_sets

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_stage_in_boxes_matches_point_polygon_test(gf):
    n = 0
    for box, pts in probe_sets(seed=2):
        want = np.array([cv2_inside(box, p) for p in pts])
        assert np.array_equal(gf.in_boxes(pts, [box]), want), box
        n += len(pts)
    rng = np.random.default_rng(3)
    sets = probe_sets(seed=4, n_boxes=200)
    for k in range(0, 200, 100):                         # 100 boxes at once, every box's probes against all of them
        boxes = [b for b, _ in sets[k:k + 100]]
        pts = np.concatenate([p for _, p in sets[k:k + 100]] + [rng.uniform(-100, 800, (500, 2)).astype(np.float32)], 0)
        want = np.array([any(cv2_inside(b, p) for b in boxes) for p in pts])
        assert np.array_equal(gf.in_boxes(pts, boxes), want)
        n += len(pts)
    assert n > 150000


def test_stage_in_boxes_limits(gf):
    from ground_fusion_b200._lib import GfError
    pts = np.zeros((4, 2), np.float32)
    assert not gf.in_boxes(pts, np.zeros((0, 4))).any()
    assert gf.in_boxes([[5, 5]], [[0, 0, 10, 10]] * 100)[0]
    with pytest.raises(GfError, match="-4"):
        gf.in_boxes(pts, [[0, 0, 10, 10]] * 101)


def _cam(w):
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    sc = w / 640.0
    return PinholeCamera(IDC_CAM["fx"] * sc, IDC_CAM["fy"] * sc, IDC_CAM["cx"] * sc, IDC_CAM["cy"] * sc,
                         IDC_CAM["k1"], IDC_CAM["k2"], IDC_CAM["p1"], IDC_CAM["p2"])


def box_schedule(st, k, w, h):
    """Detections of frame k: the moving object's box; none; 100 boxes (the object, degenerate, inverted, out-of-image, int64
    corners outside int32, random); the object plus a box over the whole image (an empty featureFrame)."""
    obj = st.boxes(k)
    kind = k % 4
    if kind == 0:
        return obj
    if kind == 1:
        return np.zeros((0, 4), np.int64)
    if kind == 3:
        return np.concatenate([obj, [[-5, -5, w + 5, h + 5]]], 0).astype(np.int64)
    rng = np.random.default_rng(1000 + k)
    x, y = rng.integers(0, w, 40), rng.integers(0, h, 40)
    fixed = [[100, 50, 100, 400], [20, 300, 600, 300], [500, 400, 300, 200], [w + 10, 0, w + 200, h], [-300, -300, -1, h],
             [2 ** 32 + 200, 2 ** 32 + 100, 2 ** 32 + 260, 2 ** 32 + 180], [-2 ** 40, 0, 2 ** 40, 30]]
    rand = np.stack([x, y, x + rng.integers(-30, 60, 40), y + rng.integers(-30, 60, 40)], 1)
    out = np.concatenate([obj, fixed, rand], 0).astype(np.int64)
    return np.concatenate([out, rng.integers(0, min(w, h), (100 - len(out), 4))], 0).astype(np.int64)


def dynamic_frames(seed, w, h, n):
    from ground_fusion_b200.synth import SyntheticStream
    st = SyntheticStream(seed=seed, width=w, height=h, dynamic=True)
    return [st.frame(k) + (box_schedule(st, k, w, h),) for k in range(n)]


def _oracle(frames, w, depth_cam=1):
    """Per frame (ids, track_cnt, status, trackImagebox frame, n_new, empty) of the cv2 oracle; empty: depth_cam without a depth
    image, where the reference returns an empty featureFrame and the library no entries."""
    ref = FeatureTrackerOracleFastBox(_cam(w), 150, 30, 1, depth_cam)
    out = []
    for t, g, d, b in frames:
        got = ref.trackImagebox(t, b, g, d) if len(b) else ref.trackImage(t, g, d)
        out.append((list(ref.ids), list(ref.track_cnt), ref.last_status.copy(), got, len(ref.last_n_pts), bool(depth_cam and d is None)))
    return out


def _check(k, want, obs, status, info, in_box):
    ids, cnt, st, frame, n_new, empty = want
    assert np.array_equal(status, st), "frame %d: inlier mask differs" % k
    if empty:
        assert len(obs) == 0 and len(in_box) == 0 and frame == {}, "frame %d" % k
        return
    assert list(obs["id"]) == [int(i) for i in ids], "frame %d: feature ids / order differ" % k
    assert list(obs["track_cnt"]) == [int(c) for c in cnt], "frame %d" % k
    assert info["n_new"] == n_new, "frame %d" % k
    kept = obs[~in_box]
    assert sorted(int(i) for i in kept["id"]) == sorted(frame), "frame %d: boxed features differ" % k
    for o in kept:
        assert np.array_equal(o["v"], frame[int(o["id"])]), "frame %d id %d" % (k, o["id"])


def _padded(a, pad):
    buf = np.full((a.shape[0], a.shape[1] + pad), np.iinfo(a.dtype).max, a.dtype)
    buf[:, :a.shape[1]] = a
    return buf[:, :a.shape[1]]


@pytest.mark.parametrize("w,h,n,pad", [(640, 480, 16, 0), (641, 481, 10, 13), (1280, 720, 8, 0)])
@pytest.mark.parametrize("depth_cam", [1, 0])
def test_trackimagebox_sequence_matches_oracle(gf, w, h, n, pad, depth_cam):
    frames = dynamic_frames(7, w, h, n)
    want = _oracle(frames, w, depth_cam)
    tr = gf.FeatureTracker(w, h, _cam(w).params8(), 150, 30, 1, depth_cam)
    boxed = 0
    for k, (t, g, d, b) in enumerate(frames):
        if pad:
            g, d = _padded(g, pad), _padded(d, pad)
        obs, in_box = tr.trackImageboxRaw(t, b, g, d)
        _check(k, want[k], obs, tr.last_status, tr.last_info, in_box)
        if k % 4 == 3:
            assert in_box.all() and len(in_box) > 50                  # the whole image is boxed: nothing reaches the estimator
        if k % 4 == 1:
            assert not in_box.any()
        boxed += int(in_box.sum())
    assert boxed > 200
    tr.close()


def test_boxes_change_in_box_only(gf):
    """A tracker fed boxes returns the same out / status / info bytes as one fed none; only in_box differs, and the next frames
    still match after a frame whose every feature was boxed."""
    frames = dynamic_frames(8, 640, 480, 14)
    a, b = (gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1) for _ in range(2))
    for k, (t, g, d, bx) in enumerate(frames):
        o1 = a.trackImageRaw(t, g, d).copy()
        s1, i1 = a.last_status.copy(), dict(a.last_info)
        o2, in_box = b.trackImageboxRaw(t, bx, g, d)
        assert o1.tobytes() == o2.tobytes() and np.array_equal(s1, b.last_status) and i1 == b.last_info, "frame %d" % k
        assert np.array_equal(in_box, closed_form(bx, o2["v"][:, 3:5])), "frame %d" % k
    a.close(); b.close()


def _submit_boxes(tr, t, g, d, boxes):
    from ground_fusion_b200._lib import check
    bx = np.ascontiguousarray(boxes, np.int64).reshape(-1, 4)
    check(tr.L.gf_tracker_submit(tr._h, float(t), g.ctypes.data, g.strides[0], d.ctypes.data if d is not None else None,
                                 d.strides[0] if d is not None else 0, 0, bx.ctypes.data if len(bx) else None, len(bx)))


def _wait_boxes(tr):
    from ground_fusion_b200._lib import TrackInfo, check
    n, info, ib = ctypes.c_int(0), TrackInfo(), np.zeros(tr.max_cnt, np.uint8)
    check(tr.L.gf_tracker_wait(tr._h, tr._obs.ctypes.data, ctypes.byref(n), ib.ctypes.data, tr._status.ctypes.data, ctypes.byref(info)))
    return tr._collect(n, info), ib[:n.value].view(np.bool_)


def test_two_frames_in_flight(gf):
    """submit t+1 with boxes before wait t: the parameter block with the boxes rotates with the frame; frames with and without
    depth and with and without boxes interleave, and gf_tracker_wait without in_box collects a boxed frame as trackImage's result."""
    frames = dynamic_frames(9, 640, 480, 17)
    frames = [(t, np.ascontiguousarray(g), (np.ascontiguousarray(d) if k % 5 != 2 else None), b) for k, (t, g, d, b) in enumerate(frames)]
    want = _oracle(frames, 640)
    tr = gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1)
    pending, k_out = 0, 0

    def collect():
        nonlocal k_out
        if k_out % 6 == 5:                               # the plain wait: trackImage's result, without the flags
            obs = tr.wait()
            ids, cnt, st, frame, n_new, empty = want[k_out]
            assert np.array_equal(tr.last_status, st) and list(obs["id"]) == ([] if empty else [int(i) for i in ids])
        else:
            obs, ib = _wait_boxes(tr)
            _check(k_out, want[k_out], obs, tr.last_status, tr.last_info, ib)
        k_out += 1

    for t, g, d, b in frames:
        _submit_boxes(tr, t, g, d, b)
        pending += 1
        if pending == 2:
            collect(); pending -= 1
    while pending:
        collect(); pending -= 1
    tr.close()


def _ptrs(frames, on_device, keep):
    import torch
    if not on_device:
        return [f[1].ctypes.data for f in frames], [f[2].ctypes.data for f in frames]
    gs = [torch.from_numpy(f[1]).cuda() for f in frames]
    ds = [torch.from_numpy(f[2].view(np.int16)).cuda() for f in frames]
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


@pytest.mark.parametrize("on_device", [False, True])
def test_batch_matches_oracle(gf, orchestration, on_device):
    if orchestration == "no-graph" and on_device:
        pytest.skip("GF_NO_GRAPH: once, host frames")
    frames = [(t, np.ascontiguousarray(g), np.ascontiguousarray(d), b) for t, g, d, b in dynamic_frames(10, 640, 480, 15)]
    want = _oracle(frames, 640)
    tr = gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1)
    keep, pos = [], 0
    for n in (1, 6, 8):                                  # batches back to back: the pipeline state carries across calls
        fr = frames[pos:pos + n]
        gp, dp = _ptrs(fr, on_device, keep)
        got = tr.trackBatch([f[0] for f in fr], gp, dp, on_device=on_device, boxes=[f[3] for f in fr])
        for k, (obs, st, info, ib) in enumerate(got):
            _check(pos + k, want[pos + k], obs, st, info, ib)
        pos += n
    tr.close()


@pytest.mark.parametrize("on_device", [False, True])
def test_batch_multi_matches_oracle(gf, orchestration, on_device):
    from ground_fusion_b200.feature_tracker import FeatureTracker
    if orchestration == "no-graph" and on_device:
        pytest.skip("GF_NO_GRAPH: once, host frames")
    S, n = 3, 9
    streams = [[(t, np.ascontiguousarray(g), np.ascontiguousarray(d), b) for t, g, d, b in dynamic_frames(40 + i, 640, 480, n)] for i in range(S)]
    streams[1] = [(t, g, d, np.zeros((0, 4), np.int64)) for t, g, d, _ in streams[1]]        # one stream without detections
    want = [_oracle(fr, 640) for fr in streams]
    trs = [gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1) for _ in range(S)]
    keep = []
    ptrs = [_ptrs(fr, on_device, keep) for fr in streams]
    got = FeatureTracker.trackBatchMulti(trs, [[f[0] for f in fr] for fr in streams], [p[0] for p in ptrs], [p[1] for p in ptrs],
                                         on_device=on_device, boxes=[[f[3] for f in fr] for fr in streams])
    for i in range(S):
        assert len(got[i]) == n
        for k, (obs, st, info, ib) in enumerate(got[i]):
            _check(k, want[i][k], obs, st, info, ib)
        assert (i == 1) == (sum(int(r[3].sum()) for r in got[i]) == 0)
    for tr in trs:
        tr.close()


def test_profiling_mode(gf):
    frames = dynamic_frames(11, 640, 480, 6)
    want = _oracle(frames, 640)
    tr = gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1)
    tr.set_profiling(True)
    for k, (t, g, d, b) in enumerate(frames):
        obs, ib = tr.trackImageboxRaw(t, b, g, d)
        _check(k, want[k], obs, tr.last_status, tr.last_info, ib)
        assert tr.last_stage_ms()["finalize"] > 0
    tr.close()


def test_argument_errors_consume_no_frame(gf):
    """101 boxes: GF_ERR_CAPACITY; a negative count or a NULL list with a count: GF_ERR_INVALID_ARG; a batch with one bad list is
    refused before its first frame.  No frame is consumed and the tracker goes on matching the oracle."""
    from ground_fusion_b200._lib import GfError, check
    frames = [(t, np.ascontiguousarray(g), np.ascontiguousarray(d), b) for t, g, d, b in dynamic_frames(12, 640, 480, 6)]
    want = _oracle(frames, 640)
    tr = gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1)
    t, g, d, b = frames[0]
    with pytest.raises(GfError, match="-4"):
        tr.trackImageboxRaw(t, np.zeros((101, 4), np.int64), g, d)
    for nb, ptr in ((-1, None), (3, None)):
        with pytest.raises(GfError, match="-1"):
            check(tr.L.gf_tracker_submit(tr._h, t, g.ctypes.data, 640, d.ctypes.data, 1280, 0, ptr, nb))
    bad = [b, np.zeros((101, 4), np.int64)]
    with pytest.raises(GfError, match="-4"):
        tr.trackBatch([f[0] for f in frames[:2]], [f[1].ctypes.data for f in frames[:2]], [f[2].ctypes.data for f in frames[:2]], boxes=bad)
    for k, (t, g, d, b) in enumerate(frames):
        if k < 3:
            obs, ib = tr.trackImageboxRaw(t, b, g, d)
            _check(k, want[k], obs, tr.last_status, tr.last_info, ib)
        else:
            (obs, st, info, ib), = tr.trackBatch([t], [g.ctypes.data], [d.ctypes.data], boxes=[b])
            _check(k, want[k], obs, st, info, ib)
    tr.close()


def test_kernels_per_frame(gf):
    """Boxes add no kernel: 11 launches per frame with and without them."""
    lib = gf._lib.lib()
    frames = dynamic_frames(13, 640, 480, 8)
    per_frame = {}
    for with_boxes in (False, True):
        tr = gf.FeatureTracker(640, 480, _cam(640).params8(), 150, 30, 1, 1)
        for t, g, d, b in frames[:2]:
            tr.trackImageRaw(t, g, d)
        n0 = lib.gf_kernel_launch_count()
        for t, g, d, b in frames[2:]:
            if with_boxes:
                tr.trackImageboxRaw(t, b, g, d)
            else:
                tr.trackImageRaw(t, g, d)
        per_frame[with_boxes] = (lib.gf_kernel_launch_count() - n0) / (len(frames) - 2)
        tr.close()
    assert per_frame == {False: 11, True: 11}, per_frame


def test_trackimagebox_through_the_cpp_adaptor(tmp_path):
    """harness fe-box: featureFrame without the boxed features, and cur_pts / ids / track_cnt with all of them, as the oracle's."""
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "adaptor")])
    exe = os.path.join(ROOT, "adaptor", "_build", "harness")
    from ground_fusion_b200.synth import idc_params8
    n, p8 = 10, idc_params8()
    frames = dynamic_frames(14, 640, 480, n)
    with open(tmp_path / "fe.bin", "wb") as f:
        f.write(struct.pack("<4i8d3i", n, 640, 480, 1, *p8, 150, 30, 1))
        for t, g, d, b in frames:
            f.write(struct.pack("<d", t)); f.write(np.ascontiguousarray(g, np.uint8).tobytes()); f.write(np.ascontiguousarray(d, np.uint16).tobytes())
            f.write(struct.pack("<i", len(b))); f.write(np.ascontiguousarray(b, np.int64).tobytes())
    subprocess.check_call([exe, "fe-box", str(tmp_path / "fe.bin"), str(tmp_path / "fe.out")], timeout=120)
    raw = open(tmp_path / "fe.out", "rb").read()
    ref = FeatureTrackerOracleFastBox(_cam(640), 150, 30, 1, 1)
    off = 0
    for t, g, d, b in frames:
        want = ref.trackImagebox(t, b, g, d)
        (m,) = struct.unpack_from("<i", raw, off); off += 4
        assert m == len(want)
        for fid in sorted(want):
            (got_id,) = struct.unpack_from("<i", raw, off); off += 4
            v = np.frombuffer(raw, np.float64, 8, off); off += 64
            assert got_id == fid and np.array_equal(v, want[fid])
        (npts,) = struct.unpack_from("<i", raw, off); off += 4
        rec = np.frombuffer(raw, np.dtype([("id", "<i4"), ("x", "<f4"), ("y", "<f4"), ("cnt", "<i4")]), npts, off); off += 16 * npts
        assert list(rec["id"]) == [int(i) for i in ref.ids] and list(rec["cnt"]) == [int(c) for c in ref.track_cnt]
        assert np.array_equal(rec["x"], ref.cur_pts[:, 0]) and np.array_equal(rec["y"], ref.cur_pts[:, 1])
        assert npts > m or len(b) == 0
    assert off == len(raw)


def test_replay_with_boxes_matches_the_oracle_pipeline(capsys):
    """USE_YOLO through the replay loop on the stream with the moving object: detections on most frames (every fifth frame has
    none and goes through trackImage).  GPU pipeline and oracle pipeline agree as in test_fm_gpu's replay test; no observation
    the estimator receives lies inside its frame's box, while without boxes some do."""
    from test_fm_gpu import _gpu_fm
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    from oracle.fe_oracle import PinholeCamera
    from oracle.fm_oracle import FeatureManagerOracle
    from oracle.replay_adapters import OracleBA
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    p8 = [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]
    n = 48
    st = SyntheticStream(seed=0, dynamic=True)
    boxes = [st.boxes(k) if k % 5 != 4 else np.zeros((0, 4), np.int64) for k in range(n)]

    class Watch:
        """Records, per frame, whether an observation handed to the estimator lies inside the frame's box."""
        def __init__(self, tr):
            self.tr, self.k, self.inside = tr, 0, []

        def _seen(self, frame):
            b = st.boxes(self.k)
            pts = np.array([v[3:5] for v in frame.values()], np.float32).reshape(-1, 2)
            self.inside.append(int(closed_form(b, pts).sum()))
            self.k += 1
            return frame

        def trackImage(self, t, g, d):
            return self._seen(self.tr.trackImage(t, g, d))

        def trackImagebox(self, t, b, g, d):
            return self._seen(self.tr.trackImagebox(t, b, g, d))

    want = replay(SyntheticStream(seed=0, dynamic=True), FeatureTrackerOracleFastBox(PinholeCamera(**cam), 150, 30, 1, 1),
                  FeatureManagerOracle(depth_threshold=4.0), OracleBA(), n, boxes=boxes)
    ate = {}
    for use_boxes in (True, False):
        w = Watch(FeatureTracker(640, 480, p8, 150, 30, 1, 1))
        gba = BundleAdjuster(0)
        got = replay(SyntheticStream(seed=0, dynamic=True), w, _gpu_fm(depth_threshold=4.0), gba, n, boxes=boxes if use_boxes else None)
        w.tr.close(); gba.close()
        ate[use_boxes] = got["ate_m"]
        if use_boxes:
            assert (got["n_margin_old"], got["n_margin_second_new"]) == (want["n_margin_old"], want["n_margin_second_new"])
            assert got["iterations"] == want["iterations"]
            d = np.linalg.norm(got["P_est"] - want["P_est"], axis=1)
            assert d.max() < 1e-4, d.max()
            assert abs(got["ate_m"] - want["ate_m"]) < 1e-4
            assert all(c == 0 for k, c in enumerate(w.inside) if k % 5 != 4)
        else:
            assert sum(w.inside) > 100, w.inside
    with capsys.disabled():
        print("\nreplay on the dynamic scene, %d frames: ATE %.3f mm with boxes, %.3f mm without" % (n, 1e3 * ate[True], 1e3 * ate[False]))
