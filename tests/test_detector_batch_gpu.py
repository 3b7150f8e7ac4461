"""gf_detector_detect_batch on the GPU: every frame of a batch gives, bit for bit, what gf_detector_detect gives for that frame
alone (letterboxed input, every layer's output, boxes, class ids, probabilities) in both precisions, for the six networks the
reference ships, at any position in a batch of any size; the handle's state across batch sizes, precisions and capacities;
and the multi-camera loop (replay_group) with the detector in it."""
import ctypes

import numpy as np
import pytest

from test_detector_gpu import files, random_bgr, synth_bgr  # noqa: F401  (files is a fixture)
from yolo_ref import CFGS, Darknet, extract, oracle_available

pytestmark = pytest.mark.gpu

PRECISIONS = ("exact", "tf32")
GF_ERR_CAPACITY = -4


def mixed_frames(n):
    """Distinct frames of different sizes: synthetic 640x480, random 1280x720, portrait 480x640, 1x1, then more synthetic ones."""
    base = [synth_bgr(0), random_bgr(2, 1280, 720), random_bgr(3, 480, 640), random_bgr(4, 16, 16)[:1, :1].copy()]
    return [base[i] if i < len(base) else synth_bgr(i) for i in range(n)]


def assert_bits(a, b, what):
    assert a.shape == b.shape, what
    bad = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
    assert bad.size == 0, "%s: %d of %d values differ, first at %d: %r vs %r" % (what, bad.size, a.size, bad[0], a.flat[bad[0]],
                                                                                b.flat[bad[0]])


def assert_same_result(got, want, what):
    for g, w, name in zip(got, want, ("boxes", "class ids", "probabilities")):
        assert g.dtype == w.dtype and np.array_equal(g, w), "%s: %s differ" % (what, name)


def check_batch_against_single(cfg, weights, frames, precision, layers=True):
    """One detect_batch over `frames` on one handle against detect on each frame alone on another."""
    from ground_fusion_b200.detector import YoloDetector
    bat = YoloDetector(cfg, weights, thresh=0.3, precision=precision)
    one = YoloDetector(cfg, weights, thresh=0.3, precision=precision)
    try:
        bat.set_max_batch(len(frames))
        got = bat.detect_batch(frames)
        boxes, start = bat.detect_batch_csr(frames)
        assert len(got) == len(frames) and len(start) == len(frames) + 1
        total = 0
        for i, bgr in enumerate(frames):
            want = one.detect(bgr)
            total += len(want[0])
            assert_same_result(got[i], want, "frame %d" % i)
            assert np.array_equal(boxes[start[i]:start[i + 1]], want[0])
            for k in range(-1, one.n_layers if layers else 0):
                assert_bits(bat.member_layer_output(i, k), one.layer_output(k), "frame %d layer %d" % (i, k))
        assert_bits(bat.layer_output(one.n_layers - 1), bat.member_layer_output(0, one.n_layers - 1), "layer_output = member 0")
        return total
    finally:
        bat.close()
        one.close()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", CFGS)
def test_every_member_equals_single_detect_at_160(name, precision, files):
    total = 0
    for n in (1, 2, 5):
        total += check_batch_against_single(*files(name), mixed_frames(n), precision)
    if name in ("yolov2-tiny", "yolov3"):
        assert total > 0


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", ["yolov2-tiny", "yolov3"])
def test_every_member_equals_single_detect_at_416(name, precision, files):
    check_batch_against_single(*files(name, 416), mixed_frames(8), precision)


@pytest.mark.skipif(not oracle_available(), reason="darknet oracle not built (oracle/darknet.mk needs darknet's sources)")
def test_exact_batch_matches_darknet(files):
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov3")
    frames = mixed_frames(4)
    det = YoloDetector(cfg, w, thresh=0.3)
    ref = Darknet(cfg, w)
    try:
        det.set_max_batch(4)
        got = det.detect_batch(frames)
        for i, bgr in enumerate(frames):
            x = ref.forward(bgr)
            bbox, _, prob = ref.detections(bgr.shape[1], bgr.shape[0], 0.3)
            b, c, p = extract(bbox, prob, bgr.shape[1], bgr.shape[0])
            assert_same_result(got[i], (np.array(b, np.int64).reshape(-1, 4), np.array(c, np.int32), np.array(p, np.float32)),
                               "frame %d" % i)
            assert_bits(det.member_layer_output(i, -1), x, "frame %d input" % i)
            for k in range(ref.n):
                assert_bits(det.member_layer_output(i, k), ref.layer_output(k), "frame %d layer %d" % (i, k))
    finally:
        det.close()
        ref.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_a_frame_has_the_same_bits_at_any_position_and_batch_size(precision, files):
    """yolov3 at 416 (its 13 x 13 and 26 x 26 layers split K in TF32): one frame at positions 0 and 7 of a batch of 8, alone, and
    last in a batch of 16."""
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov3", 416)
    x = synth_bgr(3)
    others = mixed_frames(16)[1:]
    det = YoloDetector(cfg, w, thresh=0.3, precision=precision)
    try:
        det.set_max_batch(16)
        runs = []
        for frames, pos in (([x] + others[:6] + [x], 0), ([x] + others[:6] + [x], 7), ([x], 0), (others[:15] + [x], 15)):
            if len(runs) != 1:                       # positions 0 and 7 come from the same call
                res = det.detect_batch(frames)
            runs.append((res[pos], [det.member_layer_output(pos, k) for k in range(-1, det.n_layers)]))
        (r0, l0) = runs[0]
        for r, ls in runs[1:]:
            assert_same_result(r, r0, precision)
            for k, (a, b) in enumerate(zip(ls, l0)):
                assert_bits(a, b, "layer %d" % (k - 1))
    finally:
        det.close()


def _c_batch(det, frames, cap, box_start, boxes, cls=None, prob=None):
    n = len(frames)
    vp = ctypes.c_void_p
    return det._L.gf_detector_detect_batch(det._h, n, (vp * n)(*[f.ctypes.data for f in frames]),
                                           (ctypes.c_size_t * n)(*[f.strides[0] for f in frames]),
                                           (ctypes.c_int * n)(*[f.shape[1] for f in frames]),
                                           (ctypes.c_int * n)(*[f.shape[0] for f in frames]), 0,
                                           boxes.ctypes.data if boxes is not None else None,
                                           cls.ctypes.data if cls is not None else None, prob.ctypes.data if prob is not None else None,
                                           cap, box_start.ctypes.data)


def test_capacity_errors_change_nothing(files):
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov3")
    frames = mixed_frames(3)
    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        det.set_max_batch(3)
        want = det.detect_batch(frames)
        counts = [len(r[0]) for r in want]
        assert sum(counts) > 1
        last = [det.member_layer_output(i, det.n_layers - 1) for i in range(3)]
        # more frames than max_batch
        start = np.full(5, -7, np.int32)
        boxes = np.zeros((400, 4), np.int64)
        assert _c_batch(det, frames + [frames[0]], 400, start, boxes) == GF_ERR_CAPACITY
        assert (start == -7).all() and not boxes.any()
        for i in range(3):
            assert_bits(det.member_layer_output(i, det.n_layers - 1), last[i], "after the refused call")
        # too small a cap: box_start filled, nothing written at or past cap
        cap = sum(counts) - 1
        start = np.zeros(4, np.int32)
        boxes, cls, prob = np.full((cap + 8, 4), -1, np.int64), np.full(cap + 8, -1, np.int32), np.full(cap + 8, -1, np.float32)
        assert _c_batch(det, frames, cap, start, boxes, cls, prob) == GF_ERR_CAPACITY
        assert list(np.diff(start)) == counts and start[0] == 0
        assert (boxes[cap:] == -1).all() and (cls[cap:] == -1).all() and (prob[cap:] == -1).all()
        flat = np.concatenate([r[0] for r in want])
        assert np.array_equal(boxes[:cap], flat[:cap])
        # and the handle still gives the same results
        for g, r in zip(det.detect_batch(frames), want):
            assert_same_result(g, r, "after the capacity errors")
    finally:
        det.close()


@pytest.mark.skipif(not oracle_available(), reason="darknet oracle not built (oracle/darknet.mk needs darknet's sources)")
def test_more_than_100_boxes_give_an_empty_range(files):
    """Weights that put small boxes on every cell: darknet's extraction collects more than 100 on each frame (checked against the
    oracle frame by frame), so each frame's range is empty, as detect publishes nothing for it."""
    from yolo_ref import raw_roi_count
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov2-tiny", 416, obj_bias=6.0, tw_bias=-1.0)
    frames = [synth_bgr(1), synth_bgr(2), random_bgr(5, 640, 480)]
    ref = Darknet(cfg, w)
    try:
        for f in frames:
            ref.forward(f)
            bbox, _, prob = ref.detections(f.shape[1], f.shape[0], 0.3)
            assert raw_roi_count(bbox, prob) > 100
    finally:
        ref.close()
    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        det.set_max_batch(3)
        singles = [det.detect(f) for f in frames]
        got = det.detect_batch(frames)
        _, start = det.detect_batch_csr(frames)
        assert all(len(s[0]) == 0 for s in singles) and list(start) == [0, 0, 0, 0]
        for g, s in zip(got, singles):
            assert_same_result(g, s, "crowded frame")
    finally:
        det.close()


def test_host_and_device_frames_give_the_same_results(files):
    import torch
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov3")
    frames = mixed_frames(4)
    det = YoloDetector(cfg, w, thresh=0.3, precision="tf32")
    try:
        det.set_max_batch(4)
        host = det.detect_batch(frames)
        x_host = [det.member_layer_output(i, -1) for i in range(4)]
        dev = det.detect_batch([torch.from_numpy(f).cuda() for f in frames])
        for a, b in zip(host, dev):
            assert_same_result(a, b, "device frames")
        for i in range(4):
            assert_bits(det.member_layer_output(i, -1), x_host[i], "device frame %d input" % i)
        with pytest.raises(ValueError):
            det.detect_batch([frames[0], torch.from_numpy(frames[1]).cuda()])
        assert det.last_device_ms() > 0
        assert len(det.layer_times(2)) == det.n_layers
    finally:
        det.close()


def test_interleaved_calls_equal_a_fresh_handle(files):
    """detect, detect_batch at several n, set_precision and set_max_batch (shrinking and growing) on one handle give what a
    fresh handle gives for each call."""
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov3")
    frames = mixed_frames(6)

    def fresh(precision, fs):
        d = YoloDetector(cfg, w, thresh=0.3, precision=precision)
        try:
            d.set_max_batch(max(len(fs), 1))
            return d.detect_batch(fs), d.member_layer_output(len(fs) - 1, d.n_layers - 1)
        finally:
            d.close()

    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        steps = [("batch", 6, None), ("detect", 1, None), ("batch", 3, None), ("precision", 0, "tf32"), ("batch", 6, None),
                 ("max", 2, None), ("batch", 2, None), ("detect", 1, None), ("precision", 0, "exact"), ("batch", 2, None),
                 ("max", 8, None), ("batch", 5, None), ("precision", 0, "tf32"), ("batch", 5, None), ("max", 1, None),
                 ("detect", 1, None)]
        det.set_max_batch(6)
        for s, (op, n, arg) in enumerate(steps):
            if op == "precision":
                det.set_precision(arg)
                continue
            if op == "max":
                det.set_max_batch(n)
                with pytest.raises(GfError):
                    det.member_layer_output(0, 0)                        # the last call's outputs went with the buffers
                if n < 6:
                    with pytest.raises(GfError):
                        det.detect_batch(frames[:n + 1])
                continue
            fs = frames[s % 3:s % 3 + n]
            got = [det.detect(fs[0])] if op == "detect" else det.detect_batch(fs)
            want, last = fresh(det.precision, fs)
            for g, r in zip(got, want):
                assert_same_result(g, r, "step %d" % s)
            assert_bits(det.member_layer_output(len(fs) - 1, det.n_layers - 1), last, "step %d" % s)
        with pytest.raises(GfError):
            det.set_max_batch(0)
        with pytest.raises(GfError):
            det.set_max_batch(65)
        assert det.max_batch == 1
    finally:
        det.close()


def test_libgf_b200_forwards_the_batch_entry_points(files):
    from ground_fusion_b200 import _lib
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov2-tiny")
    frames = mixed_frames(3)
    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        det.set_max_batch(3)
        want = det.detect_batch(frames)
        x = det.member_layer_output(2, det.n_layers - 1)
    finally:
        det.close()
    L = _lib.lib()
    vp, i = ctypes.c_void_p, ctypes.c_int
    L.gf_detector_create.argtypes = [ctypes.POINTER(vp), i, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_float]
    L.gf_detector_set_max_batch.argtypes = [vp, i]
    L.gf_detector_detect_batch.argtypes = [vp, i, vp, vp, vp, vp, i, vp, vp, vp, i, vp]
    L.gf_detector_member_layer_output.argtypes = [vp, i, i, vp, ctypes.c_size_t]
    L.gf_detector_destroy.argtypes = [vp]
    L.gf_detector_destroy.restype = None
    h = vp()
    _lib.check(L.gf_detector_create(ctypes.byref(h), 0, cfg.encode(), w.encode(), ctypes.c_float(0.3)))

    class Shim:
        _L, _h = L, h
    try:
        _lib.check(L.gf_detector_set_max_batch(h, 3))
        start, boxes = np.zeros(4, np.int32), np.zeros((300, 4), np.int64)
        cls, prob = np.zeros(300, np.int32), np.zeros(300, np.float32)
        _lib.check(_c_batch(Shim, frames, 300, start, boxes, cls, prob))
        out = np.empty_like(x)
        _lib.check(L.gf_detector_member_layer_output(h, 2, _n_layers(cfg) - 1, out.ctypes.data, out.size))
    finally:
        L.gf_detector_destroy(h)
    for k, r in enumerate(want):
        a, b = start[k], start[k + 1]
        assert_same_result((boxes[a:b], cls[a:b], prob[a:b]), r, "forwarded frame %d" % k)
    assert_bits(out, x, "forwarded layer output")


def _n_layers(cfg):
    from ground_fusion_b200.detector import parse_cfg
    return len(parse_cfg(cfg)[1])


def _p8():
    from ground_fusion_b200.synth import IDC_CAM
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    return [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]


def _independent(seed, n, cfg, w):
    from ground_fusion_b200.detector import YoloDetector
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import SyntheticStream
    tr, fm, ba = FeatureTracker(640, 480, _p8(), 150, 30, 1, 1), FeatureWindow(depth_threshold=4.0), BundleAdjuster(0)
    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        return replay(SyntheticStream(seed=seed), tr, fm, ba, n, detector=det)
    finally:
        tr.close(); fm.close(); ba.close(); det.close()


def _group(seeds, n, **kw):
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.feature_window import FeatureWindow
    from ground_fusion_b200.replay import replay_group
    from ground_fusion_b200.synth import SyntheticStream
    K = len(seeds)
    trs = [FeatureTracker(640, 480, _p8(), 150, 30, 1, 1) for _ in range(K)]
    wins = [FeatureWindow(depth_threshold=4.0) for _ in range(K)]
    bas = [BundleAdjuster(0) for _ in range(K)]
    try:
        return replay_group([SyntheticStream(seed=s) for s in seeds], trs, wins, bas, n, **kw)
    finally:
        for x in trs + wins + bas:
            x.close()


def test_replay_group_with_detector_matches_independent_replays(files, capsys):
    """replay_group(..., detector=) over K = 3 streams (one detect_batch per step) against three independent
    replay(..., detector=) runs, in test_fm_group_gpu's form: the solve's atomics are not ordered, so the trajectory bar is three
    times the run-to-run difference (floor 1e-9 m, cap 1e-8 m).  replay_group(..., boxes=) with each stream's boxes from detect
    gives the same result."""
    from ground_fusion_b200.detector import YoloDetector
    from ground_fusion_b200.synth import SyntheticStream
    K, n = 3, 30
    seeds = list(range(K))
    cfg, w = files("yolov2-tiny")
    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        got = _group(seeds, n, detector=det)
        assert det.max_batch == K
        boxes = [[det.detect(np.ascontiguousarray(SyntheticStream(seed=s).color(k)[..., ::-1]))[0] for k in range(n)] for s in seeds]
    finally:
        det.close()
    assert sum(len(b) > 0 for bs in boxes for b in bs) >= K * n // 2
    got_boxes = _group(seeds, n, boxes=boxes)
    d_run = d_grp = 0.0
    for s, g, gb in zip(seeds, got, got_boxes):
        a, b, c = (_independent(s, n, cfg, w) for _ in range(3))
        for grp in (g, gb):
            for f, it in enumerate(grp["iterations"]):
                ref = {a["iterations"][f], b["iterations"][f], c["iterations"][f]}
                assert it in ref, (s, f, it, ref)
            assert (grp["n_margin_old"], grp["n_margin_second_new"]) == (a["n_margin_old"], a["n_margin_second_new"]), s
            assert len(grp["P_est"]) == len(a["P_est"]) > 0
            d_grp = max(d_grp, min(np.linalg.norm(grp["P_est"] - x["P_est"], axis=1).max() for x in (a, b, c)))
        d_run = max(d_run, max(np.linalg.norm(x["P_est"] - y["P_est"], axis=1).max() for x, y in ((a, b), (a, c), (b, c))))
    with capsys.disabled():
        print("\nreplay_group K=%d, %d frames, detector: group vs independent %.3e m, run to run %.3e m" % (K, n, d_grp, d_run))
    bar = min(max(3 * d_run, 1e-9), 1e-8)
    assert d_grp <= bar, (d_grp, d_run)
