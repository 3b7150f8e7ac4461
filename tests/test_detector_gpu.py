"""The YOLO detector on the GPU against darknet's CPU build (tests/yolo_ref.py), bit for bit: the letterboxed input, every layer's
output and the boxes, class ids and probabilities darknet_ros would publish, for the six networks the reference ships, at a
reduced [net] size and at 416, on synthetic and random frames of several sizes, at two thresholds; plus the >100-boxes rule,
ties in objectness, device frames, and the replay loop with the detector in it."""
import numpy as np
import pytest

from yolo_ref import CFGS, Darknet, cfg_at, oracle_available, raw_roi_count, write_weights

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not oracle_available(), reason="darknet oracle not built (oracle/darknet.mk needs darknet's sources)")]


def synth_bgr(k=0):
    from ground_fusion_b200.synth import SyntheticStream
    return np.ascontiguousarray(SyntheticStream(seed=0).color(k)[..., ::-1])


def random_bgr(seed, w, h):
    """Smooth random colour noise (so that objectness varies over the frame) plus pixel noise."""
    import cv2
    rng = np.random.default_rng(seed)
    a = cv2.resize(rng.uniform(0, 255, (h // 16 + 2, w // 16 + 2, 3)).astype(np.float32), (w, h), interpolation=cv2.INTER_CUBIC)
    a = a + rng.normal(0, 12, a.shape)
    return np.clip(a, 0, 255).astype(np.uint8)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("yolo")
    cache = {}

    def get(name, size=160, **kw):
        key = (name, size, tuple(sorted(kw.items())))
        if key not in cache:
            cfg = cfg_at(name, str(d), size, size)
            tag = "_".join("%s%s" % kv for kv in sorted(kw.items()))
            cache[key] = (cfg, write_weights(cfg, str(d / ("%s_%d_%s.weights" % (name, size, tag))), seed=1, **kw))
        return cache[key]
    return get


def check_detector(cfg, weights, frames, thresholds=(0.3, 0.7), layers=True):
    """For each frame: the GPU's letterboxed input, (optionally) every layer's output, and the published boxes at each threshold
    equal darknet's.  Returns the box counts."""
    from ground_fusion_b200.detector import YoloDetector
    ref = Darknet(cfg, weights)
    dets = {t: YoloDetector(cfg, weights, thresh=t) for t in thresholds}
    counts = []
    try:
        for bgr in frames:
            x = ref.forward(bgr)
            for t in thresholds:
                got = dets[t].detect(bgr)
                bbox, _, prob = ref.detections(bgr.shape[1], bgr.shape[0], t)
                from yolo_ref import extract
                b, c, p = extract(bbox, prob, bgr.shape[1], bgr.shape[0])
                want = (np.array(b, np.int64).reshape(-1, 4), np.array(c, np.int32), np.array(p, np.float32))
                for g, w_, what in zip(got, want, ("boxes", "class ids", "probabilities")):
                    assert g.dtype == w_.dtype and np.array_equal(g, w_), "%s differ at thresh %.1f" % (what, t)
                counts.append((t, len(got[0]), raw_roi_count(bbox, prob)))
            det = dets[thresholds[0]]
            assert np.array_equal(det.input_image().view(np.uint32), x.view(np.uint32)), "letterboxed input differs"
            if layers:
                for k in range(ref.n):
                    g, w_ = det.layer_output(k), ref.layer_output(k)
                    assert g.shape == w_.shape
                    bad = np.flatnonzero(g.view(np.uint32) != w_.view(np.uint32))
                    assert bad.size == 0, "layer %d (%s): %d of %d values differ, first at %d: %r vs %r" % (
                        k, ref.layers[k]["type"], bad.size, g.size, bad[0], g.flat[bad[0]], w_.flat[bad[0]])
            else:
                k = ref.n - 1
                assert np.array_equal(det.layer_output(k).view(np.uint32), ref.layer_output(k).view(np.uint32))
    finally:
        for d in dets.values():
            d.close()
        ref.close()
    return counts


@pytest.mark.parametrize("name", CFGS)
def test_every_layer_and_the_boxes_match_darknet_at_160(name, files):
    counts = check_detector(*files(name), [synth_bgr(0)])
    if name in ("yolov2-tiny", "yolov3"):
        assert any(n > 1 for _, n, _ in counts), counts          # the data exercises NMS and extraction


@pytest.mark.parametrize("name", CFGS)
def test_every_layer_and_the_boxes_match_darknet_at_416(name, files):
    check_detector(*files(name, 416), [synth_bgr(2)], thresholds=(0.3,))


@pytest.mark.parametrize("name", ["yolov2-tiny", "yolov3"])
def test_frame_sizes_and_random_frames(name, files):
    """640x480, 1280x720 and portrait 480x640 (vertical letterbox padding) random frames, a 641x481 synthetic-sized crop and a
    1x1 frame."""
    frames = [random_bgr(1, 640, 480), random_bgr(2, 1280, 720), random_bgr(3, 480, 640),
              np.ascontiguousarray(np.pad(synth_bgr(5), ((0, 1), (0, 1), (0, 0)), mode="edge")), random_bgr(4, 16, 16)[:1, :1].copy()]
    check_detector(*files(name), frames, layers=False)


def test_letterbox_stage_matches_darknet(files):
    from ground_fusion_b200.detector import letterbox
    cfg, w = files("yolov2-tiny")
    ref = Darknet(cfg, w)
    try:
        for (fw, fh) in ((640, 480), (1280, 720), (480, 640), (641, 481), (160, 160), (100, 37), (2, 3)):
            bgr = random_bgr(fw * 7 + fh, fw + 16, fh + 16)[:fh, :fw]       # a view with padded rows
            for nw, nh in ((160, 160), (416, 416), (320, 192)):
                ref_net = ref if (nw, nh) == (160, 160) else None
                got = letterbox(bgr, nw, nh)
                if ref_net is not None:
                    assert np.array_equal(got.view(np.uint32), ref.letterbox(bgr).view(np.uint32)), (fw, fh)
                else:
                    assert got.shape == (3, nh, nw) and np.all(np.isfinite(got))
    finally:
        ref.close()


def test_more_than_100_boxes_publish_none(files):
    """Small boxes on every cell: the node's extraction collects more than 100 and publishes nothing."""
    cfg, w = files("yolov2-tiny", 416, obj_bias=6.0, tw_bias=-1.0)
    counts = check_detector(cfg, w, [synth_bgr(1)], thresholds=(0.3,), layers=False)
    assert counts[0][1] == 0 and counts[0][2] > 100, counts


def test_ties_in_objectness(files):
    """Zero head weights: every cell of an anchor has the same objectness and box size, so do_nms_obj's sort is full of ties
    and which box survives rests on qsort's order, as in darknet."""
    cfg, w = files("yolov2-tiny", obj_bias=2.0, tw_bias=0.5, tie=True)
    ref = Darknet(cfg, w)
    try:
        ref.forward(synth_bgr(0))
        _, obj, _ = ref.detections(640, 480, 0.3)
        nz = obj[obj > 0]
        assert len(nz) > len(np.unique(nz))
    finally:
        ref.close()
    counts = check_detector(cfg, w, [synth_bgr(0)], thresholds=(0.3, 0.7), layers=False)
    assert any(n > 0 for _, n, _ in counts), counts


def test_device_frames_match_host_frames(files):
    import torch
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov3")
    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        for bgr in (synth_bgr(0), random_bgr(9, 1280, 720)):
            host = det.detect(bgr)
            x_host = det.input_image()
            dev = det.detect(torch.from_numpy(bgr).cuda())
            for a, b in zip(host, dev):
                assert np.array_equal(a, b)
            assert np.array_equal(det.input_image(), x_host)
            assert det.last_device_ms() > 0
    finally:
        det.close()


def test_replay_with_detector_matches_replay_with_oracle_boxes(files):
    """replay(..., detector=) equals replay(..., boxes=) fed darknet's boxes for the same frames: same trajectory, and the same
    in-box masks frame by frame."""
    from test_fm_gpu import _gpu_fm
    from ground_fusion_b200.detector import YoloDetector
    from ground_fusion_b200.estimator import BundleAdjuster
    from ground_fusion_b200.feature_tracker import FeatureTracker
    from ground_fusion_b200.replay import replay
    from ground_fusion_b200.synth import IDC_CAM, SyntheticStream
    cam = dict(IDC_CAM, k1=0.0, k2=0.0, p1=0.0, p2=0.0)
    p8 = [cam[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")]
    n = 24
    cfg, w = files("yolov2-tiny")
    st = SyntheticStream(seed=0)
    ref = Darknet(cfg, w)
    try:
        oracle_boxes = [ref.detect(np.ascontiguousarray(st.color(k)[..., ::-1]), 0.3)[0] for k in range(n)]
    finally:
        ref.close()
    assert sum(len(b) > 0 for b in oracle_boxes) >= n // 2

    class Watch:
        def __init__(self, tr):
            self.tr, self.masks = tr, []

        def trackImage(self, t, g, d):
            self.masks.append(None)
            return self.tr.trackImage(t, g, d)

        def trackImagebox(self, t, b, g, d):
            obs, in_box = self.tr.trackImageboxRaw(t, b, g, d)
            self.masks.append((np.asarray(b).copy(), obs["id"].copy(), in_box.copy()))
            return {int(o["id"]): o["v"].copy() for o, inside in zip(obs, in_box) if not inside}

    runs = []
    for use_detector in (True, False):
        tr = Watch(FeatureTracker(640, 480, p8, 150, 30, 1, 1, device=0))
        ba = BundleAdjuster(0)
        det = YoloDetector(cfg, w, thresh=0.3) if use_detector else None
        try:
            out = replay(SyntheticStream(seed=0), tr, _gpu_fm(depth_threshold=4.0), ba, n,
                         detector=det, boxes=None if use_detector else oracle_boxes)
        finally:
            tr.tr.close()
            ba.close()
            if det is not None:
                det.close()
        runs.append((out, tr.masks))
    (a, ma), (b, mb) = runs
    assert np.array_equal(np.asarray(a["P_est"]), np.asarray(b["P_est"]))
    assert np.array_equal(np.asarray(a["R_est"]), np.asarray(b["R_est"]))
    assert len(ma) == len(mb) == n
    for x, y in zip(ma, mb):
        assert (x is None) == (y is None)
        if x is not None:
            for u, v in zip(x, y):
                assert np.array_equal(u, v)
    assert any(x is not None and x[2].any() for x in ma)           # some features did fall inside a detection


def test_libgf_b200_entry_points_forward_to_the_detector(files):
    """The gf_detector_* entry points libgf_b200.so exports open libgf_yolo.so and give the same boxes as calling it directly."""
    import ctypes
    from ground_fusion_b200 import _lib
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov2-tiny")
    bgr = synth_bgr(0)
    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        want = det.detect(bgr)
    finally:
        det.close()
    L = _lib.lib()
    L.gf_detector_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_float]
    L.gf_detector_detect.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 3 + [
        ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    L.gf_detector_destroy.argtypes = [ctypes.c_void_p]
    L.gf_detector_destroy.restype = None
    h = ctypes.c_void_p()
    _lib.check(L.gf_detector_create(ctypes.byref(h), 0, cfg.encode(), w.encode(), ctypes.c_float(0.3)))
    boxes, cls, prob, n = np.zeros((100, 4), np.int64), np.zeros(100, np.int32), np.zeros(100, np.float32), ctypes.c_int()
    try:
        _lib.check(L.gf_detector_detect(h, bgr.ctypes.data, bgr.strides[0], bgr.shape[1], bgr.shape[0], 0, boxes.ctypes.data,
                                        cls.ctypes.data, prob.ctypes.data, 100, ctypes.byref(n)))
    finally:
        L.gf_detector_destroy(h)
    m = n.value
    assert m == len(want[0]) > 0
    assert np.array_equal(boxes[:m], want[0]) and np.array_equal(cls[:m], want[1]) and np.array_equal(prob[:m], want[2])
