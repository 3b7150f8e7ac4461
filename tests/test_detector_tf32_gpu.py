"""The detector's TF32 mode on the GPU (include/gf_b200.h GF_DETECTOR_TF32).

- Dyadic operands: every convolution shape of the six shipped networks at 160 and 416 and edge shapes give the exact mode's bits
  (any order of summation is exact there), and a float64 reference's bits without bias, batch norm or leaky.
- Operand rounding: with K = 1 every output is float32(rna(w) rna(x)), exact in FP32; truncation or ties-to-even fail.
- Real-valued data: every convolution of a TF32 forward of each network stays within the error bound of DESIGN.md against a
  float64 restatement with TF32-rounded operands, fed the GPU's own input to the layer.
- Agreement with the exact mode's boxes, determinism, host / device frames, switching exact -> TF32 -> exact on one handle, and
  the libgf_b200.so forwarders.
"""
import ctypes

import numpy as np
import pytest

from tf32_ref import check_dyadic_operands, conv_shapes, detect_from_heads, heads_oracle_available, layer_bound_check, rna_tf32
from yolo_ref import CFGS, cfg_at, oracle_available, write_weights

pytestmark = pytest.mark.gpu


def synth_bgr(k=0):
    from ground_fusion_b200.synth import SyntheticStream
    return np.ascontiguousarray(SyntheticStream(seed=0).color(k)[..., ::-1])


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("yolo_tf32")
    cache = {}

    def get(name, size=160):
        if (name, size) not in cache:
            cfg = cfg_at(name, str(d), size, size)
            cache[name, size] = (cfg, write_weights(cfg, str(d / ("%s_%d.weights" % (name, size))), seed=1))
        return cache[name, size]
    return get


def _shapes():
    import tempfile
    from yolo_ref import cfg_path
    seen = set()
    with tempfile.TemporaryDirectory() as d:
        for name in CFGS:
            for size in (160, 416):
                seen.update(conv_shapes(cfg_at(name, d, size, size) if size != 416 else cfg_path(name)))
    # edges: M, N, K off every tile multiple, stride 2, 1x1 and 3x3, pad 0 and 1, N below one tile, K below one k-step
    seen.update({(3, 7, 5, 5, 3, 1, 1), (1, 1, 1, 1, 1, 1, 0), (5, 9, 11, 67, 3, 2, 1), (13, 10, 10, 129, 1, 1, 0),
                 (7, 12, 9, 65, 3, 2, 0), (33, 17, 19, 131, 3, 1, 1), (2, 30, 31, 200, 3, 1, 0), (70, 5, 6, 63, 1, 2, 0),
                 (9, 40, 40, 127, 3, 1, 1), (257, 3, 3, 3, 3, 1, 1)})
    return sorted(seen)


SHAPES = _shapes()


@pytest.mark.parametrize("shape", SHAPES, ids=["C%d_H%d_W%d_M%d_s%d_st%d_p%d" % s for s in SHAPES])
def test_dyadic_operands_give_the_exact_modes_bits(shape):
    check_dyadic_operands(shape)


def test_operands_are_rounded_to_nearest_ties_away():
    """K = 1: out[m][p] = rna(w[m]) rna(x[p]), a product of two 11-bit significands and so exact in FP32.  The data carries
    low mantissa bits everywhere and exact ties at the TF32 rounding point, on both even and odd kept LSBs."""
    from ground_fusion_b200.detector import conv_stage
    rng = np.random.default_rng(5)

    def values(n):
        v = rng.standard_normal(n).astype(np.float32) * np.float32(4.0)
        u = v.view(np.uint32).copy()
        u[: n // 3] = (u[: n // 3] & ~np.uint32(0x1FFF)) | np.uint32(0x1000)             # exact ties
        u[n // 3: n // 3 + 8] = (u[n // 3: n // 3 + 8] & ~np.uint32(0x3FFF)) | np.uint32(0x1000)   # ties, even kept LSB
        u[n // 3 + 8: n // 3 + 16] = (u[n // 3 + 8: n // 3 + 16] & ~np.uint32(0x3FFF)) | np.uint32(0x3000)  # ties, odd LSB
        u[n // 3 + 16: n // 3 + 24] |= np.uint32(0x7FF000)                                 # rounds up into the exponent
        return u.view(np.float32)
    for H, W, M in ((1, 1, 1), (37, 41, 131), (64, 64, 256), (13, 13, 425)):
        x = values(H * W).reshape(1, H, W)
        w = values(M).reshape(M, 1, 1, 1)
        got = conv_stage(x, w, np.zeros(M, np.float32), precision="tf32")
        want = (rna_tf32(w.reshape(M, 1)).astype(np.float64) * rna_tf32(x.reshape(1, -1)).astype(np.float64)).astype(np.float32)
        assert np.array_equal(got.reshape(M, -1).view(np.uint32), want.view(np.uint32))
        trunc = (w.reshape(M, 1).view(np.uint32) & ~np.uint32(0x1FFF)).view(np.float32).astype(np.float64) * \
            (x.reshape(1, -1).view(np.uint32) & ~np.uint32(0x1FFF)).view(np.float32).astype(np.float64)
        if M * H * W > 1:
            assert not np.array_equal(got.reshape(M, -1), trunc.astype(np.float32))


@pytest.mark.parametrize("name", CFGS)
def test_every_convolution_within_the_error_bound_at_160(name, files):
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files(name)
    det = YoloDetector(cfg, w, thresh=0.3, precision="tf32")
    try:
        det.detect(synth_bgr(0))
        worst = layer_bound_check(det, cfg, w)
    finally:
        det.close()
    print("%s at 160: largest error / bound %.4f" % (name, worst))


def test_yolov3_at_416_within_the_error_bound(files):
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov3", 416)
    det = YoloDetector(cfg, w, thresh=0.3, precision="tf32")
    try:
        det.detect(synth_bgr(3))
        worst = layer_bound_check(det, cfg, w)
    finally:
        det.close()
    print("yolov3 at 416: largest error / bound %.4f" % worst)


@pytest.mark.skipif(not (oracle_available() and heads_oracle_available()), reason="darknet oracle not built")
@pytest.mark.parametrize("name", ["yolov2-tiny", "yolov2", "yolov3"])
def test_decoding_of_the_tf32_heads_matches_darknet(name, files):
    """The boxes, classes and probabilities the TF32 mode publishes are darknet's decoding, NMS and darknet_ros's extraction
    applied to the TF32 mode's own [region] / [yolo] outputs, bit for bit."""
    from ground_fusion_b200.detector import YoloDetector
    from yolo_ref import Darknet, extract
    cfg, w = files(name)
    ref = Darknet(cfg, w)
    try:
        heads = [k for k, L in enumerate(ref.layers) if L["type"] in ("region", "yolo")]
        for thresh in (0.3, 0.7):
            det = YoloDetector(cfg, w, thresh=thresh, precision="tf32")
            try:
                for k in (0, 2):
                    bgr = synth_bgr(k)
                    got = det.detect(bgr)
                    bbox, _, prob = detect_from_heads(ref, {i: det.layer_output(i) for i in heads}, bgr.shape[1], bgr.shape[0], thresh)
                    b, c, p = extract(bbox, prob, bgr.shape[1], bgr.shape[0])
                    want = (np.array(b, np.int64).reshape(-1, 4), np.array(c, np.int32), np.array(p, np.float32))
                    for g, w_ in zip(got, want):
                        assert g.dtype == w_.dtype and np.array_equal(g, w_), (name, thresh, k)
            finally:
                det.close()
    finally:
        ref.close()


def _boxes_match(a, b, thresh, margin=0.02, iou_min=0.98):
    """Every box of a whose prob exceeds thresh by margin has a box of b of the same class with IoU >= iou_min, or with
    every corner within one pixel.  darknet_ros publishes corners truncated to whole pixels, so a difference far below a
    pixel (the heads differ by about 1e-6 relative, per the layer bound) can still move an edge by one: for a box 30 pixels
    wide that alone takes IoU to 0.967, which the first run met on yolov3-voc (0.962, two edges)."""
    (ba, ca, pa), (bb, cb, _) = a, b
    for box, c, p in zip(ba, ca, pa):
        if p < thresh + margin:
            continue
        best = 0.0
        for box2, c2 in zip(bb, cb):
            if c2 != c:
                continue
            ix = max(0, min(box[2], box2[2]) - max(box[0], box2[0]))
            iy = max(0, min(box[3], box2[3]) - max(box[1], box2[1]))
            inter = ix * iy
            uni = (box[2] - box[0]) * (box[3] - box[1]) + (box2[2] - box2[0]) * (box2[3] - box2[1]) - inter
            iou = inter / uni if uni > 0 else 0.0
            best = max(best, 1.0 if np.abs(np.asarray(box) - np.asarray(box2)).max() <= 1 else iou)
        assert best >= iou_min, (box, c, p, best)


@pytest.mark.parametrize("name", CFGS)
def test_boxes_agree_with_the_exact_mode(name, files):
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files(name)
    for thresh in (0.3, 0.7):
        ex = YoloDetector(cfg, w, thresh=thresh)
        tf = YoloDetector(cfg, w, thresh=thresh, precision="tf32")
        try:
            for k in (0, 4):
                a, b = ex.detect(synth_bgr(k)), tf.detect(synth_bgr(k))
                _boxes_match(a, b, thresh)
                _boxes_match(b, a, thresh)
        finally:
            ex.close()
            tf.close()


def test_determinism_device_frames_and_mode_switching(files):
    import torch
    from ground_fusion_b200.detector import YoloDetector
    cfg, w = files("yolov3")
    bgr = synth_bgr(1)
    fresh = YoloDetector(cfg, w, thresh=0.3)
    det = YoloDetector(cfg, w, thresh=0.3)
    try:
        want = fresh.detect(bgr)
        exact_layers = [fresh.layer_output(k) for k in range(fresh.n_layers)]
        det.detect(bgr)
        assert det.precision == "exact"
        det.set_precision("tf32")
        assert det.precision == "tf32"
        first = det.detect(bgr)
        l1 = [det.layer_output(k) for k in range(det.n_layers)]
        second = det.detect(torch.from_numpy(bgr).cuda())
        l2 = [det.layer_output(k) for k in range(det.n_layers)]
        for a, b in zip(first, second):
            assert np.array_equal(a, b)
        for a, b in zip(l1, l2):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        assert any(not np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(l1, exact_layers))
        assert det.last_device_ms() > 0
        assert np.all(det.layer_times(2) >= 0)
        det.set_precision("exact")
        again = det.detect(bgr)
        for a, b in zip(again, want):
            assert np.array_equal(a, b)
        for k in range(det.n_layers):
            assert np.array_equal(det.layer_output(k).view(np.uint32), exact_layers[k].view(np.uint32))
        with pytest.raises(ValueError):
            det.set_precision("fp16")
    finally:
        fresh.close()
        det.close()


def test_libgf_b200_forwards_the_precision_and_conv_stage(files):
    from ground_fusion_b200 import _lib
    from ground_fusion_b200.detector import YoloDetector, conv_stage
    cfg, w = files("yolov2-tiny")
    bgr = synth_bgr(0)
    det = YoloDetector(cfg, w, thresh=0.3, precision="tf32")
    try:
        want = det.detect(bgr)
    finally:
        det.close()
    L = _lib.lib()
    vp = ctypes.c_void_p
    L.gf_detector_create.argtypes = [ctypes.POINTER(vp), ctypes.c_int, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_float]
    L.gf_detector_detect.argtypes = [vp, vp, ctypes.c_size_t] + [ctypes.c_int] * 3 + [vp] * 3 + [ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    L.gf_detector_destroy.argtypes = [vp]
    L.gf_detector_destroy.restype = None
    L.gf_detector_set_precision.argtypes = [vp, ctypes.c_int]
    L.gf_detector_get_precision.argtypes = [vp, ctypes.POINTER(ctypes.c_int)]
    L.gf_stage_yolo_conv.argtypes = [ctypes.c_int, ctypes.c_int] + [vp] * 8
    h = vp()
    _lib.check(L.gf_detector_create(ctypes.byref(h), 0, cfg.encode(), w.encode(), ctypes.c_float(0.3)))
    boxes, cls, prob, n, p = np.zeros((100, 4), np.int64), np.zeros(100, np.int32), np.zeros(100, np.float32), ctypes.c_int(), ctypes.c_int()
    try:
        assert L.gf_detector_set_precision(h, 7) != 0
        _lib.check(L.gf_detector_set_precision(h, 1))
        _lib.check(L.gf_detector_get_precision(h, ctypes.byref(p)))
        assert p.value == 1
        _lib.check(L.gf_detector_detect(h, bgr.ctypes.data, bgr.strides[0], bgr.shape[1], bgr.shape[0], 0, boxes.ctypes.data,
                                        cls.ctypes.data, prob.ctypes.data, 100, ctypes.byref(n)))
    finally:
        L.gf_detector_destroy(h)
    m = n.value
    assert m == len(want[0]) > 0
    assert np.array_equal(boxes[:m], want[0]) and np.array_equal(cls[:m], want[1]) and np.array_equal(prob[:m], want[2])
    rng = np.random.default_rng(2)
    x, wt, b = rng.standard_normal((3, 9, 8)).astype(np.float32), rng.standard_normal((5, 3, 3, 3)).astype(np.float32), np.zeros(5, np.float32)
    shape = (ctypes.c_int * 9)(3, 9, 8, 5, 3, 1, 1, 0, 1)
    out = np.empty((5, 9, 8), np.float32)
    _lib.check(L.gf_stage_yolo_conv(0, 1, shape, x.ctypes.data, wt.ctypes.data, b.ctypes.data, None, None, None, out.ctypes.data))
    assert np.array_equal(out, conv_stage(x, wt, b, 1, 1, leaky=True, precision="tf32"))


def test_adaptor_set_precision_gives_the_python_detectors_boxes(files, tmp_path):
    """YoloObjectDetector::setPrecision (adaptor/yolo_check drives it on one raw frame) publishes, in either precision, the
    boxes, class ids and probabilities of YoloDetector in that precision."""
    import os
    import subprocess
    from ground_fusion_b200.detector import YoloDetector
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-s", "-C", os.path.join(root, "adaptor")])
    cfg, w = files("yolov3")
    bgr = synth_bgr(0)
    frame = tmp_path / "frame.bgr"
    frame.write_bytes(bgr.tobytes())
    for precision, code in (("tf32", 1), ("exact", 0)):
        det = YoloDetector(cfg, w, thresh=0.3, precision=precision)
        try:
            boxes, cls, prob = det.detect(bgr)
        finally:
            det.close()
        out = subprocess.check_output([os.path.join(root, "adaptor", "_build", "yolo_check"), cfg, w, "0.3", str(code), str(frame),
                                       str(bgr.shape[1]), str(bgr.shape[0])], text=True)
        rows = [ln.split() for ln in out.splitlines()]
        assert len(rows) == len(boxes) > 0, precision
        for r, b, c, p in zip(rows, boxes, cls, prob):
            assert int(r[0]) == c and np.float32(float(r[1])) == p and [int(v) for v in r[2:]] == list(b), precision
