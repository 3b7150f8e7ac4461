"""Host restatements for the detector's TF32 mode (tests only).

- rna_tf32(): cvt.rna.tf32.f32 on the uint32 view: round to the nearest value with 10 explicit mantissa bits, ties away from
  zero, the low 13 bits cleared.  Adding half an ulp (0x1000) to the magnitude bits and clearing the low 13 does exactly that,
  and a carry out of the mantissa moves into the exponent as it should.  Inf and NaN pass through.
- im2col(): darknet's im2col order, k = c size^2 + ky size + kx, for a float64 reference of a convolution.
- conv_shapes(): every convolution shape (C H W M size stride pad) of a cfg.
- detect_from_heads(): darknet's decoding and NMS of given [region] / [yolo] outputs (oracle/yolo_heads.c's
  yh_detect_from_heads, built into oracle/_ref/libyolo_heads.so).
- check_dyadic_operands(): one convolution shape on dyadic operands, where both modes must give float64's bits.
- layer_bound_check(): every convolution of a TF32 forward within DESIGN.md's error bound.
"""
import ctypes
import os

import numpy as np

HEADS_ORACLE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libyolo_heads.so")
U = 2.0 ** -24           # FP32 unit roundoff


def rna_tf32(x):
    x = np.asarray(x, np.float32)
    u = x.view(np.uint32)
    finite = (u & 0x7F800000) != 0x7F800000
    r = np.where(finite, ((u & 0x7FFFFFFF) + 0x1000) & 0x7FFFE000 | (u & 0x80000000), u).astype(np.uint32)
    return r.view(np.float32)


def im2col(x, size, stride, pad):
    """x (C, H, W) -> (C size^2, OH OW) in darknet's k order, zeros in the padding."""
    C, H, W = x.shape
    OH, OW = (H + 2 * pad - size) // stride + 1, (W + 2 * pad - size) // stride + 1
    xp = np.zeros((C, H + 2 * pad, W + 2 * pad), x.dtype)
    xp[:, pad:pad + H, pad:pad + W] = x
    cols = np.empty((C, size, size, OH, OW), x.dtype)
    for ky in range(size):
        for kx in range(size):
            cols[:, ky, kx] = xp[:, ky:ky + stride * (OH - 1) + 1:stride, kx:kx + stride * (OW - 1) + 1:stride]
    return cols.reshape(C * size * size, OH * OW), OH, OW


def conv_shapes(cfg):
    from ground_fusion_b200.detector import parse_cfg
    _, layers = parse_cfg(cfg)
    return [(L["c"], L["h"], L["w"], L["n"], L["size"], L["stride"], L["pad"]) for L in layers if L["type"] == "convolutional"]


def heads_oracle_available():
    return os.path.exists(HEADS_ORACLE)


def detect_from_heads(darknet, heads, frame_w, frame_h, thresh):
    """darknet (a yolo_ref.Darknet) with its head layers' outputs replaced by heads {layer index: array}: the detections
    after do_nms_obj as Darknet.detections returns them (bbox, objectness, probs)."""
    L = ctypes.CDLL(HEADS_ORACLE)
    vp = ctypes.c_void_p
    L.yh_detect_from_heads.argtypes = [vp, ctypes.c_int, vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_float, vp, vp, vp, ctypes.c_int]
    L.yh_detect_from_heads.restype = ctypes.c_int
    idx = np.array(sorted(heads), np.int32)
    arrs = [np.ascontiguousarray(heads[k], np.float32) for k in idx]
    ptrs = (vp * len(arrs))(*[a.ctypes.data for a in arrs])
    cap = 1 << 16
    bbox, obj = np.zeros((cap, 4), np.float32), np.zeros(cap, np.float32)
    prob = np.zeros((cap, darknet.classes), np.float32)
    n = L.yh_detect_from_heads(darknet._net, len(arrs), idx.ctypes.data, ptrs, frame_w, frame_h, ctypes.c_float(thresh),
                               bbox.ctypes.data, obj.ctypes.data, prob.ctypes.data, cap)
    assert 0 <= n <= cap
    return bbox[:n], obj[:n], prob[:n]


def _dyadic(rng, n):
    return (rng.integers(-8, 9, n) / 8.0).astype(np.float32)


def check_dyadic_operands(shape):
    """shape = (C, H, W, M, size, stride, pad).  Multiples of 1/8 in [-1, 1]: every product and partial sum is exact in FP32
    (and in TF32 operands), so both modes and a float64 reference agree bit for bit whatever the order of summation; then
    bias, batch norm and leaky give the same bits in both modes."""
    from ground_fusion_b200.detector import conv_stage
    C, H, W, M, size, stride, pad = shape
    rng = np.random.default_rng(hash(shape) % (1 << 32))
    x = _dyadic(rng, C * H * W).reshape(C, H, W)
    w = _dyadic(rng, M * C * size * size).reshape(M, C, size, size)
    zero = np.zeros(M, np.float32)
    # the sums alone: both modes and float64 agree bit for bit
    t = conv_stage(x, w, zero, stride, pad, precision="tf32")
    e = conv_stage(x, w, zero, stride, pad, precision="exact")
    cols, OH, OW = im2col(x.astype(np.float64), size, stride, pad)
    ref = (w.reshape(M, -1).astype(np.float64) @ cols).astype(np.float32).reshape(M, OH, OW)
    assert t.shape == ref.shape
    assert np.array_equal(e.view(np.uint32), ref.view(np.uint32))
    bad = np.flatnonzero(t.view(np.uint32) != ref.view(np.uint32))
    assert bad.size == 0, "%d of %d differ, first at %d: %r vs %r" % (bad.size, t.size, bad[0], t.flat[bad[0]], ref.flat[bad[0]])
    # the epilogue: bias, batch norm and leaky give the same bits in both modes
    bias = rng.standard_normal(M).astype(np.float32)
    bn = (rng.uniform(0.5, 1.5, M).astype(np.float32), rng.standard_normal(M).astype(np.float32),
          rng.uniform(0.2, 2.0, M).astype(np.float32))
    for kw in (dict(leaky=True), dict(bn=bn), dict(bn=bn, leaky=True)):
        t = conv_stage(x, w, bias, stride, pad, precision="tf32", **kw)
        e = conv_stage(x, w, bias, stride, pad, precision="exact", **kw)
        assert np.array_equal(t.view(np.uint32), e.view(np.uint32)), kw


def layer_bound_check(det, cfg, weights):
    """For every convolution: |o_gpu - o_ref| <= L K 2^-22 S + E_epi elementwise, and mean(|o_gpu - o_ref| / (L S)) <= 2^-20.
    Returns the largest error / bound ratio.

    o_ref is the layer in float64 from the GPU's own input: s = sum_k w~ x~ (w~, x~ the TF32-rounded operands), then
    normalize_cpu, scale, bias and leaky without rounding.  S = sum_k |w~| |x~|, and L = |scale| / den with batch norm, 1
    without.  K 2^-22 S is twice the first-order bound on truncated FP32 additions in any order, propagated through the
    epilogue's gain L (leaky's slope is <= 1).
    E_epi: the epilogue's own roundings, each at most U = 2^-24 of its result: the subtraction of the mean (U L |s - mu|
    once carried through den and scale), the rounding of the double division (U L |s - mu|), the product with scale
    (U L |s - mu|), the bias addition and leaky's product (U |y| each, |y| <= L |s - mu| + |b|).  That is at most
    5 U L |s - mu| + 2 U |b| to first order; E_epi = 8 U (L |s - mu| + |b|) covers it with the second-order terms and the
    difference between the GPU's sum and s (both far smaller)."""
    from ground_fusion_b200.detector import parse_cfg
    from yolo_ref import conv_params_expected
    _, layers = parse_cfg(cfg)
    params = conv_params_expected(cfg, weights)
    worst = 0.0
    for k, L_ in enumerate(layers):
        if L_["type"] != "convolutional":
            continue
        p = params[k]
        x = det.layer_output(k - 1) if k > 0 else det.input_image()
        size, M = L_["size"], L_["n"]
        cols, OH, OW = im2col(rna_tf32(x).astype(np.float64), size, L_["stride"], L_["pad"])
        wt = rna_tf32(p["weights"]).reshape(M, -1).astype(np.float64)
        s = wt @ cols
        S = np.abs(wt) @ np.abs(cols)
        K = wt.shape[1]
        b = p["biases"].astype(np.float64)[:, None]
        if L_["batch_normalize"]:
            mu = p["mean"].astype(np.float64)[:, None]
            den = np.sqrt(p["var"].astype(np.float64)) + float(np.float32(1e-6))
            gain = (np.abs(p["scales"].astype(np.float64)) / den)[:, None]
            y = (s - mu) / den[:, None] * p["scales"].astype(np.float64)[:, None] + b
        else:
            mu, gain = 0.0, np.ones((M, 1))
            y = s + b
        act = det.layer_output(k).reshape(M, -1).astype(np.float64)
        ref = np.where(y > 0, y, 0.1 * y) if is_leaky(cfg, k) else y
        err = np.abs(act - ref)
        bound = gain * K * 2.0 ** -22 * S + 8 * U * (gain * np.abs(s - mu) + np.abs(b)) + 1e-30
        ratio = float((err / bound).max())
        assert ratio <= 1.0, "layer %d: error %g exceeds its bound by %.3f" % (k, float(err.max()), ratio)
        mean_rel = float(np.mean(err / np.maximum(gain * S, 1e-30)))
        assert mean_rel <= 2.0 ** -20, "layer %d: mean relative error %g" % (k, mean_rel)
        worst = max(worst, ratio)
    return worst


def is_leaky(cfg, k):
    from ground_fusion_b200.detector import _sections
    secs = [s for s in _sections(cfg)[1:]]
    return secs[k][1].get("activation", "logistic") == "leaky"
