"""Host restatements for the detector's TF32 mode (tests only).

- rna_tf32(): cvt.rna.tf32.f32 on the uint32 view: round to the nearest value with 10 explicit mantissa bits, ties away from
  zero, the low 13 bits cleared.  Adding half an ulp (0x1000) to the magnitude bits and clearing the low 13 does exactly that,
  and a carry out of the mantissa moves into the exponent as it should.  Inf and NaN pass through.
- im2col(): darknet's im2col order, k = c size^2 + ky size + kx, for a float64 reference of a convolution.
- conv_shapes(): every convolution shape (C H W M size stride pad) of a cfg.
- detect_from_heads(): darknet's decoding and NMS of given [region] / [yolo] outputs (oracle/yolo_heads.c's
  yh_detect_from_heads, built into oracle/_ref/libyolo_heads.so).
"""
import ctypes
import os

import numpy as np

HEADS_ORACLE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libyolo_heads.so")


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
