"""gf_detector_detect_batch without a GPU: the header and both libraries carry the batch entry points, and every argument error
is refused before the library touches a device."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "ground_fusion_b200")
NEW_SYMBOLS = ("gf_detector_set_max_batch", "gf_detector_detect_batch", "gf_detector_member_layer_output")
GF_ERR_INVALID_ARG = -1


def _built(name):
    p = os.path.join(PKG, name)
    if not os.path.exists(p):
        pytest.skip("%s not built" % name)
    return p


def test_header_declares_the_batch_entry_points():
    h = open(os.path.join(ROOT, "include", "gf_b200.h")).read()
    assert "#define GF_DETECTOR_BATCH_MAX 64" in h and "#define GF_TRACKER_GROUP_MAX 64" in h
    for s in NEW_SYMBOLS:
        assert re.search(r"\bint %s\(" % s, h), s
    from ground_fusion_b200 import _lib
    assert _lib.GF_DETECTOR_BATCH_MAX == 64


@pytest.mark.parametrize("name", ["libgf_yolo.so", "libgf_b200.so"])
def test_both_libraries_export_the_batch_entry_points(name):
    L = ctypes.CDLL(_built(name))
    for s in NEW_SYMBOLS:
        assert hasattr(L, s), s


@pytest.mark.parametrize("name", ["libgf_yolo.so", "libgf_b200.so"])
def test_argument_errors_are_refused_before_any_device_call(name):
    """A null handle or null arrays: GF_ERR_INVALID_ARG from the argument checks, which run before any CUDA call (so they answer
    the same on a machine without a device)."""
    L = ctypes.CDLL(_built(name))
    vp, i = ctypes.c_void_p, ctypes.c_int
    L.gf_detector_detect_batch.argtypes = [vp, i, vp, vp, vp, vp, i, vp, vp, vp, i, vp]
    L.gf_detector_set_max_batch.argtypes = [vp, i]
    L.gf_detector_member_layer_output.argtypes = [vp, i, i, vp, ctypes.c_size_t]
    bgr = np.zeros((4, 4, 3), np.uint8)
    ptrs = (vp * 1)(bgr.ctypes.data)
    pitch = (ctypes.c_size_t * 1)(12)
    w, h = (i * 1)(4), (i * 1)(4)
    boxes, start = np.zeros((8, 4), np.int64), np.zeros(2, np.int32)
    good = [None, 1, ptrs, pitch, w, h, 0, boxes.ctypes.data, None, None, 8, start.ctypes.data]
    assert L.gf_detector_detect_batch(*good) == GF_ERR_INVALID_ARG            # null handle
    # The checks below never read the handle: the null and range checks and the per-frame checks all come before it is used
    # (its max_batch is read only after them).  So a zeroed stand-in of the handle's size class is enough, and a refusal proves
    # the check ran before any use of the handle or the device.
    stand_in = ctypes.create_string_buffer(4096)
    for k, v in ((1, 0), (1, -1), (2, None), (3, None), (4, None), (5, None), (10, -1), (7, None), (11, None)):
        a = list(good)
        a[0], a[k] = ctypes.addressof(stand_in), v
        assert L.gf_detector_detect_batch(*a) == GF_ERR_INVALID_ARG, (k, v)
    # a bad member among good ones: width, height, pitch below 3 * width, a null frame
    for what, (ww, hh, pp, ok) in {"width": (0, 4, 12, True), "height": (4, 0, 12, True), "pitch": (4, 4, 11, True),
                                   "too wide": (16385, 4, 3 * 16385, True), "null frame": (4, 4, 12, False)}.items():
        ptrs3 = (vp * 3)(bgr.ctypes.data, bgr.ctypes.data if ok else None, bgr.ctypes.data)
        pitch3 = (ctypes.c_size_t * 3)(12, pp, 12)
        w3, h3 = (i * 3)(4, ww, 4), (i * 3)(4, hh, 4)
        start3 = np.zeros(4, np.int32)
        rc = L.gf_detector_detect_batch(ctypes.addressof(stand_in), 3, ptrs3, pitch3, w3, h3, 0, boxes.ctypes.data, None, None, 8,
                                        start3.ctypes.data)
        assert rc == GF_ERR_INVALID_ARG, what
        assert not start3.any(), what
    assert L.gf_detector_set_max_batch(None, 2) == GF_ERR_INVALID_ARG
    out = np.zeros(16, np.float32)
    assert L.gf_detector_member_layer_output(None, 0, 0, out.ctypes.data, out.size) == GF_ERR_INVALID_ARG
    assert not start.any()


def test_python_batch_refuses_bad_frame_lists_before_the_library():
    from ground_fusion_b200.detector import YoloDetector
    det = YoloDetector.__new__(YoloDetector)          # no handle: the checks below must not reach the library
    det._h, det._L, det.max_batch = ctypes.c_void_p(), None, 2
    with pytest.raises(ValueError):
        det.detect_batch([])
    with pytest.raises(ValueError):
        det.detect_batch([np.zeros((4, 4), np.uint8)])
    with pytest.raises(ValueError):
        det.detect_batch_csr([np.zeros((4, 4, 3), np.float32)])


def test_batch_kernels_keep_each_precision_on_its_units():
    """The batched convolutions compile the same bodies as the single-image ones: the exact variants stay off the tensor cores,
    the TF32 variant issues TF32 HGMMA."""
    import subprocess
    lib = _built("libgf_yolo.so")
    try:
        sass = subprocess.check_output(["cuobjdump", "-sass", lib], text=True, stderr=subprocess.STDOUT)
    except (OSError, subprocess.CalledProcessError) as e:
        pytest.skip("cuobjdump unavailable: %s" % e)
    funcs = re.split(r"\n\s+Function : ", sass)
    exact = [f for f in funcs if f.startswith("_ZN3gfy17k_yolo_conv_batch")]
    tf32 = [f for f in funcs if f.startswith("_ZN3gfy22k_yolo_conv_tf32_batch")]
    assert len(exact) == 2 and not any("HGMMA" in f or "HMMA" in f for f in exact)
    assert len(tf32) == 1 and re.search(r"HGMMA\.64x64x8\.F32\.TF32", tf32[0])
