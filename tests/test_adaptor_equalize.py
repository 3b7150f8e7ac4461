"""The C++ adaptor with EQUALIZE = 1 (parameters.h:33): FeatureTracker::trackImage turns on the library's CLAHE right after
gf_tracker_create, and its feature frames equal the cv2 oracle that equalises each image before trackImage, as the reference's
getImageFromMsg does.  The harness takes the same input file as tests/test_adaptor.py, in its `fe-eq` mode."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "adaptor")])
    return os.path.join(ROOT, "adaptor", "_build", "harness")


def test_adaptor_binds_set_equalize():
    syms = subprocess.check_output(["nm", "-D", "--undefined-only", build()]).decode()
    assert " U gf_tracker_set_equalize" in syms


@pytest.mark.gpu
def test_trackimage_with_equalize_through_the_cpp_adaptor(tmp_path):
    from clahe_ref import dark_stream, make_equalizing_oracle
    from ground_fusion_b200.synth import idc_params8
    from oracle.fe_oracle import IDC_CAM, PinholeCamera
    exe = build()
    n, p8 = 10, idc_params8()
    frames = dark_stream(seed=13, w=640, h=480, n=n)
    with open(tmp_path / "fe.bin", "wb") as f:
        f.write(struct.pack("<4i8d3i", n, 640, 480, 1, *p8, 150, 30, 1))
        for t, g, d in frames:
            f.write(struct.pack("<d", t)); f.write(np.ascontiguousarray(g, np.uint8).tobytes()); f.write(np.ascontiguousarray(d, np.uint16).tobytes())
    subprocess.check_call([exe, "fe-eq", str(tmp_path / "fe.bin"), str(tmp_path / "fe.out")], timeout=120)
    raw = open(tmp_path / "fe.out", "rb").read()
    ref = make_equalizing_oracle()(PinholeCamera(**IDC_CAM), 150, 30, 1, 1)
    off = 0
    for t, g, d in frames:
        want = ref.trackImage(t, g, d)
        (m,) = struct.unpack_from("<i", raw, off); off += 4
        assert m == len(want) and m > 50
        for fid in sorted(want):
            (got_id,) = struct.unpack_from("<i", raw, off); off += 4
            v = np.frombuffer(raw, np.float64, 8, off); off += 64
            assert got_id == fid and np.array_equal(v, want[fid])
    assert off == len(raw)
