"""The reference-side C++ shim of the resident FeatureManager (adaptor/feature_manager.{h,cpp}): the reference's method names on
gf_fm_window.  CPU: it compiles and links against libgf_b200.so.  GPU: the harness's `fm` mode drives a call script through it,
and every return value and the table after every call equal the host mirror's (feature_manager.FeatureManager), bit for bit."""
import os
import struct
import subprocess

import numpy as np
import pytest

from test_fm_oracle import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "adaptor", "_build", "harness")


def build():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "adaptor")])
    return HARNESS


def test_feature_manager_shim_compiles_and_binds_the_c_abi():
    syms = subprocess.check_output(["nm", "-D", "--undefined-only", build()]).decode()
    for s in ("create", "destroy", "clear", "add_frame", "add_frame_from_tracker", "triangulate", "fill_problem", "set_depth", "remove_failures",
              "clear_depth", "remove_ids", "remove_back_shift_depth", "remove_back", "remove_front", "outliers", "predict_next", "read"):
        assert (" U gf_fm_window_" + s + "\n") in syms, s


def _poses(Ps, Rs, tic, ric):
    return struct.pack("<33d99d3d9d", *Ps.ravel(), *Rs.ravel(), *tic, *ric.ravel())


@pytest.mark.gpu
def test_call_script_through_the_cpp_adaptor(tmp_path):
    from ground_fusion_b200.feature_manager import FOCAL_LENGTH, INIT_DEPTH, FeatureManager
    from test_fm_window_gpu import ROW_BYTES, python_factor_arrays
    exe = build()
    Ps, Rs, lms, frames = scene(seed=4, n_lm=300, noise=2e-4, depth_noise=0.01)
    tic, ric = np.array([0.02, -0.01, 0.03]), np.eye(3)
    m = FeatureManager(depth_threshold=5.0)
    par = {}                    # call index -> the mirror's last_average_parallax
    ops, want = [], []          # the script, and per call (return values as bytes, the mirror's table)

    def table():
        out = struct.pack("<i", len(m.feature))
        for it in m.feature:
            out += struct.pack("<5id", it.feature_id, it.start_frame, len(it.obs), it.estimate_flag, it.solve_flag, it.estimated_depth)
            out += np.asarray(it.obs, np.float64).tobytes()
        return out

    def ids(s):
        return struct.pack("<i", len(s)) + np.array(sorted(s), np.int32).tobytes()

    def step(op, ret=b""):
        par[len(ops)] = m.last_average_parallax
        ops.append(op); want.append((ret, table()))

    for f in range(11):
        img = frames.get(f, {})
        r = m.addFeatureCheckParallax(f, img, 0.01 * f)
        step(struct.pack("<iidi", 0, f, 0.01 * f, len(img)) + b"".join(struct.pack("<i8d", k, *img[k]) for k in sorted(img)),
             struct.pack("<4i", int(r), m.last_track_num, m.new_feature_num, m.long_track_num))
    m.triangulateAll(10, Ps, Rs, tic, ric); step(struct.pack("<ii", 1, 10) + _poses(Ps, Rs, tic, ric))
    pb, n = python_factor_arrays(m)
    step(struct.pack("<i", 2), struct.pack("<2i", pb.n_visual, n) + bytes(pb.visual)[:ROW_BYTES * pb.n_visual] + pb.para_feature[:n].tobytes() + pb.feature_const[:n].tobytes())
    x = m.getDepthVector(); x[::7] *= 0.4; x[5::13] = -1.0
    m.setDepth(x); step(struct.pack("<ii", 3, len(x)) + x.tobytes())
    a = m.outliersRejection(Ps, Rs, tic, ric); step(struct.pack("<i", 9) + _poses(Ps, Rs, tic, ric), ids(a))
    b = m.movingConsistencyCheckW(Ps, Rs, tic, ric); step(struct.pack("<i", 10) + _poses(Ps, Rs, tic, ric), ids(b))
    p = m.predictPtsInNextFrame(10, Ps, Rs, tic, ric)
    step(struct.pack("<ii", 11, 10) + _poses(Ps, Rs, tic, ric), struct.pack("<i", len(p)) + b"".join(struct.pack("<i3d", k, *p[k]) for k in sorted(p)))
    m.removeOutlier(b); step(struct.pack("<ii", 5, len(b)) + np.array(sorted(b), np.int32).tobytes())
    m.removeFailures(); step(struct.pack("<i", 4))
    m.removeBackShiftDepth(Rs[0], Ps[0], Rs[1], Ps[1]); step(struct.pack("<i9d3d9d3d", 6, *Rs[0].ravel(), *Ps[0], *Rs[1].ravel(), *Ps[1]))
    img = {k: v for k, v in frames[10].items() if k in {it.feature_id for it in m.feature}}
    r = m.addFeatureCheckParallax(10, img, 0.0)
    step(struct.pack("<iidi", 0, 10, 0.0, len(img)) + b"".join(struct.pack("<i8d", k, *img[k]) for k in sorted(img)),
         struct.pack("<4i", int(r), m.last_track_num, m.new_feature_num, m.long_track_num))
    m.removeFront(10); step(struct.pack("<ii", 8, 10))
    m.removeBack(); step(struct.pack("<i", 7))
    assert a and b and p and len(m.feature) > 100 and any(v > 0 for v in par.values())
    with open(tmp_path / "fm.bin", "wb") as f:
        f.write(struct.pack("<3d2i", 10.0 / FOCAL_LENGTH, 5.0, INIT_DEPTH, 512, len(ops)) + b"".join(ops))
    subprocess.check_call([exe, "fm", str(tmp_path / "fm.bin"), str(tmp_path / "fm.out")], timeout=300)
    raw = open(tmp_path / "fm.out", "rb").read()
    off = 0
    for k, (op, (ret, tab)) in enumerate(zip(ops, want)):
        assert raw[off:off + len(ret)] == ret, ("return values of call", k); off += len(ret)
        if op[:4] == struct.pack("<i", 0):             # last_average_parallax: summed in another order than the mirror's kernel
            got, = struct.unpack("<d", raw[off:off + 8]); off += 8
            assert abs(got - par[k]) <= 1e-13 * abs(par[k]), (k, got, par[k])
        assert raw[off:off + len(tab)] == tab, ("table after call", k); off += len(tab)
    assert off == len(raw)
