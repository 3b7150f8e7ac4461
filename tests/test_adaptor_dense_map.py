"""The reference-side C++ shim of the dense colour map (adaptor/dense_map.{h,cpp}): PoseGraph's octree blocks and the node's
sampling loop on the C ABI.  CPU: it compiles and links against libgf_b200.so.  GPU: the harness's `dm` mode drives keyframes and
a pose correction through it, and the returned point_rgbd, the cloud and the filtered indices equal the sequential oracle's."""
import os
import struct
import subprocess

import numpy as np
import pytest

import dm_scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "adaptor", "_build", "harness")
P8 = [320.0, 318.5, 81.3, 59.7, 0.12, -0.3, 1.5e-3, -8e-3]


def build():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "adaptor")])
    return HARNESS


def test_dense_map_shim_compiles_and_binds_the_c_abi():
    syms = subprocess.check_output(["nm", "-D", "--undefined-only", build()]).decode()
    for s in ("gf_dense_map_create", "gf_dense_map_add_keyframe", "gf_dense_map_update_poses", "gf_dense_map_read",
              "gf_dense_map_keyframe_points", "gf_dense_map_destroy"):
        assert (" U " + s) in syms, s


@pytest.mark.gpu
def test_dense_map_through_the_cpp_adaptor(tmp_path):
    from oracle.dm_oracle import DenseMapOracle
    exe = build()
    w, h, dd, db = 160, 120, 2, 3
    ric, tic = dm_scenes.rot(0.01, -0.02, 0.015), np.array([0.03, -0.01, 0.02])
    ops = []
    for k in range(6):
        rgb, depth = dm_scenes.frame(k, w, h)
        ops.append(("add",) + dm_scenes.pose(k) + (rgb, depth))
    Rs, Ps = zip(*[dm_scenes.pose(k) for k in range(6)])
    Rn, Pn = dm_scenes.perturbed(np.array(Rs), np.array(Ps), 4)
    ops.append(("update", Rn, Pn))
    rgb, depth = dm_scenes.frame(9, w, h)
    ops.append(("add",) + dm_scenes.pose(9) + (rgb, depth))
    with open(tmp_path / "dm.bin", "wb") as f:
        f.write(struct.pack("<2i8d2i9d3d3i", w, h, *P8, dd, db, *ric.ravel(), *tic, 1 << 20, 64, len(ops)))
        for op in ops:
            if op[0] == "add":
                f.write(struct.pack("<i9d3d", 0, *op[1].ravel(), *op[2]))
                f.write(np.ascontiguousarray(op[3], np.uint8).tobytes()); f.write(np.ascontiguousarray(op[4], np.uint16).tobytes())
            else:
                f.write(struct.pack("<2i", 1, len(op[1])))
                for R, P in zip(op[1], op[2]):
                    f.write(struct.pack("<9d3d", *R.ravel(), *P))
    subprocess.check_call([exe, "dm", str(tmp_path / "dm.bin"), str(tmp_path / "dm.out")], timeout=300)
    raw = open(tmp_path / "dm.out", "rb").read()
    o = DenseMapOracle(w, h, P8, dd, db, ric, tic)
    off, n_kf = 0, 0
    for op in ops:
        if op[0] == "add":
            assert o.addKeyFrame(*op[1:]) >= 0
            (m,) = struct.unpack_from("<i", raw, off); off += 4
            got = np.frombuffer(raw, np.float32, 6 * m, off).reshape(m, 6); off += 24 * m
            assert got.tobytes() == o.keyframePoints(n_kf).tobytes()
            n_kf += 1
        else:
            o.updatePath(op[1], op[2])
        xyz, rgb = o.cloud()
        (n,) = struct.unpack_from("<i", raw, off); off += 4
        assert n == len(xyz) > 0
        assert raw[off:off + 12 * n] == xyz.tobytes(); off += 12 * n
        assert raw[off:off + 3 * n] == rgb.tobytes(); off += 3 * n
        (nf,) = struct.unpack_from("<i", raw, off); off += 4
        assert np.array_equal(np.frombuffer(raw, np.int32, nf, off), o.filtered()[2]); off += 4 * nf
    assert off == len(raw)
