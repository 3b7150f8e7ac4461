"""The reference-side C++ shim of the occupancy grid (adaptor/grid_map.{h,cpp}): the grid_mapping tool's GridMap + GridMapper and
main.cpp's per-keyframe body on the C ABI.  CPU: it compiles and links against libgf_b200.so.  GPU: the harness's `gm` mode drives
keyframes and a pose correction through it, and bel, the image and the occupancy equal the sequential oracle's shared mode."""
import os
import struct
import subprocess

import numpy as np
import pytest

import gm_scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "adaptor", "_build", "harness")


def build():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "adaptor")])
    return HARNESS


def test_grid_map_shim_compiles_and_binds_the_c_abi():
    syms = subprocess.check_output(["nm", "-D", "--undefined-only", build()]).decode()
    for s in ("gf_grid_map_create", "gf_grid_map_add_keyframe", "gf_grid_map_update_poses", "gf_grid_map_read", "gf_grid_map_destroy"):
        assert (" U " + s) in syms, s


@pytest.mark.gpu
def test_grid_map_through_the_cpp_adaptor(tmp_path):
    from oracle.gm_oracle import GridMapOracle
    exe = build()
    ric, tic = gm_scenes.camera_to_body()
    sx, sy, ix, iy, cs, p = 300, 200, 150, 100, 0.05, (0.6, 0.4, 0.5)
    ops = [("add",) + gm_scenes.body_pose(k) + (gm_scenes.keyframe_points(k, 800),) for k in range(5)]
    Rs, Ps = zip(*[gm_scenes.body_pose(k) for k in range(5)])
    ops.append(("update", [R.copy() for R in Rs], [P + np.array([0.03, -0.02, 0.0]) for P in Ps]))
    ops.append(("add",) + gm_scenes.body_pose(9) + (gm_scenes.keyframe_points(9, 800),))
    with open(tmp_path / "gm.bin", "wb") as f:
        f.write(struct.pack("<4i4d9d3d4i", sx, sy, ix, iy, cs, *p, *ric.ravel(), *tic, 1 << 16, 16, 4096, len(ops)))
        for op in ops:
            if op[0] == "add":
                f.write(struct.pack("<i9d3di", 0, *op[1].ravel(), *op[2], len(op[3])))
                f.write(np.ascontiguousarray(op[3], np.float32).tobytes())
            else:
                f.write(struct.pack("<2i", 1, len(op[1])))
                for R, P in zip(op[1], op[2]):
                    f.write(struct.pack("<9d3d", *R.ravel(), *P))
    subprocess.check_call([exe, "gm", str(tmp_path / "gm.bin"), str(tmp_path / "gm.out")], timeout=300)
    raw = open(tmp_path / "gm.out", "rb").read()
    o = GridMapOracle(ric, tic, sx, sy, ix, iy, cs, *p, mode="shared")
    off, n = 0, sx * sy
    for op in ops:
        if op[0] == "add":
            o.addKeyFrame(*op[1:])
        else:
            o.updatePath(op[1], op[2])
        assert raw[off:off + 8 * n] == np.ascontiguousarray(o.bel().T).tobytes(); off += 8 * n
        assert raw[off:off + n] == o.image().tobytes(); off += n
        assert raw[off:off + n] == o.occupancy().tobytes(); off += n
    assert off == len(raw)
    assert (o.bel() != 0.5).any()
