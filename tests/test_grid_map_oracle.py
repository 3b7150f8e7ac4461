"""The occupancy grid's CPU side: the C oracle pinned against the pure-Python witness on scenes that hit each of the tool's quirks,
the shared log / exp against mpmath, the image and occupancy conversions against cv2, the libm-vs-shared distance, and the C
ABI's config struct against its ctypes mirror."""
import math
import os
import random
import subprocess

import numpy as np
import pytest

import gm_scenes
import gm_witness
from oracle import gm_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle(cfg, mode):
    return gm_oracle.GridMapOracle(mode=mode, **cfg)


def _run(g, kfs):
    for R, P, pts in kfs:
        g.addKeyFrame(R, P, pts)
    return g


@pytest.mark.parametrize("name", [s[0] for s in gm_scenes.quirk_scenes()])
def test_oracle_libm_equals_witness(name):
    _, cfg, kfs = next(s for s in gm_scenes.quirk_scenes() if s[0] == name)
    o = _run(_oracle(cfg, "libm"), kfs)
    w = _run(gm_witness.GridWitness(**dict(dict(ric=np.eye(3), tic=np.zeros(3)), **cfg)), kfs)
    assert o.bel().tobytes() == w.bel_array().tobytes()
    bel = o.bel()
    assert (bel != 0.5).any()
    if name == "fixed_points":
        assert bel.min() == 2.0 ** -52 and bel.max() == 1 - 2.0 ** -53
    if name == "absorbing":
        assert bel.max() == 1.0 and bel.min() == 0.0
    # a rebuild with moved poses equals a fresh witness fed the moved keyframes
    moved = [(R, P + np.array([0.013, -0.021, 0.0]), pts) for R, P, pts in kfs]
    o.updatePath([m[0] for m in moved], [m[1] for m in moved])
    w2 = _run(gm_witness.GridWitness(**dict(dict(ric=np.eye(3), tic=np.zeros(3)), **cfg)), moved)
    assert o.bel().tobytes() == w2.bel_array().tobytes()


def test_quirk_scenes_reach_what_they_name():
    """The band edges keep exactly 0.1 and 0.5; the body at (-1, -1) skips the first cell of each ray."""
    edges = gm_scenes.band_edge_z()
    assert any(k for _, _, k in edges) and any(not k for _, _, k in edges)
    for h, pz, kept in edges:
        z = float(h) + pz
        assert (not (z > 0.5 or z < 0.1)) == kept
    _, cfg, kfs = next(s for s in gm_scenes.quirk_scenes() if s[0] == "body_at_minus_one")
    w = gm_witness.GridWitness(np.eye(3), np.zeros(3), **cfg)
    seen = []
    w._update = lambda x, y, kind: seen.append((x, y))
    w.addKeyFrame(*kfs[0])
    assert (-1.0, -1.0) not in seen


def test_fixed_points_of_the_update():
    for c, want, n_want in ((math.log(0.4 / 0.6), 2.0 ** -52, 88), (math.log(0.6 / 0.4), 1 - 2.0 ** -53, 90)):
        b, n = 0.5, 0
        while True:
            nb = 1.0 - 1.0 / (1 + math.exp(math.log(b / (1.0 - b)) + c))
            if nb == b:
                break
            b, n = nb, n + 1
        assert b == want and n == n_want


def _exact(f, x):
    """f(x) correctly rounded to double, gradual underflow included (mpmath's float() would round twice there)."""
    import mpmath
    with mpmath.workprec(240):
        v = f(mpmath.mpf(x))
        if v != 0 and abs(v) < mpmath.mpf(2) ** -1022:
            return math.ldexp(int(mpmath.nint(v * mpmath.mpf(2) ** 1074)), -1074)
        return float(v)


def test_shared_log_exp_correctly_rounded():
    """1e5 arguments of each over the ranges the grid meets -- bel / (1 - bel) over [2^-53, 2^53], log-odds over [-50, 50] --
    and 2e4 over the whole double range, against mpmath; then the special values.  Prints glibc's disagreement rate."""
    import mpmath
    rng = random.Random(5)
    bad, glibc, n = {"log": 0, "exp": 0}, {"log": 0, "exp": 0}, 0
    for i in range(120000):
        x = math.exp(rng.uniform(-37, 37)) if i < 100000 else math.ldexp(rng.uniform(1, 2), rng.randint(-1074, 1023))
        y = rng.uniform(-50, 50) if i < 100000 else rng.uniform(-746, 710)
        if x == 0 or math.isinf(x):
            continue
        want = _exact(mpmath.log, x)
        bad["log"] += gm_oracle.shared_log(x) != want
        glibc["log"] += math.log(x) != want
        want = _exact(mpmath.exp, y)
        bad["exp"] += gm_oracle.shared_exp(y) != want
        glibc["exp"] += (math.exp(y) if y < 709.78 else _exact(mpmath.exp, y)) != want
        n += 1
    print("shared log/exp misrounded: %s of %d; this host's libm: log %.4f %%, exp %.4f %%"
          % (bad, n, 100.0 * glibc["log"] / n, 100.0 * glibc["exp"] / n))
    assert bad == {"log": 0, "exp": 0}
    L, E = gm_oracle.shared_log, gm_oracle.shared_exp
    inf, nan = math.inf, math.nan
    assert L(0.0) == -inf and L(-0.0) == -inf and L(inf) == inf and math.isnan(L(-1.0)) and math.isnan(L(nan)) and math.isnan(L(-inf))
    assert L(1.0) == 0.0 and math.copysign(1, L(1.0)) == 1
    for x in (5e-324, 1e-310, 2.2250738585072014e-308, 1.7976931348623157e308):
        assert L(x) == _exact(mpmath.log, x)
    assert E(0.0) == 1.0 and E(-0.0) == 1.0 and E(inf) == inf and E(-inf) == 0.0 and math.isnan(E(nan))
    assert E(709.782712893384) == 1.7976931348622732e308 and E(709.7827128933841) == inf and E(710.0) == inf
    assert E(-745.1332191019411) == 5e-324 and E(-745.1332191019412) == 0.0 and E(-800.0) == 0.0
    for x in (-708.4, -720.5, -740.1, -744.44007192138122):
        assert E(x) == _exact(mpmath.exp, x)


def _scene_oracles(mode):
    out = {}
    for name, cfg, kfs in gm_scenes.quirk_scenes():
        out[name] = _run(_oracle(cfg, mode), kfs)
    ric, tic = gm_scenes.camera_to_body()
    g = _oracle(dict(ric=ric, tic=tic), mode)
    for k in range(60):
        R, P = gm_scenes.body_pose(k)
        g.addKeyFrame(R, P, gm_scenes.keyframe_points(k, 1500))
    out["vehicle_60kf"] = g
    return out


def test_image_matches_cv2_png():
    """image() equals cv2's PNG round trip of saveMap's float64 image: 1 - bel, rows = x, flipped, * 255."""
    import cv2
    for name, g in _scene_oracles("shared").items():
        m = np.flip(1.0 - g.bel(), 0) * 255
        ok, buf = cv2.imencode(".png", m)
        assert ok
        assert np.array_equal(cv2.imdecode(buf, cv2.IMREAD_UNCHANGED), g.image()), name


def _table():
    """The occupancy of each pixel value, as the node computes it (float32 p * float(1 / 255.0), value = 1 - v in double)."""
    out = []
    for p in range(256):
        v = np.float32(p) * np.float32(1 / 255.0)
        value = 1.0 - 1.0 * float(v)
        out.append(int(value * 100) if abs(value - 0.5) > 0.005 else -1)
    return np.array(out, np.int8)


def test_occupancy_table_pinned_against_cv2():
    import cv2
    u = np.arange(256, dtype=np.uint8).reshape(16, 16)
    f = cv2.normalize(u, None, 0, 1, cv2.NORM_MINMAX, cv2.CV_32F).ravel()   # convertTo(CV_32F, 1 / 255.0, 0) for 0 .. 255
    t = _table()
    for p in range(256):
        value = 1.0 - 1.0 * float(f[p])
        assert t[p] == (int(value * 100) if abs(value - 0.5) > 0.005 else -1)
    assert [t[p] for p in (51, 102, 153, 204)] == [79, 59, 39, 19]
    assert t[127] == t[128] == -1 and t[0] == 100 and t[255] == 0
    for name, g in _scene_oracles("shared").items():
        img = np.flip(g.image(), 0)                                   # back to rows = x
        assert np.array_equal(g.occupancy(), t[img].T.ravel()), name


def test_libm_versus_shared():
    """The distance of the GPU's arithmetic (shared) from the tool's (libm) on the committed scenes: the occupancy is identical and
    the image differs only as 127 <-> 128 at cells within a few ulps of 0.5."""
    a, b = _scene_oracles("libm"), _scene_oracles("shared")
    tot = dict(cells=0, bel_diff=0, max_dbel=0.0, px=0, occ=0)
    for name in a:
        ba, bb = a[name].bel(), b[name].bel()
        d = ba != bb
        tot["cells"] += ba.size
        tot["bel_diff"] += int(d.sum())
        if d.any():
            tot["max_dbel"] = max(tot["max_dbel"], float(np.abs(ba - bb).max()))
        ia, ib = a[name].image(), b[name].image()
        dp = ia != ib
        tot["px"] += int(dp.sum())
        assert set(zip(ia[dp].tolist(), ib[dp].tolist())) <= {(127, 128), (128, 127)}, name
        tot["occ"] += int((a[name].occupancy() != b[name].occupancy()).sum())
    print("libm vs shared:", tot)
    assert tot["occ"] == 0


def test_cfg_struct_layout_matches_ctypes(tmp_path):
    import ctypes
    from ground_fusion_b200 import _lib
    src = tmp_path / "l.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "gf_b200.h"\n'
                   'int main(void) { printf("%d %d\\n", (int)sizeof(gf_grid_map_cfg), (int)offsetof(gf_grid_map_cfg, max_records)); return 0; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "l"), str(src)])
    size, off = map(int, subprocess.check_output([str(tmp_path / "l")]).split())
    assert size == ctypes.sizeof(_lib.GridMapCfg) and off == _lib.GridMapCfg.max_records.offset
