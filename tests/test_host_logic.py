"""CPU tests of the host-side logic and of the C-ABI surface (no compute calls without a GPU)."""
import ctypes
import os
import re
import subprocess

import math

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from ground_fusion_b200 import _lib
    L = _lib.lib()
    names = set()
    for hdr in os.listdir(os.path.join(ROOT, "include")):
        src = open(os.path.join(ROOT, "include", hdr)).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names |= set(re.findall(r"\b(gf_[a-z0-9_]+)\s*\(", src))
    assert len(names) >= 15
    for n in sorted(names):
        assert hasattr(L, n), "libgf_b200.so does not export %s" % n
    assert b"sm_90a" in L.gf_version()


def test_no_cpu_fallback_without_gpu():
    """Without a CUDA device every entry point fails loudly (GF_ERR_NO_DEVICE), never computes on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ground_fusion_b200 import feature_tracker
    from ground_fusion_b200._lib import GfError
    with pytest.raises(GfError, match="no CUDA device|CPU fallback"):
        feature_tracker.FeatureTracker(640, 480, [600, 600, 320, 240, 0, 0, 0, 0])
    with pytest.raises(GfError):
        feature_tracker.pyr_down(np.zeros((480, 640), np.uint8))


def test_product_does_not_import_oracle_or_cv2():
    import re
    pkg = os.path.join(ROOT, "ground_fusion_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py") and fn != "synth.py":   # synth.py is data generation, not the hot path
            src = open(os.path.join(pkg, fn)).read()
            import re
            assert not re.search(r"^\s*(from|import)\s+(cv2|oracle)\b", src, re.M), fn
            assert "oracle/" not in src and "oracle." not in src and "import_module" not in src, fn   # no path / attribute access either
    for fn in os.listdir(os.path.join(pkg, "csrc")):
        if os.path.isdir(os.path.join(pkg, "csrc", fn)):
            continue
        src = open(os.path.join(pkg, "csrc", fn)).read()
        assert not re.search(r"^\s*#\s*include\s*[<\"][^>\"]*oracle", src, re.M), fn   # comments may cite the oracle files


@pytest.fixture(scope="module")
def host_sort(tmp_path_factory):
    """Host build of the device std::sort replica (same header the CUDA kernel compiles)."""
    d = tmp_path_factory.mktemp("hs")
    src = d / "hs.cpp"
    src.write_text('#include "%s/ground_fusion_b200/csrc/fe_sort.cuh"\n'
                   'extern "C" void hs(const int* c, int n, int* perm) {\n'
                   '  gf::sort_elem* e = new gf::sort_elem[n];\n'
                   '  for (int i = 0; i < n; i++) e[i] = ((gf::sort_elem)(unsigned)c[i] << 32) | (unsigned)i;\n'
                   '  gf::setmask_sort(e, n); for (int i = 0; i < n; i++) perm[i] = (int)(e[i] & 0xffffffffu); delete[] e; }\n' % ROOT)
    so = d / "hs.so"
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", str(so), str(src)])
    L = ctypes.CDLL(str(so))
    L.hs.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    return L


def test_sort_replica_matches_libstdcxx(host_sort):
    from oracle.fe_oracle import setmask_order
    rng = np.random.default_rng(0)
    for trial in range(3000):
        n = int(rng.integers(1, 700))
        span = int(rng.choice([2, 3, 8, 40, 1000]))
        tc = rng.integers(1, span + 1, n).astype(np.int32)
        if trial % 2:
            tc = np.sort(tc)[::-1].copy()      # the tracker's input is already non-increasing
        perm = np.empty(n, np.int32)
        host_sort.hs(tc.ctypes.data, n, perm.ctypes.data)
        assert np.array_equal(perm, setmask_order(tc)), (n, span)


def test_setmask_sort_is_not_stable():
    """The reason the replica exists: std::sort permutes equal keys once n > 16."""
    from oracle.fe_oracle import setmask_order
    tc = np.array([5] * 10 + [4] * 30 + [2] * 40, np.int32)
    assert not np.array_equal(setmask_order(tc), np.arange(len(tc)))


def test_obs_struct_layout():
    from ground_fusion_b200._lib import OBS_DTYPE, Obs
    assert ctypes.sizeof(Obs) == 72 and OBS_DTYPE.fields["v"][1] == 8


def test_ctypes_argtypes_match_header_arity():
    """Every function _lib.lib() declares argtypes for takes as many arguments as its prototype in include/gf_b200.h: ctypes
    passes a call with the wrong count without complaint, and the C side then reads garbage."""
    from ground_fusion_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gf_b200.h")).read(), flags=re.S)
    arity = {}
    for name, params in re.findall(r"\b(gf_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", src):
        params = params.strip()
        arity[name] = 0 if params in ("", "void") else params.count(",") + 1
    declared = {n: f.argtypes for n, f in vars(_lib.lib()).items() if isinstance(f, ctypes._CFuncPtr) and f.argtypes is not None}
    assert len(declared) >= 50 and "gf_tracker_track" in declared
    for name, argtypes in sorted(declared.items()):
        assert name in arity, "%s has argtypes but no prototype in gf_b200.h" % name
        assert len(argtypes) == arity[name], (name, len(argtypes), arity[name])


def test_double2vector_matches_numpy_restatement():
    """Estimator::double2vector (estimator.cpp:2440-2494): host-only entry point of the library against oracle/ba_glue.py,
    including the Euler-singularity branch (pitch within 1 degree of +-90)."""
    from ground_fusion_b200.ba_problem import Problem
    from ground_fusion_b200.estimator import double2vector
    from oracle import ba_glue as G
    rng = np.random.default_rng(11)
    for trial in range(20):
        F = 11
        pb = Problem(F, 1)
        q = rng.normal(size=(F, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
        if trial % 5 == 4:      # frame 0 pitched to the singular configuration
            q[0] = [0, math.sin(math.radians(89.7) / 2), 0, math.cos(math.radians(89.7) / 2)]
        pb.para_pose[:, :3] = rng.normal(0, 3, (F, 3)); pb.para_pose[:, 3:] = q
        pb.para_speed_bias[:] = rng.normal(0, 1, (F, 9))
        R0 = G.ypr2R(rng.uniform(-170, 170, 3) * [1, 0.4, 0.4]); P0 = rng.normal(0, 5, 3)
        for use_imu in (True, False):
            Rs, Ps, Vs = double2vector(pb, R0, P0, use_imu)
            Rw, Pw, Vw = G.double2vector(pb.para_pose, pb.para_speed_bias, R0, P0, use_imu)
            assert np.abs(Rs - Rw).max() < 1e-12 and np.abs(Ps - Pw).max() < 1e-12
            if use_imu:
                assert np.abs(Vs - Vw).max() < 1e-12
                # the point of the exercise: frame 0 keeps its position, and its yaw away from the singularity
                assert np.abs(Ps[0] - P0).max() < 1e-12
                if trial % 5 != 4:
                    assert abs(G.R2ypr(Rs[0])[0] - G.R2ypr(R0)[0]) < 1e-9


def test_header_is_valid_c_and_cxx_and_matches_the_ctypes_mirror(tmp_path):
    """include/gf_b200.h must compile as C99 and as C++11 on its own (it is what the reference-side adaptor includes), and
    the ctypes mirrors in ground_fusion_b200/_lib.py must agree with it on every struct size and on the offsets of the last
    members (ABI drift between the header and the Python host side is otherwise silent)."""
    import ctypes
    import subprocess
    from ground_fusion_b200 import _lib
    inc = os.path.join(ROOT, "include")
    structs = {"gf_tracker_cfg": _lib.TrackerCfg, "gf_obs": _lib.Obs, "gf_track_info": _lib.TrackInfo,
               "gf_ba_visual_factor": _lib.BaVisualFactor, "gf_ba_imu_factor": _lib.BaImuFactor, "gf_ba_wheel_factor": _lib.BaWheelFactor,
               "gf_ba_prior": _lib.BaPrior, "gf_ba_problem": _lib.BaProblem, "gf_ba_summary": _lib.BaSummary}
    last = {"gf_ba_problem": "plane_sqrt_info", "gf_ba_wheel_factor": "gyr_1", "gf_ba_prior": "linearized_residuals", "gf_ba_summary": "device_ms",
            "gf_tracker_cfg": "pinhole"}
    body = '#include <stdio.h>\n#include <stddef.h>\n#include "gf_b200.h"\nint main(void) {\n'
    for name in structs:
        body += '  printf("%s %%zu\\n", sizeof(%s));\n' % (name, name)
    for name, member in last.items():
        body += '  printf("%s.%s %%zu\\n", offsetof(%s, %s));\n' % (name, member, name, member)
    body += "  return 0;\n}\n"
    out = {}
    for comp, std, ext in (("gcc", "-std=c99", "c"), ("g++", "-std=c++11", "cpp")):
        src = tmp_path / ("abi." + ext)
        src.write_text(body)
        exe = tmp_path / ("abi_" + ext)
        subprocess.check_call([comp, std, "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", inc, str(src), "-o", str(exe)])
        out[ext] = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert out["c"] == out["cpp"]
    for name, cls in structs.items():
        assert int(out["c"][name]) == ctypes.sizeof(cls), (name, out["c"][name], ctypes.sizeof(cls))
    for name, member in last.items():
        assert int(out["c"]["%s.%s" % (name, member)]) == getattr(structs[name], member).offset, (name, member)


def test_parallel_partition_formulation_equals_unguarded_partition():
    """fe_sort.cuh replays libstdc++'s __unguarded_partition_pivot with one warp per range: L = ascending positions where
    `lo` stops, R = descending positions where `hi` stops (both on the ORIGINAL range, after the median-of-3 move), swap k
    exchanges L[k] and R[k] while L[k] < R[k], cut = min(L[k*], R[k*-1]).  This model of the kernel's index arithmetic is
    checked against the sequential algorithm on random ranges with heavy ties (the GPU test compares the kernel itself with
    std::sort)."""
    import random

    def comp(a, b):
        return a[0] > b[0]

    def sequential(v, first, last):
        v = list(v)
        mid = first + (last - first) // 2
        a, b, c = first + 1, mid, last - 1

        def sw(i, j):
            v[i], v[j] = v[j], v[i]
        if comp(v[a], v[b]):
            if comp(v[b], v[c]): sw(first, b)
            elif comp(v[a], v[c]): sw(first, c)
            else: sw(first, a)
        elif comp(v[a], v[c]): sw(first, a)
        elif comp(v[b], v[c]): sw(first, c)
        else: sw(first, b)
        after_median = list(v)
        lo, hi = first + 1, last
        while True:
            while comp(v[lo], v[first]): lo += 1
            hi -= 1
            while comp(v[first], v[hi]): hi -= 1
            if not lo < hi:
                return v, lo, after_median
            sw(lo, hi); lo += 1

    def parallel(med, first, last):
        v = list(med); pv = v[first][0]
        L = [p for p in range(first + 1, last) if not v[p][0] > pv]
        R = [p for p in range(first + 1, last) if not pv > v[p][0]][::-1]
        m = min(len(L), len(R))
        ks = sum(1 for k in range(m) if L[k] < R[k])
        for k in range(ks):
            v[L[k]], v[R[k]] = v[R[k]], v[L[k]]
        cut = 10 ** 9
        if ks < len(L): cut = L[ks]
        if ks >= 1: cut = min(cut, R[ks - 1])
        return v, cut

    random.seed(1)
    for _ in range(20000):
        n = random.randint(17, 80)
        span = random.choice([1, 2, 3, 6, 50])
        v = [(random.randint(1, span), i) for i in range(n)]
        if random.random() < 0.3:
            v.sort(key=lambda e: -e[0])
        vs, cs, med = sequential(v, 0, n)
        vp, cp = parallel(med, 0, n)
        assert vs == vp and cs == cp


def test_cell_head_rounds_equal_the_sequential_greedy_min_distance_pass():
    """Model of nms_cells (fe_select.cuh): candidates ranked by a unique key bid for the head of their r-sized cell; a head
    that outranks the heads of the 8 surrounding cells is accepted, accepted corners kill alive candidates closer than r in
    the next round.  The accepted SET must equal cv::goodFeaturesToTrack's sequential greedy (accept in rank order unless an
    accepted corner lies within d^2 < r^2)."""
    rng = np.random.default_rng(7)
    for trial in range(60):
        w, h = int(rng.integers(60, 400)), int(rng.integers(60, 300))
        r = int(rng.integers(5, 40)); cs = max(r, 16)
        n = int(rng.integers(1, 600))
        xs = rng.integers(1, w - 1, n); ys = rng.integers(1, h - 1, n)
        pts = list({(int(x), int(y)) for x, y in zip(xs, ys)})
        keys = rng.permutation(len(pts))                     # distinct ranks, larger = better
        order = sorted(range(len(pts)), key=lambda i: -keys[i])
        seq = []
        for i in order:
            x, y = pts[i]
            if all((x - a) ** 2 + (y - b) ** 2 >= r * r for a, b in seq):
                seq.append((x, y))
        alive = set(range(len(pts))); acc = []; new = []
        rounds = 0
        while alive:
            rounds += 1
            alive = {i for i in alive if all((pts[i][0] - a) ** 2 + (pts[i][1] - b) ** 2 >= r * r for a, b in new)}
            head = {}
            for i in alive:
                c = (pts[i][0] // cs, pts[i][1] // cs)
                if c not in head or keys[i] > keys[head[c]]:
                    head[c] = i
            new = []
            for c, i in head.items():
                if all(keys[head.get((c[0] + dx, c[1] + dy), i)] <= keys[i] for dx in (-1, 0, 1) for dy in (-1, 0, 1)):
                    new.append(pts[i]); alive.discard(i)
            assert new or not alive, "the globally best head can always decide"
            acc += new
            assert rounds < 200
        assert sorted(acc) == sorted(seq), (trial, len(acc), len(seq))
