"""gf_ba_solve_multi: the sliding windows of several estimators solved by one batched launch chain.  Every window of a batch
is compared with gf_ba_solve of a fresh copy of the same window.  The two run the same kernels on the same numbers, but a
solve is not bit-reproducible even against itself (the Hessian is accumulated with atomics, in whatever order the CTAs
arrive), so the bar is that of two gf_ba_solve calls of one window: identical decisions (iterations, steps, termination,
dimensions) and the blocks and cost traces equal to the last bits."""
import ctypes
import struct
import subprocess

import numpy as np
import pytest

from ground_fusion_b200 import _lib
from ground_fusion_b200._lib import BaProblem, BaSummary, GfError
from ground_fusion_b200.estimator import BundleAdjuster, solve_multi, solve_multi_structs
from ground_fusion_b200.synth_ba import make_window
from test_ba_edges_gpu import window_with_prior
from test_ba_edges_oracle import short_window, stationary_window

pytestmark = pytest.mark.gpu

PARA = ("para_pose", "para_speed_bias", "para_ex_pose", "para_feature", "para_td", "para_ex_wheel", "para_ix_wheel", "para_td_wheel",
        "para_plane_R", "para_plane_Z")
DECISIONS = ("iterations", "num_successful_steps", "termination", "reduced_dim", "n_free_landmarks", "n_residuals")
GF_ERR_INVALID_ARG = -1
MAX_MULTI = 256


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjuster(0)
    yield b
    b.close()


def handles(n, tile_caps=None, monkeypatch=None):
    out = []
    for k in range(n):
        cap = tile_caps[k] if tile_caps else None
        if cap is not None:
            monkeypatch.setenv("GF_BA_TILE_CAP", str(cap))
        out.append(BundleAdjuster(0))
        if cap is not None:
            monkeypatch.delenv("GF_BA_TILE_CAP")
    return out


def close(hs):
    for h in hs:
        h.close()


def assert_same_solve(sg, b, sw, w):
    """sg, b: batched summary and window; sw, w: the single solve of the same window.  A window stopped by its iteration cap in
    the steep phase ends on an intermediate iterate whose cost shows the summation order at the 1e-9 level (measured 2.4e-9 at
    cap 2): 1e-7 there, as test_ba_edges_gpu's capacity window; 1e-9 for a converged one.  Blocks: two solves of one window
    differ by up to 1.1e-9 (C2 velocities, measured on an H100), so 1e-8."""
    for k in DECISIONS:
        assert sg[k] == sw[k], k
    np.testing.assert_allclose(sg["cost"], sw["cost"], rtol=1e-7)
    np.testing.assert_allclose(sg["radius"], sw["radius"], rtol=1e-7)
    np.testing.assert_allclose(sg["final_cost"], sw["final_cost"], rtol=1e-7 if sw["termination"] == 0 else 1e-9)
    for k in PARA:
        np.testing.assert_allclose(getattr(b, k), getattr(w, k), rtol=0, atol=1e-8, err_msg=k)


def singles(single_handles, windows):
    out = []
    for h, pb in zip(single_handles, windows):
        w = pb.clone()
        out.append((h.optimization(w), w))
    return out


def heterogeneous_windows():
    wins = [make_window(seed=s)[0] for s in (0, 1, 2)]                               # C2
    wins.append(make_window(seed=7, with_wheel=True)[0])                               # wheel, all blocks free
    masked = make_window(seed=7, with_wheel=True, wheel_free=(True, False, True))[0]
    masked.ex_wheel_subset_mask = 0b100100
    wins.append(masked)                                                                # wheel, subset-parameterised extrinsic
    wins.append(make_window(seed=2, with_plane=True)[0])                               # plane
    wins.append(make_window(seed=4, with_plane=True, with_wheel=True)[0])              # plane + wheel: 179 unknowns
    wins.append(window_with_prior())                                                   # prior from a marginalize_old chain
    wins.append(make_window(seed=5, n_landmarks=120, free_fraction=0.0)[0])            # L = 0
    wins.append(make_window(seed=5, n_landmarks=120, free_fraction=1.0)[0])            # every landmark free
    wins.append(stationary_window())                                                   # frames_const
    wins.append(make_window(seed=7, n_landmarks=440)[0])                               # C3-sized
    for k, w in enumerate(wins):
        w.max_num_iterations = (1, 8)[k % 2]
    return wins


def test_heterogeneous_batch_equals_single_solves(ba):
    wins = heterogeneous_windows()
    want = singles([ba] * len(wins), wins)
    assert want[6][0]["reduced_dim"] == 179 and want[8][0]["n_free_landmarks"] == 0 and want[10][0]["reduced_dim"] == 0
    assert want[7][0]["n_residuals"] > 15 * 9 + 2 * wins[7].n_visual               # the prior's residuals are counted
    hs = handles(len(wins))
    try:
        got = [w.clone() for w in wins]
        sums, status = solve_multi(hs, got)
    finally:
        close(hs)
    assert status == [0] * len(wins)
    for (sw, w), sg, b in zip(want, sums, got):
        assert_same_solve(sg, b, sw, w)
        assert sg["device_ms"] == sums[0]["device_ms"] > 0                            # the time of the whole batch
    assert all(s["iterations"] <= w.max_num_iterations for s, w in zip(sums, wins)) and max(s["iterations"] for s in sums) > 1


def test_iteration_caps_stop_each_window(ba):
    """One window per cap from 0 to 16 in one batch: the loop runs to the largest cap and each window's state stops it at its own."""
    caps = [0, 1, 2, 3, 5, 8, 16]
    wins = [make_window(seed=40 + k)[0] for k in range(len(caps))]
    for w, c in zip(wins, caps):
        w.max_num_iterations = c
    want = singles([ba] * len(wins), wins)
    hs = handles(len(wins))
    try:
        got = [w.clone() for w in wins]
        sums, status = solve_multi(hs, got)
    finally:
        close(hs)
    for (sw, w), sg, b, c in zip(want, sums, got, caps):
        assert sg["iterations"] <= c
        assert_same_solve(sg, b, sw, w)
    assert sums[0]["iterations"] == 0 and np.array_equal(got[0].para_pose, wins[0].para_pose)


def test_mixed_step_instantiations(monkeypatch):
    """Handles created under GF_BA_TILE_CAP=40 take k_ba_step's spill instantiation; the others the shared-memory one."""
    caps = [40, None, 40, None, None]
    wins = [make_window(seed=60 + k)[0] for k in range(4)] + [make_window(seed=64, n_landmarks=440)[0]]
    ref = handles(len(wins), caps, monkeypatch)
    hs = handles(len(wins), caps, monkeypatch)
    try:
        want = singles(ref, wins)
        got = [w.clone() for w in wins]
        sums, status = solve_multi(hs, got)
    finally:
        close(ref); close(hs)
    for (sw, w), sg, b in zip(want, sums, got):
        assert_same_solve(sg, b, sw, w)


def test_batch_of_one_equals_gf_ba_solve(ba):
    pb = make_window(seed=3)[0]
    (sw, w), = singles([ba], [pb])
    b = pb.clone()
    sums, status = solve_multi([ba], [b])
    assert status == [0]
    assert_same_solve(sums[0], b, sw, w)


def test_largest_batch_and_one_more():
    wins = [short_window(4) for _ in range(MAX_MULTI + 1)]
    hs = handles(MAX_MULTI + 1)
    try:
        want = singles(hs[:1] * MAX_MULTI, wins[:MAX_MULTI])
        got = [w.clone() for w in wins]
        before = [w.para_pose.copy() for w in got]
        with pytest.raises(GfError, match="error -4"):
            solve_multi(hs, got)
        assert all(np.array_equal(w.para_pose, p) for w, p in zip(got, before))
        sums, status = solve_multi(hs[:MAX_MULTI], got[:MAX_MULTI])
    finally:
        close(hs)
    assert status == [0] * MAX_MULTI
    for (sw, w), sg, b in zip(want, sums, got):
        assert_same_solve(sg, b, sw, w)


def _raw_call(hs, n, p_array, sums=True, status=None):
    L = _lib.lib()
    L.gf_ba_solve_multi.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    harr = (ctypes.c_void_p * len(hs))(*[h._h.value for h in hs]) if hs is not None else None
    s = (BaSummary * max(n, 1))() if sums else None
    rc = L.gf_ba_solve_multi(harr, n, p_array, s, status)
    return rc, L.gf_last_error().decode()


def test_argument_errors_modify_nothing():
    wins = [make_window(seed=70 + k, n_landmarks=60)[0] for k in range(3)]
    hs = handles(3)
    try:
        got = [w.clone() for w in wins]
        before = [(w.para_pose.copy(), w.para_feature.copy()) for w in got]
        arr = (BaProblem * 3)(*[w.struct() for w in got])
        assert _raw_call(None, 3, arr)[0] == GF_ERR_INVALID_ARG
        assert _raw_call(hs, 3, None)[0] == GF_ERR_INVALID_ARG
        assert _raw_call(hs, 3, arr, sums=False)[0] == GF_ERR_INVALID_ARG
        for n in (0, -1):
            assert _raw_call(hs, n, arr)[0] == GF_ERR_INVALID_ARG
        rc, msg = _raw_call([hs[0], hs[1], hs[0]], 3, arr)
        assert rc == GF_ERR_INVALID_ARG and msg.startswith("window 2:")
        bad = got[1].clone()
        bad.visual[5].imu_j = 11                                                       # frame index out of range
        arr_bad = (BaProblem * 3)(got[0].struct(), bad.struct(), got[2].struct())
        rc, msg = _raw_call(hs, 3, arr_bad)
        assert rc == GF_ERR_INVALID_ARG and msg.startswith("window 1:") and "visual factor" in msg
        over = got[2].clone(); over.max_num_iterations = 17
        rc, msg = _raw_call(hs, 3, (BaProblem * 3)(got[0].struct(), got[1].struct(), over.struct()))
        assert rc == GF_ERR_INVALID_ARG and msg.startswith("window 2:")
        assert all(np.array_equal(w.para_pose, p) and np.array_equal(w.para_feature, f) for w, (p, f) in zip(got, before))
        # and the handles still work
        sums, status = solve_multi(hs, got)
        assert status == [0, 0, 0]
    finally:
        close(hs)


def test_singular_imu_covariance_fails_only_its_window(ba):
    wins = [make_window(seed=80 + k)[0] for k in range(3)]
    bad = wins[1]
    cov = np.array(bad.imu[3].covariance).reshape(15, 15)
    cov[7, :] = 0.0; cov[:, 7] = 0.0
    bad.imu[3].covariance[:] = list(cov.ravel())
    want = singles([ba, ba], [wins[0], wins[2]])
    hs = handles(3)
    try:
        got = [w.clone() for w in wins]
        sums, status = solve_multi(hs, got)
    finally:
        close(hs)
    assert status[1] == GF_ERR_INVALID_ARG and status[0] == status[2] == 0
    assert np.array_equal(got[1].para_pose, bad.para_pose) and np.array_equal(got[1].para_feature, bad.para_feature)
    assert sums[1]["iterations"] == 0 and sums[1]["final_cost"] == 0.0
    for (sw, w), k in zip(want, (0, 2)):
        assert_same_solve(sums[k], got[k], sw, w)
    L = _lib.lib()
    assert L.gf_last_error().decode().startswith("window 1:") and "covariance" in L.gf_last_error().decode()


def _launches():
    return _lib.lib().gf_kernel_launch_count()


def test_launch_count_does_not_depend_on_the_batch_size(ba, monkeypatch):
    """A batch costs the launches of its window with the largest cap; one more k_ba_step per loop pass when both step
    instantiations are needed."""
    wins = [make_window(seed=90 + k)[0] for k in range(6)]
    for w, c in zip(wins, (8, 3, 16, 1, 8, 5)):
        w.max_num_iterations = c
    c0 = _launches(); ba.optimization(wins[2].clone()); single = _launches() - c0
    hs = handles(6)
    try:
        c0 = _launches(); solve_multi(hs, [w.clone() for w in wins]); batch = _launches() - c0
    finally:
        close(hs)
    assert batch == single
    hs = handles(6, [40, None, None, None, None, None], monkeypatch)
    try:
        c0 = _launches(); solve_multi(hs, [w.clone() for w in wins]); mixed = _launches() - c0
    finally:
        close(hs)
    assert mixed == single + 16 + 1                  # the loop makes max_num_iterations + 1 passes


def test_handles_after_a_batch(ba):
    """Handles that served a batch, then gf_ba_solve / marginalize_old, give what handles that never did give; a later batch of
    larger windows grows their buffers."""
    small = [make_window(seed=100 + k, n_landmarks=60)[0] for k in range(3)]
    large = [make_window(seed=110 + k, n_landmarks=440)[0] for k in range(3)]
    hs = handles(3)
    fresh = handles(1)
    try:
        solve_multi(hs, [w.clone() for w in small])
        want = singles([fresh[0]] * 3, large)
        got = [w.clone() for w in large]
        sums, status = solve_multi(hs, got)
        for (sw, w), sg, b in zip(want, sums, got):
            assert_same_solve(sg, b, sw, w)
        # gf_ba_solve and marginalize_old on a batched handle
        for h in hs:
            pb = make_window(seed=120)[0]
            b, w = pb.clone(), pb.clone()
            sg, sw = h.optimization(b), fresh[0].optimization(w)
            assert_same_solve(sg, b, sw, w)
            pg, pw = h.marginalize_old(b), fresh[0].marginalize_old(b)
            assert pg.kinds == pw.kinds and pg.indices == pw.indices and pg.idx == pw.idx
            np.testing.assert_array_equal(pg.x0, pw.x0)
            H, Hw = pg.J.T @ pg.J, pw.J.T @ pw.J             # J0 is defined up to an orthogonal transform: compare J0^T J0
            assert np.abs((H - Hw) / (np.sqrt(np.outer(np.diag(Hw), np.diag(Hw))) + 1e-300)).max() < 1e-5
    finally:
        close(hs); close(fresh)


def test_ctypes_variant_for_prebuilt_structs():
    wins = [make_window(seed=130 + k, n_landmarks=80)[0] for k in range(2)]
    hs = handles(2)
    try:
        a = [w.clone() for w in wins]
        b = [w.clone() for w in wins]
        d1, s1 = solve_multi(hs, a)
        arr = (BaProblem * 2)(*[w.struct() for w in b])
        sums, status = solve_multi_structs(hs, arr)
    finally:
        close(hs)
    assert list(status) == [0, 0]
    for k in range(2):
        assert_same_solve(sums[k].as_dict(), b[k], d1[k], a[k])


# ---- the C++ adaptor: Estimator::optimizationMulti ----
def _dump_multi(path, chains, flags):
    from test_adaptor import _dump_window
    n_est, rounds = len(chains), len(chains[0])
    with open(path, "wb") as f:
        f.write(struct.pack("<4i3d", n_est, 11, n_est * rounds, 8, *chains[0][0].gravity))
        for r in range(rounds):
            for e in range(n_est):
                _dump_window(f, chains[e][r], flags[r])


def _read_multi(path, chains):
    raw = np.fromfile(path, np.float64)
    off, out = 0, []
    for r in range(len(chains[0])):
        for e in range(len(chains)):
            q = chains[e][r]
            F, nfeat = q.n_frames, q.n_features
            rec = {"pose": raw[off:off + 7 * F].reshape(F, 7)}; off += 7 * F
            rec["sb"] = raw[off:off + 9 * F].reshape(F, 9); off += 9 * F
            rec["feat"] = raw[off:off + nfeat]; off += nfeat
            it, cost, pdim, term = raw[off:off + 4]; off += 4
            rec.update(it=int(it), cost=cost, pdim=int(pdim), term=int(term))
            n = rec["pdim"]
            rec["r"] = raw[off:off + n]; off += n
            rec["J"] = raw[off:off + n * n].reshape(n, n); off += n * n
            out.append(rec)
    assert off == raw.size
    return out


def test_adaptor_optimization_multi(tmp_path):
    """Three estimators, two rounds (MARGIN_OLD, then MARGIN_SECOND_NEW with the prior the first left): one
    Estimator::optimizationMulti call per round against each estimator's optimization() in turn."""
    from test_adaptor import build
    exe = build()
    chains = [[make_window(seed=140 + 10 * e + r, n_landmarks=150)[0] for r in range(2)] for e in range(3)]
    _dump_multi(tmp_path / "in.bin", chains, [0, 1])
    subprocess.check_call([exe, "ba-multi", str(tmp_path / "in.bin"), str(tmp_path / "multi.out")], timeout=120)
    subprocess.check_call([exe, "ba-seq", str(tmp_path / "in.bin"), str(tmp_path / "seq.out")], timeout=120)
    got, want = _read_multi(tmp_path / "multi.out", chains), _read_multi(tmp_path / "seq.out", chains)
    for k, (g, w) in enumerate(zip(got, want)):
        assert (g["it"], g["term"], g["pdim"]) == (w["it"], w["term"], w["pdim"]) and g["pdim"] > 0
        # round 1 carries a prior taken from an unrelated window, which amplifies the last-bit differences of two solves
        # (atomic summation order) to ~1e-6 relative, as in test_adaptor
        tol = 1e-9 if k < 3 else 1e-4
        np.testing.assert_allclose(g["cost"], w["cost"], rtol=tol)
        np.testing.assert_allclose(g["pose"], w["pose"], atol=1e3 * tol)
        np.testing.assert_allclose(g["sb"], w["sb"], atol=1e4 * tol)
        H, Hw = g["J"].T @ g["J"], w["J"].T @ w["J"]          # J0 is defined up to an orthogonal transform: compare J0^T J0
        scale = np.sqrt(np.outer(np.diag(Hw), np.diag(Hw))) + 1e-300
        assert np.abs((H - Hw) / scale).max() < (1e-5 if k < 3 else 1e-3)       # measured up to 1.1e-6 in round 0
