"""gf_ba_marginalize_multi: the marginalisations of several estimators in one batched launch chain.  Every window of a batch is
compared with the single call (gf_ba_marginalize_old / _second_new) of the same window on a fresh handle, and with the CPU
oracle.  The single call is not bit-reproducible against itself (the Hessian is summed with atomics), so J0 is held to the
repeatability bar of test_ba_multi_gpu.test_handles_after_a_batch; the decisions (return value, blocks, path) and x0 must be
identical."""
import ctypes
import struct
import subprocess

import numpy as np
import pytest

from ground_fusion_b200 import _lib
from ground_fusion_b200._lib import (MARG_PATH_GENERIC, MARG_PATH_NOT_PD, MARG_PATH_REDUCED_JACOBI, MARG_PATH_WIDE, MARGIN_OLD,
                                     MARGIN_SECOND_NEW, BaPrior, BaProblem, GfError)
from ground_fusion_b200.ba_problem import Prior
from ground_fusion_b200.estimator import BundleAdjuster, marginalize_multi
from ground_fusion_b200.synth_ba import make_window
from oracle import ba_oracle as O
from test_ba_edges_oracle import short_window
from test_ba_gpu import _compare_priors
from test_marg_stages_gpu import _rows, _stationary_start

pytestmark = pytest.mark.gpu

GF_ERR_INVALID_ARG, GF_ERR_CAPACITY = -1, -4
MAX_MULTI = 256


def handles(n):
    return [BundleAdjuster(0) for _ in range(n)]


def close(hs):
    for h in hs:
        h.close()


def shifted(q, prior):
    """The window after MARGIN_OLD of the 11-frame window q: frame 0 dropped, the rest kept, `prior` attached."""
    nxt = q.clone(); nxt.n_frames = q.n_frames - 1
    nxt.para_pose = q.para_pose[1:].copy(); nxt.para_speed_bias = q.para_speed_bias[1:].copy()
    nxt.set_visual([(f.imu_i - 1, f.imu_j - 1, f.feature, list(f.pts_i), list(f.pts_j), list(f.vel_i), list(f.vel_j), f.td_i, f.td_j)
                    for f in list(q.visual)[:q.n_visual] if f.imu_i >= 1])
    nxt.set_imu([dict(i=f.i - 1, j=f.j - 1, sum_dt=f.sum_dt, delta_p=list(f.delta_p), delta_q=list(f.delta_q), delta_v=list(f.delta_v),
                      linearized_ba=list(f.linearized_ba), linearized_bg=list(f.linearized_bg),
                      jacobian=np.array(f.jacobian).reshape(15, 15), covariance=np.array(f.covariance).reshape(15, 15))
                 for f in list(q.imu)[1:q.n_imu]])
    nxt.prior = prior
    return nxt


def wide_window(seed, sb_frames=range(1, 9), weight=100.0):
    """A chained window whose prior is too wide for the fast path: solve -> MARGIN_OLD -> shift, and the prior carries the
    speed biases of sb_frames besides the chained blocks (block-diagonal information of `weight`).  MARGIN_OLD then keeps
    54 + 72 + 7 = 133 columns, MARGIN_SECOND_NEW 148 - 6 = 142: both WIDE, the reduced system by Jacobi."""
    q, _ = make_window(seed=seed)
    O.solve(q)
    pr = O.marginalize_old(q)
    nxt = shifted(q, pr)
    extra = list(sb_frames)
    n0 = pr.n
    J = np.zeros((n0 + 9 * len(extra),) * 2)
    J[:n0, :n0] = pr.J
    J[n0:, n0:] = weight * np.eye(9 * len(extra))
    x0_len = sum({0: 7, 1: 9, 2: 7, 3: 1}[k] for k in pr.kinds)               # pose, speed bias, ex_pose, td
    nxt.prior = Prior(pr.kinds + [1] * len(extra), pr.indices + extra, pr.idx + [n0 + 9 * j for j in range(len(extra))],
                      np.concatenate([pr.x0[:x0_len]] + [nxt.para_speed_bias[f] for f in extra]),
                      J, np.concatenate([pr.r, np.zeros(9 * len(extra))]))
    O.solve(nxt)
    return nxt


def no_frame0_landmarks(seed):
    """A chained window (solve -> MARGIN_OLD -> shift) without any visual factor starting in frame 0: m = 15 (pose 0 and speed
    bias 0 only).  The prior carries the information: without it, pose 0 and speed bias 0 are held by IMU(0->1) alone and
    eliminating them leaves nothing but rounding noise."""
    q, _ = make_window(seed=seed)
    O.solve(q)
    pb = shifted(q, O.marginalize_old(q))
    pb.set_visual([r for r in _rows(pb) if r[0] != 0])
    O.solve(pb)
    return pb


def solved(**kw):
    pb, _ = make_window(**kw)
    O.solve(pb)
    return pb


def second_new_pair(seed):
    """(window whose prior holds para_Pose[WINDOW_SIZE - 1], the same window with that pose taken out of the prior)."""
    pb = solved(seed=seed)
    pr = O.marginalize_old(pb)
    nxt = solved(seed=seed + 50)
    nxt.prior = pr
    O.solve(nxt)
    F = nxt.n_frames
    keep = [j for j, (k, i) in enumerate(zip(pr.kinds, pr.indices)) if not (k == 0 and i == F - 2)]
    without = nxt.clone()
    without.prior = Prior([pr.kinds[j] for j in keep], [pr.indices[j] for j in keep], [pr.idx[j] for j in keep], pr.x0, pr.J, pr.r)
    return nxt, without


def single(h, pb, mode):
    fn = h.marginalize_old if mode == MARGIN_OLD else h.marginalize_second_new
    try:
        pr = fn(pb)
        status = pr.n if pr is not None else 0
    except GfError:
        pr, status = None, GF_ERR_INVALID_ARG
    return pr, status, h.last_marg_info()


def assert_same_prior(g, w, bar=1e-5):
    """g: batched, w: single call of the same window.  The entry scale has test_ba_gpu._compare_priors' floor of bar * max|H|:
    the plane rotation's fourth column holds only rounding noise (diagonal ~1e-9 next to 1e7), which two single calls of one
    window already disagree on by 1e-2 of its own scale."""
    assert g.n == w.n and g.kinds == w.kinds and g.indices == w.indices and g.idx == w.idx
    np.testing.assert_array_equal(g.x0, w.x0)
    H, Hw = g.J.T @ g.J, w.J.T @ w.J              # J0 is defined up to an orthogonal transform: compare J0^T J0
    scale = np.sqrt(np.outer(np.diag(Hw), np.diag(Hw))) + 1e-300 + bar * np.abs(Hw).max()
    assert np.abs((H - Hw) / scale).max() < bar
    b, bw = g.J.T @ g.r, w.J.T @ w.r
    assert np.abs(b - bw).max() <= bar * np.abs(bw).max()


def check_batch(wins, modes, hs=None, ref=None):
    """Batch of wins / modes against single calls on `ref`; returns (priors, statuses, infos, single results)."""
    own = hs is None
    hs = handles(len(wins)) if own else hs
    own_ref = ref is None
    ref = BundleAdjuster(0) if own_ref else ref
    try:
        want = [single(ref, w.clone(), m) for w, m in zip(wins, modes)]
        priors, status = marginalize_multi(hs, [w.clone() for w in wins], modes)
        infos = [h.last_marg_info() for h in hs]
        ms = hs[0].last_marg_ms
    finally:
        if own:
            close(hs)
        if own_ref:
            ref.close()
    for k, ((pw, sw, iw), pg, sg, ig) in enumerate(zip(want, priors, status, infos)):
        assert sg == sw, k
        if sw > 0:
            assert ig[0] == iw[0], (k, ig, iw)
            assert_same_prior(pg, pw)
        else:
            assert pg is None
    assert all(h.last_marg_ms == ms for h in hs) and ms > 0
    return priors, status, infos, want


def test_mixed_batch_equals_single_calls_and_the_oracle():
    with_pose, without_pose = second_new_pair(8)
    stationary = solved(seed=11)
    _stationary_start(stationary, 0.5)
    wide = wide_window(4)
    cases = [  # (window, mode, oracle tolerance)
        (solved(seed=0), MARGIN_OLD, 1e-6),                                     # C2
        (solved(seed=1), MARGIN_OLD, 1e-6),
        (solved(seed=7, with_wheel=True), MARGIN_OLD, 1e-6),                     # wheel
        (solved(seed=3, with_plane=True), MARGIN_OLD, 1e-6),                     # plane
        (solved(seed=4, with_plane=True, with_wheel=True), MARGIN_OLD, 1e-6),    # plane + wheel: 179 unknowns
        (no_frame0_landmarks(5), MARGIN_OLD, 1e-6),                              # m = 15
        (solved(seed=7, n_landmarks=440), MARGIN_OLD, 1e-6),                     # C3-sized
        (stationary, MARGIN_OLD, 1e-6),                                          # NOT_PD: the literal path
        (wide, MARGIN_OLD, 1e-5),                                                # WIDE
        (with_pose, MARGIN_SECOND_NEW, 1e-6),
        (without_pose, MARGIN_SECOND_NEW, None),                                 # returns 0
        (wide, MARGIN_SECOND_NEW, 1e-5),                                         # WIDE
    ]
    wins, modes = [c[0] for c in cases], [c[1] for c in cases]
    s = BundleAdjuster(0)
    try:
        assert s.optimization(wins[4].clone())["reduced_dim"] == 179
    finally:
        s.close()
    priors, status, infos, _ = check_batch(wins, modes)
    assert status[10] == 0 and all(st > 0 for k, st in enumerate(status) if k != 10)
    assert priors[5].n > 0 and 1 in priors[5].kinds
    paths = [i[0] for i in infos]
    assert any(p == 0 for p in paths)                                            # fast path
    assert paths[7] & MARG_PATH_NOT_PD and paths[7] & MARG_PATH_GENERIC
    assert paths[8] & MARG_PATH_WIDE and paths[8] & MARG_PATH_REDUCED_JACOBI and paths[11] & MARG_PATH_WIDE
    assert 0 < infos[7][1] < 60 and 0 < infos[8][2] < 60
    for (pb, mode, tol), pr in zip(cases, priors):
        if tol is None:
            assert O.marginalize_second_new(pb) is None
            continue
        want = O.marginalize_old(pb) if mode == MARGIN_OLD else O.marginalize_second_new(pb)
        _compare_priors(pr, want, tol=tol)


def test_batch_of_one_equals_the_single_calls():
    pb = solved(seed=3)
    with_pose, _ = second_new_pair(9)
    for w, m in ((pb, MARGIN_OLD), (with_pose, MARGIN_SECOND_NEW)):
        h = BundleAdjuster(0)
        try:
            check_batch([w], [m], hs=[h])
        finally:
            h.close()


def _launches():
    return _lib.lib().gf_kernel_launch_count()


def test_launch_count_does_not_depend_on_the_batch_size():
    c2 = [solved(seed=20 + k) for k in range(4)]
    wide = [wide_window(30 + k) for k in range(3)]
    hs = handles(6)
    try:
        def count(wins):
            c0 = _launches(); marginalize_multi(hs[:len(wins)], [w.clone() for w in wins], [MARGIN_OLD] * len(wins))
            return _launches() - c0
        one, four = count(c2[:1]), count(c2)
        assert one == four
        mixed2, mixed6 = count([c2[0], wide[0]]), count([c2[0], wide[0], c2[1], wide[1], c2[2], wide[2]])
        assert mixed2 == mixed6 > one
    finally:
        close(hs)


def _raw(hs, n, p_array, modes, outs, bufs, kept):
    L = _lib.lib()
    dp = ctypes.POINTER(ctypes.c_double)
    L.gf_ba_marginalize_multi.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    harr = (ctypes.c_void_p * len(hs))(*[h._h.value for h in hs]) if hs is not None else None
    ptrs = [(dp * len(bufs))(*[b[j].ctypes.data_as(dp) if b[j] is not None else None for b in bufs]) for j in range(3)]
    m = np.ascontiguousarray(modes, np.int32) if modes is not None else None
    rc = L.gf_ba_marginalize_multi(harr, n, p_array, m.ctypes.data if m is not None else None, outs, ptrs[0], ptrs[1], ptrs[2],
                                   kept.ctypes.data if kept is not None else None, None)
    return rc, L.gf_last_error().decode()


def _outputs(wins):
    bufs = [[np.full(16 * w.n_frames + 24, 7.0), np.full((16 * w.n_frames + 24) ** 2, 7.0), np.full(16 * w.n_frames + 24, 7.0)] for w in wins]
    return (BaPrior * len(wins))(), bufs, np.full(len(wins), 99, np.int32)


def _untouched(outs, bufs, kept):
    return (all(o.n == 0 and o.n_blocks == 0 for o in outs) and all((b == 7.0).all() for bb in bufs for b in bb)
            and (kept == 99).all())


def test_argument_errors_write_nothing():
    wins = [solved(seed=70 + k, n_landmarks=60) for k in range(3)]
    hs = handles(3)
    try:
        arr = (BaProblem * 3)(*[w.struct() for w in wins])
        ok = [MARGIN_OLD] * 3
        outs, bufs, kept = _outputs(wins)
        assert _raw(None, 3, arr, ok, outs, bufs, kept)[0] == GF_ERR_INVALID_ARG
        assert _raw(hs, 3, None, ok, outs, bufs, kept)[0] == GF_ERR_INVALID_ARG
        assert _raw(hs, 3, arr, None, outs, bufs, kept)[0] == GF_ERR_INVALID_ARG
        assert _raw(hs, 3, arr, ok, None, bufs, kept)[0] == GF_ERR_INVALID_ARG
        assert _raw(hs, 3, arr, ok, outs, bufs, None)[0] == GF_ERR_INVALID_ARG
        for n in (0, -1):
            assert _raw(hs, n, arr, ok, outs, bufs, kept)[0] == GF_ERR_INVALID_ARG
        rc, msg = _raw([hs[0], hs[1], hs[0]], 3, arr, ok, outs, bufs, kept)
        assert rc == GF_ERR_INVALID_ARG and msg.startswith("window 2:")
        rc, msg = _raw(hs, 3, arr, [MARGIN_OLD, 5, MARGIN_OLD], outs, bufs, kept)
        assert rc == GF_ERR_INVALID_ARG and msg.startswith("window 1:") and "mode" in msg
        bad = wins[1].clone()
        bad.visual[5].imu_j = 11                                                       # frame index out of range
        rc, msg = _raw(hs, 3, (BaProblem * 3)(wins[0].struct(), bad.struct(), wins[2].struct()), ok, outs, bufs, kept)
        assert rc == GF_ERR_INVALID_ARG and msg.startswith("window 1:") and "visual factor" in msg
        nobuf = [bufs[0], bufs[1], [bufs[2][0], None, bufs[2][2]]]
        rc, msg = _raw(hs, 3, arr, ok, outs, nobuf, kept)
        assert rc == GF_ERR_INVALID_ARG and msg.startswith("window 2:")
        assert _untouched(outs, bufs, kept)
        check_batch(wins, ok, hs=hs)                                                   # and the handles still work
    finally:
        close(hs)


def test_largest_batch_and_one_more():
    wins = [short_window(4) for _ in range(MAX_MULTI + 1)]
    hs = handles(MAX_MULTI + 1)
    try:
        arr = (BaProblem * (MAX_MULTI + 1))(*[w.struct() for w in wins])
        outs, bufs, kept = _outputs(wins)
        rc, msg = _raw(hs, MAX_MULTI + 1, arr, [MARGIN_OLD] * (MAX_MULTI + 1), outs, bufs, kept)
        assert rc == GF_ERR_CAPACITY and _untouched(outs, bufs, kept)
        want = single(hs[0], wins[0].clone(), MARGIN_OLD)[0]
        priors, status = marginalize_multi(hs[:MAX_MULTI], [w.clone() for w in wins[:MAX_MULTI]], [MARGIN_OLD] * MAX_MULTI)
    finally:
        close(hs)
    assert status == [want.n] * MAX_MULTI
    for pr in priors:
        assert_same_prior(pr, want)


def test_singular_imu_covariance_fails_only_its_window():
    wins = [solved(seed=80 + k) for k in range(3)]
    bad = wins[1]
    cov = np.array(bad.imu[0].covariance).reshape(15, 15)                             # IMU(0->1): the factor MARGIN_OLD evaluates
    cov[7, :] = 0.0; cov[:, 7] = 0.0
    bad.imu[0].covariance[:] = list(cov.ravel())
    priors, status, _, _ = check_batch(wins, [MARGIN_OLD] * 3)
    assert status[1] == GF_ERR_INVALID_ARG and status[0] > 0 and status[2] > 0 and priors[1] is None
    msg = _lib.lib().gf_last_error().decode()
    assert msg.startswith("window 1:") and "covariance" in msg


def test_handles_after_a_batch():
    """Handles that served a batch give the same single solves and marginalisations as a fresh one; a later batch of larger
    windows grows their buffers."""
    small = [solved(seed=100 + k, n_landmarks=60) for k in range(3)]
    large = [solved(seed=110 + k, n_landmarks=440) for k in range(3)]
    hs = handles(3)
    fresh = BundleAdjuster(0)
    try:
        marginalize_multi(hs, [w.clone() for w in small], [MARGIN_OLD] * 3)
        for h in hs:
            pb = make_window(seed=120)[0]
            b, w = pb.clone(), pb.clone()
            sg, sw = h.optimization(b), fresh.optimization(w)
            assert (sg["iterations"], sg["termination"]) == (sw["iterations"], sw["termination"])
            np.testing.assert_allclose(b.para_pose, w.para_pose, rtol=0, atol=1e-8)
            assert_same_prior(h.marginalize_old(b), fresh.marginalize_old(b))
        check_batch(large, [MARGIN_OLD] * 3, hs=hs, ref=fresh)
    finally:
        close(hs); fresh.close()


# ---- the C++ adaptor: Estimator::optimizationMulti marginalises with gf_ba_marginalize_multi ----
def test_adaptor_optimization_multi_mixed_flags(tmp_path):
    """Three estimators over three rounds whose marginalization_flag differs within a round: one optimizationMulti call per
    round against each estimator's optimization() in turn, at test_ba_multi_gpu.test_adaptor_optimization_multi's bars.  Each
    estimator stays on one scene and the solves may take 16 iterations: a prior taken from an unrelated window leaves the solve
    far from converged after 8, where the last-bit differences of two runs (atomic summation order) grow to 2e-3 of the cost
    by the third round."""
    from test_adaptor import _dump_window, build
    from test_ba_multi_gpu import _read_multi
    exe = build()
    flags = [[0, 0, 0], [1, 0, 1], [0, 1, 0]]
    chains = [[make_window(seed=200 + 10 * e, n_landmarks=150)[0] for r in range(3)] for e in range(3)]
    with open(tmp_path / "in.bin", "wb") as f:
        f.write(struct.pack("<4i3d", 3, 11, 9, 16, *chains[0][0].gravity))
        for r in range(3):
            for e in range(3):
                _dump_window(f, chains[e][r], flags[r][e])
    subprocess.check_call([exe, "ba-multi", str(tmp_path / "in.bin"), str(tmp_path / "multi.out")], timeout=120)
    subprocess.check_call([exe, "ba-seq", str(tmp_path / "in.bin"), str(tmp_path / "seq.out")], timeout=120)
    got, want = _read_multi(tmp_path / "multi.out", chains), _read_multi(tmp_path / "seq.out", chains)
    for k, (g, w) in enumerate(zip(got, want)):
        assert (g["it"], g["term"], g["pdim"]) == (w["it"], w["term"], w["pdim"]) and g["pdim"] > 0
        tol = 1e-9 if k < 3 else 1e-4
        np.testing.assert_allclose(g["cost"], w["cost"], rtol=tol)
        np.testing.assert_allclose(g["pose"], w["pose"], atol=1e3 * tol)
        np.testing.assert_allclose(g["sb"], w["sb"], atol=1e4 * tol)
        H, Hw = g["J"].T @ g["J"], w["J"].T @ w["J"]
        scale = np.sqrt(np.outer(np.diag(Hw), np.diag(Hw))) + 1e-300
        assert np.abs((H - Hw) / scale).max() < (1e-5 if k < 3 else 1e-3)
