"""CPU: the marginalisation references of tests/marg_ref.py, pinned before the GPU tests (test_marg_stages_gpu.py) rely on them.

  * the longdouble / structured restatement against the literal one in mpmath on small systems;
  * both against the oracle's MARGIN_OLD (oracle/ba_oracle.c) on a real window's dense system;
  * the known-spectrum matrices against mpmath;
  * calibration: on the GPU tests' inputs the oracle's C restatements of the two eigensolvers (QL, Jacobi) stay below
    K / CALIBRATION_FACTOR of every bar, so each GPU bar K sits that factor above what the algorithms achieve in double.
"""
import numpy as np
import pytest

import marg_ref as R
from ground_fusion_b200.synth_ba import make_window
from oracle import ba_oracle as O


@pytest.mark.parametrize("c,L,n,kw", [(6, 0, 5, dict(null=2)), (6, 4, 6, dict(null=2)), (15, 3, 4, dict(null=1)),
                                      (6, 5, 5, dict(null=1, dead=(1,))), (6, 5, 5, dict(null=1, tiny=(2,))),
                                      (6, 5, 5, dict(null=1, c_eig=3e-9))])
def test_longdouble_reference_matches_mpmath(c, L, n, kw):
    A, b = R.marg_case(c, L, n, seed=c + 7 * L + n, **kw)
    ld, hp = R.marginalize_ld(A, b, c, L), R.marginalize_mp(A, b, c + L)
    assert ld["rank"] == hp["rank"] == n - kw["null"]
    s = np.abs(hp["Ar"]).max()
    assert float(np.abs(ld["Ar"] - hp["Ar"]).max()) <= 1e-17 * float(s)
    # the dropped subspace turns by (rounding of Ar) / gap, gap ~ 1e-5: the two agree to 1/1000 of the GPU bars' unit
    unit = hp["N"] * R.EPS
    assert float(np.abs(ld["JtJ"] - hp["JtJ"]).max()) <= 1e-3 * unit * hp["schur_scale"]
    assert float(np.abs(ld["Jtr"] - hp["Jtr"]).max()) <= 1e-3 * unit * hp["b_scale"]
    assert abs(float(ld["rtr"] - hp["rtr"])) <= 1e-3 * unit * hp["rtr_scale"]
    if kw.get("dead") or kw.get("tiny") or kw.get("c_eig"):
        assert ld["path"] == "generic"


def test_known_spectrum_longdouble_matches_mpmath():
    lam = np.concatenate([np.zeros(4), np.logspace(0, 9, 29)])
    A1, Q1, w1 = R.known_spectrum(lam, 3, exact="mp")
    A2, Q2, w2 = R.known_spectrum(lam, 3, exact="ld")
    assert np.abs(A1 - A2).max() <= 2 * R.EPS * 1e9
    assert float(np.abs(Q1 - Q2).max()) <= 1e-17
    assert w1 <= 33 * R.EPS * 1e9 and w2 <= 33 * R.EPS * 1e9           # the Weyl bound of the one rounding


def test_refined_eigh_is_accurate_beyond_double():
    A, lam, Q = R.eig_case("multiple", 64)
    w, X = R.refine_eigh(A.astype(R.LD))
    n = len(lam)
    assert float(np.abs(X.T @ X - np.eye(n, dtype=R.LD)).max()) < 1e-17
    assert float(np.abs(A.astype(R.LD) @ X - X * w).max()) < 1e-16 * 5


def _window_system(seed):
    """The dense (A, b) of MARGIN_OLD's factor set on a solved window, columns [pose0 | sb0 | landmarks of frame 0 | kept],
    as in test_ba_oracle.test_marginalization_is_the_schur_complement, and the oracle's prior on the same window."""
    pb, _ = make_window(seed=seed, n_landmarks=90)
    q = pb.clone(); O.solve(q)
    prior = O.marginalize_old(q)
    sub = q.clone()
    rows = [(f.imu_i, f.imu_j, f.feature, list(f.pts_i), list(f.pts_j), list(f.vel_i), list(f.vel_j), f.td_i, f.td_j)
            for f in list(q.visual)[:q.n_visual] if f.imu_i == 0]
    sub.set_visual(rows)
    sub.n_imu = 1
    sub.feature_const[:] = 0; sub.ex_pose_const = 0; sub.td_const = 0
    r, J = O.linearize(sub)
    H, g = J.T @ J, J.T @ r
    pose = lambda f: list(range(6 * f, 6 * f + 6)); sb = lambda f: list(range(66 + 9 * f, 66 + 9 * f + 9))
    lms = [c for c in range(66 + 99 + 7, J.shape[1]) if np.any(J[:, c] != 0)]
    keep = []
    for (c, k), i in sorted(zip(zip(prior.idx, prior.kinds), prior.indices)):
        keep += pose(i + 1) if k == 0 else sb(i + 1) if k == 1 else list(range(165, 171)) if k == 2 else [171]
    order = pose(0) + sb(0) + lms + keep
    A = H[np.ix_(order, order)]
    A = np.tril(A) + np.tril(A, -1).T
    lm = np.arange(15, 15 + len(lms))
    A[np.ix_(lm, lm)] = np.diag(np.diag(A)[lm])        # landmarks never share a residual: the block is diagonal up to rounding
    return A, g[order], 15, len(lms), prior


def test_reference_matches_the_oracle_on_a_window():
    A, b, c, L, prior = _window_system(5)
    ref = R.marginalize_ld(A, b, c, L)
    assert ref["path"] == "fast" and len(b) - c - L == prior.n
    assert ref["rank"] == np.count_nonzero(np.any(prior.J != 0, axis=1))
    # the oracle (Jacobi in double on the whole Amm, prior columns in block_idx order) against the reference: this Amm holds
    # eigenvalues near 1e-8 (weak landmarks), so the first-order scales of marg_ratios say little here; the entry-scaled
    # agreement test_ba_gpu asks of the GPU against the oracle (1e-6) holds for the oracle against the reference
    Hw, bw = prior.J.T @ prior.J, prior.J.T @ prior.r
    scale = np.sqrt(np.outer(np.diag(Hw), np.diag(Hw))) + 1e-300
    assert float(np.abs((ref["JtJ"].astype(np.float64) - Hw) / scale).max()) < 1e-6
    assert float(np.abs(ref["Jtr"].astype(np.float64) - bw).max()) < 1e-6 * np.abs(bw).max()


def _worst(items):
    worst = {}
    for name, r in items:
        for k, v in r.items():
            if k != "rank" and v > worst.get(k, (0.0, None))[0]:
                worst[k] = (v, name)
    return worst


@pytest.mark.parametrize("method", ["ql", "jacobi"])
def test_eigensolver_bars_are_calibrated(method):
    """Calibration of K_EIGVAL, K_ORTH, K_RESID, K_PROJ on the GPU tests' inputs (the oracle's restatement of each kernel)."""
    sizes = R.QL_SIZES if method == "ql" else R.JACOBI_SIZES
    items = []
    for n in sizes:
        for kind in R.EIG_KINDS:
            A, lam, Q = R.eig_case(kind, n)
            w, V = O.sym_eig(A, method)
            items.append(((kind, n), R.eig_ratios(A, lam, Q, w, V)))
    if method == "jacobi":
        A, lam, Q = R.eig_case_bound()
        w, V = O.sym_eig(A, method)
        items.append((("bound", R.JACOBI_BOUND), R.eig_ratios(A, lam, Q, w, V, dt=np.float64)))
    worst = _worst(items)
    print(method, worst)
    K = dict(eigval=R.K_EIGVAL, orth=R.K_ORTH, resid=R.K_RESID, proj=R.K_PROJ)
    for k, (v, where) in worst.items():
        assert v * R.CALIBRATION_FACTOR <= K[k], (k, v, where)


def test_marginalization_bars_are_calibrated():
    """Calibration of K_JTJ, K_JTR, K_RTR: the literal algorithm in double with the oracle's QL and Jacobi, on the GPU tests'
    systems; the count of kept eigenvalues matches the reference's exactly, and the reference takes the path the GPU test
    expects.  The oracle's sequential Jacobi on the 2304 x 2304 Amm of the bound case takes over ten minutes, so that case
    is calibrated with QL alone."""
    items = []
    for name, c, L, n, kw, path in R.marg_cases():
        A, b = R.marg_case(c, L, n, **kw)
        ref = R.marginalize_ld(A, b, c, L)
        assert ref["path"] == path, name
        for method in ("ql", "jacobi") if c + L <= 600 else ("ql",):
            J0, r0 = R.marginalize_f64(A, b, c + L, lambda M: O.sym_eig(M, method))
            r = R.marg_ratios(J0, r0, ref)
            assert r["rank"] == ref["rank"], (name, method)
            items.append(((name, method), r))
    worst = _worst(items)
    print(worst)
    K = dict(jtj=R.K_JTJ, jtr=R.K_JTR, rtr=R.K_RTR)
    for k, (v, where) in worst.items():
        assert v * R.CALIBRATION_FACTOR <= K[k], (k, v, where)
