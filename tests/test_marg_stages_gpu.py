"""GPU: the marginalisation stage by stage (gf_stage_sym_eig, gf_stage_marginalize) against the high-precision references of
tests/marg_ref.py, and the literal eigen path of gf_ba_marginalize_old on windows that reach it at large m.

Bars (ratio = error / (n eps scale), K calibrated in marg_ref.py against the oracle's C restatements on the same inputs):
  eigensolvers: sorted eigenvalues, ||V^T V - I||, ||A V - V diag(w)||, spectral projectors of separated clusters;
  marginalisation: J0^T J0 and J0^T r0 entry by entry, r0^T r0 = b^T A^+ b, and J0's nonzero row count exactly.
Every test asserts the path it meant to reach.
"""
import numpy as np
import pytest

import marg_ref as R
from ground_fusion_b200._lib import MARG_PATH_FORCED, MARG_PATH_GENERIC, MARG_PATH_NOT_PD, MARG_PATH_REDUCED_JACOBI, MARG_PATH_WIDE
from ground_fusion_b200.synth_ba import make_window
from oracle import ba_oracle as O

pytestmark = pytest.mark.gpu

JACOBI_SWEEP_CAP = 60


def _check_eig(method, kind, n):
    from ground_fusion_b200.estimator import sym_eig
    A, lam, Q = R.eig_case(kind, n)
    w, V, sweeps = sym_eig(A, method)
    r = R.eig_ratios(A, lam, Q, w, V)
    assert r["eigval"] <= R.K_EIGVAL and r["orth"] <= R.K_ORTH and r["resid"] <= R.K_RESID and r["proj"] <= R.K_PROJ, (r, kind, n)
    if method == "jacobi":
        assert sweeps < JACOBI_SWEEP_CAP, sweeps
    else:
        assert sweeps == 0
    return r, sweeps


@pytest.mark.parametrize("kind", R.EIG_KINDS)
@pytest.mark.parametrize("n", R.QL_SIZES)
def test_ql_against_known_spectra(n, kind):
    """k_sym_eig_ql (the reduced system's solver, n <= 128)."""
    r, _ = _check_eig("ql", kind, n)
    print("ql", n, kind, {k: round(v, 3) for k, v in r.items()})


@pytest.mark.parametrize("kind", R.EIG_KINDS)
@pytest.mark.parametrize("n", R.JACOBI_SIZES)
def test_jacobi_against_known_spectra(n, kind):
    """k_jacobi_eig in global memory (Amm of the literal path; reduced systems with n > 128).  The gauge kind has entries of
    1e9 next to exact zeros: the off-norm stalls at the rounding floor and the kernel's stall exit must end it."""
    r, sweeps = _check_eig("jacobi", kind, n)
    if kind in ("diagonal", "zero"):
        assert sweeps == 0
    print("jacobi", n, kind, sweeps, {k: round(v, 3) for k, v in r.items()})


def test_jacobi_at_the_stage_bound():
    """k_jacobi_eig at n = 2304, the largest size gf_stage_sym_eig takes: 1152 rotation pairs per round for 1024 threads,
    so some threads set up two rotations.  Three-by-three blocks scattered over random indices pair low and high indices
    in every round; the products of the bars are formed in double (see marg_ref.eig_ratios)."""
    from ground_fusion_b200.estimator import sym_eig
    A, lam, Q = R.eig_case_bound()
    w, V, sweeps = sym_eig(A, "jacobi")
    r = R.eig_ratios(A, lam, Q, w, V, dt=np.float64)
    print("jacobi", R.JACOBI_BOUND, "bound", sweeps, {k: round(v, 4) for k, v in r.items()})
    assert r["eigval"] <= R.K_EIGVAL and r["orth"] <= R.K_ORTH and r["resid"] <= R.K_RESID and r["proj"] <= R.K_PROJ, r
    assert sweeps < JACOBI_SWEEP_CAP


def test_sym_eig_rejects_sizes_it_cannot_take():
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.estimator import sym_eig
    with pytest.raises(GfError, match="bad argument"):
        sym_eig(np.eye(129), "ql")
    with pytest.raises(GfError, match="bad argument"):
        sym_eig(np.eye(R.JACOBI_BOUND + 1), "jacobi")


def _expected_bits(n, forced, ref_path):
    bits = MARG_PATH_REDUCED_JACOBI if n > 128 else 0
    if n > 127:
        return bits | MARG_PATH_GENERIC | MARG_PATH_WIDE
    if forced:
        return bits | MARG_PATH_GENERIC | MARG_PATH_FORCED
    return bits | (MARG_PATH_GENERIC | MARG_PATH_NOT_PD if ref_path == "generic" else 0)


@pytest.mark.parametrize("name,c,L,n,kw,ref_path", R.marg_cases(), ids=[x[0] for x in R.marg_cases()])
def test_marginalize_stage_against_reference(name, c, L, n, kw, ref_path):
    """gf_stage_marginalize, fast path (or the literal one where the positive-definiteness test must fail) and forced literal
    path on the same system: both against the reference, and against each other."""
    from ground_fusion_b200.estimator import marginalize_dense
    A, b = R.marg_case(c, L, n, **kw)
    ref = R.marginalize_ld(A, b, c, L)
    assert ref["path"] == ref_path
    got = {}
    # at the Jacobi bound the default run already takes the literal path (a landmark without information); a forced run
    # would repeat the same minute-long decomposition
    for forced in (False, True) if c + L < R.JACOBI_BOUND else (False,):
        J0, r0, path = marginalize_dense(A, b, c, L, force_generic=forced)
        assert path[0] == _expected_bits(n, forced, ref_path), (path, forced)
        if path[0] & MARG_PATH_GENERIC:
            assert 0 <= path[1] < JACOBI_SWEEP_CAP
        if path[0] & MARG_PATH_REDUCED_JACOBI:
            assert 0 < path[2] < JACOBI_SWEEP_CAP
        r = R.marg_ratios(J0, r0, ref)
        print(name, "forced" if forced else "default", path, ref["rank"], {k: round(v, 4) for k, v in r.items()})
        assert r["rank"] == ref["rank"] == n - kw["null"]
        assert r["jtj"] <= R.K_JTJ and r["jtr"] <= R.K_JTR and r["rtr"] <= R.K_RTR, r
        got[forced] = (J0.T @ J0, J0.T @ r0, r0 @ r0)
    if True not in got:
        return
    unit = ref["N"] * R.EPS
    assert np.abs(got[False][0] - got[True][0]).max() <= 2 * R.K_JTJ * unit * ref["schur_scale"]
    assert np.abs(got[False][1] - got[True][1]).max() <= 2 * R.K_JTR * unit * ref["b_scale"]
    assert abs(got[False][2] - got[True][2]) <= 2 * R.K_RTR * unit * ref["rtr_scale"]


def test_marginalize_stage_rejects_what_the_solver_never_builds():
    from ground_fusion_b200._lib import GfError
    from ground_fusion_b200.estimator import marginalize_dense
    A, b = R.marg_case(6, 4, 5, seed=1)
    bad = A.copy(); bad[7, 8] = bad[8, 7] = 1.0                 # two landmarks sharing information
    with pytest.raises(GfError, match="not diagonal"):
        marginalize_dense(bad, b, 6, 4)
    with pytest.raises(GfError, match="bad argument"):
        marginalize_dense(A, b, 6, 9)                            # n = 0
    with pytest.raises(GfError, match="bad argument"):
        marginalize_dense(A, b, 16, 0)                           # c > 15
    A2, b2 = R.marg_case(6, 0, 199, seed=2)
    with pytest.raises(GfError, match="bad argument"):
        marginalize_dense(A2, b2, 6, 0)                          # n > 16 * GF_BA_MAX_FRAMES + 22
    N3 = R.JACOBI_BOUND + 2
    with pytest.raises(GfError, match="bad argument"):
        marginalize_dense(np.eye(N3), np.ones(N3), 6, N3 - 7)    # m = 2305 > the Jacobi bound


# ------------------------------------------------------------------------------------------------ windows on the literal path
@pytest.fixture(scope="module")
def ba():
    from ground_fusion_b200.estimator import BundleAdjuster
    b = BundleAdjuster(0)
    yield b
    b.close()


def _rows(pb):
    return [(f.imu_i, f.imu_j, f.feature, list(f.pts_i), list(f.pts_j), list(f.vel_i), list(f.vel_j), f.td_i, f.td_j)
            for f in list(pb.visual)[:pb.n_visual]]


def _stationary_start(pb, frac):
    """Frames 0 and 1 share one pose (the robot stood still) and a fraction of the landmarks starting in frame 0 are seen
    only there, at the same bearing: their inverse depth has no information (d r / d lambda = 0, D_ll = 0)."""
    pb.para_pose[1] = pb.para_pose[0]
    rows = _rows(pb)
    firsts = sorted({r[2] for r in rows if r[0] == 0})
    flat = set(firsts[::int(round(1 / frac))])
    out = [r for r in rows if r[2] not in flat]
    for fid in sorted(flat):
        r0 = next(r for r in rows if r[2] == fid and r[0] == 0)
        out.append((0, 1, fid, r0[3], r0[3], [0, 0], [0, 0], 0.0, 0.0))
    pb.set_visual(out)
    return len(flat)


def _window_check(ba, pb, tol):
    from test_ba_gpu import _compare_priors
    want = O.marginalize_old(pb)
    got = ba.marginalize_old(pb)
    info = ba.last_marg_info()
    assert info[0] & MARG_PATH_NOT_PD and info[0] & MARG_PATH_GENERIC, info
    assert 0 < info[1] < JACOBI_SWEEP_CAP
    _compare_priors(got, want, tol=tol)
    return got, info


def test_stationary_start_window_takes_the_literal_path(ba):
    """A C2 window whose first two frames share one pose, half of frame 0's landmarks without information: Jacobi on the
    whole Amm (m ~ 190) with dozens of exact zero eigenvalues, against the oracle."""
    pb, _ = make_window(seed=11)
    O.solve(pb)
    n_flat = _stationary_start(pb, 0.5)
    got, info = _window_check(ba, pb, 1e-6)
    m = 15 + len({f.feature for f in list(pb.visual)[:pb.n_visual] if f.imu_i == 0})
    print("stationary start: m = %d (%d landmarks without information), n = %d, path %s, sweeps %d, %.3f ms"
          % (m, n_flat, got.n, info[0], info[1], ba.last_marg_ms))
    assert m > 150


def test_c3_window_on_the_literal_path(ba):
    """A C3-sized window (440 landmarks) with one landmark of frame 0 without information: the literal path at C3's m."""
    pb, _ = make_window(seed=7, n_landmarks=440)
    O.solve(pb)
    pb.para_pose[1] = pb.para_pose[0]
    k = pb.n_features
    rows = _rows(pb)
    rows.append((0, 1, k, [0.1, -0.05, 1.0], [0.1, -0.05, 1.0], [0, 0], [0, 0], 0.0, 0.0))
    pb.n_features = k + 1
    pb.para_feature = np.append(pb.para_feature[:k], 0.5)
    pb.feature_const = np.append(pb.feature_const[:k], 0).astype(np.uint8)
    pb.set_visual(rows)
    got, info = _window_check(ba, pb, 1e-5)
    m = 15 + len({f.feature for f in list(pb.visual)[:pb.n_visual] if f.imu_i == 0})
    print("C3 window: m = %d, n = %d, path %s, sweeps %d, %.3f ms" % (m, got.n, info[0], info[1], ba.last_marg_ms))
    assert m > 250
