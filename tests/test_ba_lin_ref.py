"""CPU: the reference of the solve's first iteration (tests/ba_lin_ref.py), pinned before test_ba_lin_stages_gpu.py relies on it.

  * the longdouble computation against mpmath on small windows;
  * calibration: the same computation in double, on a Jacobian evaluated with FMA contraction, stays below K / CALIBRATION_FACTOR
    of every bar on the windows and trust-region branches the GPU tests use; the IMU sqrt-information of the oracle (double)
    likewise against mpmath;
  * the oracle refuses a visual factor whose two frames are the same.
"""
import mpmath as mp
import numpy as np
import pytest

import ba_lin_ref as R
from ground_fusion_b200.synth_ba import make_window
from oracle import ba_oracle as O


def _mp_reference(pb, mu=1e-8, dps=40):
    """H' + mu D^2 and the Gauss-Newton step of the whole (unreduced) system in mpmath, from the same Jacobian."""
    blocks, pn, L = R.layout(pb)
    r, J = R.linearization(pb)
    with mp.workdps(dps):
        Jm, rm = mp.matrix(J.tolist()), mp.matrix(r.tolist())
        H = Jm.T * Jm
        g = Jm.T * rm
        n = H.rows
        s = [1 / (1 + mp.sqrt(H[a, a])) for a in range(n)]
        A = mp.matrix(n, n); b = mp.matrix(n, 1)
        for a in range(n):
            b[a] = g[a] * s[a]
            for c in range(n):
                A[a, c] = H[a, c] * s[a] * s[c]
        D2 = [min(max(A[a, a], mp.mpf(R.DIAG_MIN)), mp.mpf(R.DIAG_MAX)) for a in range(n)]
        for a in range(n):
            A[a, a] += mu * D2[a]
        y = mp.lu_solve(A, b)
        gn = np.array([float(-mp.sqrt(D2[a]) * y[a]) for a in range(n)])
        return np.array(H.tolist(), dtype=float), np.array([float(x) for x in g]), gn


@pytest.mark.parametrize("F,seed", [(4, 1), (5, 2)])
def test_longdouble_reference_matches_mpmath(F, seed):
    pb, _ = make_window(seed=seed, n_frames=F, n_landmarks=40)
    pb.n_imu = 0; pb.pose0_const = 1
    ref = R.reference(pb, radius=1e300)
    H, g, gn = _mp_reference(pb)
    nc = ref["nc"]
    assert nc == 6 * (F - 1) and ref["L"] > 0
    Hs = np.sqrt(np.outer(np.diag(H), np.diag(H)))
    assert np.abs(np.asarray(ref["H"], float) - H[:nc, :nc]).max() <= 1e-3 * R.EPS * Hs[:nc, :nc].max()
    assert np.abs(np.asarray(ref["g"], float) - g).max() <= 1e-3 * R.EPS * np.abs(ref["absJr"]).max()
    assert ref["branch"] == "gauss_newton"
    # the reference's Schur route and the whole system's LU at 40 digits: far below the GPU bar's unit eps kappa
    assert np.linalg.norm(np.asarray(ref["gn"], float) - gn) <= 1e-2 * R.EPS * ref["kappa"] * np.linalg.norm(gn)


def _calibration_cases():
    w = R.windows()
    # L_large shares its factors' arithmetic with c3 and would hold two dense Jacobians of 0.5 GB each here; the GPU tests run it
    cases = [(name, None) for name in sorted(w) if name != "L_large"]
    cases += [(name, branch) for name in ("c2_s0", "plane", "wheel", "prior", "prior_plane")
              for branch in ("gauss_newton", "cauchy", "interpolated", "large_mu")]
    return w, cases


def test_calibration_of_the_bars():
    """K >= CALIBRATION_FACTOR x the worst ratio of the double computation, bar by bar (the numbers are printed)."""
    w, cases = _calibration_cases()
    worst = {}
    for name, branch in cases:
        pb = R.prior_window() if name == "prior" else w[name]()
        if branch is None:
            radius, mu = 1e4, 1e-8
        elif branch == "large_mu":
            radius, mu = 1e4, 0.1
        else:
            radius, mu = R.branch_radii(pb)[branch], 1e-8
        ref = R.reference(pb, radius, mu)
        if branch not in (None, "large_mu"):
            assert ref["branch"] == branch
        for k, v in R.ratios(R.f64_capture(pb, radius, mu), ref).items():
            if v > worst.get(k, (0.0, ""))[0]:
                worst[k] = (v, "%s/%s" % (name, branch or "default"))
    print()
    for k in sorted(worst):
        print("bar %-13s K %-9g worst CPU ratio %.3g (%s)" % (k, R.K[k], worst[k][0], worst[k][1]))
    for k, (v, where) in worst.items():
        assert R.CALIBRATION_FACTOR * v <= R.K[k], (k, v, where)


def test_calibration_of_the_sqrt_information():
    pb, _ = make_window(seed=1)
    worst = 0.0
    for kind in R.COV_KINDS:
        if kind == "indefinite":
            continue
        for k in range(pb.n_imu):
            cov = R.imu_covariance(pb.imu[k].covariance, kind, seed=k)
            U = np.zeros(225)
            assert O.lib().gfo_sqrt_info(np.ascontiguousarray(cov).ctypes.data_as(O._dp), 15, U.ctypes.data_as(O._dp)) == 0
            worst = max(worst, R.sqrt_info_ratio(U.reshape(15, 15), cov))
    print("\nbar sqrt_info     K %-9g worst CPU ratio %.3g" % (R.K["sqrt_info"], worst))
    assert R.CALIBRATION_FACTOR * worst <= R.K["sqrt_info"]


def test_covariance_kinds():
    cov = np.array(make_window(seed=1)[0].imu[0].covariance).reshape(15, 15)
    for kind in R.COV_KINDS:
        c = R.imu_covariance(cov, kind)
        w = np.linalg.eigvalsh(c)
        if kind == "indefinite":
            assert (w < 0).sum() == 1
        else:
            assert w.min() > 0
    g = np.linalg.eigvalsh(R.imu_covariance(cov, "graded"))
    assert g.max() / g.min() > 1e11
    assert (R.imu_covariance(cov, "zeros") == 0).sum() > 100


def test_window_shapes():
    """The windows reach what they are named for: the pair sizes around k_ba_eval's 64-factor chunks, a large L, a prior with
    plane blocks and with blocks that are constant in its window."""
    from ground_fusion_b200._lib import BLOCK_EX_POSE, BLOCK_EX_WHEEL, BLOCK_PLANE_R, BLOCK_PLANE_Z, BLOCK_TD
    for N in (1, 63, 64, 65, 128, 129):
        pb = R.windows()["pair%d" % N]()
        assert sum((pb.visual[v].imu_i, pb.visual[v].imu_j) == (0, 1) for v in range(pb.n_visual)) == N
    assert R.layout(R.windows()["L_large"]())[2] > 2000
    q = R.windows()["prior_plane"]()
    assert {BLOCK_PLANE_R, BLOCK_PLANE_Z, BLOCK_EX_POSE, BLOCK_TD, BLOCK_EX_WHEEL} <= set(q.prior.kinds)
    assert q.ex_pose_const and q.td_const and q.ex_wheel_const and not q.plane_const


def test_oracle_refuses_same_frame_visual_factor():
    pb, _ = make_window(seed=0)
    pb.visual[5].imu_j = pb.visual[5].imu_i
    assert O.lib().gfo_ba_solve(pb.struct(), O.BaSummary()) == -1
    with pytest.raises(RuntimeError, match="invalid window"):
        O.linearize(pb)
    with pytest.raises(RuntimeError):
        O.marginalize_old(pb)
    assert np.isnan(O.cost(pb))
