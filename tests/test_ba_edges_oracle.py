"""CPU side of the back end's edge tests (tests/test_ba_edges_gpu.py): the window builders those tests share, proof on the oracle
(oracle/ba_oracle.c) that every window reaches the path it is meant to reach, and the oracle's visual factor with feature
velocities and time offsets pinned by a NumPy restatement and by central differences.

The windows:
  stationary    systemstationary && stationary_detect (estimator.cpp:3233-3246): every pose / speed-bias block constant, the
                landmarks without depth free -- reduced dimension 0 with free landmarks
  rough         a far start that takes rejected steps (radius halved, the dogleg re-solved from the existing factor)
  visual-only   !USE_IMU: pose 0 constant, no IMU factors, no speed-bias blocks
  velocities    pts_i / pts_j compensated by (td - td_i) vel_i and (td - td_j) vel_j, the time offset free
  outliers      pixels moved by 20-40 px: the Huber corrector stays active at the optimum
  marginalisation priors whose kept dimension sits on either side of the fast path's 127-column limit
"""
import numpy as np
import pytest

from ground_fusion_b200.ba_problem import Prior
from ground_fusion_b200.synth_ba import make_window, q_to_R
from oracle import ba_oracle as O
from oracle import dogleg_witness as W

FOCAL = 460.0                      # pixels per unit of normalised image coordinates in synth_ba
# far starts, make_window(seed, pose_noise): 4 and 5 rejected steps within 16 iterations.  (6, (0.3, 0.1)) also rejects
# steps but fails the screening below: one of its decisions flips under a 1e-12 perturbation of the start
ROUGH = {9: (0.3, 0.1), 11: (0.3, 0.1)}


# ---- window builders ---------------------------------------------------------------------------------------------------
def stationary_window(with_wheel=False):
    pb, _ = make_window(seed=6, n_landmarks=120, with_wheel=with_wheel)
    pb.frames_const = 1
    return pb


def rough_window(seed):
    pb, _ = make_window(seed=seed, pose_noise=ROUGH[seed])
    pb.max_num_iterations = 16
    return pb


def visual_only_window(F, seed=None):
    pb, _ = make_window(seed=30 + F if seed is None else seed, n_frames=F)
    pb.n_imu = 0; pb.pose0_const = 1
    return pb


def short_window(F):
    pb, _ = make_window(seed=40 + F, n_frames=F)
    return pb


def add_velocities(pb, seed, sigma=0.05, para_td=0.004):
    """Feature velocities (normalised image units per second) on both ends of every visual factor, per-factor time offsets
    td_i != td_j != para_td, and the time offset free."""
    rng = np.random.default_rng(seed)
    for f in list(pb.visual)[:pb.n_visual]:
        f.vel_i[0], f.vel_i[1] = rng.normal(0, sigma, 2)
        f.vel_j[0], f.vel_j[1] = rng.normal(0, sigma, 2)
        f.td_i, f.td_j = rng.uniform(-0.01, 0.01, 2)
    pb.para_td[0] = para_td
    pb.td_const = 0
    return pb


def add_outliers(pb, seed, fraction=0.08):
    """Moves pts_j of `fraction` of the visual factors by 20-40 px in a random direction; returns their indices."""
    rng = np.random.default_rng(seed)
    idx = np.sort(rng.choice(pb.n_visual, int(round(fraction * pb.n_visual)), replace=False))
    for k in idx:
        a, d = rng.uniform(0, 2 * np.pi), rng.uniform(20.0, 40.0) / FOCAL
        f = pb.visual[int(k)]
        f.pts_j[0] += d * np.cos(a); f.pts_j[1] += d * np.sin(a)
    return idx


def truncate_frame0_tracks(pb, last):
    """Drops the visual factors (0, j) with j > last: the landmarks of frame 0 then reach frames 1..last only."""
    rows = [(f.imu_i, f.imu_j, f.feature, list(f.pts_i), list(f.pts_j), list(f.vel_i), list(f.vel_j), f.td_i, f.td_j)
            for f in list(pb.visual)[:pb.n_visual] if not (f.imu_i == 0 and f.imu_j > last)]
    pb.set_visual(rows)


def synthetic_prior(pb, poses, speed_biases, seed, weight=100.0):
    """An SPD prior r = r0 + J0 dx over the given pose / speed-bias blocks, linearised at their current values."""
    rng = np.random.default_rng(seed)
    kinds, indices, idx, x0 = [], [], [], []
    col = 0
    for f in poses:
        kinds.append(0); indices.append(f); idx.append(col); x0.extend(pb.para_pose[f]); col += 6
    for f in speed_biases:
        kinds.append(1); indices.append(f); idx.append(col); x0.extend(pb.para_speed_bias[f]); col += 9
    J = weight * (np.eye(col) + 0.05 * np.triu(rng.standard_normal((col, col)), 1))
    return Prior(kinds, indices, idx, np.array(x0), J, rng.normal(0, 0.1, col))


def marginalization_boundary_window(kept):
    """MARGIN_OLD windows whose kept dimension is exactly 127 (the largest the structured fast path takes) or 128 (the
    smallest that goes to the generic eigen path, and still to the QL eigensolver).  Kept: poses 1..8 (48), speed biases
    1..a (9a), ex_pose + td (7) and, with wheel factors, the wheel extrinsic, sx, sy, sw and time offset (10):
    127 = 48 + 72 + 7 (a = 8),  128 = 48 + 63 + 7 + 10 (a = 7, wheel)."""
    wheel = kept == 128
    a = {127: 8, 128: 7}[kept]
    pb, _ = make_window(seed=12, with_wheel=wheel)
    O.solve(pb)
    truncate_frame0_tracks(pb, 8)
    pb.prior = synthetic_prior(pb, range(1, 9), range(2, a + 1), seed=kept)
    return pb


# ---- what a solve did ---------------------------------------------------------------------------------------------------
def decisions(s):
    """Per iteration: 'A' step accepted / '-' not; radius '<' cut, '=' kept, '>' grown."""
    out = []
    for k in range(1, s["iterations"] + 1):
        c0, c1, r0, r1 = s["cost"][k - 1], s["cost"][k], s["radius"][k - 1], s["radius"][k]
        out.append(("A" if c1 < c0 else "-") + ("<" if r1 < r0 else ">" if r1 > r0 else "="))
    return out


def rejected_steps(s):
    return decisions(s).count("-<")


def screen(pb, copies=3):
    """The accept / reject sequence, termination and iteration count of pb must not change when the initial poses move by
    1e-12 relative: then no decision sits on a knife edge (rel near 1e-3, 0.25 or 0.75, a tolerance test near its bound), and
    a second implementation whose sums differ in the last bits takes the same path."""
    s0 = O.solve(pb.clone())
    rng = np.random.default_rng(0)
    for _ in range(copies):
        q = pb.clone()
        q.para_pose[:, :3] *= 1 + 1e-12 * rng.standard_normal((q.n_frames, 3))
        s = O.solve(q)
        assert (s["iterations"], s["termination"], decisions(s)) == (s0["iterations"], s0["termination"], decisions(s0))
    return s0


def visual_residual(pb, f, sqrt_info=None):
    """ProjectionTwoFrameOneCamFactor::Evaluate's residual in NumPy (projectionTwoFrameOneCamFactor.cpp:43-70)."""
    si = pb.visual_sqrt_info if sqrt_info is None else sqrt_info
    td = pb.para_td[0]
    vi, vj = np.array([f.vel_i[0], f.vel_i[1], 0.0]), np.array([f.vel_j[0], f.vel_j[1], 0.0])
    pts_i = np.array(f.pts_i) - (td - f.td_i) * vi
    pts_j = np.array(f.pts_j) - (td - f.td_j) * vj
    Pi, Ri = pb.para_pose[f.imu_i, :3], q_to_R(pb.para_pose[f.imu_i, 3:])
    Pj, Rj = pb.para_pose[f.imu_j, :3], q_to_R(pb.para_pose[f.imu_j, 3:])
    tic, ric = pb.para_ex_pose[:3], q_to_R(pb.para_ex_pose[3:])
    pw = Ri @ (ric @ (pts_i / pb.para_feature[f.feature]) + tic) + Pi
    pc = ric.T @ (Rj.T @ (pw - Pj) - tic)
    return si * (pc[:2] / pc[2] - pts_j[:2])


def huber_s(pb):
    """s = |r|^2 of every visual factor before the Huber corrector (s > 1: the corrector is active)."""
    return np.array([(visual_residual(pb, f) ** 2).sum() for f in list(pb.visual)[:pb.n_visual]])


# GPU windows and the iteration counts they run at, screened below
SCREENED = {
    **{"stationary_%d" % it: (lambda it=it: stationary_window(), it) for it in (1, 8, 16)},
    "stationary_wheel": (lambda: stationary_window(with_wheel=True), 16),
    **{"rough_%d" % s: (lambda s=s: rough_window(s), 16) for s in ROUGH},
    **{"c2_%d" % s: (lambda s=s: make_window(seed=s)[0], 16) for s in (0, 1, 2)},
    **{"visual_only_%d" % F: (lambda F=F: visual_only_window(F), 8) for F in range(2, 12)},
    **{"short_%d" % F: (lambda F=F: short_window(F), 8) for F in (1, 2, 3, 4, 6, 10)},
    "velocities": (lambda: add_velocities(make_window(seed=33)[0], 33), 8),
    "outliers": (lambda: (lambda pb: (add_outliers(pb, 32), pb)[1])(make_window(seed=32)[0]), 16),
}


@pytest.mark.parametrize("name", sorted(SCREENED))
def test_gpu_windows_take_no_knife_edge_decision(name):
    build, it = SCREENED[name]
    pb = build(); pb.max_num_iterations = it
    screen(pb)


def test_stationary_window_has_free_landmarks_and_no_reduced_system():
    for it in (1, 8, 16):
        pb = stationary_window(); pb.max_num_iterations = it
        q = pb.clone(); s = O.solve(q)
        assert s["reduced_dim"] == 0 and s["n_free_landmarks"] == 36 and s["iterations"] >= 1
        assert np.array_equal(q.para_pose, pb.para_pose) and np.array_equal(q.para_speed_bias, pb.para_speed_bias)
        assert np.abs(q.para_feature - pb.para_feature).max() > 1e-3        # the landmarks do move
    pb = stationary_window(with_wheel=True)
    s = O.solve(pb)
    assert s["reduced_dim"] == 10 and s["n_free_landmarks"] == 36


def test_rough_windows_reject_steps():
    for seed in ROUGH:
        s = O.solve(rough_window(seed))
        assert s["iterations"] == 16 and rejected_steps(s) >= 4, decisions(s)


def test_visual_only_and_short_windows_reach_their_layouts():
    for F in range(2, 12):
        s = O.solve(visual_only_window(F))
        assert s["reduced_dim"] == 6 * (F - 1)                 # no speed-bias columns, pose 0 constant
        assert (s["n_free_landmarks"] > 0) == (F >= 4)           # a landmark needs 4 consecutive observations
    for F in (1, 2, 3, 4, 6, 10):
        s = O.solve(short_window(F))
        assert s["reduced_dim"] == 15 * F and (s["n_free_landmarks"] > 0) == (F >= 4)
        if F in (2, 3):
            assert s["termination"] == 2 and s["final_cost"] < 1e-9        # IMU only: an exact fit, CONVERGENCE_PARAMETER


def test_visual_residual_with_velocities_matches_numpy():
    """The oracle's visual residual against the NumPy restatement, Huber off (sqrt_info = 1); the velocity terms matter."""
    pb = add_velocities(make_window(seed=33, n_landmarks=60)[0], 33)
    pb.visual_sqrt_info = 1.0
    r, _ = O.linearize(pb)
    rv = r[15 * pb.n_imu:].reshape(-1, 2)
    facs = list(pb.visual)[:pb.n_visual]
    want = np.array([visual_residual(pb, f) for f in facs])
    assert np.abs(rv - want).max() < 1e-12
    # the window reaches the compensation: dropping either velocity, or swapping them, moves the residual by far more than that
    for change in ("vel_i", "vel_j", "swap"):
        q = pb.clone()
        for f in list(q.visual)[:q.n_visual]:
            a, b = list(f.vel_i), list(f.vel_j)
            if change == "vel_i": f.vel_i[:] = [0.0, 0.0]
            elif change == "vel_j": f.vel_j[:] = [0.0, 0.0]
            else: f.vel_i[:], f.vel_j[:] = b, a
        moved = np.array([visual_residual(q, f) for f in list(q.visual)[:q.n_visual]])
        assert np.abs(moved - want).max() > 1e-5, change


def test_td_and_inverse_depth_columns_match_finite_differences_with_velocities():
    """Central differences of the oracle's td and inverse-depth columns with non-zero velocities and td_i != td_j != td
    (sqrt_info = 1: the Huber corrector is off, the corrected Jacobian is dr/dx)."""
    from test_ba_oracle import fd_jacobian
    pb = add_velocities(make_window(seed=34, n_landmarks=60)[0], 34)
    pb.visual_sqrt_info = 1.0
    col_td = 11 * 6 + 11 * 9                                     # poses, speed biases, then td (ex_pose constant)
    _, J = O.linearize(pb)
    L = J.shape[1] - col_td - 1
    assert L > 10
    J, num = fd_jacobian(pb, [col_td] + list(range(col_td + 1, col_td + 1 + L)))
    rows = slice(15 * pb.n_imu, None)
    for c, g in num.items():
        scale = np.abs(J[rows, c]).max()
        assert scale > 0
        assert np.abs(g[rows] - J[rows, c]).max() <= 1e-6 * scale + 1e-7, c
    # the velocity part of the td column is well above that bar
    q = pb.clone()
    for f in list(q.visual)[:q.n_visual]:
        f.vel_i[:] = [0.0, 0.0]
    _, Jq = O.linearize(q)
    assert np.abs(Jq[rows, col_td] - J[rows, col_td]).max() > 1e3 * (1e-6 * np.abs(J[rows, col_td]).max() + 1e-7)


def test_outliers_keep_the_huber_corrector_active_at_the_optimum():
    pb, _ = make_window(seed=32)
    idx = add_outliers(pb, 32)
    pb.max_num_iterations = 16
    O.solve(pb)
    s = huber_s(pb)
    mask = np.zeros(pb.n_visual, bool); mask[idx] = True
    assert mask.sum() >= 0.05 * pb.n_visual
    assert (s[mask] > 1).all() and np.median(s[~mask]) < 1


@pytest.mark.parametrize("kept", [127, 128])
def test_marginalization_boundary_windows_have_the_kept_dimension(kept):
    pb = marginalization_boundary_window(kept)
    pr = O.marginalize_old(pb)
    assert pr.n == kept


def test_witness_agrees_on_a_window_that_rejects_steps():
    pa = rough_window(9)
    pb = pa.clone()
    so, sw = O.solve(pa), W.solve(pb)
    assert so["iterations"] == sw["iterations"] and so["num_successful_steps"] == sw["successful"] and rejected_steps(so) > 0
    np.testing.assert_allclose(so["cost"], sw["cost"], rtol=1e-7)
    np.testing.assert_allclose(so["radius"], sw["radius"], rtol=1e-6)
