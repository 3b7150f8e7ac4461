"""GPU parity tests of the back end on the windows and trust-region branches the C2-style windows of test_ba_gpu.py never
build: stationary windows (reduced dimension 0), rejected steps, visual-only and short windows, feature velocities with a
free time offset, outliers, the marginalisation's fast / generic boundary, the free-landmark capacity, and several handles.
The windows come from test_ba_edges_oracle.py, which shows on the CPU that each one reaches its path and takes no
knife-edge decision; every test here asserts again that the path was taken.  Bar: test_ba_gpu.compare."""
import threading

import numpy as np
import pytest

from ground_fusion_b200.synth_ba import make_window
from oracle import ba_oracle as O
from test_ba_edges_oracle import (ROUGH, add_outliers, add_velocities, decisions, huber_s, marginalization_boundary_window,
                                  rejected_steps, rough_window, short_window, stationary_window, visual_only_window)
from test_ba_gpu import _compare_priors, assert_matches, compare

pytestmark = pytest.mark.gpu

# IMU-only windows (F = 2, 3: no landmark has 4 observations) have an exact fit: both solvers end at a cost of rounding
# noise (1e-22 .. 1e-13) whose relative difference means nothing.  Their costs are compared to 1e-9 absolute (chi-square
# units), every parameter block to the usual 1e-6.
EXACT_FIT_ATOL = 1e-9
# The far starts fall by 6-7 decades in their first steps, which amplifies 1e-13 differences of the step (atomic summation
# order, Schur vs dense elimination) to 1e-7 in the cost trace, as in test_ba_gpu's wheel windows; after 16 iterations they
# are still far from converged and their end cost is sensitive to summation order at the 1e-8 level (two GPU runs of the
# same window differ by up to 5e-9), as in test_ba_gpu's plane windows.  Blocks keep the 1e-6 bar.
ROUGH_TOL = dict(mid_rtol=1e-6, final_rtol=1e-7)


@pytest.fixture(scope="module")
def ba():
    from ground_fusion_b200.estimator import BundleAdjuster
    b = BundleAdjuster(0)
    yield b
    b.close()


@pytest.mark.parametrize("max_iter", [1, 8, 16])
def test_stationary_window_solves_the_landmarks_alone(ba, max_iter):
    """frames_const: reduced dimension 0 with free landmarks -- k_ba_schur and k_ba_step run with nothing but the rhs row
    in the augmented system (n8 = 1).  Poses and speed biases come back bit-identical."""
    pb = stationary_window()
    b = pb.clone()
    s = compare(ba, pb, max_iter)
    assert s["reduced_dim"] == 0 and s["n_free_landmarks"] == 36 and s["num_successful_steps"] >= 1
    b.max_num_iterations = max_iter
    ba.optimization(b)
    assert np.array_equal(b.para_pose, pb.para_pose) and np.array_equal(b.para_speed_bias, pb.para_speed_bias)
    assert np.abs(b.para_feature - pb.para_feature).max() > 1e-3


def test_stationary_window_with_free_wheel_blocks(ba):
    """Every pose fixed, the wheel extrinsic / intrinsics / time offset free: nc = 10 while no pose moves."""
    pb = stationary_window(with_wheel=True)
    s = compare(ba, pb, 16)
    assert s["reduced_dim"] == 10
    b = pb.clone(); ba.optimization(b)
    assert np.array_equal(b.para_pose, pb.para_pose) and np.array_equal(b.para_speed_bias, pb.para_speed_bias)
    assert not np.array_equal(b.para_ex_wheel, pb.para_ex_wheel)


@pytest.mark.parametrize("seed", sorted(ROUGH))
def test_rejected_steps_match_the_oracle(ba, seed):
    """Far starts at GF_BA_MAX_ITERATIONS: after a rejected step the radius is halved and k_ba_step re-solves the dogleg
    from the existing factor (no new Cholesky, k_ba_eval(1)'s buffer discarded).  Cost and radius traces entry by entry."""
    pb = rough_window(seed)
    a, b = pb.clone(), pb.clone()
    so = O.solve(a); sg = ba.optimization(b)
    assert rejected_steps(so) >= 4
    assert decisions(sg) == decisions(so)
    assert_matches(sg, so, b, a, **ROUGH_TOL)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_c2_windows_at_the_iteration_limit(ba, seed):
    pb, _ = make_window(seed=seed)
    s = compare(ba, pb, 16)
    assert s["reduced_dim"] == 165 and s["iterations"] >= 7


@pytest.mark.parametrize("F", list(range(2, 12)))
def test_visual_only_window(ba, F):
    """!USE_IMU: pose 0 constant, no IMU factors, no speed-bias columns (use_sb false); pair CTAs of frame 0 have no pose
    column.  F = 2, 3 have no landmark with 4 observations and no factor at all: CONVERGENCE_GRADIENT at iteration 0."""
    pb = visual_only_window(F)
    s = compare(ba, pb, 8)
    assert s["reduced_dim"] == 6 * (F - 1)
    if F < 4:
        assert s["n_free_landmarks"] == 0 and s["iterations"] == 0 and s["termination"] == 3
    else:
        assert s["n_free_landmarks"] > 0 and s["num_successful_steps"] >= 5


def test_visual_only_marginalization(ba):
    """MARGIN_OLD on a visual-only window (cdim = 6: pose 0 alone, no speed bias), then MARGIN_SECOND_NEW on the next
    visual-only window carrying that prior."""
    pb = visual_only_window(11)
    O.solve(pb)
    want = O.marginalize_old(pb)
    got = ba.marginalize_old(pb)
    _compare_priors(got, want)
    assert 1 not in got.kinds                                  # no speed-bias block is kept
    nxt = visual_only_window(11, seed=77)
    nxt.prior = want
    O.solve(nxt)
    want2 = O.marginalize_second_new(nxt)
    got2 = ba.marginalize_second_new(nxt)
    assert want2 is not None and got2 is not None
    _compare_priors(got2, want2)


@pytest.mark.parametrize("F", [1, 2, 3, 4, 6, 10])
def test_short_window_with_imu(ba, F):
    """The initialisation phase: F = 1 has no factor (CONVERGENCE_GRADIENT at iteration 0), F = 2, 3 are IMU-only."""
    pb = short_window(F)
    a, b = pb.clone(), pb.clone()
    so = O.solve(a); sg = ba.optimization(b)
    # F >= 4: the first two steps take the cost down by 4 decades, which amplifies 1e-13 step differences to 1e-7 in
    # iterate 2, as in test_ba_gpu's wheel windows; the end point agrees to 1e-9
    assert_matches(sg, so, b, a, mid_rtol=1e-6, cost_atol=EXACT_FIT_ATOL if F in (2, 3) else 0.0)
    assert sg["reduced_dim"] == 15 * F and (sg["n_free_landmarks"] > 0) == (F >= 4)
    if F == 1:
        assert sg["iterations"] == 0 and sg["termination"] == 3
    if F in (2, 3):
        assert sg["termination"] == 2 and sg["final_cost"] < EXACT_FIT_ATOL


def test_time_offset_with_feature_velocities(ba):
    """vel_i / vel_j about 0.05 /s, td_i != td_j != para_td, the time offset free (the td column carries tmp_r vel_i / inv_dep)."""
    pb = add_velocities(make_window(seed=33)[0], 33)
    s = compare(ba, pb, 8)
    assert s["reduced_dim"] == 166
    a, b = pb.clone(), pb.clone()
    O.solve(a); ba.optimization(b)
    assert abs(a.para_td[0] - b.para_td[0]) < 1e-6 and a.para_td[0] != pb.para_td[0]


def test_outliers_keep_the_huber_corrector_active(ba):
    pb, _ = make_window(seed=32)
    idx = add_outliers(pb, 32)
    s = compare(ba, pb, 16)
    b = pb.clone(); ba.optimization(b)
    assert (huber_s(b)[idx] > 1).all() and s["iterations"] >= 5


@pytest.mark.parametrize("kept", [127, 128])
def test_marginalization_fast_and_generic_boundary(ba, kept):
    """Kept dimension 127 takes the structured fast path (k_marg_c_elim's buffer), 128 the generic eigen-truncated path."""
    pb = marginalization_boundary_window(kept)
    want = O.marginalize_old(pb)
    got = ba.marginalize_old(pb)
    assert got.n == want.n == kept
    _compare_priors(got, want)


def capacity_window(n_free):
    """A C2-like window with n_free free landmarks (the rest of its features constant)."""
    pb, _ = make_window(seed=13, n_landmarks=10500, free_fraction=1.0)
    assert pb.n_features > n_free + 1
    pb.feature_const[:] = 1
    pb.feature_const[:n_free] = 0
    return pb


def test_free_landmark_capacity(ba):
    """GF_BA_MAX_FREE_LANDMARKS = 8192 free landmarks: k_ba_schur stages 8 (L + 2 nc + 2) = 68 KB (above the 48 KB default)
    and the solve matches the oracle; one more is GF_ERR_CAPACITY before anything is enqueued, and the handle stays usable."""
    from ground_fusion_b200._lib import GfError
    pb = capacity_window(8192)
    # two iterations end on an intermediate iterate of the steep phase (cost 1e9 -> 3e6): test_ba_gpu's 1e-7 bar for those
    s = compare(ba, pb, 2, final_rtol=1e-7)
    assert s["n_free_landmarks"] == 8192 and s["reduced_dim"] == 165
    over = pb.clone()
    over.feature_const[8192] = 0
    before = over.para_pose.copy(), over.para_feature.copy()
    with pytest.raises(GfError, match="error -4: .*free landmarks"):
        ba.optimization(over)
    assert np.array_equal(over.para_pose, before[0]) and np.array_equal(over.para_feature, before[1])
    compare(ba, make_window(seed=0)[0], 8)


FLAVOURS = {
    "stationary": lambda: stationary_window(),
    "rough": lambda: rough_window(9),
    "visual_only": lambda: visual_only_window(7),
    "velocities": lambda: add_velocities(make_window(seed=33)[0], 33),
}


def test_handles_on_four_threads():
    """Four handles, one per thread, each solving its own flavour three times; every result against the oracle."""
    from ground_fusion_b200.estimator import BundleAdjuster
    windows = {k: f() for k, f in FLAVOURS.items()}
    oracle = {}
    for k, pb in windows.items():
        a = pb.clone(); oracle[k] = (O.solve(a), a)
    handles = {k: BundleAdjuster(0) for k in windows}
    results = {k: [] for k in windows}
    errors = []

    def work(k):
        try:
            for _ in range(3):
                b = windows[k].clone()
                results[k].append((handles[k].optimization(b), b))
        except Exception as e:       # surfaced below
            errors.append((k, e))

    threads = [threading.Thread(target=work, args=(k,)) for k in windows]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        for h in handles.values():
            h.close()
    assert not errors, errors
    for k in windows:
        so, a = oracle[k]
        assert len(results[k]) == 3
        for sg, b in results[k]:
            assert_matches(sg, so, b, a, **(ROUGH_TOL if k == "rough" else {}))


def window_with_prior():
    """The next window after MARGIN_OLD, as test_ba_gpu.test_solve_with_marginalization_prior builds it: frame 0 dropped,
    the rest kept and perturbed, the prior attached."""
    q, _ = make_window(seed=4)
    O.solve(q)
    prior = O.marginalize_old(q)
    nxt = q.clone(); nxt.n_frames = 10
    nxt.para_pose = q.para_pose[1:].copy(); nxt.para_speed_bias = q.para_speed_bias[1:].copy()
    nxt.set_visual([(f.imu_i - 1, f.imu_j - 1, f.feature, list(f.pts_i), list(f.pts_j), list(f.vel_i), list(f.vel_j), f.td_i, f.td_j)
                    for f in list(q.visual)[:q.n_visual] if f.imu_i >= 1])
    nxt.set_imu([dict(i=f.i - 1, j=f.j - 1, sum_dt=f.sum_dt, delta_p=list(f.delta_p), delta_q=list(f.delta_q), delta_v=list(f.delta_v),
                      linearized_ba=list(f.linearized_ba), linearized_bg=list(f.linearized_bg),
                      jacobian=np.array(f.jacobian).reshape(15, 15), covariance=np.array(f.covariance).reshape(15, 15))
                 for f in list(q.imu)[1:q.n_imu]])
    nxt.prior = prior
    nxt.para_pose[:, :3] += np.random.default_rng(0).normal(0, 0.01, (10, 3))
    return nxt


def test_one_handle_across_window_sizes():
    """One handle solving C3 -> F = 2 -> stationary -> C2 with a prior: the workspace grows once and is reused by smaller
    windows; nothing stale from an earlier window may leak into a later one."""
    from ground_fusion_b200.estimator import BundleAdjuster
    h = BundleAdjuster(0)
    try:
        s = compare(h, make_window(seed=7, n_landmarks=440)[0], 8)
        assert s["n_residuals"] > 5000
        pb = short_window(2)
        a, b = pb.clone(), pb.clone()
        so = O.solve(a); sg = h.optimization(b)
        assert_matches(sg, so, b, a, cost_atol=EXACT_FIT_ATOL)
        assert compare(h, stationary_window(), 8)["reduced_dim"] == 0
        compare(h, window_with_prior(), 8)
    finally:
        h.close()
