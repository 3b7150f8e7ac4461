"""The C oracle's trust-region loop against a separately written NumPy witness (oracle/dogleg_witness.py): per-iteration
cost and radius traces, iteration counts, termination and the solved parameters, at max_num_iterations 1 and 8 and at
every window flavour the golden fixtures hold (VERDICT r1 item 7: 'a shared misreading of Ceres passes every test')."""
import numpy as np
import pytest

from ground_fusion_b200.synth_ba import make_window
from oracle import ba_oracle as O
from oracle import dogleg_witness as W

TERM = {0: "NO_CONVERGENCE", 1: "CONVERGENCE_FUNCTION", 2: "CONVERGENCE_PARAMETER", 3: "CONVERGENCE_GRADIENT", 4: "FAILURE"}
CASES = {
    "c2": dict(seed=0),
    "prior": dict(seed=3, with_prior=True),
    "wheel": dict(seed=1, with_wheel=True),
    "plane": dict(seed=2, with_plane=True),
    "rough": dict(seed=6, pose_noise=(0.2, 0.2)),           # far start: two rejected steps (iterations 7, 8) and radius cuts
    "small": dict(seed=7, n_frames=6, n_landmarks=60),
}


@pytest.mark.parametrize("max_iter", [1, 8])
@pytest.mark.parametrize("case", sorted(CASES))
def test_trace_matches_the_numpy_witness(case, max_iter):
    pa, _ = make_window(**CASES[case])
    pa.max_num_iterations = max_iter
    pb = pa.clone()
    so = O.solve(pa)
    sw = W.solve(pb)
    assert so["iterations"] == sw["iterations"]
    assert TERM[so["termination"]] == sw["termination"]
    assert so["num_successful_steps"] == sw["successful"]
    np.testing.assert_allclose(so["cost"], sw["cost"], rtol=1e-7)
    np.testing.assert_allclose(so["radius"], sw["radius"], rtol=1e-6)
    for k in ("para_pose", "para_speed_bias", "para_feature", "para_ex_pose", "para_td", "para_ex_wheel", "para_ix_wheel", "para_plane_R", "para_plane_Z"):
        np.testing.assert_allclose(getattr(pa, k), getattr(pb, k), atol=2e-7, rtol=1e-6, err_msg=k)


def test_witness_takes_rejected_steps_somewhere():
    """The comparison above is only worth something if the interesting branches run: the "rough" case must reject a step
    (fewer successful steps than iterations, not counting a last iteration that ends in convergence) and cut the radius."""
    pb, _ = make_window(**CASES["rough"])
    pb.max_num_iterations = 8
    s = W.solve(pb)
    rad = np.array(s["radius"][:s["iterations"] + 1])
    converged_last = s["termination"] in ("CONVERGENCE_FUNCTION", "CONVERGENCE_PARAMETER")
    assert s["successful"] < s["iterations"] - (1 if converged_last else 0), s
    assert (np.diff(rad) < 0).any()
