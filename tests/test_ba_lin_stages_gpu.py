"""The bundle-adjustment solve's first iteration on the GPU, stage by stage (gf_ba_first_step), against the high-precision
reference of tests/ba_lin_ref.py: the linearisation (k_ba_eval), the scaled and reduced system (k_ba_schur), the Cholesky, the
dogleg step and the candidate point (k_ba_step), for single windows, on both factor paths, and for a batch."""
import ctypes
import os

import numpy as np
import pytest

import ba_lin_ref as R
from ground_fusion_b200 import _lib
from ground_fusion_b200._lib import GfError
from ground_fusion_b200.estimator import BundleAdjuster, first_step_multi
from ground_fusion_b200.synth_ba import make_window

pytestmark = pytest.mark.gpu

SPILL_CAP = 4          # GF_BA_TILE_CAP: every window with nc >= 16 factors out of L2
PARA = ("para_pose", "para_speed_bias", "para_ex_pose", "para_feature", "para_td", "para_ex_wheel", "para_ix_wheel", "para_td_wheel",
        "para_plane_R", "para_plane_Z")
WINDOWS = R.windows()
WORST = {}


def spill_handle():
    """A handle whose factor keeps SPILL_CAP tiles in shared memory (GF_BA_TILE_CAP is read when the handle is created)."""
    old = os.environ.get("GF_BA_TILE_CAP")
    os.environ["GF_BA_TILE_CAP"] = str(SPILL_CAP)
    try:
        return BundleAdjuster(0)
    finally:
        if old is None:
            del os.environ["GF_BA_TILE_CAP"]
        else:
            os.environ["GF_BA_TILE_CAP"] = old


def smem_handle():
    old = os.environ.pop("GF_BA_TILE_CAP", None)
    try:
        return BundleAdjuster(0)
    finally:
        if old is not None:
            os.environ["GF_BA_TILE_CAP"] = old


@pytest.fixture(scope="module")
def handles():
    h = {"smem": smem_handle(), "spill": spill_handle()}
    yield h
    for v in h.values():
        v.close()
    print("\nworst H100 ratio per bar: " + ", ".join("%s %.3g (%s)" % (k, v[0], v[1]) for k, v in sorted(WORST.items())))


def branch_of(c):
    return "gauss_newton" if (c["dogleg_a"] == 0 and c["dogleg_b"] == 1) else "cauchy" if c["dogleg_b"] == 0 else "interpolated"


def check(got, ref, pb, name, spill_cap=None):
    nc = ref["nc"]
    assert (got["nc"], got["L"], got["n"]) == (nc, ref["L"], ref["n"])
    assert got["solver_failed"] == 0 and got["done"] == 0 and got["iterations"] == 1
    ntiles = (nc + 8) // 8 * ((nc + 8) // 8 + 1) // 2
    assert got["spill"] == (int(ntiles > spill_cap) if spill_cap is not None else 0)
    assert branch_of(got) == ref["branch"]
    assert np.array_equal(got["D"] == np.sqrt(R.DIAG_MIN), ref["clamped"])            # the [1e-6, 1e32] clamp fires where it should
    assert got["step_valid"] == int(ref["model_change"] > 0)
    cf = got["col_feat"]
    assert np.array_equal(np.sort(cf[cf >= 0]), np.arange(nc, ref["n"]))
    rat = R.ratios(got, ref)
    bad = {k: v for k, v in rat.items() if not v <= R.K[k]}
    for k, v in rat.items():
        if v > WORST.get(k, (0.0, ""))[0]:
            WORST[k] = (v, name)
    assert not bad, (name, bad)
    for k in range(pb.n_imu):
        assert R.sqrt_info_ratio(got["imu_sqrt"][k], np.array(pb.imu[k].covariance)) <= R.K["sqrt_info"]


@pytest.mark.parametrize("path", ["smem", "spill"])
@pytest.mark.parametrize("name", sorted(WINDOWS))
def test_first_step_matches_reference(handles, name, path):
    pb = WINDOWS[name]()
    before = {k: getattr(pb, k).copy() for k in PARA}
    got = handles[path].first_step(pb)
    for k in PARA:
        assert np.array_equal(getattr(pb, k), before[k]), k                           # nothing is written back
    check(got, R.reference(pb), pb, name, SPILL_CAP if path == "spill" else None)


@pytest.mark.parametrize("name", ["c2_s0", "plane", "wheel", "prior", "prior_plane"])
@pytest.mark.parametrize("branch", ["gauss_newton", "cauchy", "interpolated", "large_mu"])
def test_dogleg_branches(handles, name, branch):
    pb = R.prior_window() if name == "prior" else WINDOWS[name]()
    radius, mu = (1e4, 0.1) if branch == "large_mu" else (R.branch_radii(pb)[branch], 1e-8)
    ref = R.reference(pb, radius, mu)
    if branch != "large_mu":
        assert ref["branch"] == branch
    got = handles["smem"].first_step(pb, radius=radius, mu=mu)
    assert got["mu"] == mu and got["radius"] == radius
    check(got, ref, pb, "%s/%s" % (name, branch))


def test_prior_window_both_paths(handles):
    pb = R.prior_window()
    ref = R.reference(pb)
    assert np.abs(ref["Hp"]).max() > 0
    check(handles["smem"].first_step(pb), ref, pb, "prior")
    check(handles["spill"].first_step(pb), ref, pb, "prior/spill", SPILL_CAP)


@pytest.mark.parametrize("kind", [k for k in R.COV_KINDS if k != "indefinite"])
def test_imu_sqrt_information(handles, kind):
    pb, _ = make_window(seed=1)
    for k in range(pb.n_imu):
        pb.imu[k].covariance[:] = list(R.imu_covariance(pb.imu[k].covariance, kind, seed=k).ravel())
    got = handles["smem"].first_step(pb)
    worst = max(R.sqrt_info_ratio(got["imu_sqrt"][k], np.array(pb.imu[k].covariance)) for k in range(pb.n_imu))
    if worst > WORST.get("sqrt_info", (0.0, ""))[0]:
        WORST["sqrt_info"] = (worst, kind)
    assert worst <= R.K["sqrt_info"], (kind, worst)


def test_indefinite_covariance_fails_untouched(handles):
    pb, _ = make_window(seed=1)
    pb.imu[3].covariance[:] = list(R.imu_covariance(pb.imu[3].covariance, "indefinite").ravel())
    before = {k: getattr(pb, k).copy() for k in PARA}
    with pytest.raises(GfError, match="not positive definite"):
        handles["smem"].first_step(pb)
    b = pb.clone()
    with pytest.raises(GfError, match="not positive definite"):
        handles["smem"].optimization(b)
    for k in PARA:
        assert np.array_equal(getattr(pb, k), before[k]) and np.array_equal(getattr(b, k), before[k]), k


def test_heterogeneous_batch():
    """Both k_ba_step instantiations in one batch: every other window's handle spills its factor."""
    names = ["c2_s0", "plane_wheel", "wheel_masked", "stationary", "L0", "visual_only_F5", "c3", "td_free_still", "prior_plane", "pair65"]
    wins = [WINDOWS[n]() for n in names] + [R.prior_window()]
    names.append("prior")
    hs = [spill_handle() if k % 2 else smem_handle() for k in range(len(wins))]
    try:
        got = first_step_multi(hs, wins)
    finally:
        for h in hs:
            h.close()
    assert {c["spill"] for c in got} == {0, 1}
    for k, (c, pb, n) in enumerate(zip(got, wins, names)):
        check(c, R.reference(pb), pb, "batch/" + n, SPILL_CAP if k % 2 else None)


def test_arguments_and_launches(handles):
    pb, _ = make_window(seed=0)
    for radius, mu in ((0.0, 1e-8), (-1.0, 1e-8), (1e4, 0.0), (1e4, 1.0), (1e4, -1e-8), (float("nan"), 1e-8)):
        with pytest.raises(GfError, match="radius must be"):
            handles["smem"].first_step(pb, radius=radius, mu=mu)
    L = _lib.lib()
    n0 = L.gf_kernel_launch_count()
    handles["smem"].first_step(pb)
    assert L.gf_kernel_launch_count() - n0 == 3                                         # k_ba_eval(0), k_ba_schur, k_ba_step
    n0 = L.gf_kernel_launch_count()
    handles["smem"].optimization(pb.clone())
    assert L.gf_kernel_launch_count() - n0 == 1 + 3 * pb.max_num_iterations + 2          # unchanged by the capture path


def _same_frame(pb):
    f = pb.visual[5]
    f.imu_j = f.imu_i
    return pb


def test_same_frame_visual_factor_is_an_argument_error(handles):
    """A visual factor with imu_i == imu_j would map its two pose slabs onto the same columns; every entry point refuses it."""
    pb = _same_frame(make_window(seed=0)[0])
    before = {k: getattr(pb, k).copy() for k in PARA}
    ba = handles["smem"]
    for call in (lambda: ba.optimization(pb), lambda: ba.first_step(pb), lambda: ba.marginalize_old(pb)):
        with pytest.raises(GfError, match="imu_i == imu_j"):
            call()
    # gf_ba_first_step itself (first_step asks gf_ba_step_dims first, which refuses the window too); NULL arrays are skipped
    L = _lib.lib()
    L.gf_ba_first_step.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.POINTER(_lib.BaProblem), ctypes.c_double,
                                   ctypes.c_double, ctypes.POINTER(_lib.BaStepCapture)]
    cap = _lib.BaStepCapture()
    rc = L.gf_ba_first_step((ctypes.c_void_p * 1)(ba._h.value), 1, ctypes.byref(pb.struct()), 1e4, 1e-8, ctypes.byref(cap))
    assert rc == -1 and b"imu_i == imu_j" in L.gf_last_error()
    q = R.prior_window()
    q = _same_frame(q)
    with pytest.raises(GfError, match="imu_i == imu_j"):
        ba.marginalize_second_new(q)
    from ground_fusion_b200.estimator import solve_multi
    other = BundleAdjuster(0)
    try:
        with pytest.raises(GfError, match="window 1: visual factor with imu_i == imu_j"):
            solve_multi([other, ba], [make_window(seed=1)[0], pb])
    finally:
        other.close()
    for k in PARA:
        assert np.array_equal(getattr(pb, k), before[k]), k
