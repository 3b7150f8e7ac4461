"""CPU tests of the FeatureManager references (tests/fm_ref.py): the references against ground truth, each other and the oracle
(oracle/fm_oracle.py); the bars' calibration by plain-double implementations; and a negative control showing that the DLT bar
tells the kernel's former algorithm (the eigenvector of A^T A) from a backward-stable one."""
import mpmath as mp
import numpy as np
import pytest

import fm_ref as R
from oracle.fm_oracle import FeatureManagerOracle, FeaturePerFrame, FeaturePerId

CAL = {k: v / R.CALIBRATION_FACTOR for k, v in R.K.items()}


def smallest_eigvec4_ata(A):
    """NumPy port of what k_fm_triangulate computed before it worked on A itself: M = sum of r r^T over the DLT rows, then the
    eigenvector of M's smallest eigenvalue by cyclic Jacobi (at most 30 sweeps, stopping when the off-diagonal mass is below
    1e-300); depth v2 / v3.  Forming A^T A squares the condition number."""
    M = [[0.0] * 4 for _ in range(4)]
    for r in np.asarray(A, float):
        for u in range(4):
            for v in range(4):
                M[u][v] += r[u] * r[v]
    V = [[float(i == j) for j in range(4)] for i in range(4)]
    for _ in range(30):
        if sum(M[p][q] ** 2 for p in range(4) for q in range(p + 1, 4)) < 1e-300:
            break
        for p in range(3):
            for q in range(p + 1, 4):
                if M[p][q] == 0.0:
                    continue
                th = (M[q][q] - M[p][p]) / (2.0 * M[p][q])
                with np.errstate(over="ignore"):
                    t = (1.0 if th >= 0 else -1.0) / (abs(th) + np.sqrt(np.float64(th) * th + 1.0))
                c = 1.0 / np.sqrt(t * t + 1.0); s = t * c
                for k in range(4):
                    a, b = M[k][p], M[k][q]; M[k][p] = c * a - s * b; M[k][q] = s * a + c * b
                for k in range(4):
                    a, b = M[p][k], M[q][k]; M[p][k] = c * a - s * b; M[q][k] = s * a + c * b
                for k in range(4):
                    a, b = V[k][p], V[k][q]; V[k][p] = c * a - s * b; V[k][q] = s * a + c * b
    m = min(range(4), key=lambda k: M[k][k])
    return V[2][m] / V[3][m]


def all_triangulation_scenes():
    return list(R.dlt_scenes().values()) + list(R.depth_scenes().values()) + [R.count_scene()]


def dlt_items():
    for sc in all_triangulation_scenes():
        for lm, ref in zip(sc.lms, R.triangulate_ref(sc)):
            if ref["kind"] == "dlt" and np.isfinite(ref["scale"]):
                yield sc, lm, ref


# ---- the references --------------------------------------------------------------------------------------------------
def test_dlt_reference_recovers_the_true_depth_from_noise_free_observations():
    """Noise-free observations are the true projections rounded to double: the true depth lies within the bar."""
    n = 0
    for sc in R.dlt_scenes().values():
        for lm, ref in zip(sc.lms, R.triangulate_ref(sc)):
            if ref["kind"] == "dlt" and lm["noise"] == 0 and np.isfinite(ref["scale"]):
                assert R.ratio(ref["d"], lm["z"][0], ref["scale"]) <= R.K["dlt"], (sc.name, ref["d"], lm["z"][0])
                n += 1
    assert n > 200


def test_depth_pairs_longdouble_agrees_with_mpmath():
    """triangulateWithDepth's residuals and verified depths in longdouble against the same steps at 50 digits."""
    sc = R.depth_scenes()["depth_b1e-01_o1e+04_ric"]
    with mp.workdps(50):
        tic, ric = R._mp_vec(sc.tic), R._mp_mat(sc.ric)

        def cam(f):
            Rm = R._mp_mat(sc.Rs[f])
            return R._mp_vec(sc.Ps[f]) + Rm * tic, Rm * ric
        n = 0
        for lm in sc.lms[:12]:
            for p in R.depth_pairs(sc, lm):
                s0 = lm["start"]
                tr, Rr = cam(s0); t0, R0 = cam(s0 + p["i"]); t1, R1 = cam(s0 + p["j"])
                point0 = R._mp_vec(lm["pts"][p["i"]]) * mp.mpf(float(lm["dep"][p["i"]]))
                t20, R20 = R0.T * (t1 - t0), R0.T * R1
                pp = R20.T * point0 - R20.T * t20
                res = mp.sqrt((lm["pts"][p["j"]][0] - pp[0] / pp[2]) ** 2 + (lm["pts"][p["j"]][1] - pp[1] / pp[2]) ** 2)
                z = ((Rr.T * R0) * point0 + Rr.T * (t0 - tr))[2]
                assert abs(float(p["res"]) - float(res)) <= 1e-16 * (1 + float(res)) * 1e3
                assert abs(float(p["z"]) - float(z)) <= 1e-16 * p["scale"]
                n += 1
    assert n > 100


def _oracle_fm(sc):
    fm = FeatureManagerOracle(depth_threshold=sc.depth_threshold)
    for k, lm in enumerate(sc.lms):
        it = FeaturePerId(k, lm["start"])
        for p, d in zip(lm["pts"], lm["dep"]):
            it.feature_per_frame.append(FeaturePerFrame([p[0], p[1], p[2], 0, 0, 0, 0, d], 0.0))
        it.estimated_depth, it.estimate_flag = float(lm["est"]), int(lm["flag"])
        fm.feature.append(it)
    return fm


@pytest.mark.parametrize("name", ["b1e-01_o0e+00", "b1e-03_o1e+03_ric", "b1e-06_o1e+04_ric", "depth_b1e-01_o0e+00",
                                  "depth_b1e-02_o1e+03_ric", "depth_backwards"])
def test_triangulation_reference_matches_the_oracle(name):
    """oracle/fm_oracle.py (LAPACK's SVD, plain double) lands on every pinned decision of the reference and within its bars."""
    sc = {**R.dlt_scenes(), **R.depth_scenes()}[name]
    fm = _oracle_fm(sc)
    fm.triangulateAll(10, sc.Ps, sc.Rs, sc.tic, sc.ric)
    for it, lm, ref in zip(fm.feature, sc.lms, R.triangulate_ref(sc)):
        if ref["kind"] == "skip":
            assert (it.estimated_depth, it.estimate_flag) == (lm["est"], lm["flag"])
            continue
        k = R.K["dlt"] if ref["kind"] == "dlt" else R.K["depth_mean"]
        if R.flag_pinned(ref, k):
            assert it.estimate_flag == ref["flag"], (name, it.feature_id)
        if it.estimate_flag in (1, 2):
            assert R.ratio(it.estimated_depth, ref["d"], ref["scale"]) <= k / R.CALIBRATION_FACTOR
        else:
            assert it.estimated_depth == R.INIT_DEPTH


def test_parallax_back_shift_reprojection_and_prediction_references_match_the_oracle():
    o = FeatureManagerOracle()
    pi, pj = R.parallax_case(300, 1, near_plane=True)
    ref, s = R.parallax_ref(pi, pj)
    got = 0.0
    for a, b in zip(pi, pj):
        it = FeaturePerId(0, 0)
        it.feature_per_frame = [FeaturePerFrame(list(a) + [0, 0, 0, 0, 1.0], 0), FeaturePerFrame(list(b) + [0, 0, 0, 0, 1.0], 0)]
        got += o.compensatedParallax2(it, 2)
    assert R.ratio(got, ref, s) <= CAL["parallax"]
    uv, d, mR, mP, nR, nP = R.back_shift_case(200, 1e3, 2)
    z, s = R.back_shift_ref(uv, d, mR, mP, nR, nP)
    fm = FeatureManagerOracle()
    for k in range(len(d)):
        it = FeaturePerId(k, 0)
        it.feature_per_frame = [FeaturePerFrame(list(uv[k]) + [0, 0, 0, 0, 1.0], 0)] * 3
        it.estimated_depth = d[k]
        fm.feature.append(it)
    fm.removeBackShiftDepth(mR, mP, nR, nP)
    for it, zz, ss in zip(fm.feature, z, s):
        if abs(zz) > R.K["back_shift"] * R.EPS * ss:
            assert (it.estimated_depth == R.INIT_DEPTH) if zz <= 0 else R.ratio(it.estimated_depth, zz, ss) <= CAL["back_shift"]
    sc = R.reproj_case(150, 1e3, True, 4)
    fm = _oracle_fm(sc)
    for it, (e2, e3, c, s2, s3) in zip(fm.feature, R.reproj_ref(sc)):
        w2, w3, wc = fm._errors(it, sc.Ps, sc.Rs, sc.tic, sc.ric)
        assert wc == c and R.ratio(w2, e2, s2) <= CAL["reproj2d"] and R.ratio(w3, e3, s3) <= CAL["reproj3d"]
    sc, first, uv, dep = R.predict_case(100, 1e4, True, 5)
    ref, s = R.predict_ref(sc, first, uv, dep, 10)
    fm = FeatureManagerOracle()
    for k in range(len(first)):
        it = FeaturePerId(k, int(first[k]))
        it.feature_per_frame = [FeaturePerFrame(list(uv[k]) + [0, 0, 0, 0, 1.0], 0)] * (11 - int(first[k]))
        it.estimated_depth = dep[k]
        fm.feature.append(it)
    pred = fm.predictPtsInNextFrame(10, sc.Ps, sc.Rs, sc.tic, sc.ric)
    for k, (r, ss) in enumerate(zip(ref, s)):
        if k in pred:
            assert np.abs(pred[k] - r).max() <= CAL["predict"] * R.EPS * ss
    assert len(pred) > 5


def test_prediction_reference_lands_on_the_landmark_under_constant_velocity():
    """nextT of the reference: with poses that really move at constant velocity the carried point is the landmark seen from
    the next pose."""
    dR, dP = R.rot([0.2, 1.0, -0.1], 0.03), np.array([0.1, 0.01, 0.02])
    Rs, Ps = [R.rot([1, 2, 3], 0.5)], [np.array([1e3, -2e3, 50.0])]
    for _ in range(11):
        Ps.append(Ps[-1] + Rs[-1] @ dP); Rs.append(Rs[-1] @ dR)
    sc = R.Scene("cv", np.array(Ps), np.array(Rs), R.TIC, R.RIC, 3.0, [])
    rng = np.random.default_rng(0)
    first = rng.integers(0, 11, 20).astype(np.int32)
    X = np.array(Ps[10]) + rng.uniform(-5, 5, (20, 3))
    uv, dep = [], []
    for f, x in zip(first, X):
        t, Rm = R.cam_pose(sc.Ps, sc.Rs, sc.tic, sc.ric, f)
        pc = Rm.T @ (x - t)
        uv.append(pc / pc[2]); dep.append(pc[2])
    ref, s = R.predict_ref(sc, first, np.array(uv), np.array(dep), 10)
    for x, r in zip(X, ref):
        t, Rm = Ps[11] + Rs[11] @ R.TIC, Rs[11] @ R.RIC
        assert np.abs(Rm.T @ (x - t) - r).max() < 1e-9


# ---- cases -----------------------------------------------------------------------------------------------------------
def test_cases_pin_every_decision_and_reach_every_outcome():
    outcomes = set()
    for sc in all_triangulation_scenes():
        for lm, ref in zip(sc.lms, R.triangulate_ref(sc)):
            for p in R.depth_pairs(sc, lm):
                assert p["pinned"], (sc.name, p["i"], p["j"], float(p["res"]))
            if ref["kind"] == "dlt":
                outcomes.add(("dlt", "negative" if ref["d"] < 0 else "below 0.1" if ref["d"] < 0.1 else "accepted"))
            elif ref["kind"] == "depth":
                outcomes.add(("depth", ref["flag"]))
    assert outcomes == {("dlt", "negative"), ("dlt", "below 0.1"), ("dlt", "accepted"), ("depth", 0), ("depth", 1)}
    # the RGB-D bounds: exactly 0.1 and depth_threshold are usable depths, one ulp outside them is not
    for sc in R.depth_scenes().values():
        if sc.name == "depth_backwards":
            continue
        refs = R.triangulate_ref(sc)
        for lm, ref in zip(sc.lms, refs):
            nz = lm["dep"][lm["dep"] != 0]
            if len(nz) == 1 and nz[0] in (0.1, sc.depth_threshold):
                assert ref["kind"] == "depth"
            if len(nz) == 1 and nz[0] in (np.nextafter(0.1, 0.0), np.nextafter(sc.depth_threshold, np.inf)):
                assert ref["kind"] == "dlt"
    # every list length 1 .. 11, each ending in the last frame
    ms = {len(lm["dep"]) for sc in R.dlt_scenes().values() for lm in sc.lms}
    assert ms == set(range(1, 12)) and all(lm["start"] + len(lm["dep"]) == R.N_FRAMES for sc in R.dlt_scenes().values() for lm in sc.lms)


# ---- calibration -------------------------------------------------------------------------------------------------------
def test_dlt_bar_is_calibrated_by_lapack_and_the_kernel_algorithm():
    worst_l = worst_k = 0.0
    sweeps = 0
    for sc, lm, ref in dlt_items():
        A = R.dlt_matrix_f64(sc, lm)
        worst_l = max(worst_l, R.ratio(R.dlt_lapack(A), ref["d"], ref["scale"]))
        d, sw = R.dlt_kernel_port(A)
        worst_k = max(worst_k, R.ratio(d, ref["d"], ref["scale"]))
        sweeps = max(sweeps, sw)
    assert worst_l <= CAL["dlt"] and worst_k <= CAL["dlt"], (worst_l, worst_k)
    assert sweeps <= 8


def test_dlt_negative_control_the_eigenvector_of_AtA_exceeds_the_bar():
    """The former kernel algorithm passes the well-conditioned scenes and fails every small-baseline one: the bar separates
    eps kappa(A) from eps kappa(A)^2."""
    over = {}
    for sc in R.dlt_scenes().values():
        worst = 0.0
        for lm, ref in zip(sc.lms, R.triangulate_ref(sc)):
            if ref["kind"] == "dlt" and np.isfinite(ref["scale"]):
                worst = max(worst, R.ratio(smallest_eigvec4_ata(R.dlt_matrix_f64(sc, lm)), ref["d"], ref["scale"]))
        over[sc.name] = worst
    small = [n for n in over if n.startswith(("b1e-03_o0e+00", "b1e-04_o0e+00", "b1e-05_o0e+00", "b1e-06_o0e+00", "b1e-06_o1e+03"))]
    assert len(small) == 10
    assert all(over[n] > R.K["dlt"] for n in small), {n: over[n] for n in small}
    assert all(over[n] <= R.K["dlt"] for n in over if n.startswith("b1e-01")), over


def test_other_bars_are_calibrated_by_plain_double():
    for sc in list(R.depth_scenes().values()) + [R.count_scene()]:
        for lm, ref in zip(sc.lms, R.triangulate_ref(sc)):
            if ref["kind"] == "depth":
                assert R.ratio(R.depth_mean_f64(sc, lm), ref["d"], ref["scale"]) <= CAL["depth_mean"], sc.name
    for n in R.COUNTS:
        for near in (False, True):
            pi, pj = R.parallax_case(n, n, near)
            ref, s = R.parallax_ref(pi, pj)
            assert R.ratio(R.parallax_f64(pi, pj), ref, s) <= CAL["parallax"], n
    for o in R.OFFSETS:
        case = R.back_shift_case(3000, o, 3)
        z, s = R.back_shift_ref(*case)
        got = R.back_shift_f64(*case)
        pinned = np.abs(z) > R.K["back_shift"] * R.EPS * s
        assert np.all((got[pinned] > 0) == (z[pinned] > 0))
        assert (np.abs(got - z) / (R.EPS * s))[pinned].max() <= CAL["back_shift"]
        for ext in (False, True):
            for near in (False, True):
                sc = R.reproj_case(300, o, ext, 5, near)
                for (e2, e3, c, s2, s3), (g2, g3, gc) in zip(R.reproj_ref(sc), R.reproj_f64(sc)):
                    assert gc == c and R.ratio(g2, e2, s2) <= CAL["reproj2d"] and R.ratio(g3, e3, s3) <= CAL["reproj3d"]
            sc, first, uv, dep = R.predict_case(200, o, ext, 3)
            for fc in (1, 5, 10):
                ref, s = R.predict_ref(sc, first, uv, dep, fc)
                got = R.predict_f64(sc, first, uv, dep, fc)
                assert (np.abs(got - ref).max(1) / (R.EPS * s)).max() <= CAL["predict"]
