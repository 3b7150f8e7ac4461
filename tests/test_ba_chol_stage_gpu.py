"""The back end's dense SPD solve on its own (gf_stage_spd_solve: chol_factor + chol_backsubst of ba_chol.cuh) against the
references and bars of tests/chol_ref.py, at every size boundary of its tiling, with the factor in shared memory, partly
spilled to L2 and wholly spilled, plus exact results over the exponent range, failures and the solver's own systems."""
import numpy as np
import pytest

import chol_ref as C
from ground_fusion_b200._lib import GfError
from ground_fusion_b200.estimator import spd_solve

pytestmark = pytest.mark.gpu

SIZES = list(range(1, 65)) + [207, 208, 215, 216, 223, 224, 231, 255, 256, 300, 375, 376, 382, 383]
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst H100 ratio per bar (closest to its bar): "
          + ", ".join("%s %.3g (K %g, %.2f of it, %s)" % (k, v[1], v[2], v[0], v[3]) for k, v in sorted(WORST.items())))


def caps(n, full):
    """tile_cap values worth running at size n: the default (-1), everything from L2 (0), caps that cut the middle and the
    last block row, and (full) caps that put the bulk copy's tile count (64 tiles per 32 KB copy) on either side of a
    multiple of 64, and 375; only caps below the tile count, the others equal the default."""
    nt, m8 = C.ntiles(n), C.n8(n)
    out = {-1, 0, C.tix(m8 // 2, m8 // 4) + 1, C.tix(m8 - 1, (m8 - 1) // 2)}
    if full:
        out |= {63, 64, 65, 127, 128, 129, 320, 321, 375}
    return sorted(c for c in out if c == -1 or 0 <= c < min(nt, C.TILE_CAP))


def check(A, b, x, xr, kappa, fam, where):
    """x within the family's bars; WORST keeps, per bar, the ratio closest to its bar."""
    m = C.metrics(A, b, x, xr, kappa)
    for k, v in m.items():
        if v / C.K[fam][k] > WORST.get(k, (0.0,))[0]:
            WORST[k] = (v / C.K[fam][k], v, C.K[fam][k], where)
    bad = {k: v for k, v in m.items() if not v <= C.K[fam][k]}
    assert not bad, (where, bad, C.K[fam])


def solve_all_caps(A, b, n, full, where):
    """x per instantiation; within one instantiation every cap must give the same bits (only where the tiles live differs)."""
    got = {}
    for cap in caps(n, full):
        x = spd_solve(A, b, tile_cap=cap)
        key = "spill" if C.spills(n, cap) else "smem"
        if key in got:
            assert np.array_equal(x, got[key][1]), (where, cap, got[key][0])
        else:
            got[key] = (cap, x)
    return got


@pytest.mark.parametrize("n", SIZES)
def test_families_every_size(n):
    big = n > 64
    for name in C.FAMILIES:
        A, b = C.family(name, n)
        xr, kap = C.solve_ref(A, b), C.equilibrated_kappa(A)
        got = solve_all_caps(A, b, n, big and name in ("random", "block"), "%s n=%d" % (name, n))
        assert set(got) == ({"spill"} if C.spills(n) else {"smem", "spill"})
        for key, (cap, x) in got.items():
            check(A, b, x, xr, kap, name, "%s n=%d %s" % (name, n, key))


def test_window_systems():
    for name, (S, rhs, _) in C.window_systems().items():
        n = len(rhs)
        got = solve_all_caps(S, rhs, n, False, name)
        xr, kap = C.solve_ref(S, rhs), C.equilibrated_kappa(S)
        for key, (cap, x) in got.items():
            check(S, rhs, x, xr, kap, "window", "window %s %s" % (name, key))


@pytest.mark.parametrize("odd", [False, True])
def test_diagonal_exact_over_the_exponent_range(odd):
    """diag(4^k): x = b / 4^k bit for bit (sqrt_rsqrt is exact on even exponents, every product then exact); diag(2 4^k):
    within 3 ulps.  The exponents 2k run over -1000 .. 1000, in shuffled order, on both instantiations."""
    ex = np.random.default_rng(3).permutation(C.diag_exponents())
    for part, cap_list in ((ex[:383], (-1, 0, 100)), (ex[383:766], (-1, 0, 321)), (ex[766:], (-1, 0, 37))):
        A, b = C.diag_system(part, odd)
        want = b / np.diag(A)
        for cap in cap_list:
            x = spd_solve(A, b, tile_cap=cap)
            if odd:
                assert C.ulps(x, want).max() <= 3, (cap, C.ulps(x, want).max())
            else:
                assert np.array_equal(x, want), (cap, np.flatnonzero(x != want)[:8])


def _indefinite_after_elimination(n, p, rng):
    """SPD except that the pivot at p turns negative only through the elimination of column p - 9 (another block)."""
    A = C.family("random", n)[0]
    q = p - 9
    A[p, q] = A[q, p] = 2.0 * np.sqrt(A[p, p] * A[q, q])
    assert np.all(np.diag(A) > 0) and np.linalg.eigvalsh(A).min() < 0
    return A


@pytest.mark.parametrize("n,cap", [(64, -1), (64, 0), (200, -1), (200, 40), (300, -1), (383, 0)])
def test_non_positive_pivots_are_errors(n, cap):
    rng = np.random.default_rng(n)
    last = 8 * ((n - 1) // 8)
    b = rng.standard_normal(n)
    positions = [16, 19, 23, last, n - 1]          # first, middle and last column of a block; the last genuine block
    for p in positions:
        for v in (0.0, -1.0):
            A = C.family("random", n)[0]
            A[p, p] = v
            with pytest.raises(GfError, match="not positive definite"):
                spd_solve(A, b, tile_cap=cap)
    for p in (20, n - 1):
        with pytest.raises(GfError, match="not positive definite"):
            spd_solve(_indefinite_after_elimination(n, p, rng), b, tile_cap=cap)


def _correct_or_error(A, b, cap=-1):
    """The solve either refuses the system or returns x within the bars; never a wrong x."""
    try:
        x = spd_solve(A, b, tile_cap=cap)
    except GfError as e:
        return str(e)
    xr = C.solve_ref(A, b)
    assert np.all(np.isfinite(x))
    check(A, b, x, xr, C.equilibrated_kappa(A), "random", "edge n=%d" % len(b))
    return None


def test_subnormal_pivots_are_refused():
    assert "not positive definite" in _correct_or_error(1e-310 * np.eye(3), np.full(3, 1e-300))
    a = 2.0 ** -1000
    A = a * np.array([[1.0, 1.0 - 2.0 ** -30], [1.0 - 2.0 ** -30, 1.0]])      # the second pivot is subnormal after elimination
    assert "not positive definite" in _correct_or_error(A, np.array([a, a]))
    A, b = C.family("random", 300)
    A[250, :] = 0; A[:, 250] = 0; A[250, 250] = 1e-310
    for cap in (-1, 0):
        assert "not positive definite" in _correct_or_error(A, b, cap)
    A = np.diag(np.ldexp(1.0, -1022 + np.arange(40)))                            # the smallest normal pivots still solve
    assert _correct_or_error(A, np.ones(40)) is None


@pytest.mark.parametrize("what", ["inf_diag", "inf_lower", "nan_diag", "nan_lower", "inf_b", "nan_b"])
@pytest.mark.parametrize("n", [5, 64, 300])
def test_non_finite_input_is_refused(what, n):
    A, b = C.family("random", n)
    i, j = n - 1, max(n - 3, 0)
    v = np.inf if what.startswith("inf") else np.nan
    if what.endswith("diag"):
        A[i, i] = v
    elif what.endswith("lower"):
        A[i, j] = A[j, i] = v
    else:
        b[i] = v
    with pytest.raises(GfError, match="not finite"):
        spd_solve(A, b)


def test_upper_triangle_is_not_read():
    """A NaN in the strict upper triangle (inside a diagonal tile and in an off-diagonal one) changes nothing."""
    for n, cap in ((64, -1), (300, -1), (64, 0)):
        A, b = C.family("random", n)
        x = spd_solve(A, b, tile_cap=cap)
        B = A.copy()
        B[0, 1] = B[8, 15] = B[n - 2, n - 1] = B[0, n - 1] = np.nan
        assert np.array_equal(spd_solve(B, b, tile_cap=cap), x)


def test_stage_solve_equals_the_solvers_reduced_solution():
    """The stage solve of the reduced system S and right-hand side that gf_ba_first_step captured equals the solver's own
    reduced solution bit for bit, on the same instantiation and cap.  The solver keeps gn = -D y (y the reduced solution),
    so the comparison is gn[:nc] == -(D[:nc] * x)."""
    import os

    import ba_lin_ref as R
    from ground_fusion_b200.estimator import BundleAdjuster
    w = R.windows()
    for cap_env, cap in ((None, -1), ("4", 4)):
        old = os.environ.pop("GF_BA_TILE_CAP", None)
        if cap_env:
            os.environ["GF_BA_TILE_CAP"] = cap_env
        try:
            ba = BundleAdjuster(0)
        finally:
            os.environ.pop("GF_BA_TILE_CAP", None)
            if old is not None:
                os.environ["GF_BA_TILE_CAP"] = old
        try:
            for name in ("stationary_wheel", "visual_only_F6", "c2_s0", "plane_wheel", "c3"):
                got = ba.first_step(w[name]())
                nc = got["nc"]
                assert got["solver_failed"] == 0 and got["mu"] == 1e-8         # the first factorisation succeeded
                assert got["spill"] == int(C.spills(nc, cap))
                S = got["S"]
                A = np.tril(S[:nc, :nc]) + np.tril(S[:nc, :nc], -1).T
                x = spd_solve(A, S[nc, :nc], tile_cap=cap)
                assert np.array_equal(got["gn"][:nc], -(got["D"][:nc] * x)), (name, cap)
        finally:
            ba.close()


def test_arguments():
    with pytest.raises(GfError):
        spd_solve(np.eye(384), np.ones(384))
    x = spd_solve(np.eye(383) * 4.0, np.ones(383), tile_cap=10 ** 6)          # a cap above the default is the default
    assert np.array_equal(x, np.full(383, 0.25))
