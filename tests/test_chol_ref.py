"""CPU: the references, test matrices and bars of the dense SPD solve (tests/chol_ref.py), pinned before
test_ba_chol_stage_gpu.py relies on them.

  * the longdouble reference against mpmath;
  * calibration: the NumPy port of the kernel's algorithm and LAPACK stay below K / CALIBRATION_FACTOR on every family and
    on the windows' reduced systems (the worst ratios are printed beside the bars);
  * negative control: the port with sqrt_rsqrt one Newton step short exceeds the bars;
  * the families reach what they are named for, and the restated sqrt_rsqrt is exact on 4^k and shows the defects of a
    subnormal or infinite pivot that the kernel's pivot rule now refuses.
"""
import numpy as np
import pytest

import chol_ref as C
from marg_ref import EPS


@pytest.mark.parametrize("name,n", [("random", 5), ("graded1e8", 17), ("graded1e14", 24), ("dad", 40), ("block", 33),
                                    ("near_singular", 16), ("scale-1000", 12), ("scale+500", 9), ("graded1e12", 64)])
def test_longdouble_reference_matches_mpmath(name, n):
    A, b = C.family(name, n)
    x_mp = C.solve_mp(A, b)
    x_ld = C.solve_ref(A, b)
    E = np.sqrt(np.diag(A).astype(C.LD))
    err = float(np.sqrt((((x_ld - x_mp) * E) ** 2).sum()) / np.sqrt(((x_mp * E) ** 2).sum()))
    # far below the forward bar's unit eps kappa
    assert err <= 1e-3 * EPS * C.equilibrated_kappa(A), (err, C.equilibrated_kappa(A))


def test_reference_is_exact_on_diagonal_systems():
    A, b = C.diag_system(C.diag_exponents()[::7], odd=False)
    assert np.array_equal(np.asarray(C.solve_ref(A, b), np.float64), b / np.diag(A))


def _cases():
    for name in C.FAMILIES:
        for n in C.CAL_SIZES:
            yield name, n, C.family(name, n)
    for name, (S, rhs, _) in C.window_systems().items():
        yield "window", name, (S, rhs)


def test_calibration_of_the_bars():
    """K[family][bar] >= CALIBRATION_FACTOR x the worst ratio of the port and of LAPACK."""
    worst = {}
    for fam, where, (A, b) in _cases():
        xr, kap = C.solve_ref(A, b), C.equilibrated_kappa(A)
        for who, x in (("port", C.port_solve(A, b)), ("LAPACK", C.lapack_solve(A, b))):
            assert x is not None, (who, fam, where)
            for k, v in C.metrics(A, b, x, xr, kap).items():
                if v > worst.get((fam, k), (0.0, ""))[0]:
                    worst[(fam, k)] = (v, "%s, %s" % (who, where))
    print()
    for (fam, k) in sorted(worst):
        print("bar %-13s %-6s K %-4g worst CPU ratio %.3g (%s)" % (fam, k, C.K[fam][k], *worst[(fam, k)]))
    for (fam, k), (v, where) in worst.items():
        assert C.CALIBRATION_FACTOR * v <= C.K[fam][k], (fam, k, v, where)


def _over(m, fam):
    return max(m[k] / C.K[fam][k] for k in C.BARS)


def test_negative_control_exceeds_the_bars():
    """sqrt_rsqrt one Newton step short, from a seed at MUFU.RSQ's 2^-22: ~2^-44 relative error in every root.  The bars
    catch it at every size of every family but the graded spectra with kappa 1e12 and 1e14, where the rounding error the
    bars allow hides it at most sizes, and on every window."""
    hidden = {}
    for name in C.FAMILIES:
        for n in C.NEG_SIZES:
            A, b = C.family(name, n)
            m = C.metrics(A, b, C.port_solve(A, b, steps=1, seed_err=2.0 ** -22), C.solve_ref(A, b), C.equilibrated_kappa(A))
            if _over(m, name) <= 1.0:
                hidden.setdefault(name, []).append(n)
    print("\nnegative control inside the bars at " + (str(hidden) if hidden else "no case"))
    assert set(hidden) <= {"graded1e12", "graded1e14"}, hidden
    for name, (S, rhs, _) in C.window_systems().items():
        m = C.metrics(S, rhs, C.port_solve(S, rhs, steps=1, seed_err=2.0 ** -22), C.solve_ref(S, rhs), C.equilibrated_kappa(S))
        assert _over(m, "window") > 4.0, (name, m)


def test_families_reach_what_they_name():
    n = 120
    for name, e in C.GRADED.items():
        A, _ = C.family(name, n)
        w = np.linalg.eigvalsh(A)
        assert 0.5 * 10.0 ** e <= w.max() / w.min() <= 2 * 10.0 ** e, (name, w.max() / w.min())
    A, b = C.family("dad", n)
    d = np.log2(np.diag(A))
    assert d.max() - d.min() > 155 and 0.3 < (np.diff(d) > 0).mean() < 0.7       # D^2 spans 2^+-80, in shuffled order
    A0 = C.family("random", n)[0]
    assert C.equilibrated_kappa(A) < 10 * C.equilibrated_kappa(A0) and np.linalg.cond(A) > 1e40
    A, _ = C.family("block", n)
    for J in range(0, n, 8):
        assert np.linalg.cond(A[J:J + 8, J:J + 8]) > 1e6
    # the diagonal tiles the kernel factors (after the left-looking update) stay as ill-conditioned
    L = np.linalg.cholesky(A)
    for J in range(8, n, 8):
        T = L[J:J + 8, J:J + 8] @ L[J:J + 8, J:J + 8].T
        assert np.linalg.cond(T) > 1e6
    for m in (8, 64, 383):
        A, b = C.family("near_singular", m)
        w = np.linalg.eigvalsh(A)
        assert 0 < w.min() < 1e-11 and C.port_solve(A, b) is not None
        B = A - 2 * w.min() * np.eye(m)                     # the same system just below the failure point
        assert C.port_solve(B, b) is None
    for name, p in C.SCALES.items():
        A, _ = C.family(name, 64)
        assert np.all(np.abs(np.log2(np.abs(A[A != 0])) - p) < 40) and np.abs(A).min() >= 0
        assert np.diag(A).min() >= C.DBL_MIN
    assert C.family("scale-1000", 8)[0].min() < 2.0 ** -990
    ex = C.diag_exponents()
    assert len(ex) == 1001 and ex.min() == -1000 and ex.max() == 1000 and np.all(ex % 2 == 0)


def test_sqrt_rsqrt_restatement():
    """Exact on 4^k and within one ulp on 2 4^k over the whole normal range; the subnormal and infinite pivots get the
    wrong roots the kernel's pivot rule has to refuse."""
    for e in range(-1022, 1024):
        x = np.ldexp(1.0, e)
        sq, rs = C.sqrt_rsqrt(x)
        if e % 2 == 0:
            assert sq == np.ldexp(1.0, e // 2) and rs == np.ldexp(1.0, -e // 2), e
        else:
            assert C.ulps(sq, np.sqrt(x)) <= 1 and C.ulps(rs, 1 / np.sqrt(x)) <= 1, e
    sq, _ = C.sqrt_rsqrt(1e-310)
    assert abs(sq / 1e-155 - 1) > 0.05                      # 1.057e-154 instead of 1e-155
    assert np.isfinite(C.sqrt_rsqrt(np.inf)[0])             # 2^512: a finite root of +inf
    for bad in (1e-310, 5e-324, np.inf, np.nan, 0.0, -1.0, -np.inf):
        assert not C.pivot_ok(bad)
    for good in (C.DBL_MIN, C.DBL_MAX, 1.0):
        assert C.pivot_ok(good)


def test_port_exact_on_diagonal_systems():
    ex = C.diag_exponents()
    A, b = C.diag_system(ex[:120], odd=False)
    assert np.array_equal(C.port_solve(A, b), b / np.diag(A))
    A, b = C.diag_system(ex[-120:], odd=True)
    assert C.ulps(C.port_solve(A, b), b / np.diag(A)).max() <= 3


def test_port_refuses_subnormal_pivots():
    assert C.port_solve(1e-310 * np.eye(3), np.full(3, 1e-300)) is None
    a = 2.0 ** -1000
    A = a * np.array([[1.0, 1.0 - 2.0 ** -30], [1.0 - 2.0 ** -30, 1.0]])      # the second pivot is subnormal
    assert C.port_solve(A, np.array([a, a])) is None


def test_tile_geometry():
    """Where the factor stops fitting the 376 shared-memory tiles: 26 block rows (nc <= 207)."""
    assert (C.n8(207), C.ntiles(207), C.spills(207)) == (26, 351, False)
    assert (C.n8(208), C.ntiles(208), C.spills(208)) == (27, 378, True)
    assert C.spills(215) and C.spills(383) and not C.spills(64) and C.spills(64, 0)
    assert C.n8(223) == 28 and C.n8(224) == 29
