"""References, test matrices and calibrated bars for the back end's dense SPD solve on its own (ba_chol.cuh: chol_factor +
chol_backsubst, reached through gf_stage_spd_solve / estimator.spd_solve), CPU only.

  * families(): the test systems (A, b): random, graded spectra, D A D with D spanning 2^+-40, ill-conditioned 8x8 diagonal
    blocks, near-singular, uniform scalings 2^-1000 .. 2^+500, diag(4^k) / diag(2 4^k) over the normal exponent range, and
    the reduced systems S of ba_lin_ref's windows.
  * solve_ref(): x = A^-1 b in np.longdouble by iterative refinement (residual in longdouble, corrections from LAPACK's
    factor); solve_mp(): the same in mpmath (small n; test_chol_ref.py pins the first against the second).
  * metrics(): normwise backward error eta = ||b - A x||_inf / (||A||_inf ||x||_inf + ||b||_inf), componentwise backward
    error omega = max_i |b - A x|_i / (|A| |x| + |b|)_i and the forward error of the equilibrated system
    fwd = ||E (x - x_ref)||_2 / (kappa_2(E^-1 A E^-1) ||E x_ref||_2), E = diag(sqrt(a_ii)) (Cholesky is invariant under a
    symmetric diagonal scaling, so this is the kappa that governs its error), each in units of eps, computed in longdouble.
  * port_solve(): the kernel's algorithm in NumPy: the (n+1)-row augmented system with b as row n and identity padding,
    left-looking on 8x8 tiles, each diagonal tile factored by the kernel's straight-line chol8_inv (sqrt_rsqrt restated bit
    by bit: exponent scaling, a single-precision rsqrt seed, two coupled Newton steps and a last correction; padding columns
    as identity; its pivot rule), the explicit inverse of L_JJ built row by row, the TRSM and the back substitution through
    that inverse.  With steps=1 and a seed at MUFU.RSQ's 2^-22 accuracy it is the negative control: sqrt_rsqrt then loses
    one Newton step (~2^-44 relative error), which the bars must catch.

Bars, per family: K[family][bar] = CALIBRATION_FACTOR x the worst ratio of the port and of LAPACK (scipy cho_factor /
cho_solve) over the family at every size 1 .. 64 and at 120 .. 383, rounded up to one digit (test_chol_ref.py recomputes
the worst ratios and prints them).  Systems outside the families (edge cases) are held to the "random" bars.
"""
import struct

import mpmath as mp
import numpy as np
import scipy.linalg

from marg_ref import EPS, LD

CALIBRATION_FACTOR = 8
TILE_CAP = 376                 # ba_chol.cuh: factor tiles resident in shared memory
MAX_NC = 383
SMEM_ROWS = 28                 # (MAXR / 2) * CH_BULK: block rows of the shared-memory instantiation
DBL_MIN = float(np.finfo(np.float64).tiny)
DBL_MAX = float(np.finfo(np.float64).max)
# family -> bar -> K.  eta: normwise backward error / eps; omega: componentwise backward error / eps; fwd: forward error of the
# equilibrated system / (eps kappa).  The graded spectra at kappa 1e12 need the most: the explicit inverse of an
# ill-conditioned 8x8 factor (the kernel's TRSM and back substitution) is where it loses to LAPACK's substitution.
K = {
    "random": {"eta": 4, "omega": 20, "fwd": 8},            # worst CPU eta 0.496 (LAPACK, n=1), omega 1.62 (LAPACK, n=256), fwd 0.992 (LAPACK, n=1)
    "graded1e4": {"eta": 5, "omega": 10, "fwd": 3},         # worst CPU eta 0.512 (port, n=2), omega 1.24 (port, n=9), fwd 0.303 (port, n=2)
    "graded1e8": {"eta": 8, "omega": 40, "fwd": 2},         # worst CPU eta 0.882 (port, n=5), omega 3.87 (port, n=9), fwd 0.147 (port, n=23)
    "graded1e12": {"eta": 60, "omega": 200, "fwd": 4},      # worst CPU eta 6.83 (port, n=10), omega 24.5 (port, n=10), fwd 0.405 (LAPACK, n=2)
    "graded1e14": {"eta": 6, "omega": 70, "fwd": 2},        # worst CPU eta 0.655 (port, n=17), omega 7.92 (port, n=10), fwd 0.243 (port, n=12)
    "dad": {"eta": 5, "omega": 7, "fwd": 9},                # worst CPU eta 0.513 (LAPACK, n=1), omega 0.867 (port, n=62), fwd 1.03 (LAPACK, n=1)
    "block": {"eta": 5, "omega": 10, "fwd": 3},             # worst CPU eta 0.535 (port, n=3), omega 1.24 (LAPACK, n=25), fwd 0.367 (port, n=1)
    "near_singular": {"eta": 10, "omega": 20, "fwd": 8},    # worst CPU eta 1.14 (port, n=6), omega 2.44 (LAPACK, n=383), fwd 0.931 (port, n=1)
    "scale-1000": {"eta": 4, "omega": 20, "fwd": 7},        # worst CPU eta 0.393 (LAPACK, n=1), omega 1.28 (LAPACK, n=216), fwd 0.787 (LAPACK, n=1)
    "scale-500": {"eta": 4, "omega": 9, "fwd": 6},          # worst CPU eta 0.425 (LAPACK, n=2), omega 1.04 (LAPACK, n=22), fwd 0.679 (port, n=1)
    "scale+250": {"eta": 4, "omega": 7, "fwd": 6},          # worst CPU eta 0.465 (LAPACK, n=5), omega 0.852 (port, n=383), fwd 0.747 (port, n=3)
    "scale+500": {"eta": 6, "omega": 9, "fwd": 20},         # worst CPU eta 0.728 (LAPACK, n=1), omega 1.03 (port, n=207), fwd 1.46 (LAPACK, n=1)
    "window": {"eta": 4, "omega": 60, "fwd": 2},            # worst CPU eta 0.422 (port, visual_only_F6), omega 6.75 (port, plane_wheel), fwd 0.182 (port, stationary_wheel)
}
BARS = ("eta", "omega", "fwd")
CAL_SIZES = tuple(range(1, 65)) + (120, 207, 216, 256, 300, 383)
NEG_SIZES = (1, 2, 7, 8, 9, 16, 33, 64, 120, 207, 216, 383)


# ---- tile geometry ----------------------------------------------------------------------------------------------------
def n8(n):
    return (n + 8) // 8


def ntiles(n):
    return n8(n) * (n8(n) + 1) // 2


def tix(I, J):
    return I * (I + 1) // 2 + J


def spills(n, tile_cap=-1):
    """True when gf_stage_spd_solve takes the <MAXR, true> instantiation (the factor does not fit the shared tiles)."""
    cap = tile_cap if 0 <= tile_cap < TILE_CAP else TILE_CAP
    return not (ntiles(n) <= cap and n8(n) <= SMEM_ROWS)


# ---- sqrt_rsqrt and chol8_inv, restated --------------------------------------------------------------------------------
def _hl(x):
    b = struct.unpack("<q", struct.pack("<d", x))[0]
    return b >> 32, b & 0xffffffff


def _d(hi, lo):
    v = ((hi & 0xffffffff) << 32) | lo
    return struct.unpack("<d", struct.pack("<Q", v & 0xffffffffffffffff))[0]


def _fma(a, b, c):
    return float(LD(a) * LD(b) + LD(c))


def sqrt_rsqrt(x, steps=2, seed_err=0.0):
    """ba_chol.cuh's sqrt_rsqrt on a double: (sqrt(x), 1/sqrt(x)) for a positive normal x, garbage otherwise (as on the
    device).  steps / seed_err: the negative control's weakened variant."""
    hi, lo = _hl(float(x))
    e = ((((hi >> 20) & 0x7ff) - 1023) & ~1)
    xs = _d(hi - (e << 20), lo)
    with np.errstate(all="ignore"):
        y = float(np.float32(1) / np.sqrt(np.float32(xs))) * (1.0 + seed_err)
    g, h = xs * y, 0.5 * y
    for _ in range(steps):
        r = _fma(-g, h, 0.5)
        g, h = _fma(g, r, g), _fma(h, r, h)
    r = _fma(-g, g, xs)
    g = _fma(r, h, g)
    h = h + h
    he = (e >> 1) << 20
    gh, gl = _hl(g)
    hh, hlo = _hl(h)
    return _d(gh + he, gl), _d(hh - he, hlo)


def pivot_ok(dk):
    """chol8_inv's pivot rule: positive and normal."""
    return DBL_MIN <= dk <= DBL_MAX


def chol8_inv(S8, ncol, steps=2, seed_err=0.0):
    """(L, inverse of L, ok) of one updated 8x8 diagonal tile (lower triangle read), as the diagonal warp computes them."""
    a = np.tril(np.asarray(S8, np.float64)).copy()
    ok = True
    inv = np.zeros(8)
    with np.errstate(all="ignore"):
        for k in range(8):
            live = k < ncol
            dk = float(a[k, k]) if live else 1.0
            ok = ok and pivot_ok(dk)
            sq, r = sqrt_rsqrt(dk, steps, seed_err)
            inv[k] = r
            a[k, k] = sq
            a[k + 1:, k] = a[k + 1:, k] * r if live else 0.0
            c = a[k + 1:, k].astype(LD)
            a[k + 1:, k + 1:] = np.tril(a[k + 1:, k + 1:].astype(LD) - np.outer(c, c)).astype(np.float64)
        li = np.zeros((8, 8))
        for r in range(8):
            for c in range(r):
                s0 = s1 = 0.0
                for m in range(c, r, 2):
                    s0 = _fma(a[r, m], li[m, c], s0)
                    if m + 1 < r:
                        s1 = _fma(a[r, m + 1], li[m + 1, c], s1)
                li[r, c] = -(s0 + s1) * inv[r]
            li[r, r] = inv[r]
    return np.tril(a), li, ok


def port_solve(A, b, steps=2, seed_err=0.0):
    """x = A^-1 b by the kernel's algorithm (module docstring); None where the kernel reports a failed pivot."""
    A = np.asarray(A, np.float64)
    b = np.asarray(b, np.float64)
    n = len(b)
    m8 = n8(n)
    N = 8 * m8
    M = np.eye(N)
    M[:n, :n] = np.tril(A) + np.tril(A, -1).T
    M[n, :n] = b
    L = np.zeros((N, N))
    Linv = []
    ok = True
    with np.errstate(all="ignore"):
        for J in range(m8):
            s = slice(8 * J, 8 * J + 8)
            Lj, li, okj = chol8_inv(M[s, s] - L[s, :8 * J] @ L[s, :8 * J].T, min(8, n - 8 * J), steps, seed_err)
            ok = ok and okj
            L[s, s] = Lj
            Linv.append(li)
            for I in range(J + 1, m8):
                t = slice(8 * I, 8 * I + 8)
                L[t, s] = (M[t, s] - L[t, :8 * J] @ L[s, :8 * J].T) @ li.T
        if not ok:
            return None
        z = L[n, :n]
        y = np.zeros(N)
        for J in range((n - 1) // 8, -1, -1):
            c0, m = 8 * J, min(8, n - 8 * J)
            rhs = np.zeros(8)
            rhs[:m] = z[c0:c0 + m] - L[c0 + 8:n, c0:c0 + 8][:, :m].T @ y[c0 + 8:n]
            y[c0:c0 + m] = (Linv[J].T @ rhs)[:m]
    return y[:n]


def lapack_solve(A, b):
    return scipy.linalg.cho_solve(scipy.linalg.cho_factor(A, lower=True), b)


# ---- references ---------------------------------------------------------------------------------------------------------
def solve_ref(A, b, iters=8):
    """x = A^-1 b in longdouble: LAPACK's Cholesky in double, then refinement with longdouble residuals until the correction
    is below longdouble's resolution.  Exact systems (diagonal A) come out exact."""
    A64 = np.tril(A) + np.tril(A, -1).T
    Al, bl = A64.astype(LD), np.asarray(b, LD)
    cf = scipy.linalg.cho_factor(A64, lower=True)
    x = np.asarray(scipy.linalg.cho_solve(cf, np.asarray(b, np.float64)), LD)
    for _ in range(iters):
        r = bl - Al @ x
        rs = float(np.abs(r).max())
        if rs == 0.0:
            break
        sc = 2.0 ** -np.floor(np.log2(rs))          # keeps the correction's right-hand side away from underflow
        dx = np.asarray(scipy.linalg.cho_solve(cf, np.asarray(r * LD(sc), np.float64)), LD) / LD(sc)
        x = x + dx
        if float(np.abs(dx).max()) <= 1e-21 * float(np.abs(x).max()):
            break
    return x


def solve_mp(A, b, dps=60):
    """x = A^-1 b in mpmath (LU at `dps` digits), as longdouble."""
    A64 = np.tril(A) + np.tril(A, -1).T
    with mp.workdps(dps):
        x = mp.lu_solve(mp.matrix(A64.tolist()), mp.matrix(np.asarray(b, np.float64).tolist()))
        return np.array([LD(mp.nstr(v, 30)) for v in x])


def equilibrated_kappa(A):
    A64 = np.tril(A) + np.tril(A, -1).T
    e = 1.0 / np.sqrt(np.diag(A64))
    w = np.linalg.eigvalsh(A64 * e[:, None] * e[None, :])
    return float(w.max() / w.min()) if w.min() > 0 else np.inf


def metrics(A, b, x, xref, kappa):
    """{eta, omega, fwd} of the solution x in units of eps (module docstring); kappa: equilibrated_kappa(A)."""
    A64 = np.tril(A) + np.tril(A, -1).T
    Al, bl, xl = A64.astype(LD), np.asarray(b, LD), np.asarray(x, LD)
    r = np.abs(bl - Al @ xl)
    aA = np.abs(Al)
    eta = r.max() / (aA.sum(1).max() * np.abs(xl).max() + np.abs(bl).max())
    den = aA @ np.abs(xl) + np.abs(bl)
    omega = np.where(den > 0, r / np.where(den > 0, den, 1), np.where(r > 0, np.inf, 0)).max()
    E = np.sqrt(np.diag(Al))
    fe = np.sqrt((((xl - xref) * E) ** 2).sum()) / np.sqrt(((xref * E) ** 2).sum()) if np.any(xref != 0) else LD(0)
    return {"eta": float(eta) / EPS, "omega": float(omega) / EPS, "fwd": float(fe) / (EPS * kappa)}


# ---- test matrices ------------------------------------------------------------------------------------------------------
GRADED = {"graded1e4": 4, "graded1e8": 8, "graded1e12": 12, "graded1e14": 14}
SCALES = {"scale-1000": -1000, "scale-500": -500, "scale+250": 250, "scale+500": 500}
FAMILIES = ("random", *GRADED, "dad", "block", "near_singular", *SCALES)
BLOCK_BUMP = 1e8


def _orth(rng, n):
    Q, R_ = np.linalg.qr(rng.standard_normal((n, n)))
    return Q * np.sign(np.diag(R_))


def _spectral(rng, w):
    Q = _orth(rng, len(w))
    A = (Q * w) @ Q.T
    return np.tril(A) + np.tril(A, -1).T


def _wishart(rng, n):
    B = rng.standard_normal((n, n + 5))
    return B @ B.T + np.eye(n)


def family(name, n, seed=0):
    """(A, b) of family `name` at size n (A symmetric, both exactly as passed to the solver)."""
    rng = np.random.default_rng([seed, n, FAMILIES.index(name)])
    b = rng.standard_normal(n)
    if name == "random":
        A = _wishart(rng, n)
    elif name in GRADED:
        A = _spectral(rng, np.logspace(0, GRADED[name], n) if n > 1 else np.ones(1))
    elif name == "dad":                                     # D A0 D, D = 2^k with k spanning -40 .. 40 in shuffled order
        d = 2.0 ** np.round(np.linspace(-40, 40, n)) if n > 1 else np.full(1, 2.0 ** 40)
        rng.shuffle(d)
        A = _wishart(rng, n) * d[:, None] * d[None, :]
        b = b * d
    elif name == "block":                                   # a rank-1 bump of 1e8 inside every 8x8 diagonal block
        A = _wishart(rng, n)
        for J in range(0, n, 8):
            m = min(8, n - J)
            v = rng.standard_normal(m)
            A[J:J + m, J:J + m] += BLOCK_BUMP * np.outer(v, v)
    elif name == "near_singular":                           # one eigenvalue 64 n eps above 0, the others in [0.5, 1]
        w = rng.uniform(0.5, 1.0, n)
        w[rng.integers(n)] = 64 * max(n, 8) * EPS
        A = _spectral(rng, w)
    elif name in SCALES:
        A = _wishart(rng, n) * 2.0 ** SCALES[name]
    else:
        raise ValueError(name)
    return A, b


def diag_exponents():
    """The 1001 exponents 2k of 4^k covering -1000 .. 1000 (even) and, with the factor 2, the odd ones -999 .. 1001."""
    return np.arange(-1000, 1001, 2)


def diag_system(exps, odd, seed=0):
    """A = diag(4^k) (odd=False) or diag(2 4^k) for the exponents 2k in `exps`, b in [1, 2): x = b / a exactly
    representable for 4^k."""
    rng = np.random.default_rng([seed, len(exps), int(odd)])
    a = np.ldexp(1.0, np.asarray(exps) + (1 if odd else 0))
    b = rng.uniform(1.0, 2.0, len(a))
    return np.diag(a), b


def window_systems(names=("stationary_wheel", "visual_only_F6", "c2_s0", "plane_wheel")):
    """name -> (S, rhs, ref) of the reduced systems ba_lin_ref.reference builds for the stage-test windows (S's lower triangle
    and rhs rounded to double; nc = 10, 30, 165, 179)."""
    import ba_lin_ref as R
    w = R.windows()
    out = {}
    for name in names:
        ref = R.reference(w[name]())
        S = np.asarray(ref["S"], np.float64)
        out[name] = (np.tril(S) + np.tril(S, -1).T, np.asarray(ref["rhs"], np.float64), ref)
    return out


def ulps(x, want):
    """|x - want| in units in the last place of want (elementwise)."""
    x, want = np.asarray(x, np.float64), np.asarray(want, np.float64)
    return np.abs(x - want) / np.spacing(np.abs(want))
