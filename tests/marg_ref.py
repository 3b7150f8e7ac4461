"""The marginalisation's arithmetic, restated at high precision for the tests: MarginalizationInfo::marginalize
(marginalization_factor.cpp:272-302) and the symmetric eigendecompositions it performs, plus the test matrices.

Two restatements of the same steps -- symmetrise Amm, take its eigen-truncated inverse (eigenvalues <= 1e-8 dropped), form
the Schur complement A = Arr - Arm Amm^+ Amr, b = brr - Arm Amm^+ bmm, decompose A from its lower triangle, J0 = sqrt(S) V^T,
r0 = sqrt(S^-1) V^T b:
  * marginalize_mp: literally, in mpmath (small sizes only: mpmath.eigsy costs about a second at n = 40);
  * marginalize_ld: in np.longdouble (64-bit significand) using the structure the device code relies on -- the landmark
    block is diagonal, landmarks are 1x1 pivots, the c x c block is solved in mpmath -- and, when Amm - 1e-8 I is not
    positive definite, a refined eigendecomposition of the whole Amm.  Eigenvectors come from LAPACK in double and are
    refined in longdouble (Ogita & Aishima, "Iterative refinement for symmetric eigenvalue decomposition", Japan J. Indust.
    Appl. Math. 35, 2018), which converges quadratically, clusters included.
Matrices with a known spectrum are A = Q diag(lam) Q^T with Q a product of Householder reflectors, formed once at high
precision and rounded to double; the eigenvalues of the rounded matrix are then lam within the Weyl bound of that rounding.

Bars: ratio = error / (n eps scale).  The GPU tests assert ratio <= K; on the same inputs the oracle's C restatements of the
two eigensolvers (oracle/ba_oracle.c) stay below K / CALIBRATION_FACTOR (tests/test_marg_stages_ref.py), so K sits a fixed
factor above what the algorithms achieve in double on a CPU.
"""
import mpmath as mp
import numpy as np

EPS_MARG = 1e-8            # marginalization_factor.cpp:280, 294
EPS = np.finfo(np.float64).eps
LD = np.longdouble
DPS = 40

CALIBRATION_FACTOR = 8
# worst ratio of the oracle's QL / Jacobi over every eigen case of the GPU tests (CPU, gcc -O2 -ffp-contract=off), rounded up,
# times CALIBRATION_FACTOR:
K_EIGVAL = 24.0            # |sort(w) - lam|_max / (n eps ||A||_2)                    worst CPU 2.63 (Jacobi, n = 520)
K_ORTH = 48.0              # ||V^T V - I||_2 / (n eps)                                 worst CPU 5.82 (Jacobi, n = 520)
K_RESID = 24.0             # ||A V - V diag(w)||_2 / (n eps ||A||_2)                   worst CPU 2.63 (Jacobi, n = 520)
K_PROJ = 16.0              # ||P - P_exact||_2 gap / (n eps ||A||_2), separated clusters   worst CPU 1.22 (QL, n = 3)
# worst ratio of the literal algorithm in double with the oracle's QL or Jacobi over the marginalisation cases, rounded up
# to one digit, times CALIBRATION_FACTOR:
K_JTJ = 16.0               # |J0^T J0 - JtJ|_max / (N eps schur_scale)       worst CPU 1.05 (Jacobi, c6_L1_n76)
K_JTR = 0.24               # |J0^T r0 - Jtr|_max / (N eps b_scale)           worst CPU 0.024 (QL, c6_L0_n1)
K_RTR = 0.24               # |r0^T r0 - b^T A^+ b| / (N eps rtr_scale)       worst CPU 0.022 (QL, c6_L1_n1)


def ld_to_mp(x):
    """A longdouble as an exact mpf (double head + double tail)."""
    hi = float(x)
    return mp.mpf(hi) + mp.mpf(float(LD(x) - LD(hi)))


def mp_to_ld(x):
    hi = float(x)
    return LD(hi) + LD(float(x - mp.mpf(hi)))


def _to_ld(M, r, c):
    return np.array([[mp_to_ld(M[i, j]) for j in range(c)] for i in range(r)], dtype=LD).reshape(r, c)


# ------------------------------------------------------------------------------------------------ known spectra
def known_spectrum(lam, seed, k=3, exact="auto"):
    """A = Q diag(lam) Q^T, Q = H_1 ... H_k, H_i = I - 2 v v^T / v^T v with float64 v (exactly orthogonal as a real matrix).
    Formed in mpmath (exact="mp", the default up to n = 33) or in longdouble, rounded to double once.
    Returns (A float64 exactly symmetric, Q longdouble: columns = eigenvectors of the unrounded matrix, ||A - A_exact||_F)."""
    lam = np.asarray(lam, np.float64)
    n = len(lam)
    rng = np.random.default_rng(seed)
    vs = [rng.standard_normal(n) for _ in range(k)]
    if exact == "auto":
        exact = "mp" if n <= 33 else "ld"
    if exact == "mp":
        mp.mp.dps = DPS
        M = mp.diag([mp.mpf(float(x)) for x in lam])
        Qm = mp.eye(n)
        for v in reversed(vs):                        # M <- H M H, innermost reflector first
            vm = mp.matrix([mp.mpf(float(x)) for x in v]); s = (vm.T * vm)[0]
            Mv = M * vm; vMv = (vm.T * Mv)[0]
            M = M - (2 / s) * (vm * Mv.T + Mv * vm.T) + (4 * vMv / (s * s)) * (vm * vm.T)
        for v in vs:
            vm = mp.matrix([mp.mpf(float(x)) for x in v]); s = (vm.T * vm)[0]
            Qm = Qm - (2 / s) * ((Qm * vm) * vm.T)
        Ahi, Q = _to_ld(M, n, n), _to_ld(Qm, n, n)
    else:
        Ahi = np.diag(lam.astype(LD))
        for v in reversed(vs):
            v = v.astype(LD); s = v @ v
            Av = Ahi @ v; vAv = v @ Av
            Ahi = Ahi - (2 / s) * (np.outer(v, Av) + np.outer(Av, v)) + (4 * vAv / (s * s)) * np.outer(v, v)
        Q = np.eye(n, dtype=LD)
        for v in vs:
            v = v.astype(LD); s = v @ v
            Q = Q - (2 / s) * np.outer(Q @ v, v)
    Ahi = (Ahi + Ahi.T) / 2
    A = Ahi.astype(np.float64)
    A = np.tril(A) + np.tril(A, -1).T
    return A, Q, float(np.sqrt(((A.astype(LD) - Ahi) ** 2).sum()))


EIG_KINDS = ("spd", "graded", "gauge", "zero_row", "diagonal", "multiple", "indefinite", "zero")


def eig_case(kind, n, seed=0):
    """(A, lam ascending, Q longdouble with the matching eigenvectors in its columns) for one input kind:
    spd: random SPD; graded: spectrum 1e-3 .. 1e9 (VIO scale); gauge: PSD at ||A|| ~ 1e9 with a 4-dimensional null space;
    zero_row: a zero row and column (tred2's scale == 0 branch, like the plane rotation's unused fourth column);
    diagonal; multiple: eigenvalues of multiplicity 3 to 10; indefinite; zero: the zero matrix."""
    rng = np.random.default_rng(1000 * seed + 16 * n + EIG_KINDS.index(kind))
    sub = seed * 100003 + 31 * n + EIG_KINDS.index(kind)
    if kind == "diagonal":
        lam = rng.uniform(-3.0, 3.0, n) * 10.0 ** rng.uniform(-2, 2, n)
        A, Q = np.diag(lam), np.eye(n, dtype=LD)
    elif kind == "zero":
        lam, A, Q = np.zeros(n), np.zeros((n, n)), np.eye(n, dtype=LD)
    elif kind == "zero_row":
        k = int(rng.integers(0, n))
        lsub = rng.uniform(0.5, 50.0, n - 1)
        idx = [i for i in range(n) if i != k]
        A, Q = np.zeros((n, n)), np.zeros((n, n), LD)
        if n > 1:
            As, Qs, _ = known_spectrum(lsub, sub)
            A[np.ix_(idx, idx)] = As
            Q[np.ix_(idx, list(range(n - 1)))] = Qs
        Q[k, n - 1] = 1
        lam = np.concatenate([lsub, [0.0]])
    else:
        if kind == "spd":
            lam = rng.uniform(0.1, 10.0, n)
        elif kind == "graded":
            lam = np.logspace(-3, 9, n) * rng.uniform(0.9, 1.1, n)
        elif kind == "gauge":
            z = min(4, n - 1)
            lam = np.concatenate([np.zeros(z), np.logspace(0, 9, n - z)])
        elif kind == "indefinite":
            lam = rng.uniform(-10.0, 10.0, n)
        elif kind == "multiple":
            vals = []
            while len(vals) < n:
                vals += [float(np.round(rng.uniform(-5, 5), 3))] * int(rng.integers(3, 11))
            lam = np.array(vals[:n])
        else:
            raise ValueError(kind)
        A, Q, _ = known_spectrum(lam, sub)
    order = np.argsort(lam, kind="stable")
    return A, np.asarray(lam, np.float64)[order], Q[:, order]


JACOBI_BOUND = 2304        # the largest Jacobi size gf_stage_sym_eig / gf_stage_marginalize take (above 2048: > 1 rotation per thread)


def eig_case_bound(n=JACOBI_BOUND, seed=0):
    """The Jacobi bound case: 3 x 3 known-spectrum blocks (eigenvalues 1e-3 .. 1e9 and a 4-dimensional null space, as the
    gauge and graded kinds) scattered over random index triples, so that rotations pair low and high indices in every round.
    Returns (A, lam ascending, Q) like eig_case."""
    rng = np.random.default_rng(seed + 77)
    lam = np.concatenate([np.zeros(4), np.logspace(-3, 9, n - 4) * rng.uniform(0.9, 1.1, n - 4)])
    lam = lam[rng.permutation(n)]
    perm = rng.permutation(n)
    A, Q = np.zeros((n, n)), np.zeros((n, n), LD)
    for k in range(n // 3):
        idx = perm[3 * k:3 * k + 3]
        Ab, Qb, _ = known_spectrum(lam[3 * k:3 * k + 3], seed + k, exact="ld")
        A[np.ix_(idx, idx)] = Ab
        Q[np.ix_(idx, np.arange(3 * k, 3 * k + 3))] = Qb
    order = np.argsort(lam, kind="stable")
    return A, lam[order], Q[:, order]


def clusters(lam, norm, rel_gap=1e-3):
    """Index ranges [lo, hi) of ascending lam whose neighbours lie more than rel_gap * norm away, with that gap; the whole
    spectrum (projector = I) is left out."""
    n = len(lam)
    cuts = [0] + [i for i in range(1, n) if lam[i] - lam[i - 1] > rel_gap * norm] + [n]
    out = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        if b - a < n:
            left = lam[a] - lam[a - 1] if a > 0 else np.inf
            right = lam[b] - lam[b - 1] if b < n else np.inf
            out.append((a, b, min(left, right)))
    return out


def eig_ratios(A, lam, Q, w, V, dt=LD):
    """The four eigensolver bars' ratios for a computed decomposition (w, V) of A (exact eigenpairs lam, Q).  The products
    are formed in longdouble; dt=np.float64 is for the bound case (n = 2304), whose A and Q have three nonzeros per row
    and column, so that double's rounding of V^T V (~ sqrt(n) eps) stays far below the bars (K n eps)."""
    n = len(lam)
    norm = float(np.abs(lam).max())
    order = np.argsort(w, kind="stable")
    w, V = np.asarray(w, np.float64)[order], np.asarray(V, np.float64)[:, order]
    unit = n * EPS
    Vl = V.astype(dt)
    Q = Q.astype(dt)
    orth = np.linalg.norm((Vl.T @ Vl - np.eye(n, dtype=dt)).astype(np.float64), 2) / unit
    if norm == 0.0:
        exact = 0.0 if np.all(w == 0) else np.inf
        return dict(eigval=exact, orth=orth, resid=exact, proj=0.0)
    eigval = np.abs(w - lam).max() / (unit * norm)
    resid = np.linalg.norm((A.astype(dt) @ Vl - Vl * w.astype(dt)).astype(np.float64), 2) / (unit * norm)
    proj = 0.0
    M = (Q.T @ Vl).astype(np.float64)                  # ||P - P_exact||_2 = ||Q_out^T V_in||_2 for orthonormal bases
    for a, b, gap in clusters(lam, norm):
        out = np.r_[0:a, b:n]
        proj = max(proj, np.linalg.norm(M[np.ix_(out, np.r_[a:b])], 2) * gap / (unit * norm))
    return dict(eigval=eigval, orth=orth, resid=resid, proj=proj)


# ------------------------------------------------------------------------------------------------ refined eigh
def refine_eigh(A, iters=3):
    """Eigendecomposition of a symmetric longdouble matrix: LAPACK in double, then Ogita-Aishima refinement in longdouble.
    Eigenvalues within 1e-10 ||A|| of each other are refined as one cluster (the invariant subspace is accurate, the basis
    inside it is any orthonormal one).  Returns (w ascending, X), longdouble."""
    A = np.asarray(A, LD)
    n = A.shape[0]
    w, X = np.linalg.eigh(A.astype(np.float64))
    X = X.astype(LD)
    normA = max(float(np.abs(w).max()), 1e-300)
    I = np.eye(n, dtype=LD)
    lam = w.astype(LD)
    for _ in range(iters):
        R = I - X.T @ X
        S = X.T @ A @ X
        lam = np.diag(S) / (1 - np.diag(R))
        delta = 2 * (np.linalg.norm((S - np.diag(lam)).astype(np.float64), 2) + normA * np.linalg.norm(R.astype(np.float64), 2))
        delta = max(delta, 1e-10 * normA)     # closer eigenvalues form one cluster: its subspace converges, not its vectors
        dl = lam[None, :] - lam[:, None]                            # lam_j - lam_i
        sep = np.abs(dl.astype(np.float64)) > delta
        E = np.where(sep, (S + lam[None, :] * R) / np.where(sep, dl, LD(1)), R / 2)
        X = X + X @ E
    order = np.argsort(lam.astype(np.float64), kind="stable")
    return lam[order], X[:, order]


# ------------------------------------------------------------------------------------------------ marginalisation
def _outputs(Ar, br, w, V, eps=EPS_MARG):
    """J0^T J0 = V_k S V_k^T, J0^T r0 = V_k V_k^T b, r0^T r0 = b^T A^+ b and the number of kept eigenvalues (nonzero rows of
    J0) from the reduced system's decomposition."""
    keep = w > eps
    Vk, wk = V[:, keep], w[keep]
    y = Vk.T @ br
    return dict(Ar=Ar, br=br, w=w, V=V, rank=int(keep.sum()), JtJ=(Vk * wk) @ Vk.T, Jtr=Vk @ y, rtr=(y * y / wk).sum(),
                x=Vk @ (y / wk))


def marginalize_mp(A, b, m, eps=EPS_MARG):
    """marginalization_factor.cpp:272-302 in mpmath, literally.  Returns longdouble arrays (see _outputs)."""
    mp.mp.dps = DPS
    N = len(b); n = N - m
    Am = mp.matrix([[mp.mpf(float(x)) for x in row] for row in A])
    bm = mp.matrix([mp.mpf(float(x)) for x in b])
    Amm = mp.matrix(m, m)
    for i in range(m):
        for j in range(m):
            Amm[i, j] = (Am[i, j] + Am[j, i]) / 2
    E, Qe = mp.eigsy(Amm)
    Ainv = mp.matrix(m, m)
    for k in range(m):
        if E[k] > eps:
            col = Qe[:, k]
            Ainv += (col * col.T) / E[k]
    T = Am[m:N, 0:m] * Ainv
    Ar = Am[m:N, m:N] - T * Am[0:m, m:N]
    br = bm[m:N, 0] - T * bm[0:m, 0]
    Al = mp.matrix(n, n)
    for i in range(n):
        for j in range(i + 1):
            Al[i, j] = Al[j, i] = Ar[i, j]               # SelfAdjointEigenSolver reads the lower triangle
    E2, Q2 = mp.eigsy(Al)
    w = np.array([mp_to_ld(E2[k]) for k in range(n)], dtype=LD)
    V = _to_ld(Q2, n, n)
    order = np.argsort(w.astype(np.float64), kind="stable")
    out = _outputs(_to_ld(Al, n, n), _to_ld(br, n, 1)[:, 0], w[order], V[:, order], eps)
    out.update(scales(A, b, m, out), N=N)
    return out


def _mp_min_eig(C):
    mp.mp.dps = DPS
    return float(min(mp.eigsy(mp.matrix([[ld_to_mp(x) for x in row] for row in C]), eigvals_only=True)))


def _mp_solve(C, R):
    """C^-1 R for a small longdouble C (c x c) and R (c x k), in mpmath."""
    mp.mp.dps = DPS
    X = mp.inverse(mp.matrix([[ld_to_mp(x) for x in row] for row in C])) * mp.matrix([[ld_to_mp(x) for x in row] for row in R])
    return _to_ld(X, X.rows, X.cols)


def marginalize_ld(A, b, c, L, eps=EPS_MARG):
    """The same in longdouble for a symmetric A with a diagonal landmark block.  Landmarks whose row of Amm is zero (no
    information) carry an exact zero eigenvalue of Amm and drop out of the eigen-truncated inverse.  If the rest passes
    Amm - eps I > 0 (landmark pivots > eps and the eps-shifted c x c Schur complement positive definite, decided in mpmath)
    the truncated inverse is the inverse and the two-stage elimination (landmarks, then the c x c block in mpmath) is exact;
    otherwise Amm is decomposed whole (refine_eigh).  Returns longdouble arrays (see _outputs), the error scales (see
    scales) and 'path': 'fast' when the structured test passes on the whole Amm, else 'generic'."""
    A = np.asarray(A, np.float64); b = np.asarray(b, np.float64)
    assert np.array_equal(A, A.T)
    N = len(b); m = c + L; n = N - m
    Al = A.astype(LD); bl = b.astype(LD)
    lm = np.arange(c, m)
    assert np.count_nonzero(A[np.ix_(lm, lm)] - np.diag(np.diag(A)[lm])) == 0, "the landmark block must be diagonal"
    dead = [l for l in lm if not np.any(A[l, :m] != 0)]
    live = np.array([l for l in lm if l not in set(dead)], dtype=int)
    D = np.diag(Al)[live]
    kept = np.arange(m, N)
    structured = bool(np.all(D > eps))
    if structured:
        cols = np.concatenate([np.arange(c), kept])
        Acl = Al[np.ix_(cols, live)]
        Qs = Al[np.ix_(cols, cols)] - (Acl / D) @ Acl.T
        qb = bl[cols] - (Acl / D) @ bl[live]
        Ceps = Al[:c, :c] - (Acl[:c] / (D - LD(eps))) @ Acl[:c].T - LD(eps) * np.eye(c, dtype=LD)
        structured = _mp_min_eig(Ceps) > 0
    if structured:
        X = _mp_solve(Qs[:c, :c], np.concatenate([Qs[:c, c:], qb[:c, None]], axis=1))
        Ar = Qs[c:, c:] - Qs[c:, :c] @ X[:, :n]
        br = qb[c:] - Qs[c:, :c] @ X[:, n]
    else:
        w, Vm = refine_eigh(Al[:m, :m])
        keep = w > eps
        Ainv = (Vm[:, keep] / w[keep]) @ Vm[:, keep].T
        T = Al[m:, :m] @ Ainv
        Ar = Al[m:, m:] - T @ Al[:m, m:]
        br = bl[m:] - T @ bl[:m]
    Ar = np.tril(Ar) + np.tril(Ar, -1).T
    w2, V2 = refine_eigh(Ar)
    out = _outputs(Ar, br, w2, V2, eps)
    out["path"] = "fast" if structured and not dead else "generic"
    out.update(scales(A, b, m, out), N=N)
    return out


def scales(A, b, m, out):
    """First-order error scales of the marginalisation in double.  schur_scale: of the reduced matrix (Arr, the product
    Arm Amm^+ Amr and its sensitivity to Amm); b_scale: of the reduced vector, plus the turn of the kept eigenspace by
    schur_scale / gap when eigenvalues are dropped; rtr_scale: of b^T A^+ b = |x|^2 terms, same gap term."""
    Amm = 0.5 * (A[:m, :m] + A[:m, :m].T)
    wm = np.linalg.eigvalsh(Amm)
    inv = 1.0 / wm[wm > EPS_MARG].min() if np.any(wm > EPS_MARG) else 0.0
    nArm = np.linalg.norm(A[m:, :m], 2)
    schur = np.linalg.norm(A[m:, m:], 2) + nArm ** 2 * inv + np.linalg.norm(Amm, 2) * (nArm * inv) ** 2
    bsc = np.linalg.norm(b[m:]) + nArm * inv * np.linalg.norm(b[:m]) * (1 + np.linalg.norm(Amm, 2) * inv)
    w = out["w"].astype(np.float64)
    kept, dropped = w[w > EPS_MARG], w[w <= EPS_MARG]
    turn = 0.0
    if len(kept) and len(dropped):
        turn = schur / (kept.min() - dropped.max())
    br = np.linalg.norm(out["br"].astype(np.float64))
    x = np.linalg.norm(out["x"].astype(np.float64))
    return dict(schur_scale=schur, b_scale=bsc + turn * br, rtr_scale=schur * x * x + 2 * bsc * x + turn * br * x)


def marginalize_f64(A, b, m, eig):
    """The literal algorithm in double with a given eigensolver eig(A) -> (w, V): J0, r0 as the reference forms them."""
    A = np.asarray(A, np.float64); b = np.asarray(b, np.float64)
    Amm = 0.5 * (A[:m, :m] + A[:m, :m].T)
    w, V = eig(Amm)
    Ainv = (V * np.where(w > EPS_MARG, 1 / np.where(w > EPS_MARG, w, 1), 0)) @ V.T
    T = A[m:, :m] @ Ainv
    Ar = A[m:, m:] - T @ A[:m, m:]
    br = b[m:] - T @ b[:m]
    Ar = np.tril(Ar) + np.tril(Ar, -1).T
    w2, V2 = eig(Ar)
    S = np.where(w2 > EPS_MARG, w2, 0); Si = np.where(w2 > EPS_MARG, 1 / np.where(w2 > EPS_MARG, w2, 1), 0)
    return np.sqrt(S)[:, None] * V2.T, np.sqrt(Si) * (V2.T @ br)


def marg_ratios(J0, r0, ref):
    """The three marginalisation bars' ratios of a computed (J0, r0) against a reference, and J0's nonzero row count."""
    unit = ref["N"] * EPS
    JtJ, Jtr, rtr = J0.T @ J0, J0.T @ r0, r0 @ r0
    return dict(jtj=float(np.abs(JtJ - ref["JtJ"].astype(np.float64)).max()) / (unit * ref["schur_scale"]),
                jtr=float(np.abs(Jtr - ref["Jtr"].astype(np.float64)).max()) / (unit * ref["b_scale"]),
                rtr=abs(float(rtr) - float(ref["rtr"])) / (unit * ref["rtr_scale"]),
                rank=int(np.count_nonzero(np.any(J0 != 0, axis=1))))


# ------------------------------------------------------------------------------------------------ test systems
def marg_case(c, L, n, seed, null=0, scale=1.0, dead=(), tiny=(), c_eig=None):
    """A symmetric system [c dense | L landmarks | n kept] whose Schur complement has a prescribed spectrum: `null`
    eigenvalues 0 (after rounding |lam| ~ 1e-13, far below 1e-8) and the rest in [1e-5, 1e2] * scale, so that with ||A|| <= 1e3
    the truncation decision is clear on both sides.  Amm = [[C, B], [B^T, D]] with D diagonal (landmarks couple to the c
    block and to the kept columns, never to each other).
      dead: landmarks without information (zero rows and columns: D_ll = 0)
      tiny: landmarks with D_ll = 5e-9 and couplings of 1e-6
      c_eig: an eigenvalue c_eig in (0, 1e-8) of Amm along a direction of the c block the landmarks do not see (Amm is
             positive definite, Amm - 1e-8 I is not)."""
    rng = np.random.default_rng(seed)
    m = c + L; N = m + n
    G = rng.standard_normal((c, c + 3))
    C = (G @ G.T / (c + 3) + 0.5 * np.eye(c)) * scale
    B = rng.standard_normal((c, L)) * 0.1 * np.sqrt(scale / max(L, 1))      # ||B D^-1 B^T|| < 0.5 scale: Amm stays positive definite
    D = rng.uniform(1.0, 4.0, L) * scale
    if c_eig is not None:
        u = rng.standard_normal(c); u /= np.linalg.norm(u)
        P = np.eye(c) - np.outer(u, u)
        C = P @ C @ P + c_eig * np.outer(u, u)
        B = P @ B
    Amr = rng.standard_normal((m, n)) * 0.3 * np.sqrt(scale)
    for l in tiny:
        B[:, l] *= 1e-6 / np.abs(B[:, l]).max(); D[l] = 5e-9
        Amr[c + l] *= 1e-6 / np.abs(Amr[c + l]).max()
    Amm = np.zeros((m, m)); Amm[:c, :c] = 0.5 * (C + C.T); Amm[:c, c:] = B; Amm[c:, :c] = B.T; Amm[c:, c:] = np.diag(D)
    for l in dead:
        Amm[c + l, :] = 0; Amm[:, c + l] = 0; Amr[c + l] = 0
    mu = np.concatenate([np.zeros(null), np.logspace(-5, 2, n - null) * rng.uniform(0.5, 1.0, n - null)]) * scale
    _, Q, _ = known_spectrum(mu, seed + 1, exact="ld")
    # Arr = Sred + Arm Amm^+ Amr in double: the reduced system of the rounded input then has the spectrum mu to ~1e-13
    w, Vm = np.linalg.eigh(Amm)
    keep = w > EPS_MARG
    Arr = ((Q * mu.astype(LD)) @ Q.T).astype(np.float64) + Amr.T @ ((Vm[:, keep] / w[keep]) @ Vm[:, keep].T) @ Amr
    A = np.zeros((N, N))
    A[:m, :m] = Amm; A[:m, m:] = Amr; A[m:, :m] = Amr.T; A[m:, m:] = np.tril(Arr) + np.tril(Arr, -1).T
    b = rng.standard_normal(N) * np.sqrt(scale)
    for l in dead:
        b[c + l] = 0.0
    return A, b


# ------------------------------------------------------------------------------------------------ the cases of the tests
QL_SIZES = (1, 2, 3, 7, 8, 31, 32, 33, 64, 76, 91, 127, 128)
JACOBI_SIZES = (1, 2, 3, 33, 128, 129, 157, 198, 315, 520)        # 520: about Amm of a C4 window


def marg_cases():
    """(id, c, L, n, marg_case keywords, expected reference path).  The size grid takes the structured fast path (null = n // 3
    reduced eigenvalues below 1e-8); the rest fails the positive-definiteness test in each way it can."""
    out = []
    for c in (6, 15):
        for L in (0, 1, 40, 300):
            for n in (1, 6, 76, 127, 128, 129, 198):
                out.append(("c%d_L%d_n%d" % (c, L, n), c, L, n, dict(seed=1000 * c + 10 * L + n, null=n // 3), "fast"))
    out += [("dead_L40", 15, 40, 76, dict(seed=5, null=10, dead=(3, 17)), "generic"),
            ("dead_L300", 15, 300, 76, dict(seed=6, null=10, dead=tuple(range(0, 300, 7))), "generic"),
            ("tiny_L40", 15, 40, 76, dict(seed=7, null=10, tiny=(5,)), "generic"),
            ("c_eig_c6", 6, 40, 76, dict(seed=8, null=10, c_eig=3e-9), "generic"),
            ("c_eig_c15_n129", 15, 40, 129, dict(seed=9, null=10, c_eig=3e-9), "generic"),
            # small n with a weak landmark past the first (c + n)^2 threads of k_marg_lm_elim
            ("tiny_hi_c6_n1", 6, 300, 1, dict(seed=11, null=0, tiny=(299,)), "generic"),
            ("tiny_hi_c15_n1", 15, 300, 1, dict(seed=12, null=0, tiny=(280,)), "generic"),
            ("tiny_hi_c6_n6", 6, 300, 6, dict(seed=13, null=2, tiny=(250,)), "generic"),
            ("dead_hi_c6_n6", 6, 300, 6, dict(seed=14, null=2, dead=(290,)), "generic"),
            # Amm at the stage's Jacobi bound
            ("bound_m2304", 6, JACOBI_BOUND - 6, 6, dict(seed=15, null=2, dead=(JACOBI_BOUND - 20,)), "generic")]
    return out
