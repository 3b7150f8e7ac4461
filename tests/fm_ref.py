"""High-precision references of the FeatureManager kernels (csrc/fm_kernels.cu), their error bars and their test cases, CPU
only.

Each operation is restated on the exact double inputs:
  * triangulate (DLT, feature_manager.cpp:668-723): A (2m x 4) is formed in mpmath from the exact poses and observations and
    its smallest right singular vector taken with mp.svd_r at DPS digits; the depth is v2 / v3;
  * triangulateWithDepth (:726-799): every pair's residual norm and verified depth in np.longdouble, then their mean;
  * the keyframe parallax sum, the back-shift depth transfer, the reprojection-error sums and the constant-velocity
    prediction in np.longdouble (the prediction's nextT in mpmath, in the oracle's 4x4-transform form).
Each reference returns the value and an error scale; a kernel result passes when ratio = |got - ref| / (EPS scale) <= K.
K is CALIBRATION_FACTOR times the worst ratio a plain-double CPU implementation reaches over the cases below, rounded up
(tests/test_fm_ref.py: LAPACK's SVD and a NumPy port of the kernel's Givens-QR + one-sided Jacobi for the DLT, plain double
restatements for the rest).

The DLT scale is the first-order sensitivity of v2 / v3 to a backward perturbation of A of size eps s_A,
  s_A / (sigma_3 - sigma_4) * sqrt(1 + d^2) / |v3|,   s_A = ||A||_2 + max_k |P_k + R_k tic|,
whose second term covers the rounding of t1 - t0 at large world coordinates, which no backward-stable SVD removes.
"""
import functools

import mpmath as mp
import numpy as np

from marg_ref import EPS, LD, mp_to_ld

CALIBRATION_FACTOR = 8
DPS = 50
N_FRAMES = 11                       # GF_BA_MAX_FRAMES: every list ends in the window's last frame
INIT_DEPTH = 5.0                    # parameters.cpp:478
BAR = 10.0 / 460                    # triangulateWithDepth's re-projection test
# bar -> K (CALIBRATION_FACTOR x the worst plain-double CPU ratio over the cases of this module, rounded up)
K = {
    "dlt": 30.0,              # |d - ref| / (eps dlt scale)          worst CPU 3.74 (LAPACK, depth_b1e-01_o0e+00); Givens-QR + Jacobi port 0.488
    "depth_mean": 13.0,       # |mean - ref| / (eps mean_k (|point0_k| + |t0_k| + |tr| + |z_k|))      worst CPU 1.58 (depth_b1e-01_o0e+00)
    "parallax": 1.0,          # |sum - ref| / (eps (log2(n) sum |terms| + sum_i (|u_i| + |v_i| + |u_j| + |v_j|)))   worst CPU 0.122 (n = 3000)
    "back_shift": 4.5,        # |z - ref| / (eps (sum_k |new_R_k2| (|marg_R_k| |uv d| + |marg_P_k| + |new_P_k|) + |z|))   worst CPU 0.557 (offset 0)
    "reproj2d": 2.3,          # |e2 - ref| / (eps sum_j 2-D term scale, reproj_ref)     worst CPU 0.28 (offset 0, extrinsic, near the camera plane)
    "reproj3d": 6.1,          # |e3 - ref| / (eps sum_j 3-D term scale, reproj_ref)     worst CPU 0.755 (offset 0, extrinsic)
    "predict": 6.3,           # max_k |c_k - ref_k| / (eps carried-point scale)        worst CPU 0.782 (offset 0, extrinsic)
}


# ---- geometry ------------------------------------------------------------------------------------------------------------
def rot(axis, ang):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    K_ = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K_ + (1 - np.cos(ang)) * (K_ @ K_)


RIC = rot([0.3, -1.0, 0.2], 0.4)
TIC = np.array([0.07, -0.031, 0.113])


class Scene:
    """One call's inputs: the window's poses, the extrinsic and a list of landmarks {start, pts (m x 3), dep (m,), est, flag}."""

    def __init__(self, name, Ps, Rs, tic, ric, depth_threshold, lms):
        self.name, self.Ps, self.Rs, self.tic, self.ric, self.depth_threshold, self.lms = name, Ps, Rs, tic, ric, depth_threshold, lms
        self.P_cam = max(float(np.abs(Ps[f] + Rs[f] @ tic).max()) for f in range(len(Ps)))

    def arrays(self, idx=None):
        lms = self.lms if idx is None else [self.lms[i] for i in idx]
        nobs = np.array([len(l["dep"]) for l in lms], np.int32)
        off = np.zeros(len(lms), np.int32); off[1:] = np.cumsum(nobs)[:-1]
        pts = np.ascontiguousarray(np.concatenate([l["pts"] for l in lms]).reshape(-1, 3), np.float64)
        dep = np.ascontiguousarray(np.concatenate([l["dep"] for l in lms]), np.float64)
        start = np.array([l["start"] for l in lms], np.int32)
        est = np.array([l["est"] for l in lms], np.float64)
        flag = np.array([l["flag"] for l in lms], np.int32)
        return start, nobs, off, pts, dep, est, flag


def window_poses(baseline, offset, seed, stationary=False):
    """11 poses moving `baseline` per frame along a fixed direction (or not at all), turning slowly, `offset` metres from the
    origin.  stationary: every pose bit-identical."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=3)
    d /= np.linalg.norm(d)
    P0 = offset * np.array([0.6, -0.48, 0.64]) + rng.uniform(-1, 1, 3)
    R0 = rot(rng.normal(size=3), rng.uniform(0, np.pi))
    w = rng.normal(size=3)
    Ps, Rs = [], []
    for k in range(N_FRAMES):
        kk = 0 if stationary else k
        Ps.append(P0 + baseline * kk * d)
        Rs.append(R0 @ rot(w, 0.01 * kk * min(1.0, baseline / 0.1)))
    return np.array(Ps), np.array(Rs)


def cam_pose(Ps, Rs, tic, ric, f):
    return Ps[f] + Rs[f] @ tic, Rs[f] @ ric


def observe(Ps, Rs, tic, ric, X, start, m, noise, rng):
    """Normalised observations (x, y, 1) and true depths of world point X in frames start .. start + m - 1."""
    pts, z = [], []
    for f in range(start, start + m):
        t, R = cam_pose(Ps, Rs, tic, ric, f)
        pc = R.T @ (X - t)
        pts.append([pc[0] / pc[2] + rng.normal(0, noise) if noise else pc[0] / pc[2],
                    pc[1] / pc[2] + rng.normal(0, noise) if noise else pc[1] / pc[2], 1.0])
        z.append(pc[2])
    return np.array(pts), np.array(z)


def landmark(Ps, Rs, tic, ric, depth, m, noise, rng, dep=None, est=-1.0, flag=0):
    """A landmark at `depth` in its start frame (start = N_FRAMES - m), seen in every later frame.  dep: the RGB-D depths
    (None: 0, i.e. no depth measurement)."""
    start = N_FRAMES - m
    t, R = cam_pose(Ps, Rs, tic, ric, start)
    ray = np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.3, 0.3), 1.0])
    X = t + R @ (ray * depth)
    pts, z = observe(Ps, Rs, tic, ric, X, start, m, noise, rng)
    return dict(start=start, pts=pts, dep=np.zeros(m) if dep is None else np.asarray(dep(z), float), est=est, flag=flag, z=z, noise=noise)


BASELINES = (0.1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6)
OFFSETS = (0.0, 1e3, 1e4)
DEPTHS = (0.15, 0.5, 2.0, 5.0, 30.0, 100.0)
NOISES = (0.0, 1e-6, 1e-3)


def _untouched(Ps, Rs, tic, ric, rng, out):
    """Landmarks both loops skip: fewer than 4 observations, or a depth already (estimate flags arbitrary on purpose)."""
    for m, est, flag in ((1, -1.0, 7), (2, -1.0, 0), (3, -2.5, 3), (6, 3.7, 1), (11, 1e-300, 2), (4, np.inf, -9)):
        out.append(landmark(Ps, Rs, tic, ric, 4.0, m, 0.0, rng, dep=lambda z: z, est=est, flag=flag))


@functools.lru_cache(None)
def dlt_scenes():
    """Geometry grid of the DLT path: baseline x world offset x extrinsic; in each, depths 0.15 .. 100 m, list lengths 4 .. 11,
    pixel noise 0 / 1e-6 / 1e-3, two landmarks behind the camera and the skipped kinds.  No RGB-D depth is valid
    (depth_threshold 0.05), so every landmark with >= 4 observations goes to the DLT."""
    out = {}
    for bi, b in enumerate(BASELINES):
        for oi, o in enumerate(OFFSETS):
            for ext in (False, True):
                seed = 100 * bi + 10 * oi + ext
                rng = np.random.default_rng(seed)
                tic, ric = (TIC, RIC) if ext else (np.zeros(3), np.eye(3))
                Ps, Rs = window_poses(b, o, seed)
                lms = []
                for k, depth in enumerate(DEPTHS):
                    for j in range(2):
                        m = 4 + (2 * k + j + bi) % 8
                        lms.append(landmark(Ps, Rs, tic, ric, depth, m, NOISES[(k + j + oi) % 3], rng))
                for depth in (-5.0, -0.5):                                       # behind the camera: negative DLT depth
                    lms.append(landmark(Ps, Rs, tic, ric, depth, 11 - bi, 0.0, rng))
                lms.append(landmark(Ps, Rs, tic, ric, 0.06, 7, 0.0, rng))        # d < 0.1
                _untouched(Ps, Rs, tic, ric, rng, lms)
                name = "b%.0e_o%.0e%s" % (b, o, "_ric" if ext else "")
                out[name] = Scene(name, Ps, Rs, tic, ric, 0.05, lms)
    return out


@functools.lru_cache(None)
def depth_scenes():
    """triangulateWithDepth: RGB-D depths valid in some frames (exact, noisy or wrong by a factor, so that some pairs are
    rejected), at the exact bounds 0.1 and depth_threshold and one ulp outside them, and a window moving backwards whose
    verified depths transfer below 0.1 into the start frame."""
    out = {}
    for b, o, ext, seed in ((0.1, 0.0, False, 1), (0.1, 1e4, True, 2), (1e-2, 1e3, True, 3), (1e-4, 0.0, True, 4), (0.05, 1e3, False, 5)):
        rng = np.random.default_rng(seed)
        tic, ric = (TIC, RIC) if ext else (np.zeros(3), np.eye(3))
        Ps, Rs = window_poses(b, o, seed)
        thr = 3.0
        lms = []
        for k in range(40):
            depth = rng.uniform(0.3, 6.0)
            m = 4 + k % 8
            kind = k % 4
            if kind == 0:
                dep = lambda z: z                                                # exact depths
            elif kind == 1:
                dep = lambda z: z * (1 + rng.normal(0, 0.01, len(z)))            # noisy
            elif kind == 2:
                dep = lambda z: z * np.where(rng.uniform(size=len(z)) < 0.5, rng.uniform(0.3, 2.0, len(z)), 1.0)   # some wrong
            else:
                dep = lambda z: np.where(rng.uniform(size=len(z)) < 0.7, 0.0, z)  # mostly missing
            lms.append(landmark(Ps, Rs, tic, ric, depth, m, NOISES[k % 3] if b > 1e-3 else 0.0, rng, dep=dep))
        # the depth bounds: one observation carries the only usable depth, at or just outside 0.1 / depth_threshold
        for v in (0.1, thr, np.nextafter(0.1, 0.0), np.nextafter(thr, np.inf)):
            for m in (4, 9):
                def dep(z, v=v):
                    d = np.zeros(len(z)); d[0] = v
                    return d
                lm = landmark(Ps, Rs, tic, ric, v, m, 0.0, rng, dep=dep)
                lms.append(lm)
        _untouched(Ps, Rs, tic, ric, rng, lms)
        name = "depth_b%.0e_o%.0e%s" % (b, o, "_ric" if ext else "")
        out[name] = Scene(name, Ps, Rs, tic, ric, thr, lms)
    # moving backwards along the optical axis: a landmark 0.06 m in front of the start frame is seen at 0.1 .. 0.3 m later on
    rng = np.random.default_rng(9)
    Ps = np.array([[0, 0, -0.02 * k] for k in range(N_FRAMES)], float) + 3.0
    Rs = np.array([np.eye(3)] * N_FRAMES)
    lms = []
    for k in range(12):
        m = 4 + k % 8
        lms.append(landmark(Ps, Rs, np.zeros(3), np.eye(3), rng.uniform(0.04, 0.08), m, 0.0, rng, dep=lambda z: z))
        lms.append(landmark(Ps, Rs, np.zeros(3), np.eye(3), rng.uniform(0.3, 1.0), m, 0.0, rng, dep=lambda z: z))
    out["depth_backwards"] = Scene("depth_backwards", Ps, Rs, np.zeros(3), np.eye(3), 3.0, lms)
    for sc in out.values():
        _pin_decisions(sc)
    return out


@functools.lru_cache(None)
def stationary_scenes():
    """Bit-identical poses across the window: A has a two-dimensional null space and the depth is not determined."""
    out = {}
    for o, ext, seed in ((0.0, False, 11), (1e3, True, 12), (1e4, True, 13)):
        rng = np.random.default_rng(seed)
        tic, ric = (TIC, RIC) if ext else (np.zeros(3), np.eye(3))
        Ps, Rs = window_poses(0.1, o, seed, stationary=True)
        lms = [landmark(Ps, Rs, tic, ric, d, m, nz, rng) for d in (0.5, 5.0, 50.0) for m in (4, 8, 11) for nz in (0.0, 1e-6)]
        name = "stationary_o%.0e%s" % (o, "_ric" if ext else "")
        out[name] = Scene(name, Ps, Rs, tic, ric, 0.05, lms)
    return out


COUNTS = (1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 3000)


@functools.lru_cache(None)
def count_scene():
    """A pool of 260 distinct landmarks (DLT, RGB-D and skipped ones mixed) for the calls whose landmark count straddles the
    64-thread blocks; the first n of the pool, repeated for n > 260."""
    rng = np.random.default_rng(77)
    tic, ric = TIC, RIC
    Ps, Rs = window_poses(0.03, 1e3, 77)
    lms = []
    while len(lms) < 260:
        k = len(lms)
        kind = k % 5
        if kind == 4:
            lms.append(landmark(Ps, Rs, tic, ric, 4.0, 1 + k % 3, 0.0, rng, est=(-1.0 if k % 2 else 2.5), flag=k % 3))
        else:
            dep = (lambda z: z) if kind == 1 else (lambda z: z * 1.7) if kind == 2 else None
            lms.append(landmark(Ps, Rs, tic, ric, rng.uniform(0.5, 40.0), 4 + k % 8, NOISES[k % 3], rng, dep=dep))
    sc = Scene("count", Ps, Rs, tic, ric, 3.0, lms)
    _pin_decisions(sc)
    return sc


def count_index(n):
    return np.arange(n) % len(count_scene().lms)


def _pin_decisions(sc):
    """Keeps every re-projection decision of triangulateWithDepth at least 1e-9 relative (and the double-evaluation error)
    away from 10/460, by dropping the RGB-D depth of an observation whose pairs come closer."""
    for lm in sc.lms:
        for _ in range(lm["pts"].shape[0]):
            pairs = depth_pairs(sc, lm)
            close = [p for p in pairs if not p["pinned"]]
            if not close:
                break
            lm["dep"] = lm["dep"].copy(); lm["dep"][close[0]["i"]] = 0.0


# ---- triangulateWithDepth ------------------------------------------------------------------------------------------------
def _cam_ld(sc, f):
    Ps, Rs, tic, ric = (np.asarray(x, LD) for x in (sc.Ps, sc.Rs, sc.tic, sc.ric))
    return Ps[f] + Rs[f] @ tic, Rs[f] @ ric


def depth_pairs(sc, lm):
    """Every pair (i, j) of triangulateWithDepth in longdouble: residual norm, verified depth, and whether the accept decision
    is pinned (the exact residual lies outside both 1e-9 relative and the double-evaluation error of 10/460)."""
    s0, m = lm["start"], len(lm["dep"])
    if m < 4 or lm["est"] > 0:
        return []
    tr, Rr = _cam_ld(sc, s0)
    out = []
    for i in range(m):
        di = lm["dep"][i]
        if di < 0.1 or di > sc.depth_threshold:
            continue
        t0, R0 = _cam_ld(sc, s0 + i)
        point0 = np.asarray(lm["pts"][i], LD) * LD(di)
        t2r, R2r = Rr.T @ (t0 - tr), Rr.T @ R0
        z = (R2r @ point0 + t2r)[2]
        for j in range(m):
            if i == j:
                continue
            t1, R1 = _cam_ld(sc, s0 + j)
            t20, R20 = R0.T @ (t1 - t0), R0.T @ R1
            pp = R20.T @ point0 - R20.T @ t20
            u = np.asarray(lm["pts"][j][:2], LD) - pp[:2] / pp[2]
            res = np.sqrt((u * u).sum())
            mag = float(np.linalg.norm(np.asarray(point0, float)) + np.linalg.norm(np.asarray(t20, float)) + 2 * sc.P_cam)
            err = 64 * EPS * mag / abs(float(pp[2])) * (1 + float(np.abs(pp[:2] / pp[2]).sum()))
            gap = abs(float(res) - BAR)
            out.append(dict(i=i, j=j, res=res, z=z, accept=bool(res < BAR), pinned=gap > max(1e-9 * BAR, err),
                            scale=float(np.linalg.norm(np.asarray(point0, float)) + np.linalg.norm(np.asarray(t0, float))
                                        + np.linalg.norm(np.asarray(tr, float)) + abs(float(z)))))
    return out


# ---- triangulate (DLT) ---------------------------------------------------------------------------------------------------
def _mp_mat(a):
    return mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.asarray(a, float)])


def _mp_vec(a):
    return mp.matrix([mp.mpf(float(x)) for x in np.asarray(a, float)])


def dlt_matrix_mp(sc, lm):
    """A of feature_manager.cpp:680-705 from the exact double inputs, in mpmath."""
    s0, m = lm["start"], len(lm["dep"])
    tic, ric = _mp_vec(sc.tic), _mp_mat(sc.ric)

    def cam(f):
        R = _mp_mat(sc.Rs[f])
        return _mp_vec(sc.Ps[f]) + R * tic, R * ric
    t0, R0 = cam(s0)
    A = mp.matrix(2 * m, 4)
    for k in range(m):
        t1, R1 = cam(s0 + k)
        t = R0.T * (t1 - t0); R = R0.T * R1
        P = mp.matrix(3, 4)
        nt = -(R.T * t)
        for r in range(3):
            for c in range(3):
                P[r, c] = R[c, r]
            P[r, 3] = nt[r]
        p = [mp.mpf(float(x)) for x in lm["pts"][k]]
        nrm = mp.sqrt(p[0] ** 2 + p[1] ** 2 + p[2] ** 2)
        f = [x / nrm for x in p]
        for c in range(4):
            A[2 * k, c] = f[0] * P[2, c] - f[2] * P[0, c]
            A[2 * k + 1, c] = f[1] * P[2, c] - f[2] * P[1, c]
    return A


def dlt_ref(sc, lm):
    """(depth v2 / v3, scale, sigma) of the DLT at DPS digits; scale inf when the null space is not one-dimensional."""
    with mp.workdps(DPS):
        A = dlt_matrix_mp(sc, lm)
        _, S, V = mp.svd_r(A, compute_uv=True)
        order = sorted(range(4), key=lambda k: S[k], reverse=True)
        s = [S[k] for k in order]
        v = [V[order[3], c] for c in range(4)]
        d = v[2] / v[3] if v[3] != 0 else mp.inf
        gap = s[2] - s[3]
        s_A = float(s[0]) + sc.P_cam
        scale = float(s_A / gap * mp.sqrt(1 + d * d) / abs(v[3])) if gap > 0 and v[3] != 0 else np.inf
        return float(d), scale, [float(x) for x in s]


def dlt_matrix_f64(sc, lm):
    """A in double, in the kernel's order of operations (t = Ps + Rs tic, R = Rs ric, P = [R^T | -R^T t], f = p / |p|)."""
    s0, m = lm["start"], len(lm["dep"])

    def cam(f):
        return sc.Ps[f] + sc.Rs[f] @ sc.tic, sc.Rs[f] @ sc.ric
    t0, R0 = cam(s0)
    A = np.zeros((2 * m, 4))
    for k in range(m):
        t1, R1 = cam(s0 + k)
        t = R0.T @ (t1 - t0); R = R0.T @ R1
        P = np.zeros((3, 4)); P[:, :3] = R.T; P[:, 3] = -(R.T @ t)
        p = lm["pts"][k]
        f = p / np.sqrt(p @ p)
        A[2 * k] = f[0] * P[2] - f[2] * P[0]
        A[2 * k + 1] = f[1] * P[2] - f[2] * P[1]
    return A


def dlt_lapack(A):
    v = np.linalg.svd(A, full_matrices=False)[2][-1]
    return v[2] / v[3]


def qr_add_row4(R, r):
    """Givens rotations folding row r into the upper-triangular R (k_fm_triangulate's qr_add_row4)."""
    r = list(r)
    for k in range(4):
        if r[k] == 0.0:
            continue
        h = float(np.hypot(R[k][k], r[k])); c = R[k][k] / h; s = r[k] / h
        R[k][k] = h
        for j in range(k + 1, 4):
            a, b = R[k][j], r[j]
            R[k][j] = c * a + s * b; r[j] = c * b - s * a


def smallest_right_sv4(R, max_sweeps=20):
    """One-sided Jacobi on R's columns (k_fm_triangulate's smallest_right_sv4); returns (v, sweeps)."""
    V = [[float(i == j) for j in range(4)] for i in range(4)]
    sweeps = 0
    for sweeps in range(1, max_sweeps + 1):
        rotated = False
        for p in range(3):
            for q in range(p + 1, 4):
                a = sum(R[k][p] * R[k][p] for k in range(4)); b = sum(R[k][q] * R[k][q] for k in range(4))
                g = sum(R[k][p] * R[k][q] for k in range(4))
                if abs(g) <= EPS * np.sqrt(a) * np.sqrt(b):
                    continue
                zeta = (b - a) / (2.0 * g)
                t = (1.0 if zeta >= 0 else -1.0) / (abs(zeta) + float(np.hypot(1.0, zeta)))
                c = 1.0 / np.sqrt(t * t + 1.0); s = t * c
                for M in (R, V):
                    for k in range(4):
                        x, y = M[k][p], M[k][q]
                        M[k][p] = c * x - s * y; M[k][q] = s * x + c * y
                rotated = True
        if not rotated:
            break
    n2 = [sum(R[k][j] * R[k][j] for k in range(4)) for j in range(4)]
    mi = 0
    for j in range(1, 4):
        if n2[j] < n2[mi]:
            mi = j
    return [V[k][mi] for k in range(4)], sweeps


def dlt_kernel_port(A):
    """(depth, sweeps) of the kernel's DLT on A: Givens QR streamed row by row, then one-sided Jacobi."""
    R = [[0.0] * 4 for _ in range(4)]
    for row in np.asarray(A, float):
        qr_add_row4(R, [float(x) for x in row])
    v, sweeps = smallest_right_sv4(R)
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(v[2]) / np.float64(v[3])), sweeps


# ---- triangulate the whole list ------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def triangulate_ref(sc):
    return [triangulate_ref_one(sc, lm) for lm in sc.lms]


def triangulate_ref_one(sc, lm):
    """What gf_fm_triangulate must produce for one landmark:
    kind 'skip': depth and flag unchanged; 'depth': flag 1 mean (or INIT_DEPTH / 0 below 0.1); 'dlt': v2 / v3 (flag 2 from 0.1)."""
    m = len(lm["dep"])
    if m < 4 or lm["est"] > 0:
        return dict(kind="skip")
    pairs = depth_pairs(sc, lm)
    acc = [p for p in pairs if p["accept"]]
    if acc:
        zs = np.array([p["z"] for p in acc], LD)
        d = zs.sum() / len(zs)
        return dict(kind="depth", d=float(d), scale=float(sum(p["scale"] for p in acc) / len(acc)), cnt=len(acc),
                    pinned=all(p["pinned"] for p in pairs), flag=1 if d >= 0.1 else 0)
    d, scale, sig = dlt_ref(sc, lm)
    return dict(kind="dlt", d=d, scale=scale, sigma=sig, flag=2 if d >= 0.1 else 0)


def flag_pinned(ref, k):
    """The 0.1 decision is pinned when the exact depth is more than the bar away from 0.1."""
    return abs(ref["d"] - 0.1) > k * EPS * ref["scale"]


def ratio(got, ref, scale):
    err = abs(float(got) - float(ref))
    if scale == 0:
        return 0.0 if err == 0 else np.inf
    return err / (EPS * scale)


def depth_mean_f64(sc, lm):
    """triangulateWithDepth's mean for one landmark in plain double (the calibration's stand-in); None if nothing verifies."""
    s0, m = lm["start"], len(lm["dep"])
    tr, Rr = cam_pose(sc.Ps, sc.Rs, sc.tic, sc.ric, s0)
    zs = []
    for i in range(m):
        if lm["dep"][i] < 0.1 or lm["dep"][i] > sc.depth_threshold:
            continue
        t0, R0 = cam_pose(sc.Ps, sc.Rs, sc.tic, sc.ric, s0 + i)
        point0 = lm["pts"][i] * lm["dep"][i]
        t2r, R2r = Rr.T @ (t0 - tr), Rr.T @ R0
        for j in range(m):
            if i == j:
                continue
            t1, R1 = cam_pose(sc.Ps, sc.Rs, sc.tic, sc.ric, s0 + j)
            t20, R20 = R0.T @ (t1 - t0), R0.T @ R1
            pp = R20.T @ point0 - R20.T @ t20
            if np.linalg.norm(lm["pts"][j][:2] - pp[:2] / pp[2]) < BAR:
                zs.append((R2r @ point0 + t2r)[2])
    return sum(zs) / len(zs) if zs else None


# ---- parallax ------------------------------------------------------------------------------------------------------------
def parallax_case(n, seed, near_plane=False):
    """pts_i (x, y, z) with z away from 1 (the kernel divides by it) and pts_j (x, y, 1); near_plane: some z of 1e-3 .. 1e-2."""
    rng = np.random.default_rng(seed)
    pi = np.stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.5, 3.0, n)], 1)
    if near_plane:
        pi[::3, 2] = rng.uniform(1e-3, 1e-2, len(pi[::3]))
    pj = np.stack([pi[:, 0] / pi[:, 2] + rng.normal(0, 0.02, n), pi[:, 1] / pi[:, 2] + rng.normal(0, 0.02, n), np.ones(n)], 1)
    return np.ascontiguousarray(pi), np.ascontiguousarray(pj)


def parallax_ref(pi, pj):
    a, b = np.asarray(pi, LD), np.asarray(pj, LD)
    u, v = a[:, 0] / a[:, 2], a[:, 1] / a[:, 2]
    terms = np.sqrt((u - b[:, 0]) ** 2 + (v - b[:, 1]) ** 2)
    n = len(terms)
    scale = float(max(np.log2(n), 1.0) * np.abs(terms).sum() + (np.abs(u) + np.abs(v) + np.abs(b[:, 0]) + np.abs(b[:, 1])).sum())
    return float(terms.sum()), scale


def parallax_f64(pi, pj):
    s = 0.0
    for a, b in zip(pi, pj):
        du, dv = a[0] / a[2] - b[0], a[1] / a[2] - b[1]
        s += np.sqrt(du * du + dv * dv)
    return s


# ---- back shift ------------------------------------------------------------------------------------------------------------
def back_shift_case(n, offset, seed):
    """uv (x, y, 1), depths (some negative, some near the new camera plane) and the marginalised / new first poses."""
    rng = np.random.default_rng(seed)
    mR, nR = rot(rng.normal(size=3), 0.7), rot(rng.normal(size=3), 0.9)
    base = offset * np.array([0.6, -0.48, 0.64])
    mP = base + rng.uniform(-1, 1, 3); nP = mP + rng.normal(0, 0.3, 3)
    uv = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.4, 0.4, n), np.ones(n)], 1)
    d = rng.uniform(0.2, 30.0, n)
    d[::7] *= -1
    # some points close to the new camera's plane: z_j = 0 at a depth found in double, then nudged by a few 1e-12 m
    for i in range(3, n, 11):
        w_dir, w0 = mR @ uv[i], mP - nP
        lam = -(nR[:, 2] @ w0) / (nR[:, 2] @ w_dir)
        d[i] = lam * (1 + rng.choice([-1, 1]) * 1e-12 * rng.integers(0, 5))
    return np.ascontiguousarray(uv), d, mR, mP, nR, nP


def back_shift_ref(uv, d, mR, mP, nR, nP):
    a = [np.asarray(x, LD) for x in (uv, d, mR, mP, nR, nP)]
    uvl, dl, mRl, mPl, nRl, nPl = a
    pts = uvl * dl[:, None]
    w = pts @ mRl.T + mPl - nPl
    z = w @ nRl[:, 2]
    mag = np.abs(pts) @ np.abs(np.asarray(mR, float)).T + np.abs(mP) + np.abs(nP)
    scale = np.asarray(np.abs(np.asarray(mag, float)) @ np.abs(nR[:, 2]), float) + np.abs(np.asarray(z, float))
    return np.asarray(z, float), scale


def back_shift_f64(uv, d, mR, mP, nR, nP):
    return np.array([(nR.T @ (mR @ (u * di) + mP - nP))[2] for u, di in zip(uv, d)])


# ---- reprojection errors ---------------------------------------------------------------------------------------------------
def reproj_case(n, offset, ext, seed, near_plane=False):
    """Landmarks with 1 .. 11 observations ending anywhere in the window, depths right or wrong by a factor; near_plane: a
    window that turns so that later observations see the point almost in the camera plane."""
    rng = np.random.default_rng(seed)
    tic, ric = (TIC, RIC) if ext else (np.zeros(3), np.eye(3))
    Ps, Rs = window_poses(0.2, offset, seed)
    if near_plane:
        Rs = np.array([Rs[0] @ rot([0, 1, 0], 0.14 * k) for k in range(N_FRAMES)])
    lms = []
    for k in range(n):
        m = 1 + k % 11
        start = int(rng.integers(0, N_FRAMES - m + 1))
        t, R = cam_pose(Ps, Rs, tic, ric, start)
        ray = np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.3, 0.3), 1.0])
        depth = rng.uniform(0.3, 20.0)
        X = t + R @ (ray * depth)
        pts, _ = observe(Ps, Rs, tic, ric, X, start, m, 1e-3, rng)
        est = depth * (1.0 if k % 3 else rng.uniform(0.3, 2.0))
        lms.append(dict(start=start, pts=pts, dep=np.zeros(m), est=est, flag=2))
    return Scene("reproj", Ps, Rs, tic, ric, 3.0, lms)


def reproj_ref(sc):
    """Per landmark (e2, e3, count, scale2, scale3) in longdouble."""
    out = []
    Ps, Rs, tic, ric = (np.asarray(x, LD) for x in (sc.Ps, sc.Rs, sc.tic, sc.ric))
    for lm in sc.lms:
        fi, d = lm["start"], LD(lm["est"])
        uvi = np.asarray(lm["pts"][0], LD)
        pw = Rs[fi] @ (ric @ (d * uvi) + tic) + Ps[fi]
        s_pw = float(abs(lm["est"]) * np.linalg.norm(lm["pts"][0]) + np.linalg.norm(sc.tic) + np.linalg.norm(sc.Ps[fi]))
        e2 = e3 = LD(0); s2 = s3 = 0.0
        for j in range(1, len(lm["dep"])):
            fj = lm["start"] + j
            pc = ric.T @ (Rs[fj].T @ (pw - Ps[fj]) - tic)
            uvj = np.asarray(lm["pts"][j], LD)
            r = pc[:2] / pc[2] - uvj[:2]
            e2 += np.sqrt((r * r).sum())
            e3 += np.sqrt(((pc - uvj) ** 2).sum()) / d
            s_pc = s_pw + float(np.linalg.norm(sc.Ps[fj]) + np.linalg.norm(sc.tic) + np.linalg.norm(np.asarray(pw, float)))
            q = np.abs(np.asarray(pc[:2] / pc[2], float))
            s2 += s_pc * (2 + q.sum()) / abs(float(pc[2])) + float(q.sum() + np.abs(lm["pts"][j][:2]).sum() + np.sqrt(float((r * r).sum())))
            s3 += (s_pc + float(np.linalg.norm(np.asarray(pc, float)) + np.linalg.norm(lm["pts"][j]))) / abs(lm["est"])
        out.append((float(e2), float(e3), len(lm["dep"]) - 1, s2, s3))
    return out


def reproj_f64(sc):
    out = []
    for lm in sc.lms:
        fi, d = lm["start"], lm["est"]
        pw = sc.Rs[fi] @ (sc.ric @ (d * lm["pts"][0]) + sc.tic) + sc.Ps[fi]
        e2 = e3 = 0.0
        for j in range(1, len(lm["dep"])):
            fj = fi + j
            pc = sc.ric.T @ (sc.Rs[fj].T @ (pw - sc.Ps[fj]) - sc.tic)
            e2 += float(np.hypot(pc[0] / pc[2] - lm["pts"][j][0], pc[1] / pc[2] - lm["pts"][j][1]))
            e3 += float(np.linalg.norm(pc - lm["pts"][j])) / d
        out.append((e2, e3, len(lm["dep"]) - 1))
    return out


# ---- predict_next ------------------------------------------------------------------------------------------------------------
def _T_mp(R, P):
    T = mp.eye(4)
    for i in range(3):
        for j in range(3):
            T[i, j] = mp.mpf(float(R[i][j]))
        T[i, 3] = mp.mpf(float(P[i]))
    return T


def predict_ref(sc, first, uv, dep, frame_count):
    """Carried points inv(nextT Tbc) Tws_i Tbc (d uv, 1), nextT = cur (prev^-1 cur) with exact 4x4 inverses (the oracle's
    form): nextT and the inverse at DPS digits, the per-landmark products in longdouble; and their scale per landmark."""
    with mp.workdps(DPS):
        cur, prev = _T_mp(sc.Rs[frame_count], sc.Ps[frame_count]), _T_mp(sc.Rs[frame_count - 1], sc.Ps[frame_count - 1])
        nxt = cur * (mp.inverse(prev) * cur)
        M = mp.inverse(nxt * _T_mp(sc.ric, sc.tic))
        Minv = np.array([[mp_to_ld(M[i, j]) for j in range(4)] for i in range(4)], dtype=LD)
        nP = float(mp.sqrt(nxt[0, 3] ** 2 + nxt[1, 3] ** 2 + nxt[2, 3] ** 2))
    Tbc = np.eye(4, dtype=LD); Tbc[:3, :3] = np.asarray(sc.ric, LD); Tbc[:3, 3] = np.asarray(sc.tic, LD)
    out, scale = [], []
    motion = float(np.linalg.norm(sc.Ps[frame_count]) + np.linalg.norm(sc.Ps[frame_count - 1]))
    for f, u, d in zip(first, uv, dep):
        Tw = np.eye(4, dtype=LD); Tw[:3, :3] = np.asarray(sc.Rs[f], LD); Tw[:3, 3] = np.asarray(sc.Ps[f], LD)
        pw = Tw @ Tbc @ np.append(LD(d) * np.asarray(u, LD), LD(1))
        c = (Minv @ pw)[:3]
        out.append(np.asarray(c, float))
        scale.append(float(abs(d) * np.linalg.norm(u) + np.linalg.norm(sc.tic) + np.linalg.norm(sc.Ps[f]) + nP + 2 * motion
                           + np.linalg.norm(np.asarray(pw[:3], float))))
    return np.array(out), np.array(scale)


def predict_f64(sc, first, uv, dep, frame_count):
    """The oracle's 4x4 form in double (the calibration's stand-in)."""
    def T(R, P):
        t = np.eye(4); t[:3, :3] = R; t[:3, 3] = P
        return t
    cur, prev = T(sc.Rs[frame_count], sc.Ps[frame_count]), T(sc.Rs[frame_count - 1], sc.Ps[frame_count - 1])
    nxt = cur @ (np.linalg.inv(prev) @ cur)
    Tbc = T(sc.ric, sc.tic)
    inv = np.linalg.inv(nxt @ Tbc)
    return np.array([(inv @ T(sc.Rs[f], sc.Ps[f]) @ Tbc @ np.append(d * np.asarray(u), 1.0))[:3] for f, u, d in zip(first, uv, dep)])


def predict_case(n, offset, ext, seed):
    rng = np.random.default_rng(seed)
    tic, ric = (TIC, RIC) if ext else (np.zeros(3), np.eye(3))
    Ps, Rs = window_poses(0.15, offset, seed)
    sc = Scene("predict", Ps, Rs, tic, ric, 3.0, [])
    first = rng.integers(0, N_FRAMES, n).astype(np.int32)
    uv = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.4, 0.4, n), np.ones(n)], 1)
    dep = rng.uniform(0.2, 50.0, n)
    return sc, first, np.ascontiguousarray(uv), dep
