"""High-precision reference of the bundle-adjustment solve's first iteration (gf_ba_first_step), CPU only.

Everything starts from the oracle's dense, loss-corrected, locally parameterised linearisation (oracle/ba_oracle.c
gfo_ba_linearize, pinned by finite differences in test_ba_oracle.py) and is then computed in np.longdouble: the cost,
J^T J split into the camera block H, the prior block Hp, the landmark terms W and h_ll, the gradient g, the Jacobi scale,
D^2 with its [1e-6, 1e32] clamp, the reduced system (H' + mu D^2 with the landmarks eliminated) and its right-hand side, the
Cauchy step, the Gauss-Newton step (Cholesky with one refinement step, then the landmark back substitution), the dogleg branch,
the model cost change, delta and x (+) delta.  The IMU sqrt-information LLT(cov^-1).L^T is computed in mpmath.

`reference(..., dt=np.float64, lin=fma_linearization)` runs the same computation in plain double on a Jacobian evaluated with
FMA contraction (nvcc contracts, the oracle is built without): that is what an FP64 implementation of these stages achieves, and
what the bars below are calibrated on (test_ba_lin_ref.py).

Bars: ratio = error / (EPS * scale); a GPU result passes when ratio <= K.  K = CALIBRATION_FACTOR x the worst ratio of the
double computation over the calibration windows, rounded up.
"""
import ctypes
import os
import platform
import subprocess

import mpmath as mp
import numpy as np
import scipy.linalg

from marg_ref import EPS, LD
from oracle import ba_oracle as O

CALIBRATION_FACTOR = 8
DIAG_MIN, DIAG_MAX = 1e-6, 1e32          # Ceres' min_lm_diagonal / max_lm_diagonal
# bar -> K (see the module docstring; scales in ratios())
K = {
    "cost": 170.0,            # |c - c_ref| / (eps c_ref)   worst CPU 20.9 (visual_only_F6)
    "H": 1200.0,              # |H_ab - ref| / (eps sqrt(H_aa H_bb))          (camera block without the prior)   worst CPU 140 (visual_only_F6)
    "Hp": 32.0,             # same with the prior's own diagonal   worst CPU 3.93 (prior)
    "W": 400.0,              # |W_la - ref| / (eps sqrt(h_ll H_aa))   worst CPU 49.9 (visual_only_F11)
    "hll": 2900.0,            # relative   worst CPU 361 (visual_only_F6)
    "g": 2800.0,  # |g_a - ref| / (eps (|J|^T rm)_a), rm = |r|, prior rows |r0| + |J0| (|dx| + |x0|), IMU rows |U| (terms before cancellation)   worst CPU 338 (prior)
    "scale": 1400.0,           # relative   worst CPU 172 (visual_only_F6)
    "D": 70.0,               # relative   worst CPU 8.41 (visual_only_F6)
    "gs": 2600.0,  # |gs_a - ref| / (eps s_a (|J|^T rm)_a / D_a)   worst CPU 320 (prior)
    "e_l": 140.0,            # relative   worst CPU 17.2 (visual_only_F6)
    "S": 320.0,              # |S_ab - ref| / (eps sqrt(S^_aa S^_bb)), S^ = H' + mu D^2 before the elimination   worst CPU 38.6 (ex_td_free)
    "rhs": 1200.0,  # |b_a - ref| / (eps (s_a gm_a + sum_l |A_al| e_l s_l gm_l)), gm = the g bar's scale   worst CPU 144 (visual_only_F6)
    "cauchy_num": 310.0,      # relative   worst CPU 38 (visual_only_F6)
    "cauchy_den": 30.0,     # |den - ref| / (eps (sum_a |v_a| sqrt(H'_aa))^2)   worst CPU 3.7 (visual_only_F6)
    "gn_backward": 7.0,     # ||S y - b|| / (n eps (||S|| ||y|| + ||b||)), y = the captured reduced solution   worst CPU 0.822 (stationary_wheel)
    "gn_forward": 120.0,      # ||gn - ref|| / (eps kappa(S) ||ref||)   worst CPU 14.5 (stationary)
    "model_change": 50.0,   # |m - ref| / (eps (|s^T g'| + |s^T H' s| / 2 + [GN part] kappa ||s|| ||g' + H' s||))   worst CPU 6.18 (visual_only_F6)
    "delta": 140.0,           # max |delta - ref| / (eps kappa_step ||delta_ref||), kappa_step = kappa(S) when the step has a GN part, else 1   worst CPU 16.3 (plane_wheel)
    "alpha": 2.0,  # |alpha - ref| / (eps alpha (1 + den scale / den))   worst CPU 0.245 (visual_only_F6)
    "grad_max": 16.0,  # |x - x (+) -g|_inf, / (eps (|x|_inf + grad_max + |g bar scale|_inf))   worst CPU 1.93 (visual_only_F6)
    "x_norm": 7.0,  # relative   worst CPU 0.861 (prior_plane)
    "step_norm": 10.0,  # against |Xc - x| of the captured Xc, / (eps (step_norm + sqrt(m) |x|_inf))   worst CPU 1.18 (plane)
    "dogleg_norm": 7.0,  # against |a gs + b gn| of the captured vectors, / (eps (|a| |gs| + |b| |gn|))   worst CPU 0.826 (plane)
    "Xc": 8.0,  # against x (+) delta of the captured delta (oracle Plus), / (eps (|x (+) delta| + |delta|_inf))   worst CPU 0.945 (prior)
    "sqrt_info": 6e-4,      # max |U - ref| / (eps ||U||_2 kappa(cov))   worst CPU 6.74e-05 (oracle, graded)
}


# ---- linearisation ----------------------------------------------------------------------------------------------------
def layout(pb):
    """(row block sizes in the oracle's row order, pn, L): prior | IMU | wheel | plane | visual."""
    pn = pb.prior.n if pb.prior is not None else 0
    blocks = ([pn] if pn else []) + [15] * pb.n_imu + [6] * pb.n_wheel + [3] * pb.n_plane + [2] * pb.n_visual
    free = {int(pb.visual[v].feature) for v in range(pb.n_visual) if not pb.feature_const[pb.visual[v].feature]}
    return blocks, pn, len(free)


def linearization(pb, lib=None):
    """(r, J) of the oracle at pb's values; lib: another build of oracle/ba_oracle.c (fma_oracle())."""
    blocks, _, _ = layout(pb)
    rows = sum(blocks)
    cols = 16 * pb.n_frames + 24 + pb.n_features
    if lib is None:
        return O.linearize(pb, cap_rows=max(rows, 1), cap_cols=cols)
    p = pb.struct()
    r = np.zeros(max(rows, 1)); J = np.zeros(max(rows, 1) * cols); nc = ctypes.c_int(0)
    got = lib.gfo_ba_linearize(ctypes.byref(p), r.ctypes.data_as(O._dp), J.ctypes.data_as(O._dp), ctypes.byref(nc), max(rows, 1), cols)
    assert got == rows, got
    return r[:rows].copy(), J[:rows * nc.value].reshape(rows, nc.value).copy()


_FMA = None


def fma_oracle():
    """oracle/ba_oracle.c built with FMA contraction (-ffp-contract=fast; on x86-64 also -mfma, which the baseline ISA lacks),
    next to the oracle's own build."""
    global _FMA
    if _FMA is None:
        src = os.path.join(os.path.dirname(O.__file__), "ba_oracle.c")
        so = os.path.join(os.path.dirname(O._SO), "libgf_oracle_ba_fma.so")
        if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
            os.makedirs(os.path.dirname(so), exist_ok=True)
            arch = ["-mfma"] if platform.machine() in ("x86_64", "AMD64") else []
            subprocess.check_call(["gcc", "-O2", *arch, "-ffp-contract=fast", "-shared", "-fPIC", "-o", so, src, "-lm"])
        lib = ctypes.CDLL(so)
        lib.gfo_ba_linearize.argtypes = O.lib().gfo_ba_linearize.argtypes
        lib.gfo_ba_plus.argtypes = O.lib().gfo_ba_plus.argtypes
        lib.gfo_ba_plus.restype = None
        _FMA = lib
    return _FMA


def plus(pb, delta, lib=None):
    """x (+) delta of the oracle (lib: fma_oracle()) on a copy of pb, in packed_x order."""
    q = pb.clone()
    if lib is None:
        O.plus(q, delta)
    else:
        p = q.struct()
        d = np.ascontiguousarray(delta, np.float64)
        lib.gfo_ba_plus(ctypes.byref(p), d.ctypes.data_as(O._dp))
    return packed_x(q)


def _imu_magnitudes(pb, row0):
    """(rows, scale) of the IMU residuals before their cancellation: |U| times the magnitude of the terms each raw residual
    sums (positions, velocity * dt, gravity * dt^2, the preintegrated deltas, biases).  Near an optimum the residuals
    themselves are tiny, while their rounding follows these terms."""
    rows, mags = [], []
    G = float(np.linalg.norm(pb.gravity))
    for k in range(pb.n_imu):
        f = pb.imu[k]
        i, j, dt = f.i, f.j, f.sum_dt
        P, V = pb.para_pose[[i, j], :3], pb.para_speed_bias[[i, j], :3]
        ba, bg = pb.para_speed_bias[[i, j], 3:6], pb.para_speed_bias[[i, j], 6:9]
        m = np.empty(15)
        m[0:3] = np.abs(P).sum(0).max() + np.abs(V[0]).max() * dt + 0.5 * G * dt * dt + np.abs(f.delta_p).max()
        m[3:6] = 2.0
        m[6:9] = np.abs(V).sum(0).max() + G * dt + np.abs(f.delta_v).max()
        m[9:12] = np.abs(ba).sum(0).max()
        m[12:15] = np.abs(bg).sum(0).max()
        U = np.zeros(225)
        O.lib().gfo_sqrt_info(np.ascontiguousarray(f.covariance, np.float64).ctypes.data_as(O._dp), 15, U.ctypes.data_as(O._dp))
        rows.append(np.arange(row0 + 15 * k, row0 + 15 * k + 15))
        mags.append(np.abs(U.reshape(15, 15)) @ m)
    return rows, mags


def _gram(J, r, blocks, dt, row=0):
    """J^T J and J^T r of the row blocks `blocks` starting at `row`, summed factor by factor over each factor's nonzero columns
    (J is block-sparse by rows)."""
    n = J.shape[1]
    G = np.zeros((n, n), dt); g = np.zeros(n, dt)
    for b in blocks:
        Jb = J[row:row + b]
        nz = np.flatnonzero(np.any(Jb != 0, axis=0))
        if len(nz):
            Jz = Jb[:, nz].astype(dt)
            G[np.ix_(nz, nz)] += Jz.T @ Jz
            g[nz] += Jz.T @ r[row:row + b].astype(dt)
        row += b
    return G, g


def _chol_solve(A, b, dt):
    """A x = b for SPD A: longdouble Cholesky with one refinement step, or scipy's in double."""
    if dt == np.float64:
        return scipy.linalg.cho_solve(scipy.linalg.cho_factor(A, lower=True), b)
    n = len(b)
    Lm = np.zeros((n, n), dt)
    for j in range(n):
        v = A[j:, j] - Lm[j:, :j] @ Lm[j, :j]
        if not v[0] > 0:
            raise np.linalg.LinAlgError("not positive definite")
        Lm[j:, j] = v / np.sqrt(v[0])

    def solve(rhs):
        y = np.zeros(n, dt)
        for i in range(n):
            y[i] = (rhs[i] - Lm[i, :i] @ y[:i]) / Lm[i, i]
        x = np.zeros(n, dt)
        for i in range(n - 1, -1, -1):
            x[i] = (y[i] - Lm[i + 1:, i] @ x[i + 1:]) / Lm[i, i]
        return x
    x = solve(b)
    return x + solve(b - A @ x)


def reference(pb, radius=1e4, mu=1e-8, dt=LD, lin=None):
    """Every quantity gf_ba_first_step captures, computed from the oracle's linearisation in `dt`.  lin: (r, J) to use."""
    blocks, pn, L = layout(pb)
    r, J = lin if lin is not None else linearization(pb)
    n = J.shape[1]
    nc = n - L
    cost = _huber_cost(r, pb.n_visual, dt)
    G, g = _gram(J, r, blocks[1:] if pn else blocks, dt, row=pn)  # without the prior
    Gp, gp = _gram(J, r, blocks[:1], dt) if pn else (np.zeros((n, n), dt), np.zeros(n, dt))
    # rounding scale of each residual: |r|, except the prior's r = r0 + J0 dx: dx = x - x0 carries the rounding of x, and
    # the sum cancels
    rmag = np.abs(r)
    if pn:
        J0, r0 = pb.prior.J, pb.prior.r
        dx = np.linalg.lstsq(J0, r[:pn] - r0, rcond=None)[0]
        rmag[:pn] = np.abs(r0) + np.abs(J0) @ (np.abs(dx) + np.abs(pb.prior.x0).max())
    for rw, mg in zip(*_imu_magnitudes(pb, pn)):
        rmag[rw] = np.maximum(rmag[rw], mg)
    absJr = _gram(np.abs(J), rmag, blocks, dt)[1]
    g = g + gp
    Ht = G + Gp                                                     # the whole J^T J
    d = np.diag(Ht)
    scale = dt(1) / (dt(1) + np.sqrt(d))
    Hs = Ht * scale[:, None] * scale[None, :]
    g1 = g * scale
    D2 = np.clip(np.diag(Hs), dt(DIAG_MIN), dt(DIAG_MAX))
    D = np.sqrt(D2)
    gs = g1 / D
    v = gs / D
    num = gs @ gs
    den = v @ (Hs @ v)
    alpha = num / den
    A = Hs + np.diag(dt(mu) * D2)
    e_l = dt(1) / np.diag(A)[nc:]
    Acl = A[:nc, nc:]
    S = A[:nc, :nc] - (Acl * e_l[None, :]) @ Acl.T
    rhs = g1[:nc] - Acl @ (e_l * g1[nc:])
    y = np.zeros(n, dt)
    if nc:
        y[:nc] = _chol_solve(S, rhs, dt)
    y[nc:] = e_l * (g1[nc:] - Acl.T @ y[:nc])
    gn = -D * y
    gnorm, gnn = np.sqrt(num), np.sqrt(gn @ gn)
    if gnn <= radius:
        branch, ca, cb = "gauss_newton", dt(0), dt(1)
    elif gnorm * alpha >= radius:
        branch, ca, cb = "cauchy", -dt(radius) / gnorm, dt(0)
    else:
        branch = "interpolated"
        b_dot_a = -alpha * (gs @ gn)
        a2 = (alpha * gnorm) ** 2
        bma2 = a2 - 2 * b_dot_a + gnn * gnn
        cc = b_dot_a - a2
        dd = np.sqrt(cc * cc + bma2 * (dt(radius) ** 2 - a2))
        beta = (dd - cc) / bma2 if cc <= 0 else (dt(radius) ** 2 - a2) / (dd + cc)
        ca, cb = -alpha * (1 - beta), beta
    step = ca * gs + cb * gn
    s = step / D
    sg, sHs = s @ g1, s @ (Hs @ s)
    model_change = -(sg + sHs / 2)
    # first-order sensitivity of the model change to the Gauss-Newton part of the step (forward error ~ eps kappa)
    kappa = float(np.linalg.cond(np.asarray(S, np.float64))) if nc else 1.0
    gn_part = kappa * float(np.linalg.norm(np.asarray(s, np.float64))) * float(np.linalg.norm(np.asarray(g1 + Hs @ s, np.float64))) if cb != 0 else 0.0
    delta = s * scale
    fm = free_mask(pb)
    x = packed_x(pb)
    plib = fma_oracle() if dt == np.float64 else None          # the calibration's stand-in for the kernel's own Plus
    xg = plus(pb, -np.asarray(g, np.float64), plib)
    hat = np.sqrt(np.abs(np.diag(A)))[:nc]
    return dict(nc=nc, L=L, n=n, cost=cost, H=G[:nc, :nc], Hp=Gp[:nc, :nc], g=g, W=G[nc:, :nc], hll=np.diag(G)[nc:].copy(),
                Hfull_diag=np.diag(Ht), Hd=np.diag(G), Hpd=np.diag(Gp), absJr=absJr, scale=scale, D=D, D2=D2, gs=gs, e_l=e_l,
                S=S, rhs=rhs, S_hat=hat, rhs_scale=(scale * absJr)[:nc] + np.abs(Acl) @ (e_l * (scale * absJr)[nc:]),
                cauchy_num=num, cauchy_den=den, cauchy_den_scale=(np.abs(v) @ np.sqrt(np.diag(Hs))) ** 2, alpha=alpha,
                gn=gn, y=y, kappa=kappa, branch=branch, dogleg_a=ca, dogleg_b=cb, dogleg_norm=np.sqrt(step @ step),
                model_change=model_change, model_scale=abs(sg) + abs(sHs) / 2 + gn_part, delta=delta,
                Xc=plus(pb, np.asarray(delta, np.float64), plib), Xc_mask=packed_mask(pb), free_mask=fm, pb=pb,
                grad_max=np.abs(x - xg)[fm].max() if fm.any() else 0.0, x_norm=np.sqrt((x[fm].astype(dt) ** 2).sum()), clamped=(np.diag(Hs) < DIAG_MIN) | (np.diag(Hs) > DIAG_MAX))


def _huber_cost(r, n_visual, dt):
    """1/2 sum rho: the oracle's visual rows carry the loss-corrected sqrt(rho'(s)) r, from which rho(s) is rebuilt."""
    nvis = 2 * n_visual
    rl = r.astype(dt)
    c = rl[:len(r) - nvis] @ rl[:len(r) - nvis] / 2
    rv = rl[len(r) - nvis:].reshape(-1, 2)
    q = (rv * rv).sum(1)                                   # rho'(s) s = s (inliers) | sqrt(s) (outliers, s > 1)
    rho = np.where(q > 1, 2 * q - 1, q)                    # outliers: s = q^2, rho = 2 sqrt(s) - 1 = 2 q - 1
    return c + rho.sum() / 2


def packed_x(pb):
    """x in gf_ba_step_capture.Xc's order."""
    return np.concatenate([pb.para_pose.ravel(), pb.para_speed_bias.ravel(), pb.para_ex_pose, pb.para_td, pb.para_ex_wheel,
                           pb.para_ix_wheel, pb.para_td_wheel, pb.para_plane_R, pb.para_plane_Z, pb.para_feature[:pb.n_features]])


def free_mask(pb):
    """Entries of packed_x that belong to a free block (the ambient coordinates the solve's norms run over)."""
    F, o = pb.n_frames, 16 * pb.n_frames
    m = np.zeros(16 * F + 24 + pb.n_features, bool)
    for f in range(F):
        m[7 * f:7 * f + 7] = not (pb.frames_const or (f == 0 and pb.pose0_const))
        m[7 * F + 9 * f:7 * F + 9 * f + 9] = not (pb.frames_const or pb.pose0_const)
    m[o:o + 7] = not pb.ex_pose_const
    m[o + 7] = not pb.td_const
    m[o + 8:o + 15] = (pb.n_wheel > 0 or pb.n_plane > 0) and not pb.ex_wheel_const
    m[o + 15:o + 18] = pb.n_wheel > 0 and not pb.ix_wheel_const
    m[o + 18] = pb.n_wheel > 0 and not pb.td_wheel_const
    m[o + 19:o + 24] = pb.n_plane > 0 and not pb.plane_const
    for v in range(pb.n_visual):
        k = pb.visual[v].feature
        m[o + 24 + k] = not pb.feature_const[k]
    return m


def packed_mask(pb):
    """Entries of packed_x the solve uses (blocks of absent factor kinds hold defaults on the device)."""
    F = pb.n_frames
    m = np.ones(16 * F + 24 + pb.n_features, bool)
    o = 16 * F + 8
    m[o:o + 7] = pb.n_wheel > 0 or pb.n_plane > 0
    m[o + 7:o + 11] = pb.n_wheel > 0
    m[o + 11:o + 16] = pb.n_plane > 0
    return m


# ---- IMU sqrt-information -----------------------------------------------------------------------------------------------
def sqrt_info_mp(cov, dps=50):
    """LLT(cov^-1).matrixL().transpose() at `dps` digits; (U, ||U||_2, kappa(cov)) in double."""
    with mp.workdps(dps):
        C = mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.asarray(cov).reshape(15, 15)])
        Lm = mp.cholesky(mp.inverse(C))
        U = np.array([[float(Lm[j, i]) for j in range(15)] for i in range(15)])
    w = np.linalg.eigvalsh(np.asarray(cov, np.float64).reshape(15, 15))
    return U, float(np.linalg.norm(U, 2)), float(np.abs(w).max() / np.abs(w).min())


def sqrt_info_ratio(U, cov):
    ref, nu, kc = sqrt_info_mp(cov)
    return float(np.abs(U - ref).max() / (EPS * nu * kc))


# ---- ratios ------------------------------------------------------------------------------------------------------------
def _safe(err, sc):
    err = np.abs(np.asarray(err, np.float64)); sc = np.asarray(sc, np.float64)
    out = np.where(sc > 0, err / np.where(sc > 0, sc, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(out.max()) / EPS if out.size else 0.0


def ratios(got, ref):
    """Ratio per bar of the captured quantities `got` (a first_step dict, or reference(dt=float64)) against the reference."""
    f = lambda k: np.asarray(ref[k], np.float64)
    nc = ref["nc"]
    out = {}
    out["cost"] = _safe(got["initial_cost"] - f("cost"), f("cost"))
    Hd, Hpd = f("Hd"), f("Hpd")
    out["H"] = _safe(got["H"] - f("H"), np.sqrt(np.outer(Hd[:nc], Hd[:nc])))
    out["Hp"] = _safe(got["Hp"] - f("Hp"), np.sqrt(np.outer(Hpd[:nc], Hpd[:nc])))
    out["W"] = _safe(got["W"] - f("W"), np.sqrt(np.outer(Hd[nc:], Hd[:nc])))
    out["hll"] = _safe(got["hll"] - f("hll"), f("hll"))
    out["g"] = _safe(got["g"] - f("g"), f("absJr"))
    for k in ("scale", "D", "e_l"):
        out[k] = _safe(got[k] - f(k), np.abs(f(k)))
    out["gs"] = _safe(got["gs"] - f("gs"), f("scale") * f("absJr") / f("D"))
    S = np.tril(got["S"][:nc, :nc])
    hat = f("S_hat")
    out["S"] = _safe(S - np.tril(f("S")), np.tril(np.outer(hat, hat)))
    out["rhs"] = _safe(got["S"][nc, :nc] - f("rhs"), f("rhs_scale"))
    out["cauchy_num"] = _safe(got["cauchy_num"] - f("cauchy_num"), f("cauchy_num"))
    out["cauchy_den"] = _safe(got["cauchy_den"] - f("cauchy_den"), f("cauchy_den_scale"))
    if nc:
        yc = -np.asarray(got["gn"][:nc]) / np.asarray(got["D"][:nc])
        Sr, b = np.asarray(ref["S"], LD), np.asarray(ref["rhs"], LD)
        res = Sr @ yc.astype(LD) - b
        nS = float(np.linalg.norm(np.asarray(Sr, np.float64), 2))
        out["gn_backward"] = float(np.linalg.norm(np.asarray(res, np.float64)) / (nS * np.linalg.norm(yc) + float(np.linalg.norm(np.asarray(b, np.float64))))) / (nc * EPS)
    else:
        out["gn_backward"] = 0.0
    gn = f("gn")
    out["gn_forward"] = float(np.linalg.norm(got["gn"] - gn) / (EPS * ref["kappa"] * max(np.linalg.norm(gn), 1e-300)))
    out["model_change"] = _safe(got["model_change"] - f("model_change"), f("model_scale"))
    kst = ref["kappa"] if ref["branch"] != "cauchy" else 1.0
    nd = float(np.linalg.norm(f("delta")))
    out["delta"] = _safe(got["delta"] - f("delta"), np.full(len(gn), kst * nd))
    den_rel = f("cauchy_den_scale") / f("cauchy_den")
    out["alpha"] = _safe(got["alpha"] - f("alpha"), f("alpha") * (1.0 + den_rel))
    # x (+) delta of the captured delta, by the oracle: pins k_ba_step's Plus to a few eps whatever the conditioning
    m, fm, pb = ref["Xc_mask"], ref["free_mask"], ref["pb"]
    x, dcap = packed_x(pb), np.asarray(got["delta"], np.float64)
    xp = plus(pb, dcap)
    out["Xc"] = _safe((got["Xc"] - xp)[m], np.abs(xp[m]) + np.abs(dcap).max())
    step = (np.asarray(got["Xc"], LD) - x.astype(LD))[fm]
    out["step_norm"] = _safe(got["step_norm"] - float(np.sqrt((step * step).sum())), np.full(1, got["step_norm"] + EPS * np.abs(x[fm]).max() * np.sqrt(fm.sum())))
    dn = got["dogleg_a"] * np.asarray(got["gs"], LD) + got["dogleg_b"] * np.asarray(got["gn"], LD)
    out["dogleg_norm"] = _safe(got["dogleg_norm"] - float(np.sqrt((dn * dn).sum())),
                               abs(got["dogleg_a"]) * np.linalg.norm(got["gs"]) + abs(got["dogleg_b"]) * np.linalg.norm(got["gn"]))
    out["grad_max"] = _safe(got["grad_max"] - f("grad_max"), np.abs(x[fm]).max() + f("grad_max") + f("absJr").max() if fm.any() else 0.0)
    out["x_norm"] = _safe(got["x_norm"] - f("x_norm"), f("x_norm"))
    return out


def f64_capture(pb, radius=1e4, mu=1e-8):
    """The captured quantities computed in double on the FMA-contracted Jacobian: the calibration's stand-in for the GPU."""
    lin = linearization(pb, fma_oracle())
    c = reference(pb, radius, mu, dt=np.float64, lin=lin)
    nc = c["nc"]
    Saug = np.zeros((nc + 1, nc + 1))
    Saug[:nc, :nc] = np.tril(c["S"]); Saug[nc, :nc] = c["rhs"]; Saug[nc, nc] = 1.0
    x, fm = packed_x(pb), c["free_mask"]
    step_norm = float(np.linalg.norm((c["Xc"] - x)[fm]))
    return dict(c, initial_cost=c["cost"], S=Saug, step_norm=step_norm, dogleg_norm=float(c["dogleg_norm"]))


# ---- windows -------------------------------------------------------------------------------------------------------------
def with_free_landmarks(pb, L):
    """Exactly the first L features free (every feature of make_window has visual factors)."""
    assert pb.n_features >= L
    pb.feature_const[:] = 1
    pb.feature_const[:L] = 0
    return pb


def with_pair_size(pb, N, pair=(0, 1)):
    """Keeps only the first N visual factors of pose pair `pair` (k_ba_eval cuts a pair's factors into chunks of 64)."""
    rows, kept = [], 0
    for f in list(pb.visual)[:pb.n_visual]:
        if (f.imu_i, f.imu_j) == pair:
            if kept == N:
                continue
            kept += 1
        rows.append((f.imu_i, f.imu_j, f.feature, list(f.pts_i), list(f.pts_j), list(f.vel_i), list(f.vel_j), f.td_i, f.td_j))
    assert kept == N
    pb.set_visual(rows)
    return pb


def prior_plane_window():
    """A plane window whose prior comes from MARGIN_OLD of a plane window: it carries the plane rotation (4 prior columns, 3
    local) and height, and blocks that are constant here (ex pose, td, wheel extrinsic)."""
    from ground_fusion_b200.synth_ba import make_window
    q, _ = make_window(seed=3, with_plane=True)
    O.solve(q)
    nxt, _ = make_window(seed=53, with_plane=True)
    nxt.prior = O.marginalize_old(q)
    return nxt


def windows():
    """name -> builder of the stage tests' windows; nc + 1 covers every residue mod 8 (the 8x8 tiles of the reduced system)."""
    from ground_fusion_b200.synth_ba import make_window
    from test_ba_edges_oracle import add_outliers, add_velocities, stationary_window, visual_only_window

    def mw(**kw):
        return lambda: make_window(**kw)[0]

    def td_free_still():                       # td free, every feature velocity zero: its column is empty, D^2 clamps to 1e-6
        pb = make_window(seed=3)[0]; pb.td_const = 0
        for f in list(pb.visual)[:pb.n_visual]:
            f.vel_i[0] = f.vel_i[1] = f.vel_j[0] = f.vel_j[1] = 0.0
        return pb

    def ex_td_free():
        pb = add_velocities(make_window(seed=3)[0], 3); pb.ex_pose_const = 0
        return pb

    def masked_wheel():
        pb = make_window(seed=7, with_wheel=True, wheel_free=(True, False, True))[0]; pb.ex_wheel_subset_mask = 0b100100
        return pb

    def outliers():
        pb = make_window(seed=8)[0]; add_outliers(pb, 8)
        return pb

    def plane_wheel_masked():
        pb = make_window(seed=4, with_plane=True, with_wheel=True)[0]; pb.plane_r_subset_mask = 0b011
        return pb

    w = {"c2_s0": mw(seed=0), "c2_s1": mw(seed=1), "c2_s2": mw(seed=2),                     # nc 165
         "c3": mw(seed=7, n_landmarks=440),
         "td_free_still": td_free_still,                                                         # 166
         "velocities_td": lambda: add_velocities(make_window(seed=3)[0], 3),                     # 166
         "ex_td_free": ex_td_free,                                                               # 172
         "plane": mw(seed=2, with_plane=True),                                                   # 169
         "wheel": mw(seed=7, with_wheel=True),                                                   # 175
         "wheel_masked": masked_wheel,                                                           # 172
         "plane_wheel": plane_wheel_masked,                                                      # 179
         "outliers": outliers,
         "stationary": stationary_window,                                                        # 0
         "stationary_wheel": lambda: stationary_window(with_wheel=True)}                         # 10
    for F in range(4, 12):                                                                      # 6 (F - 1)
        w["visual_only_F%d" % F] = (lambda F=F: visual_only_window(F))
    for L in (0, 1, 63, 64, 65, 128, 129):
        w["L%d" % L] = (lambda L=L: with_free_landmarks(make_window(seed=7, n_landmarks=440)[0], L))
    w["L_large"] = mw(seed=7, n_landmarks=2150, free_fraction=1.0)                              # L = 2003
    for N in (1, 63, 64, 65, 128, 129):                                                         # factors of pose pair (0, 1)
        w["pair%d" % N] = (lambda N=N: with_pair_size(make_window(seed=7, n_landmarks=440)[0], N))
    w["prior_plane"] = prior_plane_window
    return w


def prior_window():
    from test_ba_edges_gpu import window_with_prior
    return window_with_prior()


def branch_radii(pb, mu=1e-8):
    """Trust-region radii that put the first dogleg step in each branch, well away from the switch points."""
    ref = reference(pb, 1e300, mu, dt=np.float64)
    cauchy_len = float(ref["alpha"] * np.sqrt(ref["cauchy_num"]))
    gn_len = float(np.linalg.norm(ref["gn"]))
    assert cauchy_len < 0.8 * gn_len, (cauchy_len, gn_len)
    return {"gauss_newton": 2.0 * gn_len, "cauchy": 0.5 * cauchy_len, "interpolated": float(np.sqrt(cauchy_len * gn_len))}


# IMU covariances the sqrt-information kernel is tested on (transformations of a real one)
COV_KINDS = ("real", "scaled_up", "scaled_down", "graded", "permuted", "zeros", "indefinite")


def imu_covariance(cov, kind, seed=0):
    cov = np.asarray(cov, np.float64).reshape(15, 15)
    rng = np.random.default_rng(seed)
    if kind == "real":
        return cov.copy()
    if kind == "scaled_up":
        return cov * 1e6
    if kind == "scaled_down":
        return cov * 1e-6
    if kind == "graded":                       # kappa ~ 1e12: the real matrix graded by 1e5 .. 1e0 per side
        g = np.logspace(5, 0, 15)
        out = cov * g[:, None] * g[None, :]
        return (out + out.T) / 2
    if kind == "permuted":                     # the same matrix with rows and columns reordered: another pivot sequence
        p = rng.permutation(15)
        return cov[np.ix_(p, p)]
    if kind == "zeros":                        # exact zeros off the diagonal blocks (position / rotation / velocity / biases)
        out = np.zeros_like(cov)
        for a, b in ((0, 3), (3, 6), (6, 9), (9, 12), (12, 15)):
            out[a:b, a:b] = cov[a:b, a:b]
        return out
    if kind == "indefinite":                   # invertible, one negative eigenvalue
        w, V = np.linalg.eigh(cov)
        w[7] = -w[7]
        out = V @ np.diag(w) @ V.T
        return (out + out.T) / 2
    raise ValueError(kind)
