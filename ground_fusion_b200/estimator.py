"""Host-side mirror of the reference's Estimator::optimization() (estimator.h:147, estimator.cpp:2890-3636)
over the C ABI (gf_ba_*): the ceres::Solve it performs runs on the GPU; there is no CPU fallback.
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import BaPrior, BaProblem, BaSummary, check


def double2vector(problem, R0_before, P0_before, use_imu=True):
    """Estimator::double2vector (estimator.cpp:2440-2494): Rs [F,3,3], Ps [F,3], Vs [F,3] from the solved para_* arrays,
    with frame 0's yaw and position restored to their values before the solve.  Host-only (no GPU needed)."""
    L = _lib.lib()
    dp = ctypes.POINTER(ctypes.c_double)
    L.gf_ba_double2vector.argtypes = [ctypes.POINTER(BaProblem), dp, dp, ctypes.c_int, dp, dp, dp]
    F = problem.n_frames
    R0 = np.ascontiguousarray(R0_before, np.float64).reshape(3, 3); P0 = np.ascontiguousarray(P0_before, np.float64).reshape(3)
    Rs, Ps, Vs = np.zeros((F, 3, 3)), np.zeros((F, 3)), np.zeros((F, 3))
    p = problem.struct()
    check(L.gf_ba_double2vector(ctypes.byref(p), R0.ctypes.data_as(dp), P0.ctypes.data_as(dp), 1 if use_imu else 0,
                                Rs.ctypes.data_as(dp), Ps.ctypes.data_as(dp), Vs.ctypes.data_as(dp)))
    return Rs, Ps, Vs


def spd_solve(A, b, device=0, tile_cap=-1):
    """x = A^-1 b through the back end's own dense solver (gf_stage_spd_solve: 8x8-tile Cholesky on FP64 tensor-core MMAs)."""
    L = _lib.lib()
    dp = ctypes.POINTER(ctypes.c_double)
    L.gf_stage_spd_solve.argtypes = [ctypes.c_int, dp, dp, ctypes.c_int, dp, ctypes.c_int]
    A = np.ascontiguousarray(A, np.float64); b = np.ascontiguousarray(b, np.float64)
    n = len(b)
    assert A.shape == (n, n)
    x = np.zeros(n)
    check(L.gf_stage_spd_solve(int(device), A.ctypes.data_as(dp), b.ctypes.data_as(dp), n, x.ctypes.data_as(dp), int(tile_cap)))
    return x


SYM_EIG_METHODS = {"ql": 0, "jacobi": 1}


def sym_eig(A, method, device=0):
    """Eigendecomposition of a symmetric matrix (lower triangle read) by one of the marginalisation's eigensolvers
    (gf_stage_sym_eig): "ql" = k_sym_eig_ql (n <= 128), "jacobi" = k_jacobi_eig.  Returns (w, V, sweeps): eigenvalues
    unsorted, eigenvectors in the columns of V, Jacobi's sweep count (0 for QL)."""
    L = _lib.lib()
    dp = ctypes.POINTER(ctypes.c_double)
    L.gf_stage_sym_eig.argtypes = [ctypes.c_int, dp, ctypes.c_int, ctypes.c_int, dp, dp, ctypes.POINTER(ctypes.c_int)]
    A = np.ascontiguousarray(A, np.float64)
    n = A.shape[0]
    assert A.shape == (n, n)
    w, V, sw = np.zeros(n), np.zeros((n, n)), ctypes.c_int(0)
    check(L.gf_stage_sym_eig(int(device), A.ctypes.data_as(dp), n, SYM_EIG_METHODS[method], w.ctypes.data_as(dp), V.ctypes.data_as(dp),
                             ctypes.byref(sw)))
    return w, V, sw.value


def marginalize_dense(A, b, c, L, force_generic=False, device=0):
    """MarginalizationInfo::marginalize on a dense system (gf_stage_marginalize, the device code of the marginalisation):
    columns [c dense | L landmarks (diagonal block) | n kept].  Returns (J0 n x n, r0 n, path) with
    path = (GF_MARG_PATH_* bits, Jacobi sweeps on Amm, Jacobi sweeps on the reduced system)."""
    lib = _lib.lib()
    dp = ctypes.POINTER(ctypes.c_double)
    lib.gf_stage_marginalize.argtypes = [ctypes.c_int, dp, dp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, dp, dp,
                                         ctypes.POINTER(ctypes.c_int)]
    A = np.ascontiguousarray(A, np.float64); b = np.ascontiguousarray(b, np.float64)
    N = len(b)
    assert A.shape == (N, N)
    n = N - c - L
    J0, r0, path = np.zeros((max(n, 0), max(n, 0))), np.zeros(max(n, 0)), (ctypes.c_int * 3)()
    check(lib.gf_stage_marginalize(int(device), A.ctypes.data_as(dp), b.ctypes.data_as(dp), N, int(c), int(L), 1 if force_generic else 0,
                                   J0.ctypes.data_as(dp), r0.ctypes.data_as(dp), path))
    return J0, r0, tuple(path)


def _solve_multi_fn():
    L = _lib.lib()
    L.gf_ba_solve_multi.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.POINTER(BaProblem), ctypes.POINTER(BaSummary),
                                    ctypes.POINTER(ctypes.c_int32)]
    return L.gf_ba_solve_multi


def solve_multi_structs(adjusters, p_array):
    """gf_ba_solve_multi for a pre-built ctypes array of gf_ba_problem (BaProblem * n), e.g. in timing loops: window k is
    p_array[k] on adjusters[k] (distinct BundleAdjusters on one device).  Returns (BaSummary * n, status int32 array): status[k]
    < 0 marks a window whose IMU covariance is singular (its blocks are left untouched); argument errors raise GfError."""
    n = len(adjusters)
    handles = (ctypes.c_void_p * n)(*[a._h.value for a in adjusters])
    sums, status = (BaSummary * n)(), np.zeros(n, np.int32)
    rc = _solve_multi_fn()(handles, n, p_array, sums, status.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)))
    if rc != 0 and not (status < 0).any():
        check(rc)
    return sums, status


def solve_multi(adjusters, problems):
    """Estimator::optimization() of several windows in one batched call (gf_ba_solve_multi): problems[k]
    (ground_fusion_b200.ba_problem.Problem) is solved on adjusters[k] and updated in place.  Returns (summary dicts, statuses);
    status k < 0: window k's IMU covariance is singular and its blocks are untouched.  device_ms is the time of the whole batch."""
    assert len(adjusters) == len(problems)
    p_array = (BaProblem * len(problems))(*[p.struct() for p in problems])
    sums, status = solve_multi_structs(adjusters, p_array)
    return [s.as_dict() for s in sums], [int(v) for v in status]


def _capture_buffers(adjuster, problem):
    """A gf_ba_step_capture whose arrays are numpy buffers sized for `problem` (gf_ba_step_dims), and those buffers."""
    L = _lib.lib()
    L.gf_ba_step_dims.argtypes = [ctypes.c_void_p, ctypes.POINTER(BaProblem), ctypes.POINTER(ctypes.c_int)]
    dims = (ctypes.c_int * 3)()
    p = problem.struct()
    check(L.gf_ba_step_dims(adjuster._h, ctypes.byref(p), dims))
    nc, nl, n = dims
    shapes = {"imu_sqrt": (problem.n_imu, 15, 15), "H": (nc, nc), "Hp": (nc, nc), "g": (n,), "W": (nl, nc), "hll": (nl,), "scale": (n,),
              "D": (n,), "gs": (n,), "e_l": (nl,), "S": (nc + 1, nc + 1), "gn": (n,), "delta": (n,),
              "Xc": (16 * problem.n_frames + 24 + problem.n_features,)}
    bufs = {k: np.zeros(v) for k, v in shapes.items()}
    bufs["col_feat"] = np.zeros(max(problem.n_features, 1), np.int32)
    c = _lib.BaStepCapture()
    for k in _lib.BaStepCapture.ARRAYS:
        setattr(c, k, bufs[k].ctypes.data_as(ctypes.POINTER(ctypes.c_double)) if bufs[k].size else None)
    c.col_feat = bufs["col_feat"].ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
    return c, bufs


def _capture_dict(c, bufs, problem):
    out = {k: getattr(c, k) for k, _ in c._fields_ if k not in _lib.BaStepCapture.ARRAYS and k != "col_feat"}
    for k in ("col_pose", "col_sb", "col_ix"):
        out[k] = list(out[k])
    out["col_pose"], out["col_sb"] = out["col_pose"][:problem.n_frames], out["col_sb"][:problem.n_frames]
    out.update({k: v for k, v in bufs.items() if k != "col_feat"})
    out["col_feat"] = bufs["col_feat"][:problem.n_features].copy()
    return out


def first_step_multi(adjusters, problems, radius=1e4, mu=1e-8):
    """gf_ba_first_step: the chain of solve_multi from the trust-region state (radius, mu), stopped after the first dogleg step.
    Returns one dict per window with the linearisation (H, Hp, g, W, hll, imu_sqrt), the scaling (scale, D, gs, e_l), the
    reduced system S (lower triangle, rhs in row nc), the Cauchy terms, the Gauss-Newton and dogleg step (gn, dogleg_a/b,
    delta, model_change) and the candidate Xc.  No parameter block is modified."""
    assert len(adjusters) == len(problems)
    n = len(adjusters)
    caps = [_capture_buffers(a, p) for a, p in zip(adjusters, problems)]
    L = _lib.lib()
    L.gf_ba_first_step.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.POINTER(BaProblem), ctypes.c_double,
                                   ctypes.c_double, ctypes.POINTER(_lib.BaStepCapture)]
    handles = (ctypes.c_void_p * n)(*[a._h.value for a in adjusters])
    p_array = (BaProblem * n)(*[p.struct() for p in problems])
    out = (_lib.BaStepCapture * n)(*[c for c, _ in caps])
    check(L.gf_ba_first_step(handles, n, p_array, float(radius), float(mu), out))
    return [_capture_dict(out[k], caps[k][1], problems[k]) for k in range(n)]


class BundleAdjuster:
    """One solver workspace bound to one GPU (gf_ba).  optimization(problem) updates the para_* arrays of
    `problem` (ground_fusion_b200.ba_problem.Problem) in place, like Estimator::optimization() does with
    its para_Pose / para_SpeedBias / para_Feature members, and returns the solver summary."""

    def __init__(self, device=0):
        self.L = _lib.lib()
        self.L.gf_ba_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int]
        self.L.gf_ba_destroy.argtypes = [ctypes.c_void_p]
        self.L.gf_ba_destroy.restype = None
        self.L.gf_ba_solve.argtypes = [ctypes.c_void_p, ctypes.POINTER(BaProblem), ctypes.POINTER(BaSummary)]
        self._h = ctypes.c_void_p()
        check(self.L.gf_ba_create(ctypes.byref(self._h), int(device)))

    def optimization(self, problem):
        p = problem.struct()
        s = BaSummary()
        check(self.L.gf_ba_solve(self._h, ctypes.byref(p), ctypes.byref(s)))
        return s.as_dict()

    def _marginalize(self, problem, fn_name):
        from .ba_problem import Prior
        dp = ctypes.POINTER(ctypes.c_double)
        fn = getattr(self.L, fn_name)
        fn.argtypes = [ctypes.c_void_p, ctypes.POINTER(BaProblem), ctypes.POINTER(BaPrior), dp, dp, dp, ctypes.POINTER(ctypes.c_float)]
        p = problem.struct()
        cap = 16 * problem.n_frames + 24
        x0 = np.zeros(cap); J = np.zeros(cap * cap); r = np.zeros(cap)
        out = BaPrior(); ms = ctypes.c_float(0)
        n = fn(self._h, ctypes.byref(p), ctypes.byref(out), x0.ctypes.data_as(dp), J.ctypes.data_as(dp), r.ctypes.data_as(dp), ctypes.byref(ms))
        if n < 0:
            check(n)
        if n == 0:
            return None
        self.last_marg_ms = float(ms.value)
        nb = out.n_blocks
        return Prior(list(out.block_kind)[:nb], list(out.block_index)[:nb], list(out.block_idx)[:nb], x0.copy(),
                     J[:n * n].reshape(n, n).copy(), r[:n].copy())

    def marginalize_old(self, problem):
        """MARGIN_OLD on the GPU (estimator.cpp:3334-3535): returns the ba_problem.Prior for the next window (block indices
        already shifted by one frame).  last_marg_ms holds the CUDA-event time."""
        return self._marginalize(problem, "gf_ba_marginalize_old")

    def marginalize_second_new(self, problem):
        """MARGIN_SECOND_NEW on the GPU (estimator.cpp:3536-3631): the last prior with para_Pose[WINDOW_SIZE - 1] marginalised;
        None when the prior does not hold that pose (the reference then keeps the prior as it is)."""
        return self._marginalize(problem, "gf_ba_marginalize_second_new")

    def last_marg_info(self):
        """(GF_MARG_PATH_* bits, Jacobi sweeps on Amm, Jacobi sweeps on the reduced system) of the last marginalisation."""
        info = (ctypes.c_int * 3)()
        self.L.gf_ba_last_marg_info.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
        check(self.L.gf_ba_last_marg_info(self._h, info))
        return tuple(info)

    def first_step(self, problem, radius=1e4, mu=1e-8):
        """The solve's first iteration on this handle, captured stage by stage (see first_step_multi)."""
        return first_step_multi([self], [problem], radius, mu)[0]

    def solve_struct(self, p_struct):
        """Same, for a pre-built ctypes gf_ba_problem (avoids rebuilding it in timing loops)."""
        s = BaSummary()
        check(self.L.gf_ba_solve(self._h, ctypes.byref(p_struct), ctypes.byref(s)))
        return s

    def close(self):
        if self._h:
            self.L.gf_ba_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
