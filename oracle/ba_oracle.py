"""ctypes wrapper of oracle/ba_oracle.c -- TEST INFRASTRUCTURE ONLY (CPU oracle of the back end)."""
import ctypes
import os
import subprocess

import numpy as np

from ground_fusion_b200._lib import BaImuFactor, BaPrior, BaProblem, BaSummary, BaVisualFactor, BaWheelFactor
from ground_fusion_b200.ba_problem import Prior

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libgf_oracle_ba.so")
_LIB = None
_dp = ctypes.POINTER(ctypes.c_double)


def lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(_HERE, "ba_oracle.c")
        hdr = os.path.join(_HERE, "..", "include", "gf_b200.h")
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", _SO, src, "-lm"])
        L = ctypes.CDLL(_SO)
        L.gfo_ba_solve.argtypes = [ctypes.POINTER(BaProblem), ctypes.POINTER(BaSummary)]
        L.gfo_ba_cost.argtypes = [ctypes.POINTER(BaProblem)]
        L.gfo_ba_cost.restype = ctypes.c_double
        L.gfo_ba_linearize.argtypes = [ctypes.POINTER(BaProblem), _dp, _dp, ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.c_int]
        L.gfo_ba_plus.argtypes = [ctypes.POINTER(BaProblem), _dp]
        L.gfo_ba_plus.restype = None
        L.gfo_ba_marginalize_old.argtypes = [ctypes.POINTER(BaProblem), ctypes.POINTER(BaPrior), _dp, _dp, _dp]
        L.gfo_ba_set_tolerances.argtypes = [ctypes.c_double] * 3
        L.gfo_ba_set_tolerances.restype = None
        L.gfo_sqrt_info.argtypes = [_dp, ctypes.c_int, _dp]
        L.gfo_sym_eig.argtypes = [_dp, ctypes.c_int, _dp, _dp, ctypes.c_int]
        L.gfo_sym_eig.restype = None
        L.gfo_eval_plane.argtypes = [_dp, _dp, _dp, ctypes.c_double, _dp, _dp, _dp, _dp, _dp, _dp]
        L.gfo_eval_plane.restype = None
        L.gfo_eval_wheel.argtypes = [ctypes.POINTER(BaWheelFactor), _dp, _dp, _dp] + [ctypes.c_double] * 4 + [_dp] * 8
        _LIB = L
    return _LIB


def solve(pb):
    """ceres::Solve restatement; updates pb's para_* arrays in place, returns the summary dict."""
    s = BaSummary()
    p = pb.struct()
    rc = lib().gfo_ba_solve(ctypes.byref(p), ctypes.byref(s))
    if rc:
        raise RuntimeError("oracle solve failed: %d" % rc)
    return s.as_dict()


def cost(pb):
    p = pb.struct()
    return lib().gfo_ba_cost(ctypes.byref(p))


def linearize(pb, cap_rows=6000, cap_cols=600):
    p = pb.struct()
    r = np.zeros(cap_rows); J = np.zeros((cap_rows * cap_cols,))
    nc = ctypes.c_int(0)
    rows = lib().gfo_ba_linearize(ctypes.byref(p), r.ctypes.data_as(_dp), J.ctypes.data_as(_dp), ctypes.byref(nc), cap_rows, cap_cols)
    if rows < 0:
        raise RuntimeError("oracle linearisation failed: %d (-1: invalid window, -4: capacity)" % rows)
    n = nc.value
    return r[:rows].copy(), J[:rows * n].reshape(rows, n).copy()


def plus(pb, delta):
    p = pb.struct()
    d = np.ascontiguousarray(delta, np.float64)
    lib().gfo_ba_plus(ctypes.byref(p), d.ctypes.data_as(_dp))


def marginalize_old(pb):
    """MARGIN_OLD: returns the Prior for the next window (block indices already shifted by one frame)."""
    p = pb.struct()
    F = pb.n_frames
    cap = 16 * F + 24
    x0 = np.zeros(cap); J = np.zeros(cap * cap); r = np.zeros(cap)
    out = BaPrior()
    n = lib().gfo_ba_marginalize_old(ctypes.byref(p), ctypes.byref(out), x0.ctypes.data_as(_dp), J.ctypes.data_as(_dp), r.ctypes.data_as(_dp))
    if n <= 0:
        raise RuntimeError("marginalisation failed: %d" % n)
    nb = out.n_blocks
    return Prior(list(out.block_kind)[:nb], list(out.block_index)[:nb], list(out.block_idx)[:nb], x0.copy(), J[:n * n].reshape(n, n).copy(), r[:n].copy())


def marginalize_second_new(pb):
    """MARGIN_SECOND_NEW (estimator.cpp:3536-3631): the last prior with para_Pose[WINDOW_SIZE - 1] (frame n_frames - 2)
    marginalised; None when the prior does not hold that pose (the reference then leaves the prior untouched)."""
    p = pb.struct()
    F = pb.n_frames
    cap = 16 * F + 24
    x0 = np.zeros(cap); J = np.zeros(cap * cap); r = np.zeros(cap)
    out = BaPrior()
    n = lib().gfo_ba_marginalize_second_new(ctypes.byref(p), ctypes.byref(out), x0.ctypes.data_as(_dp), J.ctypes.data_as(_dp), r.ctypes.data_as(_dp))
    if n < 0:
        raise RuntimeError("marginalisation failed: %d" % n)
    if n == 0:
        return None
    nb = out.n_blocks
    return Prior(list(out.block_kind)[:nb], list(out.block_index)[:nb], list(out.block_idx)[:nb], x0.copy(), J[:n * n].reshape(n, n).copy(), r[:n].copy())


def set_tolerances(function=1e-6, gradient=1e-10, parameter=1e-8):
    lib().gfo_ba_set_tolerances(function, gradient, parameter)


def eval_wheel(f, pose_i, pose_j, exw, sx, sy, sw, td, jac=True):
    """WheelFactor::Evaluate restatement: returns (res[6], [J_pose_i 6x7, J_pose_j 6x7, J_ex 6x7, J_sx, J_sy, J_sw, J_td (6,)])."""
    a = [np.ascontiguousarray(v, np.float64) for v in (pose_i, pose_j, exw)]
    res = np.zeros(6)
    Js = [np.zeros((6, 7)), np.zeros((6, 7)), np.zeros((6, 7)), np.zeros(6), np.zeros(6), np.zeros(6), np.zeros(6)]
    ptrs = [j.ctypes.data_as(_dp) if jac else None for j in Js]
    rc = lib().gfo_eval_wheel(ctypes.byref(f), a[0].ctypes.data_as(_dp), a[1].ctypes.data_as(_dp), a[2].ctypes.data_as(_dp),
                              float(sx), float(sy), float(sw), float(td), res.ctypes.data_as(_dp), *ptrs)
    if rc:
        raise RuntimeError("wheel covariance not positive definite")
    return res, Js


def eval_plane(pose_i, exw, qpw, zpw, sinfo, jac=True):
    """PlaneFactor::Evaluate restatement: (res[3], [J_pose 3x7, J_ex 3x7, J_qpw 3x4, J_zpw (3,)])."""
    a = [np.ascontiguousarray(v, np.float64) for v in (pose_i, exw, qpw, sinfo)]
    res = np.zeros(3)
    Js = [np.zeros((3, 7)), np.zeros((3, 7)), np.zeros((3, 4)), np.zeros(3)]
    ptrs = [j.ctypes.data_as(_dp) if jac else None for j in Js]
    lib().gfo_eval_plane(a[0].ctypes.data_as(_dp), a[1].ctypes.data_as(_dp), a[2].ctypes.data_as(_dp), float(zpw), a[3].ctypes.data_as(_dp),
                         res.ctypes.data_as(_dp), *ptrs)
    return res, Js


def sym_eig(A, method="ql"):
    """Eigendecomposition of a symmetric matrix by the oracle's solvers: "jacobi" (cyclic Jacobi, used by marginalize_old) or
    "ql" (Householder tridiagonalisation + implicit QL, the algorithm of the reference's Eigen solver).  Returns (w, V)."""
    A = np.ascontiguousarray(A, np.float64)
    n = A.shape[0]
    w = np.zeros(n); V = np.zeros((n, n))
    lib().gfo_sym_eig(A.ctypes.data_as(_dp), n, w.ctypes.data_as(_dp), V.ctypes.data_as(_dp), 0 if method == "jacobi" else 1)
    return w, V
