"""ctypes glue of oracle/gm_oracle.c -- TEST AND MEASUREMENT INFRASTRUCTURE ONLY.

GridMapOracle has the interface of ground_fusion_b200.grid_map.GridMap and restates the grid_mapping tool one point and one ray
step at a time.  mode "libm": the tool's arithmetic (this host's log / exp); mode "shared": the log / exp of
ground_fusion_b200/csrc/gm_math.h, which the GPU grid uses."""
import ctypes
import os

import numpy as np

_LIB = None
_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "libgf_oracle_gm.so")


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(_PATH)
        vp, i, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
        L.gmo_create.restype = vp
        L.gmo_create.argtypes = [i, i, i, i, d, d, d, d, vp, vp, i]
        L.gmo_destroy.argtypes = [vp]
        L.gmo_destroy.restype = None
        L.gmo_add_keyframe.argtypes = [vp, vp, vp, vp, i, i]
        L.gmo_update_poses.argtypes = [vp, i, vp, vp]
        L.gmo_n_keyframes.argtypes = [vp]
        for f in (L.gmo_read_bel, L.gmo_image, L.gmo_occupancy):
            f.argtypes = [vp, vp]
            f.restype = None
        L.gmo_log.argtypes = L.gmo_exp.argtypes = [d]
        L.gmo_log.restype = L.gmo_exp.restype = d
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def shared_log(x):
    """gm_math.h's log of one double."""
    return lib().gmo_log(float(x))


def shared_exp(x):
    return lib().gmo_exp(float(x))


class GridMapOracle:
    def __init__(self, ric=np.eye(3), tic=np.zeros(3), size_x=1500, size_y=500, init_x=750, init_y=250, cell_size=0.05, p_occ=0.6,
                 p_free=0.4, p_prior=0.5, mode="shared"):
        if mode not in ("libm", "shared"):
            raise ValueError("mode is 'libm' or 'shared'")
        self.sx, self.sy = size_x, size_y
        self._m = lib().gmo_create(size_x, size_y, init_x, init_y, float(cell_size), float(p_occ), float(p_free), float(p_prior),
                                   _p(np.ascontiguousarray(ric, np.float64).reshape(9)), _p(np.ascontiguousarray(tic, np.float64).reshape(3)),
                                   int(mode == "shared"))

    def close(self):
        if self._m:
            lib().gmo_destroy(self._m)
            self._m = None

    __del__ = close

    def addKeyFrame(self, R, P, points):
        R = np.ascontiguousarray(R, np.float64).reshape(9)
        P = np.ascontiguousarray(P, np.float64).reshape(3)
        points = np.ascontiguousarray(points, np.float32)
        points = points.reshape(len(points), -1)
        lib().gmo_add_keyframe(self._m, _p(R), _p(P), _p(points), len(points), points.shape[1] if len(points) else 3)

    def updatePath(self, Rs, Ps):
        Rs = np.ascontiguousarray(Rs, np.float64).reshape(-1, 9)
        Ps = np.ascontiguousarray(Ps, np.float64).reshape(-1, 3)
        if lib().gmo_update_poses(self._m, len(Rs), _p(Rs), _p(Ps)) < 0:
            raise ValueError("keyframe count differs")

    def size(self):
        return self.sx, self.sy, lib().gmo_n_keyframes(self._m)

    def bel(self):
        out = np.zeros((self.sy, self.sx), np.float64)
        lib().gmo_read_bel(self._m, _p(out))
        return out.T

    def image(self):
        out = np.zeros((self.sx, self.sy), np.uint8)
        lib().gmo_image(self._m, _p(out))
        return out

    def occupancy(self):
        out = np.zeros(self.sx * self.sy, np.int8)
        lib().gmo_occupancy(self._m, _p(out))
        return out
