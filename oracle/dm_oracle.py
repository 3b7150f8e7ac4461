"""ctypes glue of oracle/dm_oracle.c -- TEST AND MEASUREMENT INFRASTRUCTURE ONLY.

DenseMapOracle has the interface of ground_fusion_b200.dense_map.DenseMap and restates dense_map's colour map one point at a
time (pose_graph_node.cpp:598-623, pose_graph.cpp:191-239 and 997-1058)."""
import ctypes
import os

import numpy as np

_LIB = None
_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "libgf_oracle_dm.so")


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(_PATH)
        vp, i, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
        L.dmo_create.restype = vp
        L.dmo_create.argtypes = [i, i, vp, i, i, vp, vp]
        L.dmo_destroy.argtypes = [vp]
        L.dmo_destroy.restype = None
        L.dmo_add_keyframe.argtypes = [vp, vp, vp, vp, sz, vp, sz, i]
        L.dmo_update_poses.argtypes = [vp, i, vp, vp, i]
        L.dmo_filter.argtypes = [vp]
        L.dmo_filter.restype = None
        L.dmo_size.argtypes = [vp, ctypes.POINTER(i), ctypes.POINTER(i), ctypes.POINTER(i)]
        L.dmo_size.restype = None
        L.dmo_read.argtypes = [vp, vp, vp, vp]
        L.dmo_read.restype = None
        L.dmo_keyframe_points.argtypes = [vp, i, vp]
        L.dmo_radius_filter.argtypes = [vp, i, ctypes.c_double, i, vp]
        L.dmo_radius_filter.restype = None
        L.dmo_anchor.argtypes = [i, vp, vp]
        L.dmo_anchor.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def anchor(rebuild):
    """(min, max) of the octree's box after PCL's recentring: the constructor's box (rebuild=False) or updatePath's."""
    mn, mx = np.zeros(3), np.zeros(3)
    lib().dmo_anchor(int(bool(rebuild)), _p(mn), _p(mx))
    return mn, mx


def radius_filter(xyz, radius=0.8, min_pts=10):
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    keep = np.zeros(len(xyz), np.uint8)
    lib().dmo_radius_filter(_p(xyz), len(xyz), float(radius), int(min_pts), _p(keep))
    return keep.astype(bool)


class DenseMapOracle:
    def __init__(self, width, height, pinhole, depth_dist, depth_boundary, ric, tic):
        self.width, self.height = width, height
        self._m = lib().dmo_create(width, height, _p(np.ascontiguousarray(pinhole, np.float64)), depth_dist, depth_boundary,
                                   _p(np.ascontiguousarray(ric, np.float64).reshape(9)), _p(np.ascontiguousarray(tic, np.float64)))

    def close(self):
        if self._m:
            lib().dmo_destroy(self._m)
            self._m = None

    __del__ = close

    def addKeyFrame(self, R, P, rgb, depth, filter=True):
        """One keyframe; returns the number of points inserted.  filter=False defers the radius filter to filter()."""
        R = np.ascontiguousarray(R, np.float64)
        P = np.ascontiguousarray(P, np.float64)
        rgb = np.ascontiguousarray(rgb, np.uint8)
        depth = np.ascontiguousarray(depth, np.uint16)
        n = lib().dmo_add_keyframe(self._m, _p(R), _p(P), _p(rgb), rgb.strides[0], _p(depth), depth.strides[0], int(filter))
        if n < 0:
            raise ValueError("a point of the keyframe falls outside the octree's bounding box")
        return n

    def filter(self):
        lib().dmo_filter(self._m)

    def updatePath(self, Rs, Ps, filter=True):
        Rs = np.ascontiguousarray(Rs, np.float64)
        Ps = np.ascontiguousarray(Ps, np.float64)
        if lib().dmo_update_poses(self._m, len(Rs), _p(Rs), _p(Ps), int(filter)) < 0:
            raise ValueError("keyframe count differs or a point falls outside the octree's bounding box")

    def size(self):
        a, b, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        lib().dmo_size(self._m, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
        return a.value, b.value, c.value

    def _read(self):
        n = self.size()[0]
        xyz, rgb, keep = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.uint8), np.zeros(n, np.uint8)
        lib().dmo_read(self._m, _p(xyz), _p(rgb), _p(keep))
        return xyz, rgb, keep.astype(bool)

    def cloud(self):
        xyz, rgb, _ = self._read()
        return xyz, rgb

    def filtered(self):
        """(xyz, rgb, idx) of the points the radius filter keeps, idx = their cloud indices."""
        xyz, rgb, keep = self._read()
        idx = np.flatnonzero(keep).astype(np.int32)
        return xyz[idx], rgb[idx], idx

    def keyframePoints(self, k):
        n = lib().dmo_keyframe_points(self._m, k, None)
        if n < 0:
            raise IndexError(k)
        out = np.zeros((n, 6), np.float32)
        lib().dmo_keyframe_points(self._m, k, _p(out))
        return out
