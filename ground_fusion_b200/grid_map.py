"""Occupancy grid on the GPU: the 2-D log-odds grid of the reference's grid_mapping tool (support_files/grid_mapping: main.cpp,
grid_mapper.cpp, grid_map.cpp), built online from the dense map's keyframe points and rebuilt after a pose correction.

GridMap wraps gf_grid_map_* (include/gf_b200.h).  There is no CPU fallback."""
import ctypes

import numpy as np

from . import _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _points(points):
    """(pointer, n, stride in floats, on_device, the array kept alive) of the points addKeyFrame takes."""
    if hasattr(points, "is_cuda") and points.is_cuda:
        import torch
        if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] < 3 or (len(points) and points.stride(1) != 1):
            raise ValueError("points must be float32 (n, >= 3) with packed rows")
        n, stride = points.shape[0], (points.stride(0) if len(points) > 1 else points.shape[1])
        return ctypes.c_void_p(points.data_ptr()), n, stride, 1, points
    points = np.asarray(points)
    if points.dtype != np.float32 or points.ndim != 2 or points.shape[1] < 3:
        raise ValueError("points must be float32 (n, >= 3)")
    points = np.ascontiguousarray(points)
    return _p(points), len(points), points.shape[1], 0, points


class GridMap:
    """ric (3x3), tic (3): camera to body.  The grid has size_x x size_y cells of cell_size metres, world (0, 0) in cell
    (init_x, init_y); p_occ / p_free / p_prior: the inverse sensor model.  Defaults are the tool's.  max_points bounds the points
    of all keyframes together, max_keyframes the keyframes, max_records the ray steps sorted at once (more are processed in
    chunks)."""

    def __init__(self, ric=np.eye(3), tic=np.zeros(3), size_x=1500, size_y=500, init_x=750, init_y=250, cell_size=0.05, p_occ=0.6,
                 p_free=0.4, p_prior=0.5, max_points=1 << 22, max_keyframes=8192, max_records=1 << 24, device=0):
        cfg = _lib.GridMapCfg()
        cfg.size_x, cfg.size_y, cfg.init_x, cfg.init_y = size_x, size_y, init_x, init_y
        cfg.cell_size, cfg.p_occ, cfg.p_free, cfg.p_prior = cell_size, p_occ, p_free, p_prior
        cfg.ric[:] = [float(v) for v in np.asarray(ric, float).reshape(9)]
        cfg.tic[:] = [float(v) for v in np.asarray(tic, float).reshape(3)]
        cfg.max_points, cfg.max_keyframes, cfg.max_records = max_points, max_keyframes, max_records
        self._m = ctypes.c_void_p()
        _lib.check(_lib.lib().gf_grid_map_create(ctypes.byref(self._m), device, ctypes.byref(cfg)))

    def close(self):
        if self._m:
            _lib.lib().gf_grid_map_destroy(self._m)
            self._m = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def addKeyFrame(self, R, P, points):
        """One keyframe with body pose (R, P): points (n, >= 3) float32 camera-frame x y z first -- keyframePoints' (n, 6) rows as
        they are -- a numpy array or a CUDA tensor."""
        R = np.ascontiguousarray(R, np.float64).reshape(9)
        P = np.ascontiguousarray(P, np.float64).reshape(3)
        ptr, n, stride, on_device, _ = _points(points)
        _lib.check(_lib.lib().gf_grid_map_add_keyframe(self._m, _p(R), _p(P), ptr, n, stride, on_device))

    def updatePath(self, Rs, Ps):
        """The rebuild after a pose correction: Rs (n, 3, 3), Ps (n, 3), one pose per keyframe added."""
        Rs = np.ascontiguousarray(Rs, np.float64).reshape(-1, 9)
        Ps = np.ascontiguousarray(Ps, np.float64).reshape(-1, 3)
        if len(Rs) != len(Ps):
            raise ValueError("Rs and Ps differ in length")
        _lib.check(_lib.lib().gf_grid_map_update_poses(self._m, len(Rs), _p(Rs), _p(Ps)))

    def size(self):
        """(size_x, size_y, keyframes, points)."""
        v = [ctypes.c_int() for _ in range(4)]
        _lib.check(_lib.lib().gf_grid_map_size(self._m, *[ctypes.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def _read(self, which, dtype, shape):
        out = np.zeros(shape, dtype)
        _lib.check(_lib.lib().gf_grid_map_read(self._m, which, _p(out)))
        return out

    def bel(self):
        """float64 (size_x, size_y): bel(x, y), the tool's Eigen matrix."""
        sx, sy = self.size()[:2]
        return self._read(_lib.GRID_MAP_BEL, np.float64, (sy, sx)).T

    def image(self):
        """uint8 (size_x, size_y): the pixels GridMap::saveMap writes to map.png."""
        sx, sy = self.size()[:2]
        return self._read(_lib.GRID_MAP_IMAGE, np.uint8, (sx, sy))

    def occupancy(self):
        """int8 (size_x * size_y,): the OccupancyGrid data the mapping node publishes from that image, cell (x, y) at x + size_x * y."""
        sx, sy = self.size()[:2]
        return self._read(_lib.GRID_MAP_OCCUPANCY, np.int8, sx * sy)

    def stats(self):
        """Of the last call: dict(records, applied, skipped, longest_run)."""
        out = np.zeros(4, np.int64)
        _lib.check(_lib.lib().gf_grid_map_stats(self._m, _p(out)))
        return dict(zip(("records", "applied", "skipped", "longest_run"), (int(v) for v in out)))


class GridMapGroup:
    """gf_grid_map_group: one keyframe for each of several GridMaps with one launch chain per call.  Every member's grid afterwards
    is bit-equal to the same GridMap.addKeyFrame on it alone; the grids stay usable on their own between group calls."""

    def __init__(self, grids):
        self.members = list(grids)
        self.K = len(self.members)
        self._h = ctypes.c_void_p()
        h = (ctypes.c_void_p * self.K)(*[g._m for g in self.members])
        _lib.check(_lib.lib().gf_grid_map_group_create(ctypes.byref(self._h), h, self.K))

    def close(self):
        if self._h:
            _lib.lib().gf_grid_map_group_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _done(rc, st):
        if rc != 0 and not st.any():                  # per-member failures are reported in st; anything else changed nothing
            _lib.check(rc)
        return st

    def addKeyFrames(self, members, Rs, Ps, points):
        """Member members[j] takes pose (Rs[j], Ps[j]) and points[j] as GridMap.addKeyFrame takes them (all numpy or all CUDA).
        Returns the status per entry: 0, or the error code the single call would have raised (the member is then unchanged)."""
        from .dense_map import _members, _poses
        mb = _members(members, self.K)
        m = len(mb)
        Rs, Ps = _poses(Rs, Ps, m)
        if len(points) != m:
            raise ValueError("one point set per member")
        pp = [_points(x) for x in points]
        if len({x[3] for x in pp}) != 1:
            raise ValueError("points must be all host arrays or all CUDA tensors")
        ptrs = (ctypes.c_void_p * m)(*[x[0] for x in pp])
        n, stride = np.array([x[1] for x in pp], np.int32), np.array([x[2] for x in pp], np.int32)
        st = np.zeros(m, np.int32)
        rc = _lib.lib().gf_grid_map_group_add_keyframes(self._h, _p(mb), m, _p(Rs), _p(Ps), ptrs, _p(n), _p(stride), pp[0][3], _p(st))
        return self._done(rc, st)

    def addDenseKeyFrames(self, dense_group, members, Rs, Ps):
        """Member k takes the keyframe that member k of dense_group (a DenseMapGroup) added last, read on the device, with pose
        (Rs[j], Ps[j]) for k = members[j].  Returns the status per entry, as addKeyFrames."""
        from .dense_map import _members, _poses
        mb = _members(members, self.K)
        m = len(mb)
        Rs, Ps = _poses(Rs, Ps, m)
        st = np.zeros(m, np.int32)
        rc = _lib.lib().gf_grid_map_group_add_dense_keyframes(self._h, dense_group._h, _p(mb), m, _p(Rs), _p(Ps), _p(st))
        return self._done(rc, st)
