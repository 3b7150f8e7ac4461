"""Dense colour map on the GPU: the keyframe point map of the reference's dense_map node (PoseGraph's octree blocks,
dense_map/src/pose_graph.cpp:191-239 and 997-1058, fed by the node's sampling loop, pose_graph_node.cpp:598-623).

DenseMap wraps gf_dense_map_* (include/gf_b200.h); method names follow the reference.  There is no CPU fallback."""
import ctypes

import numpy as np

from . import _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class DenseMap:
    """width, height, pinhole (fx fy cx cy k1 k2 p1 p2): cam0_calib; depth_dist / depth_boundary: DEPTH_DIST / DEPTH_BOUNDARY;
    ric (3x3), tic (3): camera to body.  max_points bounds the points all keyframes keep together, max_keyframes the keyframes."""

    def __init__(self, width, height, pinhole, depth_dist=10, depth_boundary=10, ric=np.eye(3), tic=np.zeros(3),
                 max_points=1 << 20, max_keyframes=4096, device=0):
        cfg = _lib.DenseMapCfg()
        cfg.width, cfg.height, cfg.depth_dist, cfg.depth_boundary = width, height, depth_dist, depth_boundary
        cfg.pinhole[:] = [float(v) for v in pinhole]
        cfg.ric[:] = [float(v) for v in np.asarray(ric, float).reshape(9)]
        cfg.tic[:] = [float(v) for v in np.asarray(tic, float).reshape(3)]
        cfg.max_points, cfg.max_keyframes = max_points, max_keyframes
        self.width, self.height = width, height
        self._m = ctypes.c_void_p()
        _lib.check(_lib.lib().gf_dense_map_create(ctypes.byref(self._m), device, ctypes.byref(cfg)))

    def close(self):
        if self._m:
            _lib.lib().gf_dense_map_destroy(self._m)
            self._m = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _frame(self, rgb, depth):
        """(rgb pointer, rgb pitch, depth pointer, depth pitch, on_device) of a frame addKeyFrame takes."""
        h, w = self.height, self.width
        if tuple(rgb.shape) != (h, w, 3) or tuple(depth.shape) != (h, w):
            raise ValueError("rgb must be (%d, %d, 3) and depth (%d, %d)" % (h, w, h, w))
        if hasattr(rgb, "is_cuda") and rgb.is_cuda:
            import torch
            if rgb.dtype != torch.uint8 or depth.dtype not in (torch.int16, torch.uint16) or not depth.is_cuda:
                raise ValueError("CUDA frames: rgb uint8, depth int16 / uint16 (the millimetres' bits), both on the device")
            if rgb.stride(2) != 1 or rgb.stride(1) != 3 or depth.stride(1) != 1:
                raise ValueError("rows must be packed pixels")
            return ctypes.c_void_p(rgb.data_ptr()), rgb.stride(0), ctypes.c_void_p(depth.data_ptr()), depth.stride(0) * 2, 1
        if rgb.dtype != np.uint8 or depth.dtype != np.uint16:
            raise ValueError("rgb must be uint8 and depth uint16")
        if rgb.strides[1:] != (3, 1) or depth.strides[1] != 2:
            raise ValueError("rows must be packed pixels")
        return _p(rgb), rgb.strides[0], _p(depth), depth.strides[0], 0

    def addKeyFrame(self, R, P, rgb, depth):
        """One keyframe with body pose (R, P): rgb (H, W, 3) uint8 and depth (H, W) uint16 millimetres, numpy arrays (rows may be
        padded) or CUDA tensors.  Returns the number of points inserted."""
        R = np.ascontiguousarray(R, np.float64).reshape(9)
        P = np.ascontiguousarray(P, np.float64).reshape(3)
        n = ctypes.c_int()
        args = self._frame(rgb, depth)
        _lib.check(_lib.lib().gf_dense_map_add_keyframe(self._m, _p(R), _p(P), *args, ctypes.byref(n)))
        return n.value

    def updatePath(self, Rs, Ps):
        """The rebuild after a pose-graph correction: Rs (n, 3, 3), Ps (n, 3), one pose per keyframe added."""
        Rs = np.ascontiguousarray(Rs, np.float64).reshape(-1, 9)
        Ps = np.ascontiguousarray(Ps, np.float64).reshape(-1, 3)
        if len(Rs) != len(Ps):
            raise ValueError("Rs and Ps differ in length")
        _lib.check(_lib.lib().gf_dense_map_update_poses(self._m, len(Rs), _p(Rs), _p(Ps)))

    def size(self):
        """(points in the cloud, points the filter keeps, keyframes)."""
        a, b, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        _lib.check(_lib.lib().gf_dense_map_size(self._m, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
        return a.value, b.value, c.value

    def _read(self, which, n):
        xyz, rgb, idx = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.uint8), np.zeros(n, np.int32)
        _lib.check(_lib.lib().gf_dense_map_read(self._m, which, _p(xyz), _p(rgb), _p(idx)))
        return xyz, rgb, idx

    def cloud(self):
        """(xyz float32 (n, 3), rgb uint8 (n, 3)) of the accumulated cloud, in insertion order."""
        xyz, rgb, _ = self._read(_lib.DENSE_MAP_CLOUD, self.size()[0])
        return xyz, rgb

    def filtered(self):
        """(xyz, rgb, idx) of the points RadiusOutlierRemoval keeps, in cloud order; idx = their indices in cloud()."""
        return self._read(_lib.DENSE_MAP_FILTERED, self.size()[1])

    def keyframePoints(self, k):
        """Keyframe k's kept points (KeyFrame::point_rgbd): float32 (n, 6), camera-frame x y z and r g b."""
        n = ctypes.c_int()
        _lib.check(_lib.lib().gf_dense_map_keyframe_points(self._m, k, None, ctypes.byref(n)))
        out = np.zeros((n.value, 6), np.float32)
        _lib.check(_lib.lib().gf_dense_map_keyframe_points(self._m, k, _p(out), ctypes.byref(n)))
        return out


def _members(members, K):
    """members as int32, checked on the host: distinct indices in [0, K), at least one."""
    mb = np.ascontiguousarray(members, np.int32).reshape(-1)
    if len(mb) == 0:
        raise ValueError("no member given")
    if mb.min() < 0 or mb.max() >= K:
        raise ValueError("member index out of range [0, %d)" % K)
    if len(np.unique(mb)) != len(mb):
        raise ValueError("a member is listed twice")
    return mb


def _poses(Rs, Ps, m):
    Rs = np.ascontiguousarray(Rs, np.float64).reshape(-1, 9)
    Ps = np.ascontiguousarray(Ps, np.float64).reshape(-1, 3)
    if len(Rs) != m or len(Ps) != m:
        raise ValueError("one pose per member: Rs (m, 3, 3), Ps (m, 3)")
    return Rs, Ps


class DenseMapGroup:
    """gf_dense_map_group: one keyframe for each of several DenseMaps (one per estimator) with one launch chain and one host
    synchronisation per call.  Every member's map afterwards is bit-equal to the same DenseMap.addKeyFrame on it alone; the maps
    stay usable on their own between group calls.  The maps must share width, height, depth_dist and depth_boundary."""

    def __init__(self, maps):
        self.members = list(maps)
        self.K = len(self.members)
        self._h = ctypes.c_void_p()
        h = (ctypes.c_void_p * self.K)(*[m._m for m in self.members])
        _lib.check(_lib.lib().gf_dense_map_group_create(ctypes.byref(self._h), h, self.K))

    def close(self):
        if self._h:
            _lib.lib().gf_dense_map_group_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def addKeyFrames(self, members, Rs, Ps, rgbs, depths):
        """Member members[j] takes pose (Rs[j], Ps[j]) and frame (rgbs[j], depths[j]), as DenseMap.addKeyFrame takes them (all
        numpy or all CUDA).  Returns (points inserted, status) per entry: status[j] is 0 or the error code the single call
        would have raised for that member, which is then unchanged.  Argument errors raise and change nothing."""
        mb = _members(members, self.K)
        m = len(mb)
        Rs, Ps = _poses(Rs, Ps, m)
        if len(rgbs) != m or len(depths) != m:
            raise ValueError("one frame per member")
        fr = [self.members[k]._frame(r, d) for k, r, d in zip(mb, rgbs, depths)]
        if len({f[4] for f in fr}) != 1:
            raise ValueError("frames must be all host arrays or all CUDA tensors")
        vp = ctypes.c_void_p * m
        rgb, dep = vp(*[f[0] for f in fr]), vp(*[f[2] for f in fr])
        rp, dp = np.array([f[1] for f in fr], np.uint64), np.array([f[3] for f in fr], np.uint64)
        n, st = np.zeros(m, np.int32), np.zeros(m, np.int32)
        rc = _lib.lib().gf_dense_map_group_add_keyframes(self._h, _p(mb), m, _p(Rs), _p(Ps), rgb, _p(rp), dep, _p(dp), fr[0][4], _p(n), _p(st))
        if rc != 0 and not st.any():                  # per-member failures are reported in st; anything else changed nothing
            _lib.check(rc)
        return n, st


def radius_filter(xyz, radius=0.8, min_pts=10, device=0):
    """The map's radius filter over any float32 point set (gf_stage_radius_filter): bool keep mask."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    keep = np.zeros(len(xyz), np.uint8)
    _lib.check(_lib.lib().gf_stage_radius_filter(device, _p(xyz), len(xyz), float(radius), int(min_pts), _p(keep)))
    return keep.astype(bool)
