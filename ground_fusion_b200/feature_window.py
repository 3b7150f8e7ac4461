"""FeatureWindow: the reference's FeatureManager (vins_estimator/src/estimator/feature_manager.{h,cpp}) with its landmark table
resident on the GPU (gf_fm_window, csrc/fm_window.cu).

Same method names and return values as feature_manager.FeatureManager, whose lists live in Python: replay() takes either.  On
top of those, addFrameFromTracker ingests the frame a FeatureTracker just returned from where it lies on the device, and
fillProblem writes the visual factors, para_feature and feature_const of a ba_problem.Problem in one device pass.  The table
never crosses to the host except through read().  There is no CPU fallback.
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import OBS_DTYPE, BaVisualFactor, FmWindowCfg, check
from .feature_manager import FOCAL_LENGTH, INIT_DEPTH

_ROWS, _RD = _lib.FM_WINDOW_ROWS, _lib.FM_WINDOW_ROW_DOUBLES


def _poses(Ps, Rs, tic, ric):
    """Ps [11][3], Rs [11][9], tic [3], ric [9] as contiguous doubles (a shorter window is padded with its last pose)."""
    P = np.ascontiguousarray(Ps, np.float64).reshape(-1, 3); R = np.ascontiguousarray(Rs, np.float64).reshape(-1, 9)
    if len(P) < _ROWS:
        P = np.concatenate([P, np.repeat(P[-1:], _ROWS - len(P), 0)]); R = np.concatenate([R, np.repeat(R[-1:], _ROWS - len(R), 0)])
    return (np.ascontiguousarray(P[:_ROWS]), np.ascontiguousarray(R[:_ROWS]), np.ascontiguousarray(tic, np.float64).reshape(3),
            np.ascontiguousarray(ric, np.float64).reshape(9))


class FeatureWindow:
    """Method names and argument meaning as in feature_manager.h:90-150 (and FeatureManager of this package)."""

    def __init__(self, min_parallax_px=10.0, depth_threshold=3.0, window_size=10, device=0, max_features=2048):
        self.L = _lib.lib()
        self.MIN_PARALLAX = min_parallax_px / FOCAL_LENGTH       # parameters.cpp:345-346
        self.depth_threshold = float(depth_threshold)
        self.WINDOW_SIZE = int(window_size)
        self.device, self.max_features = int(device), int(max_features)
        cfg = FmWindowCfg(self.max_features, self.WINDOW_SIZE, self.MIN_PARALLAX, self.depth_threshold, INIT_DEPTH)
        self._h = ctypes.c_void_p()
        check(self.L.gf_fm_window_create(ctypes.byref(self._h), self.device, ctypes.byref(cfg)))
        self.last_track_num = self.new_feature_num = self.long_track_num = 0
        self.last_average_parallax = 0.0
        self._ids = np.zeros(self.max_features, np.int32)
        self._xyz = np.zeros((self.max_features, 3))
        self._feat = np.zeros(self.max_features)
        self._const = np.zeros(self.max_features, np.uint8)
        self._n_upper = 0          # landmarks after the last frame added: removals only lower the count

    def close(self):
        if self._h:
            self.L.gf_fm_window_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def clearState(self):
        check(self.L.gf_fm_window_clear(self._h))
        self._n_upper = 0

    # ---- addFeatureCheckParallax (feature_manager.cpp:57-116) ----
    def _added(self, rc, margin, cnt, par):
        check(rc)
        self.last_track_num, self.new_feature_num, self.long_track_num = int(cnt[0]), int(cnt[1]), int(cnt[2])
        self.last_average_parallax = par.value
        self._n_upper = int(cnt[3])
        return bool(margin.value)

    def addFeatureCheckParallax(self, frame_count, image, td):
        """image: {id: v[8]} as trackImage returns it."""
        obs = np.zeros(len(image), OBS_DTYPE)
        if len(image):
            obs["id"] = list(image.keys())
            obs["v"] = np.asarray(list(image.values()), np.float64)[:, :8]
        return self.addFrame(frame_count, obs, None, td)

    def addFrame(self, frame_count, obs, in_box, td):
        """obs: the structured gf_obs array trackImageRaw / trackImageboxRaw return; in_box: the latter's mask (entries set are left out)."""
        obs = np.ascontiguousarray(obs, OBS_DTYPE)
        ib = None if in_box is None else np.ascontiguousarray(in_box, np.uint8)
        margin, cnt, par = ctypes.c_int(0), np.zeros(4, np.int32), ctypes.c_double(0)
        rc = self.L.gf_fm_window_add_frame(self._h, int(frame_count), obs.ctypes.data if len(obs) else None, len(obs),
                                           ib.ctypes.data if ib is not None and len(ib) else None, float(td), ctypes.byref(margin), cnt.ctypes.data,
                                           ctypes.byref(par))
        return self._added(rc, margin, cnt, par)

    def addFrameFromTracker(self, tracker, frame_count, td):
        """addFeatureCheckParallax with the frame `tracker` (a FeatureTracker) returned last, read on the device."""
        margin, cnt, par = ctypes.c_int(0), np.zeros(4, np.int32), ctypes.c_double(0)
        rc = self.L.gf_fm_window_add_frame_from_tracker(self._h, tracker._h, int(frame_count), float(td), ctypes.byref(margin), cnt.ctypes.data,
                                                        ctypes.byref(par))
        return self._added(rc, margin, cnt, par)

    # ---- the solve's view of the table ----
    def fillProblem(self, pb):
        """The factor loop of Estimator::optimization (estimator.cpp:3268-3297): pb.visual / n_visual, pb.para_feature,
        pb.feature_const and pb.n_features from the landmarks with >= 4 observations.  Returns n_features."""
        nv, nf = ctypes.c_int(0), ctypes.c_int(0)
        cap = max(self._n_upper * self.WINDOW_SIZE, 1)
        pb.visual = (BaVisualFactor * cap)()            # the rows land here directly; pb.n_visual says how many count
        check(self.L.gf_fm_window_fill_problem(self._h, pb.visual, cap, ctypes.byref(nv), self._feat.ctypes.data, self._const.ctypes.data, ctypes.byref(nf)))
        n = nf.value
        pb.n_features, pb.n_visual = n, nv.value
        pb.para_feature = np.ones(max(n, 1)); pb.para_feature[:n] = self._feat[:n]
        pb.feature_const = np.zeros(max(n, 1), np.uint8); pb.feature_const[:n] = self._const[:n]
        return n

    def getDepthVector(self):
        nf = ctypes.c_int(0)
        check(self.L.gf_fm_window_fill_problem(self._h, None, 0, None, self._feat.ctypes.data, None, ctypes.byref(nf)))
        return self._feat[:nf.value].copy()

    def getFeatureCount(self):
        return len(self.getDepthVector())

    def setDepth(self, x):
        x = np.ascontiguousarray(x, np.float64)
        check(self.L.gf_fm_window_set_depth(self._h, x.ctypes.data if len(x) else None, len(x)))

    def iter_ba_features(self):
        """As FeatureManager.iter_ba_features, from a read() of the table (fillProblem is the path that stays on the device)."""
        for it in self.read():
            if it["n_obs"] >= 4:
                o = it["obs"]
                yield it["start_frame"], [(r[0:3], r[5:7], r[8]) for r in o], it["estimated_depth"], it["estimate_flag"]

    def triangulateAll(self, frameCnt, Ps, Rs, tic, ric):
        P, R, t, r = _poses(Ps, Rs, tic, ric)
        check(self.L.gf_fm_window_triangulate(self._h, int(frameCnt), P.ctypes.data, R.ctypes.data, t.ctypes.data, r.ctypes.data))

    def clearDepth(self):
        check(self.L.gf_fm_window_clear_depth(self._h))

    # ---- removals ----
    def removeFailures(self):
        check(self.L.gf_fm_window_remove_failures(self._h))

    def removeOutlier(self, outlierIndex):
        ids = np.array(sorted(outlierIndex), np.int32)
        check(self.L.gf_fm_window_remove_ids(self._h, ids.ctypes.data if len(ids) else None, len(ids)))

    def removeBackShiftDepth(self, marg_R, marg_P, new_R, new_P):
        a = [np.ascontiguousarray(v, np.float64).ravel() for v in (marg_R, marg_P, new_R, new_P)]
        check(self.L.gf_fm_window_remove_back_shift_depth(self._h, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, a[3].ctypes.data))

    def removeBack(self):
        check(self.L.gf_fm_window_remove_back(self._h))

    def removeFront(self, frame_count):
        check(self.L.gf_fm_window_remove_front(self._h, int(frame_count)))

    # ---- the loops that feed the front end back (estimator.cpp:3853-4011) ----
    def _outliers(self, Ps, Rs, tic, ric, mode):
        P, R, t, r = _poses(Ps, Rs, tic, ric)
        n = ctypes.c_int(0)
        check(self.L.gf_fm_window_outliers(self._h, P.ctypes.data, R.ctypes.data, t.ctypes.data, r.ctypes.data, mode, self._ids.ctypes.data, ctypes.byref(n)))
        self.last_outlier_ids = [int(v) for v in self._ids[:n.value]]       # list order
        return set(self.last_outlier_ids)

    def outliersRejection(self, Ps, Rs, tic, ric):
        return self._outliers(Ps, Rs, tic, ric, _lib.FM_OUTLIERS_REPROJECTION)

    def movingConsistencyCheckW(self, Ps, Rs, tic, ric):
        return self._outliers(Ps, Rs, tic, ric, _lib.FM_OUTLIERS_MOVING)

    def predictPtsInNextFrame(self, frame_count, Ps, Rs, tic, ric):
        P, R, t, r = _poses(Ps, Rs, tic, ric)
        n = ctypes.c_int(0)
        check(self.L.gf_fm_window_predict_next(self._h, int(frame_count), P.ctypes.data, R.ctypes.data, t.ctypes.data, r.ctypes.data, self._ids.ctypes.data,
                                               self._xyz.ctypes.data, ctypes.byref(n)))
        return {int(self._ids[k]): self._xyz[k].copy() for k in range(n.value)}

    # ---- the table on the host ----
    def size(self):
        n = ctypes.c_int(0)
        check(self.L.gf_fm_window_size(self._h, ctypes.byref(n)))
        return n.value

    def read(self):
        """The table in list order: dicts with feature_id, start_frame, n_obs, estimated_depth, estimate_flag, solve_flag and
        obs ((n_obs, 9) rows [x y z u v vx vy depth td])."""
        c = max(self._n_upper, 1)
        ints = [np.zeros(c, np.int32) for _ in range(5)]
        est = np.zeros(c); obs = np.zeros((c, _ROWS, _RD))
        n = ctypes.c_int(0)
        check(self.L.gf_fm_window_read(self._h, ints[0].ctypes.data, ints[1].ctypes.data, ints[2].ctypes.data, est.ctypes.data, ints[3].ctypes.data,
                                       ints[4].ctypes.data, obs.ctypes.data, c, ctypes.byref(n)))
        return [dict(feature_id=int(ints[0][i]), start_frame=int(ints[1][i]), n_obs=int(ints[2][i]), estimated_depth=float(est[i]),
                     estimate_flag=int(ints[3][i]), solve_flag=int(ints[4][i]), obs=obs[i, :ints[2][i]].copy()) for i in range(n.value)]

    def last_device_ms(self):
        ms = ctypes.c_float(0)
        check(self.L.gf_fm_window_last_device_ms(self._h, ctypes.byref(ms)))
        return ms.value


def _stack_poses(poses):
    """[(Ps, Rs, tic, ric)] per member -> contiguous [K][11][3], [K][11][9], [K][3], [K][9]"""
    p = [_poses(*x) for x in poses]
    return tuple(np.ascontiguousarray(np.stack([q[j] for q in p])) for j in range(4))


def _ptrs(arrays):
    return (ctypes.c_void_p * len(arrays))(*[a.ctypes.data if a is not None else None for a in arrays])


class FeatureWindowGroup:
    """gf_fm_window_group: the FeatureManager calls of several FeatureWindows (one per estimator) with one set of kernel
    launches per call.  Every method takes and returns per-member lists, and every member's results, table and Python-side
    caches are what the same FeatureWindow method would give, so the members stay usable on their own between group calls."""

    def __init__(self, windows):
        self.members = list(windows)
        self.L = _lib.lib()
        self._h = ctypes.c_void_p()
        h = (ctypes.c_void_p * len(self.members))(*[w._h for w in self.members])
        check(self.L.gf_fm_window_group_create(ctypes.byref(self._h), h, len(self.members)))
        self.K = len(self.members)
        self.last_status = np.zeros(self.K, np.int32)

    def close(self):
        if self._h:
            self.L.gf_fm_window_group_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- addFeatureCheckParallax ----
    def _added(self, rc, margin, cnt, par, status):
        self.last_status = status
        for i, w in enumerate(self.members):
            if status[i] == 0:
                w.last_track_num, w.new_feature_num, w.long_track_num = int(cnt[i, 0]), int(cnt[i, 1]), int(cnt[i, 2])
                w.last_average_parallax = float(par[i])
                w._n_upper = int(cnt[i, 3])
        check(rc)
        return [bool(m) for m in margin]

    def _out(self):
        # status starts non-zero: an argument error returns before the library writes it, and then no member changed
        return np.zeros(self.K, np.int32), np.zeros((self.K, 4), np.int32), np.zeros(self.K), np.ones(self.K, np.int32)

    def addFrames(self, frame_counts, obs, in_box, tds):
        """obs / in_box: per member the arrays FeatureWindow.addFrame takes (in_box None: no boxes).  Returns the keyframe flags.
        A member that fails on the device raises after the others are applied; last_status says which."""
        obs = [np.ascontiguousarray(o, OBS_DTYPE) for o in obs]
        start = np.zeros(self.K + 1, np.int32); start[1:] = np.cumsum([len(o) for o in obs])
        allo = np.ascontiguousarray(np.concatenate(obs) if start[-1] else np.zeros(1, OBS_DTYPE))
        ib = None
        if in_box is not None:
            ib = np.ascontiguousarray(np.concatenate([np.zeros(len(o), np.uint8) if b is None else np.asarray(b, np.uint8)
                                                      for o, b in zip(obs, in_box)]) if start[-1] else np.zeros(1, np.uint8))
        fc, td = np.asarray(frame_counts, np.int32), np.asarray(tds, np.float64)
        margin, cnt, par, st = self._out()
        rc = self.L.gf_fm_window_group_add_frame(self._h, fc.ctypes.data, allo.ctypes.data, start.ctypes.data, ib.ctypes.data if ib is not None else None,
                                                 td.ctypes.data, margin.ctypes.data, cnt.ctypes.data, par.ctypes.data, st.ctypes.data)
        return self._added(rc, margin, cnt, par, st)

    def addFeatureCheckParallaxes(self, frame_counts, images, tds):
        obs = []
        for image in images:
            o = np.zeros(len(image), OBS_DTYPE)
            if len(image):
                o["id"] = list(image.keys()); o["v"] = np.asarray(list(image.values()), np.float64)[:, :8]
            obs.append(o)
        return self.addFrames(frame_counts, obs, None, tds)

    def addFramesFromTrackerGroup(self, group, frame_counts, tds):
        """Member i ingests member i of `group` (a TrackerGroup) from the step group.wait() returned last, on the device."""
        fc, td = np.asarray(frame_counts, np.int32), np.asarray(tds, np.float64)
        margin, cnt, par, st = self._out()
        rc = self.L.gf_fm_window_group_add_frame_from_tracker_group(self._h, group._h, fc.ctypes.data, td.ctypes.data, margin.ctypes.data,
                                                                    cnt.ctypes.data, par.ctypes.data, st.ctypes.data)
        return self._added(rc, margin, cnt, par, st)

    # ---- the solve's view ----
    def fillProblems(self, problems):
        """FeatureWindow.fillProblem for every member into problems[i]; returns the n_features."""
        caps = np.array([max(w._n_upper * w.WINDOW_SIZE, 1) for w in self.members], np.int32)
        for pb, c in zip(problems, caps):
            pb.visual = (BaVisualFactor * int(c))()
        vis = (ctypes.c_void_p * self.K)(*[ctypes.addressof(pb.visual) for pb in problems])
        nv, nf, st = np.zeros(self.K, np.int32), np.zeros(self.K, np.int32), np.zeros(self.K, np.int32)
        rc = self.L.gf_fm_window_group_fill_problem(self._h, vis, caps.ctypes.data, nv.ctypes.data, _ptrs([w._feat for w in self.members]),
                                                    _ptrs([w._const for w in self.members]), nf.ctypes.data, st.ctypes.data)
        self.last_status = st
        check(rc)
        for w, pb, n, v in zip(self.members, problems, nf, nv):
            n = int(n)
            pb.n_features, pb.n_visual = n, int(v)
            pb.para_feature = np.ones(max(n, 1)); pb.para_feature[:n] = w._feat[:n]
            pb.feature_const = np.zeros(max(n, 1), np.uint8); pb.feature_const[:n] = w._const[:n]
        return [int(n) for n in nf]

    def setDepths(self, xs):
        xs = [np.ascontiguousarray(x, np.float64) for x in xs]
        n = np.array([len(x) for x in xs], np.int32)
        check(self.L.gf_fm_window_group_set_depth(self._h, _ptrs([x if len(x) else None for x in xs]), n.ctypes.data))

    def triangulateAll(self, frame_counts, poses):
        """poses: per member (Ps, Rs, tic, ric)"""
        P, R, t, r = _stack_poses(poses)
        fc = np.asarray(frame_counts, np.int32)
        check(self.L.gf_fm_window_group_triangulate(self._h, fc.ctypes.data, P.ctypes.data, R.ctypes.data, t.ctypes.data, r.ctypes.data))

    def clearDepth(self):
        check(self.L.gf_fm_window_group_clear_depth(self._h))

    # ---- removals ----
    def removeFailures(self):
        check(self.L.gf_fm_window_group_remove_failures(self._h))

    def removeOutliers(self, outlier_sets):
        ids = [np.array(sorted(s), np.int32) for s in outlier_sets]
        start = np.zeros(self.K + 1, np.int32); start[1:] = np.cumsum([len(x) for x in ids])
        allids = np.ascontiguousarray(np.concatenate(ids) if start[-1] else np.zeros(1, np.int32))
        check(self.L.gf_fm_window_group_remove_ids(self._h, allids.ctypes.data, start.ctypes.data))

    def remove(self, ops, frame_counts, shifts=None):
        """ops[i]: _lib.FM_REMOVE_*; frame_counts[i]: the member's frame_count (WINDOW_SIZE for FM_REMOVE_FRONT); shifts[i]:
        (marg_R, marg_P, new_R, new_P) for FM_REMOVE_BACK_SHIFT_DEPTH members (else None)."""
        op, fc = np.asarray(ops, np.int32), np.asarray(frame_counts, np.int32)
        sh = np.zeros((self.K, 24))
        if shifts is not None:
            for i, s in enumerate(shifts):
                if s is not None:
                    sh[i] = np.concatenate([np.ascontiguousarray(v, np.float64).ravel() for v in s])
        check(self.L.gf_fm_window_group_remove(self._h, op.ctypes.data, fc.ctypes.data, sh.ctypes.data))

    # ---- the loops that feed the front ends back ----
    def _outliers(self, poses, mode):
        P, R, t, r = _stack_poses(poses)
        n = np.zeros(self.K, np.int32)
        check(self.L.gf_fm_window_group_outliers(self._h, P.ctypes.data, R.ctypes.data, t.ctypes.data, r.ctypes.data, mode,
                                                 _ptrs([w._ids for w in self.members]), n.ctypes.data))
        out = []
        for w, k in zip(self.members, n):
            w.last_outlier_ids = [int(v) for v in w._ids[:k]]
            out.append(set(w.last_outlier_ids))
        return out

    def outliersRejections(self, poses):
        return self._outliers(poses, _lib.FM_OUTLIERS_REPROJECTION)

    def movingConsistencyCheckW(self, poses):
        return self._outliers(poses, _lib.FM_OUTLIERS_MOVING)

    def predictPtsInNextFrame(self, frame_counts, poses):
        P, R, t, r = _stack_poses(poses)
        fc, n = np.asarray(frame_counts, np.int32), np.zeros(self.K, np.int32)
        check(self.L.gf_fm_window_group_predict_next(self._h, fc.ctypes.data, P.ctypes.data, R.ctypes.data, t.ctypes.data, r.ctypes.data,
                                                     _ptrs([w._ids for w in self.members]), _ptrs([w._xyz for w in self.members]),
                                                     n.ctypes.data))
        return [{int(w._ids[k]): w._xyz[k].copy() for k in range(m)} for w, m in zip(self.members, n)]

    def last_device_ms(self):
        ms = ctypes.c_float(0)
        check(self.L.gf_fm_window_group_last_device_ms(self._h, ctypes.byref(ms)))
        return ms.value
