"""Host-side mirror of the reference's FeatureTracker class
(/root/reference/vins_estimator/src/featureTracker/feature_tracker.h:43-99) over the C ABI of
libgf_b200.so.  Method names and argument meaning follow the reference; all arithmetic runs in the
CUDA library (no OpenCV, no CPU fallback).
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import OBS_DTYPE, TrackInfo, TrackerCfg, check

# stage-level wrappers -----------------------------------------------------------------------------


def _u8(a):
    a = np.ascontiguousarray(a, np.uint8)
    assert a.ndim == 2
    return a


def pyr_down(img, device=0):
    img = _u8(img)
    h, w = img.shape
    out = np.empty(((h + 1) // 2, (w + 1) // 2), np.uint8)
    check(_lib.lib().gf_stage_pyr_down(device, img.ctypes.data, w, h, out.ctypes.data))
    return out


def clahe(img, clip_limit=40.0, tile_grid=(8, 8), device=0):
    """cv2.createCLAHE(clip_limit, tile_grid).apply(img) for u8 images (the kernels of the tracker's equalize option).
    Row-padded views are passed with their row pitch."""
    img = FeatureTracker._rows(img, np.uint8)
    h, w = img.shape
    out = np.empty((h, w), np.uint8)
    check(_lib.lib().gf_stage_clahe(device, img.ctypes.data, img.strides[0], w, h, float(clip_limit), int(tile_grid[0]),
                                    int(tile_grid[1]), out.ctypes.data))
    return out


def corner_min_eigen_val(img, device=0):
    img = _u8(img)
    h, w = img.shape
    out = np.empty((h, w), np.float32)
    nfix = ctypes.c_int(0)
    check(_lib.lib().gf_stage_min_eig(device, img.ctypes.data, w, h, out.ctypes.data, ctypes.byref(nfix)))
    return out, nfix.value


def calc_optical_flow_pyr_lk(prev, nxt, prev_pts, max_level=3, init=None, device=0, roles=True):
    """roles: the LK form of a tracker alone on its device (two warp roles); False: the form of several trackers."""
    prev, nxt = _u8(prev), _u8(nxt)
    h, w = prev.shape
    p = np.ascontiguousarray(prev_pts, np.float32).reshape(-1, 2)
    q = np.ascontiguousarray(init, np.float32).reshape(-1, 2).copy() if init is not None else np.zeros_like(p)
    st = np.zeros(len(p), np.uint8)
    check(_lib.lib().gf_stage_lk(device, prev.ctypes.data, nxt.ctypes.data, w, h, p.ctypes.data, q.ctypes.data,
                                 len(p), int(max_level), int(init is not None), st.ctypes.data, int(bool(roles))))
    return q, st


def good_features_to_track(img, max_corners, min_dist, kept_pts=None, device=0):
    img = _u8(img)
    h, w = img.shape
    kp = np.zeros((0, 2), np.float32) if kept_pts is None else np.ascontiguousarray(kept_pts, np.float32).reshape(-1, 2)
    out = np.zeros((max(max_corners, 1), 2), np.float32)
    n = ctypes.c_int(0)
    info = TrackInfo()
    check(_lib.lib().gf_stage_gftt(device, img.ctypes.data, w, h, kp.ctypes.data if len(kp) else None, len(kp),
                                   int(max_corners), int(min_dist), out.ctypes.data, ctypes.byref(n), ctypes.byref(info)))
    return out[:n.value].copy(), info.as_dict()


def box_array(boxes):
    """Detections as the (m, 4) int64 array of gf_box (xmin, ymin, xmax, ymax: the fields of darknet_ros_msgs/BoundingBox)."""
    b = np.ascontiguousarray(np.zeros((0, 4)) if boxes is None or len(boxes) == 0 else boxes, np.int64).reshape(-1, 4)
    return b


def in_boxes(pts, boxes, device=0):
    """trackImagebox's test on its own (gf_stage_in_boxes): 1 where pointPolygonTest(box contour, pt, true) > 0 for a box."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    b = box_array(boxes)
    out = np.zeros(len(p), np.uint8)
    check(_lib.lib().gf_stage_in_boxes(device, p.ctypes.data if len(p) else None, len(p), b.ctypes.data if len(b) else None, len(b),
                                       out.ctypes.data if len(p) else None))
    return out.view(np.bool_)


def _box_csr(boxes):
    """Per-frame box lists -> (gf_box array, n + 1 offsets)."""
    arrs = [box_array(b) for b in boxes]
    start = np.zeros(len(arrs) + 1, np.int32)
    start[1:] = np.cumsum([len(a) for a in arrs])
    flat = np.concatenate(arrs, 0) if arrs else np.zeros((0, 4), np.int64)
    return np.ascontiguousarray(flat, np.int64), start


def setmask_order(track_cnt, device=0):
    tc = np.ascontiguousarray(track_cnt, np.int32)
    perm = np.empty(len(tc), np.int32)
    check(_lib.lib().gf_stage_setmask_order(device, tc.ctypes.data, len(tc), perm.ctypes.data))
    return perm


# the class ----------------------------------------------------------------------------------------


class FeatureTracker:
    """trackImage / trackImagebox / setPrediction / removeOutliers as in feature_tracker.h:47,48,70,72.

    readIntrinsicParameter is folded into the constructor (pinhole = fx fy cx cy k1 k2 p1 p2).  equalize: the config key
    EQUALIZE -- every frame goes through cv::createCLAHE(clahe_clip, clahe_grid) first, as getImageFromMsg does."""

    def __init__(self, width, height, pinhole, max_cnt=150, min_dist=30, flow_back=1, depth_cam=1, device=0,
                 equalize=False, clahe_clip=40.0, clahe_grid=(8, 8)):
        self.L = _lib.lib()
        cfg = TrackerCfg(int(max_cnt), int(min_dist), int(flow_back), int(depth_cam), (ctypes.c_double * 8)(*pinhole))
        self._h = ctypes.c_void_p()
        check(self.L.gf_tracker_create(ctypes.byref(self._h), int(device), int(width), int(height), ctypes.byref(cfg)))
        if equalize:
            try:
                check(self.L.gf_tracker_set_equalize(self._h, float(clahe_clip), int(clahe_grid[0]), int(clahe_grid[1])))
            except Exception:
                self.close()
                raise
        self.width, self.height, self.max_cnt = width, height, int(max_cnt)
        self._obs = np.zeros(self.max_cnt, OBS_DTYPE)
        self._status = np.zeros(self.max_cnt, np.uint8)
        self.last_status = np.zeros(0, np.uint8)
        self.last_info = {}
        g, d = ctypes.c_void_p(), ctypes.c_void_p()
        check(self.L.gf_tracker_host_buffers(self._h, ctypes.byref(g), ctypes.byref(d)))
        self.pinned_gray = np.ctypeslib.as_array(ctypes.cast(g, ctypes.POINTER(ctypes.c_uint8)), (height, width))
        self.pinned_depth = np.ctypeslib.as_array(ctypes.cast(d, ctypes.POINTER(ctypes.c_uint16)), (height, width))

    def close(self):
        if self._h:
            self.L.gf_tracker_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _collect(self, n, info):
        self.last_info = info.as_dict()
        self.last_status = self._status[:info.n_prev].copy()
        return self._obs[:n.value].copy()

    @staticmethod
    def _rows(a, dtype):
        """a itself when its rows are contiguous (any row pitch, e.g. a view into a wider buffer), else a contiguous copy."""
        if isinstance(a, np.ndarray) and a.dtype == dtype and a.ndim == 2 and a.strides[1] == a.itemsize and a.strides[0] >= a.shape[1] * a.itemsize:
            return a
        return np.ascontiguousarray(a, dtype)

    def _track(self, cur_time, img, depth, on_device=False, boxes=None):
        """One blocking gf_tracker_track call: host frames are arrays, device frames integer addresses of tightly packed frames.
        boxes: None for trackImage (returns obs), else an (m, 4) gf_box array for trackImagebox (returns (obs, in_box))."""
        if on_device:
            frame = (img, 0, depth, 0)
        else:
            img = self._rows(img, np.uint8)
            assert img.shape == (self.height, self.width)
            if depth is not None:
                depth = self._rows(depth, np.uint16)
            frame = (img.ctypes.data, img.strides[0], None if depth is None else depth.ctypes.data, 0 if depth is None else depth.strides[0])
        nb = 0 if boxes is None else len(boxes)
        in_box = None if boxes is None else np.zeros(self.max_cnt, np.uint8)
        n, info = ctypes.c_int(0), TrackInfo()
        check(self.L.gf_tracker_track(self._h, float(cur_time), *frame, int(bool(on_device)), boxes.ctypes.data if nb else None, nb,
                                      self._obs.ctypes.data, ctypes.byref(n), None if in_box is None else in_box.ctypes.data,
                                      self._status.ctypes.data, ctypes.byref(info)))
        obs = self._collect(n, info)
        return obs if in_box is None else (obs, in_box[:n.value].view(np.bool_))

    def trackImageRaw(self, cur_time, img, depth=None):
        """Returns the structured array of gf_obs in the tracker's internal (cur_pts) order.  Row-padded views are passed
        with their row pitch, as a cv::Mat with a larger step is in the reference."""
        return self._track(cur_time, img, depth)

    def trackImage(self, cur_time, img, depth=None):
        """map<int, vector<pair<int, Matrix<double,8,1>>>> as {id: v[8]} (camera id is always 0)."""
        obs = self.trackImageRaw(cur_time, img, depth)
        return {int(o["id"]): o["v"].copy() for o in obs}

    def trackImageboxRaw(self, cur_time, boxes, img, depth=None):
        """trackImagebox (feature_tracker.cpp:374-678): (obs, in_box).  obs is exactly what trackImageRaw returns for the frame;
        in_box[i] marks the features that trackImagebox leaves out of featureFrame because they lie strictly inside one of the
        boxes ((m, 4) xmin, ymin, xmax, ymax).  Those features stay in the tracker and are tracked on the next frame."""
        return self._track(cur_time, img, depth, boxes=box_array(boxes))

    def trackImagebox(self, cur_time, boxes, img, depth=None):
        """{id: v[8]} of trackImage without the features strictly inside a box (Estimator::inputImagebox's front end)."""
        obs, in_box = self.trackImageboxRaw(cur_time, boxes, img, depth)
        return {int(o["id"]): o["v"].copy() for o in obs[~in_box]}

    def trackDevice(self, cur_time, d_gray_ptr, d_depth_ptr=None):
        return self._track(cur_time, d_gray_ptr, d_depth_ptr, on_device=True)

    @staticmethod
    def _frame(img, dtype, shape):
        if not (isinstance(img, np.ndarray) and img.dtype == dtype and img.shape == shape and img.strides[1] == img.itemsize):
            raise ValueError("frame must be a %s array of shape %s with contiguous rows" % (np.dtype(dtype).name, shape))
        return img

    def submit(self, cur_time, img, depth=None):
        """Asynchronous trackImage: up to two frames may be in flight; collect them in order with wait().
        The arrays are read by the copy engine after this call returns: keep them alive and unchanged until wait()."""
        img = self._frame(img, np.uint8, (self.height, self.width))
        if depth is not None:
            depth = self._frame(depth, np.uint16, (self.height, self.width))
        dp, dpitch = (depth.ctypes.data, depth.strides[0]) if depth is not None else (None, 0)
        check(self.L.gf_tracker_submit(self._h, float(cur_time), img.ctypes.data, img.strides[0], dp, dpitch, 0, None, 0))

    def trackBatch(self, times, gray_ptrs, depth_ptrs=None, on_device=False, gray_pitch=None, depth_pitch=None, want=True, boxes=None):
        """n consecutive trackImage calls in ONE library call (gf_tracker_track_batch: two frames in flight inside the
        library).  gray_ptrs / depth_ptrs: integer addresses of the frames (host, ideally pinned, or device).  Returns a
        list of (obs, status, info) per frame when `want`, else None (bench loops that only need the work done).
        boxes: one (m, 4) box list per frame (empty: trackImage); the frames then go through trackImagebox and every result
        gains in_box: (obs, status, info, in_box)."""
        r = _track_streams(lambda *a: self.L.gf_tracker_track_batch(self._h, *a), [self], [times], [gray_ptrs],
                           None if depth_ptrs is None else [depth_ptrs], on_device, gray_pitch, depth_pitch, want,
                           None if boxes is None else [boxes])
        return r[0] if want else None

    @staticmethod
    def trackBatchMulti(trackers, times, gray_ptrs, depth_ptrs=None, on_device=False, gray_pitch=None, depth_pitch=None, want=True, boxes=None):
        """gf_tracker_track_batch_multi: n frames on each of S independent trackers in one call, fed by one host thread.
        times / gray_ptrs / depth_ptrs: per tracker lists of n entries.  Returns per tracker what trackBatch returns.
        boxes: per tracker lists of n box lists (results gain in_box as in trackBatch)."""
        h = (ctypes.c_void_p * len(trackers))(*[tr._h for tr in trackers])
        return _track_streams(lambda *a: trackers[0].L.gf_tracker_track_batch_multi(h, len(trackers), *a), trackers, times, gray_ptrs,
                              depth_ptrs, on_device, gray_pitch, depth_pitch, want, boxes)

    def submitDevice(self, cur_time, d_gray_ptr, d_depth_ptr=None):
        check(self.L.gf_tracker_submit(self._h, float(cur_time), d_gray_ptr, 0, d_depth_ptr, 0, 1, None, 0))

    def wait(self):
        n, info = ctypes.c_int(0), TrackInfo()
        check(self.L.gf_tracker_wait(self._h, self._obs.ctypes.data, ctypes.byref(n), None, self._status.ctypes.data, ctypes.byref(info)))
        return self._collect(n, info)

    def timer_start(self):
        check(self.L.gf_tracker_timer_start(self._h))

    def timer_stop(self):
        ms = ctypes.c_float(0)
        check(self.L.gf_tracker_timer_stop(self._h, ctypes.byref(ms)))
        return float(ms.value)

    def setPrediction(self, predictPts):
        ids = np.array(sorted(predictPts.keys()), np.int32)
        xyz = np.array([predictPts[int(i)] for i in ids], np.float64).reshape(-1, 3)
        check(self.L.gf_tracker_set_prediction(self._h, ids.ctypes.data if len(ids) else None,
                                               xyz.ctypes.data if len(ids) else None, len(ids)))

    def removeOutliers(self, removePtsIds):
        ids = np.array(sorted(removePtsIds), np.int32)
        check(self.L.gf_tracker_remove_ids(self._h, ids.ctypes.data if len(ids) else None, len(ids)))

    def set_equalize(self, clip_limit=40.0, tile_grid=(8, 8)):
        """gf_tracker_set_equalize: only before the first frame; tile_grid (0, 0) turns it off."""
        check(self.L.gf_tracker_set_equalize(self._h, float(clip_limit), int(tile_grid[0]), int(tile_grid[1])))

    def set_profiling(self, on=True):
        check(self.L.gf_tracker_set_profiling(self._h, int(bool(on))))

    STAGES = ("upload", "pyramid", "lk", "setmask", "gftt_select", "finalize", "download", "min_eig_aux")

    def last_stage_ms(self):
        ms = (ctypes.c_float * 8)()
        check(self.L.gf_tracker_last_stage_ms(self._h, ms))
        return dict(zip(self.STAGES, [float(v) for v in ms]))

    def last_device_ms(self):
        ms = ctypes.c_float(0)
        check(self.L.gf_tracker_last_device_ms(self._h, ctypes.byref(ms)))
        return ms.value


class TrackerGroup:
    """gf_tracker_group: several FeatureTrackers of one geometry and configuration (a multi-camera rig, several robots) that
    track frame k of their streams in lockstep with one set of kernel launches per step.  Every member's results and state are
    exactly what its own trackBatch would give; the members stay usable on their own between steps.

    Frames are given as integer addresses, as for trackBatch: host (ideally pinned) or device (on_device, tightly packed)."""

    def __init__(self, trackers):
        self.members = list(trackers)
        self.L = _lib.lib()
        self._h = ctypes.c_void_p()
        h = (ctypes.c_void_p * len(self.members))(*[tr._h for tr in self.members])
        check(self.L.gf_tracker_group_create(ctypes.byref(self._h), h, len(self.members)))
        self.max_cnt = self.members[0].max_cnt
        S = len(self.members)
        self._obs = np.zeros((S, self.max_cnt), OBS_DTYPE)
        self._status = np.zeros((S, self.max_cnt), np.uint8)
        self._in_box = np.zeros((S, self.max_cnt), np.uint8)

    def close(self):
        if self._h:
            self.L.gf_tracker_group_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def submit(self, times, gray_ptrs, depth_ptrs=None, on_device=False, gray_pitch=None, depth_pitch=None, boxes=None):
        """One step: member i tracks (times[i], gray_ptrs[i], depth_ptrs[i] or None) with the (m, 4) detections boxes[i].
        Up to two steps may be in flight; collect them in order with wait().  Host frames are read after this call returns:
        keep them unchanged until wait()."""
        S = len(self.members)
        assert len(times) == S and len(gray_ptrs) == S
        t = np.ascontiguousarray(times, np.float64)
        g = (ctypes.c_void_p * S)(*[int(p) for p in gray_ptrs])
        d = (ctypes.c_void_p * S)(*[(int(p) if p else None) for p in depth_ptrs]) if depth_ptrs is not None else None
        bx, start = _box_csr(boxes) if boxes is not None else (np.zeros((0, 4), np.int64), None)
        w = self.members[0].width
        check(self.L.gf_tracker_group_submit(self._h, t.ctypes.data, g, int(gray_pitch or w), d, int(depth_pitch or 2 * w), int(bool(on_device)),
                                             bx.ctypes.data if len(bx) else None, start.ctypes.data if start is not None else None))

    def wait(self):
        """The oldest step: per member (obs, status, info, in_box), as trackImageboxRaw plus the status and info of the frame."""
        S = len(self.members)
        cnt = np.zeros(S, np.int32)
        info = (TrackInfo * S)()
        check(self.L.gf_tracker_group_wait(self._h, self._obs.ctypes.data, cnt.ctypes.data, self._in_box.ctypes.data,
                                           self._status.ctypes.data, info))
        out = []
        for i, tr in enumerate(self.members):
            tr.last_info = info[i].as_dict()
            tr.last_status = self._status[i, :info[i].n_prev].copy()
            out.append((self._obs[i, :cnt[i]].copy(), tr.last_status.copy(), tr.last_info,
                        self._in_box[i, :cnt[i]].view(np.bool_).copy()))
        return out

    def trackBatch(self, times, gray_ptrs, depth_ptrs=None, on_device=False, gray_pitch=None, depth_pitch=None, want=True, boxes=None):
        """n steps in one call (gf_tracker_group_track_batch, two steps in flight).  times / gray_ptrs / depth_ptrs / boxes: per
        member lists of n entries, and the return value, as FeatureTracker.trackBatchMulti on the members."""
        return _track_streams(lambda *a: self.L.gf_tracker_group_track_batch(self._h, *a), self.members, times, gray_ptrs, depth_ptrs,
                              on_device, gray_pitch, depth_pitch, want, boxes)


def _track_streams(call, trackers, times, gray_ptrs, depth_ptrs, on_device, gray_pitch, depth_pitch, want, boxes):
    """n frames on each of the S streams `trackers` in one library call: call(n, times, gray, ...) takes the arguments of
    gf_tracker_track_batch from n on, with stream i's frame k at i*n + k.  Returns per stream a list of n (obs, status, info)
    (with boxes: (obs, status, info, in_box)) when `want`, else None; updates every tracker's batch_infos / last_info."""
    S, n = len(trackers), len(times[0])
    a = trackers[0]
    assert len(times) == S and all(len(x) == n for x in times)
    assert all(tr.max_cnt == a.max_cnt and tr.width == a.width for tr in trackers)
    t = np.ascontiguousarray(times, np.float64).reshape(S * n)
    g = (ctypes.c_void_p * (S * n))(*[int(p) for row in gray_ptrs for p in row])
    d = (ctypes.c_void_p * (S * n))(*[(int(p) if p else None) for row in depth_ptrs for p in row]) if depth_ptrs is not None else None
    obs = np.zeros((S, n, a.max_cnt), OBS_DTYPE) if want else None
    st = np.zeros((S, n, a.max_cnt), np.uint8) if want else None
    cnt = np.zeros((S, n), np.int32)
    info = (TrackInfo * (S * n))()
    bx, start, ib = np.zeros((0, 4), np.int64), None, None
    if boxes is not None:
        assert len(boxes) == S and all(len(x) == n for x in boxes)
        bx, start = _box_csr([b for row in boxes for b in row])
        ib = np.zeros((S, n, a.max_cnt), np.uint8) if want else None
    check(call(n, t.ctypes.data, g, int(gray_pitch or a.width), d, int(depth_pitch or 2 * a.width), int(bool(on_device)),
               bx.ctypes.data if len(bx) else None, None if start is None else start.ctypes.data, None if obs is None else obs.ctypes.data,
               cnt.ctypes.data, None if ib is None else ib.ctypes.data, None if st is None else st.ctypes.data, info))
    for i, tr in enumerate(trackers):
        tr.batch_infos = [info[i * n + k].as_dict() for k in range(n)]
        tr.last_info = tr.batch_infos[-1] if n else {}
    if obs is None:
        return None
    return [[(obs[i, k, :cnt[i, k]].copy(), st[i, k, :info[i * n + k].n_prev].copy(), info[i * n + k].as_dict())
             + (() if ib is None else (ib[i, k, :cnt[i, k]].view(np.bool_).copy(),)) for k in range(n)] for i in range(S)]
