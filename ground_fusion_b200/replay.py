"""Bag-free replay loop: FeatureTracker -> FeatureManager -> Estimator::optimization() (+ marginalisation, window slide) over a
synthetic RGB-D + IMU stream, modelled on the reference's offline driver (vins_estimator/src/KITTIOdomTest.cpp:82-121: read a
frame, inputImage, write the pose) and on Estimator::{processIMU, processImage, optimization, slideWindow}
(vins_estimator/src/estimator/estimator.cpp:743-783, 843-1163, 2890-3636, 3638-3806).

The three components are passed in (duck-typed): the product wires the CUDA FeatureTracker / FeatureManager / BundleAdjuster;
tests and bench.py wire the CPU oracles through the same loop to get the reference pipeline's trajectory and the ATE
(BASELINE.json metric: "ATE mm").  What is NOT replayed: initialisation (SURVEY 8(f) row 4) -- the first WINDOW_SIZE + 1 frames
take their states from the ground truth, as the text of DESIGN.md says -- wheel / GNSS inputs, failure detection.
"""
import math

import numpy as np

from .ba_problem import Problem
from .synth_ba import Preintegration, R_to_q, q_to_R

WINDOW_SIZE = 10
G = np.array([0.0, 0.0, 9.805])      # parameters.cpp:74, groundchallenge.yaml g_norm


class ImuFromStream:
    """IMU samples consistent with SyntheticStream.pose: body frame = camera frame (ric = I, tic = 0), specific force
    a_m = R_wb^T (a_w + G), body rate from the rotation; derivatives by central differences of the analytic pose."""

    def __init__(self, stream, h=1e-3):
        self.st, self.h = stream, h

    def pose_t(self, t):
        R, C = self.st.pose(t * self.st.fps)          # pose(k) evaluates the trajectory at k / fps
        return R.T, C                                 # R_wb, P

    def sample(self, t):
        h = self.h
        R0, P0 = self.pose_t(t); Rp, Pp = self.pose_t(t + h); Rm, Pm = self.pose_t(t - h)
        a_w = (Pp - 2 * P0 + Pm) / (h * h)
        W = R0.T @ (Rp - Rm) / (2 * h)
        gyr = np.array([W[2, 1] - W[1, 2], W[0, 2] - W[2, 0], W[1, 0] - W[0, 1]]) * 0.5
        return R0.T @ (a_w + G), gyr

    def velocity(self, t):
        h = self.h
        return (self.pose_t(t + h)[1] - self.pose_t(t - h)[1]) / (2 * h)


class WindowEstimator:
    """Estimator's sliding window (estimator.h:229-341) with the NON_LINEAR branch of processImage."""

    def __init__(self, fm, ba, imu_propagate=True, max_iter=8, tracker=None, use_mcc=False):
        """tracker: the front end, when the estimator feeds it back as the reference does with MULTIPLE_THREAD 0 (removeOutliers +
        setPrediction after every optimisation, estimator.cpp:1132-1136); None: no feedback (MULTIPLE_THREAD 1).  use_mcc: USE_MCC."""
        W = WINDOW_SIZE
        self.fm, self.ba = fm, ba
        self.tracker, self.use_mcc = tracker, use_mcc
        self.n_removed = self.n_predicted = 0
        self.Ps = np.zeros((W + 1, 3)); self.Rs = np.tile(np.eye(3), (W + 1, 1, 1)); self.Vs = np.zeros((W + 1, 3))
        self.Bas = np.zeros((W + 1, 3)); self.Bgs = np.zeros((W + 1, 3))
        self.pre = [None] * (W + 1); self.bufs = [[] for _ in range(W + 1)]
        self.tic, self.ric, self.td = np.zeros(3), np.eye(3), 0.0
        self.frame_count = 0; self.first_imu = False; self.acc_0 = self.gyr_0 = None
        self.prior = None
        self.imu_propagate, self.max_iter = imu_propagate, max_iter
        self.nonlinear = False
        self.last_summary = None; self.n_old = self.n_second_new = 0

    # estimator.cpp:743-783 (imu_propagate restores the state propagation this fork leaves to the wheel dead reckoning)
    def processIMU(self, dt, acc, gyr):
        fc = self.frame_count
        if not self.first_imu:
            self.first_imu = True; self.acc_0, self.gyr_0 = acc.copy(), gyr.copy()
        if self.pre[fc] is None:
            self.pre[fc] = Preintegration(self.acc_0, self.gyr_0, self.Bas[fc], self.Bgs[fc])
        if fc != 0:
            self.pre[fc].push_back(dt, acc, gyr); self.bufs[fc].append((dt, acc.copy(), gyr.copy()))
            if self.imu_propagate:
                j = fc
                un_acc_0 = self.Rs[j] @ (self.acc_0 - self.Bas[j]) - G
                un_gyr = 0.5 * (self.gyr_0 + gyr) - self.Bgs[j]
                th = un_gyr * dt
                dq = np.array([th[0] / 2, th[1] / 2, th[2] / 2, 1.0]); dq /= np.linalg.norm(dq)       # Utility::deltaQ
                self.Rs[j] = self.Rs[j] @ q_to_R(dq)
                un_acc_1 = self.Rs[j] @ (acc - self.Bas[j]) - G
                un_acc = 0.5 * (un_acc_0 + un_acc_1)
                self.Ps[j] = self.Ps[j] + dt * self.Vs[j] + 0.5 * dt * dt * un_acc
                self.Vs[j] = self.Vs[j] + dt * un_acc
        self.acc_0, self.gyr_0 = acc.copy(), gyr.copy()

    def set_state(self, fc, R, P, V):
        self.Rs[fc], self.Ps[fc], self.Vs[fc] = R, P, V

    # estimator.cpp:843-1163
    def processImage(self, image):
        fc = self.frame_count
        self.margin_old = bool(self.fm.addFeatureCheckParallax(fc, image, self.td))
        if not self.frame_added():
            return None
        self.fm.triangulateAll(fc, self.Ps, self.Rs, self.tic, self.ric)
        removeIndex = set()
        if self.use_mcc:                                  # estimator.cpp:1104-1109
            removeIndex = self.fm.movingConsistencyCheckW(self.Ps, self.Rs, self.tic, self.ric)
            self.fm.removeOutlier(removeIndex)
        self.optimization()
        return self.after_optimization(removeIndex)

    def frame_added(self):
        """processImage after addFeatureCheckParallax set margin_old: False while the window fills (the frame is taken and the
        next one starts from it), True when the nonlinear branch runs."""
        fc = self.frame_count
        if not self.nonlinear:
            if fc < WINDOW_SIZE:
                self.frame_count += 1
                nf = self.frame_count                    # slideWindow is not run while the window fills: the new frame starts from the last one
                self.Ps[nf], self.Rs[nf], self.Vs[nf], self.Bas[nf], self.Bgs[nf] = self.Ps[fc].copy(), self.Rs[fc].copy(), self.Vs[fc].copy(), self.Bas[fc].copy(), self.Bgs[fc].copy()
                return False
            self.nonlinear = True
        return True

    def after_optimization(self, removeIndex):
        """processImage after optimization(): the consistency check, the feedback to the tracker, the slide."""
        if not self.use_mcc:                              # :1123-1129 -- this set shadows the outer one: the tracker is not told about it
            self.fm.removeOutlier(self.fm.movingConsistencyCheckW(self.Ps, self.Rs, self.tic, self.ric))
        if self.tracker is not None:                      # :1131-1136 (MULTIPLE_THREAD 0)
            self.tracker.removeOutliers(removeIndex)
            pred = self.fm.predictPtsInNextFrame(self.frame_count, self.Ps, self.Rs, self.tic, self.ric)
            self.tracker.setPrediction(pred)
            self.n_removed += len(removeIndex); self.n_predicted += len(pred)
        self.slideWindow()
        self.fm.removeFailures()
        return self.Ps[WINDOW_SIZE].copy(), self.Rs[WINDOW_SIZE].copy()

    # estimator.cpp:2890-3636
    def optimization(self):
        pb, n_feat = self.build_problem()
        if n_feat is None:
            n_feat = self.fm.fillProblem(pb)
        R0_before, P0_before = self.Rs[0].copy(), self.Ps[0].copy()
        self.last_summary = self.ba.optimization(pb)
        self.fm.setDepth(self.adopt_solution(pb, n_feat, R0_before, P0_before))
        if self.margin_old:
            self.adopt_prior(self.ba.marginalize_old(pb))
        else:
            self.adopt_prior(self.ba.marginalize_second_new(pb))

    def build_problem(self):
        """vector2double, the visual factors of a host manager, the IMU factors and the prior.  Returns (problem, n_features); with
        a FeatureWindow the visual part is left to its fillProblem (or a FeatureWindowGroup's) and n_features is None."""
        W = WINDOW_SIZE
        on_device = hasattr(self.fm, "fillProblem")      # FeatureWindow: the visual factors come from the resident table
        feats = [] if on_device else list(self.fm.iter_ba_features())
        pb = Problem(W + 1, len(feats))
        for i in range(W + 1):                           # vector2double (estimator.cpp:2276-2353)
            pb.para_pose[i, :3] = self.Ps[i]; pb.para_pose[i, 3:] = R_to_q(self.Rs[i])
            pb.para_speed_bias[i] = np.concatenate([self.Vs[i], self.Bas[i], self.Bgs[i]])
        pb.para_ex_pose[:3] = self.tic; pb.para_ex_pose[3:] = R_to_q(self.ric)
        pb.para_td[0] = self.td
        pb.ex_pose_const = 1; pb.td_const = 1            # ESTIMATE_EXTRINSIC 0, ESTIMATE_TD 0
        pb.max_num_iterations = self.max_iter
        rows = []
        for k, (start, obs, est_depth, flag) in enumerate(feats):
            pb.para_feature[k] = 1.0 / est_depth
            pb.feature_const[k] = 1 if flag == 1 else 0   # depth from the depth image: SetParameterBlockConstant (estimator.cpp:3291-3292)
            p0, v0, t0 = obs[0]
            for a in range(1, len(obs)):
                pj, vj, tj = obs[a]
                rows.append((start, start + a, k, p0, pj, v0, vj, t0, tj))
        n_feat = None
        if not on_device:
            pb.set_visual(rows); n_feat = len(feats)
        pb.set_imu([self.pre[j].as_dict(j - 1, j) for j in range(1, W + 1) if self.pre[j] is not None and self.pre[j].sum_dt <= 10.0])
        pb.prior = self.prior
        return pb, n_feat

    def adopt_solution(self, pb, n_feat, R0_before, P0_before):
        """double2vector (estimator.cpp:2440-2569) of the solved problem; then the blocks are re-read for the marginalisation.
        Returns the depth vector setDepth takes."""
        W = WINDOW_SIZE
        from .estimator import double2vector
        Rs, Ps, Vs = double2vector(pb, R0_before, P0_before, True)
        self.Rs, self.Ps, self.Vs = Rs, Ps, Vs
        self.Bas = pb.para_speed_bias[:, 3:6].copy(); self.Bgs = pb.para_speed_bias[:, 6:9].copy()
        x = pb.para_feature[:n_feat]
        # the prior of the next window is linearised at the solved blocks as they stand (vector2double at estimator.cpp:3337 re-reads
        # the rotated state; the rotation is the identity up to the yaw fix of a window that has a prior)
        for i in range(W + 1):
            pb.para_pose[i, :3] = self.Ps[i]; pb.para_pose[i, 3:] = R_to_q(self.Rs[i])
            pb.para_speed_bias[i, :3] = self.Vs[i]
        return x

    def adopt_prior(self, prior):
        """The marginalisation's result as margin_old says: MARGIN_OLD always replaces the prior, MARGIN_SECOND_NEW only when it
        returned one (None: the prior stays)."""
        if self.margin_old:
            self.prior = prior; self.n_old += 1
        else:
            if prior is not None:
                self.prior = prior
            self.n_second_new += 1

    # estimator.cpp:3638-3806
    def slideWindow(self):
        shift = self.slide_states()
        if shift is not None:
            self.fm.removeBackShiftDepth(*shift)                  # slideWindowOld (estimator.cpp:3808-3837)
        else:
            self.fm.removeFront(self.frame_count)                 # slideWindowNew (estimator.cpp:3839-3851)

    def slide_states(self):
        """slideWindow's shift of the window's states and pre-integrations.  Returns the camera poses (R0, P0, R1, P1) of
        removeBackShiftDepth after MARGIN_OLD, None after MARGIN_SECOND_NEW (removeFront)."""
        W = WINDOW_SIZE
        if self.margin_old:
            back_R0, back_P0 = self.Rs[0].copy(), self.Ps[0].copy()
            for i in range(W):
                self.Rs[i], self.Ps[i], self.Vs[i], self.Bas[i], self.Bgs[i] = self.Rs[i + 1].copy(), self.Ps[i + 1].copy(), self.Vs[i + 1].copy(), self.Bas[i + 1].copy(), self.Bgs[i + 1].copy()
                self.pre[i], self.bufs[i] = self.pre[i + 1], self.bufs[i + 1]
            self.pre[W] = Preintegration(self.acc_0, self.gyr_0, self.Bas[W], self.Bgs[W]); self.bufs[W] = []
            R0, R1 = back_R0 @ self.ric, self.Rs[0] @ self.ric
            P0, P1 = back_P0 + back_R0 @ self.tic, self.Ps[0] + self.Rs[0] @ self.tic
            return R0, P0, R1, P1
        else:
            self.Ps[W - 1], self.Rs[W - 1] = self.Ps[W].copy(), self.Rs[W].copy()
            for dt, acc, gyr in self.bufs[W]:
                self.pre[W - 1].push_back(dt, acc, gyr); self.bufs[W - 1].append((dt, acc, gyr))
            self.Vs[W - 1], self.Bas[W - 1], self.Bgs[W - 1] = self.Vs[W].copy(), self.Bas[W].copy(), self.Bgs[W].copy()
            self.pre[W] = Preintegration(self.acc_0, self.gyr_0, self.Bas[W], self.Bgs[W]); self.bufs[W] = []
            return None


def replay(stream, tracker, fm, ba, n_frames, imu_per_frame=7, imu_propagate=True, max_iter=8, feedback=False, use_mcc=False, boxes=None,
           dense_map=None, grid_map=None, detector=None):
    """Runs n_frames of `stream` through tracker -> fm -> ba.  Returns dict(t, P_est, P_gt, R_est, R_gt, keyframes, ...).
    tracker.trackImage(t, gray, depth) -> {id: v[8]};  fm / ba: see WindowEstimator.  feedback: the estimator calls the tracker's
    removeOutliers / setPrediction after every optimisation (the reference with MULTIPLE_THREAD 0).
    boxes: USE_YOLO -- the detections of frame k in boxes[k] ((m, 4) xmin, ymin, xmax, ymax).  A frame with detections goes
    through tracker.trackImagebox(t, boxes[k], gray, depth), one without through trackImage, as sync_process does
    (rosNodeTest.cpp:433-439, 519-540).
    detector: USE_YOLO with the detector in the loop (a YoloDetector, or anything with detect(bgr) -> (boxes, class_ids, probs)):
    frame k's boxes are detector.detect(BGR of stream.color(k)), computed before frame k is tracked, so they belong to frame k.
    The darknet_ros node's three-slot asynchronous buffer, and the frames of latency it adds, are not reproduced.  Exclusive
    with boxes.
    dense_map: a map with addKeyFrame(R, P, rgb, depth) (DenseMap, or the oracle's), fed as pubKeyframe feeds the mapping node
    (visualization.cpp): after every MARGIN_OLD, the pose of window frame WINDOW_SIZE - 2 with that frame's colour and depth
    images (stream.color / stream.frame), unless its position equals the previous keyframe's exactly, as the node skips it.  It is returned under "dense_map".
    grid_map: an occupancy grid with addKeyFrame(R, P, points) (GridMap, or the oracle's); requires dense_map.  After dense-map
    keyframe k it gets the same pose and dense_map.keyframePoints(k), the point_rgbd the grid_mapping tool reads.  It is returned
    under "grid_map"."""
    if grid_map is not None and dense_map is None:
        raise ValueError("grid_map requires dense_map")
    if detector is not None and boxes is not None:
        raise ValueError("boxes and detector are exclusive")
    imu = ImuFromStream(stream)
    est = WindowEstimator(fm, ba, imu_propagate=imu_propagate, max_iter=max_iter, tracker=tracker if feedback else None, use_mcc=use_mcc)
    out_t, out_P, out_R, gt_P, gt_R, iters = [], [], [], [], [], []
    t_prev = None
    slot = [0] * (WINDOW_SIZE + 1)                      # stream frame held by each window slot (Headers[])
    last_P = None                                       # position of the last keyframe fed to dense_map
    n_dm = 0                                            # keyframes fed to dense_map
    for k in range(n_frames):
        t, gray, depth = stream.frame(k)
        if t_prev is not None:                          # IMU samples of (t_prev, t]
            dt = (t - t_prev) / imu_per_frame
            for s in range(1, imu_per_frame + 1):
                acc, gyr = imu.sample(t_prev + s * dt)
                est.processIMU(dt, acc, gyr)
        else:
            acc, gyr = imu.sample(t); est.processIMU(0.0, acc, gyr)
        frame_boxes = boxes[k] if boxes is not None else None
        if detector is not None:
            frame_boxes = detector.detect(np.ascontiguousarray(stream.color(k)[..., ::-1]))[0]
        if frame_boxes is not None and len(frame_boxes) > 0:
            image = tracker.trackImagebox(t, frame_boxes, gray, depth)
        else:
            image = tracker.trackImage(t, gray, depth)
        if not est.nonlinear:                           # initialisation is out of scope: ground-truth states while the window fills
            R_wb, P = imu.pose_t(t)
            est.set_state(est.frame_count, R_wb, P, imu.velocity(t))
        slot[est.frame_count] = k
        res = est.processImage(image)
        t_prev = t
        if res is not None:                             # the window slid: slideWindow's shift of Headers[]
            if est.margin_old:
                slot[:WINDOW_SIZE] = slot[1:]
            else:
                slot[WINDOW_SIZE - 1] = slot[WINDOW_SIZE]
            # the node skips a keyframe whose position equals the previous one exactly (pose_graph_node.cpp:660, SKIP_DIS 0)
            if dense_map is not None and est.margin_old and not np.array_equal(est.Ps[WINDOW_SIZE - 2], last_P):
                j = slot[WINDOW_SIZE - 2]
                last_P = est.Ps[WINDOW_SIZE - 2].copy()
                dense_map.addKeyFrame(est.Rs[WINDOW_SIZE - 2], last_P, stream.color(j), stream.frame(j)[2])
                if grid_map is not None:
                    grid_map.addKeyFrame(est.Rs[WINDOW_SIZE - 2], last_P, dense_map.keyframePoints(n_dm))
                n_dm += 1
        if res is not None:
            R_wb, P = imu.pose_t(t)
            out_t.append(t); out_P.append(res[0]); out_R.append(res[1]); gt_P.append(P); gt_R.append(R_wb)
            iters.append(est.last_summary["iterations"] if isinstance(est.last_summary, dict) else est.last_summary.get("iterations"))
    P_est, P_gt = np.array(out_P), np.array(gt_P)
    ate = float(np.sqrt(np.mean(np.sum((P_est - P_gt) ** 2, axis=1)))) if len(P_est) else float("nan")
    out = {"t": np.array(out_t), "P_est": P_est, "P_gt": P_gt, "R_est": np.array(out_R), "R_gt": np.array(gt_R), "ate_m": ate,
           "n_margin_old": est.n_old, "n_margin_second_new": est.n_second_new, "iterations": iters,
           "n_removed": est.n_removed, "n_predicted": est.n_predicted}
    if dense_map is not None:
        out["dense_map"] = dense_map
    if grid_map is not None:
        out["grid_map"] = grid_map
    return out


def slide_slots(slot, margin_old):
    """slideWindow's shift of the stream frames held by the window slots (Headers[]), in place."""
    if margin_old:
        slot[:WINDOW_SIZE] = slot[1:]
    else:
        slot[WINDOW_SIZE - 1] = slot[WINDOW_SIZE]


def keyframe_members(ests, last_P):
    """The estimators that add a map keyframe after this step's slide, as replay() decides it for one: MARGIN_OLD, and the pose
    of window frame WINDOW_SIZE - 2 not at the previous keyframe's position exactly (last_P[i]: None before the first)."""
    return [i for i, e in enumerate(ests) if e.margin_old and not np.array_equal(e.Ps[WINDOW_SIZE - 2], last_P[i])]


def replay_group(streams, trackers, windows, adjusters, n_frames, imu_per_frame=7, imu_propagate=True, max_iter=8, feedback=False,
                 boxes=None, detector=None, dense_maps=None, grid_maps=None, use_mcc=False):
    """K estimators in lockstep, one per stream, each step with one call per stage for all of them: the TrackerGroup over
    `trackers` tracks frame k of every stream, the FeatureWindowGroup over `windows` ingests the step on the device and
    triangulates, fills the K problems, estimator.solve_multi solves them on `adjusters`, setDepth follows, then
    estimator.marginalize_multi with each estimator's own mode, the consistency check and removal, the feedback to each member
    tracker (feedback=True, between tracker-group steps) and the slide.  The host logic is WindowEstimator's, as in replay();
    returns one result dict per stream in replay()'s format.
    boxes: USE_YOLO as in replay(), per stream: boxes[i][k] are the detections of frame k of stream i.  They go into the tracker
    group's step, and the window group takes the features inside them out on the device.
    detector: USE_YOLO with the detector in the loop, as in replay(): step k runs one detector.detect_batch over the K streams'
    colour frames before the tracker group's step (its max_batch is raised to K if smaller).  Exclusive with boxes.
    dense_maps: one DenseMap per stream (sharing the frame geometry), fed as replay() feeds its dense_map, with one
    DenseMapGroup call per step for the members that add a keyframe; grid_maps: one GridMap per stream (requires dense_maps),
    each fed on the device with the keyframe its stream's dense map just added (GridMapGroup.addDenseKeyFrames).  They are
    returned under "dense_map" / "grid_map" of each stream's dict.
    use_mcc: USE_MCC as in replay(): the moving-consistency check and removal before the solve, none after it; with feedback the
    removed ids reach each member's tracker."""
    from . import _lib
    from .estimator import marginalize_multi, solve_multi
    from .feature_tracker import TrackerGroup
    from .feature_window import FeatureWindowGroup
    K = len(streams)
    assert len(trackers) == len(windows) == len(adjusters) == K
    if detector is not None and boxes is not None:
        raise ValueError("boxes and detector are exclusive")
    if grid_maps is not None and dense_maps is None:
        raise ValueError("grid_maps requires dense_maps")
    if (dense_maps is not None and len(dense_maps) != K) or (grid_maps is not None and len(grid_maps) != K):
        raise ValueError("one dense map and one grid map per stream")
    if detector is not None and detector.max_batch < K:
        detector.set_max_batch(K)
    tg, wg = TrackerGroup(trackers), FeatureWindowGroup(windows)
    dg = gg = None
    imus = [ImuFromStream(s) for s in streams]
    ests = [WindowEstimator(windows[i], adjusters[i], imu_propagate=imu_propagate, max_iter=max_iter, tracker=trackers[i] if feedback else None,
                            use_mcc=use_mcc) for i in range(K)]
    rec = [{"t": [], "P": [], "R": [], "gP": [], "gR": [], "it": []} for _ in range(K)]
    t_prev = [None] * K
    slots = [[0] * (WINDOW_SIZE + 1) for _ in range(K)]  # stream frame held by each window slot, per stream
    last_P = [None] * K                                 # position of the last keyframe fed to each dense map
    try:
        if dense_maps is not None:
            from .dense_map import DenseMapGroup
            dg = DenseMapGroup(dense_maps)
        if grid_maps is not None:
            from .grid_map import GridMapGroup
            gg = GridMapGroup(grid_maps)
        for k in range(n_frames):
            frames = [s.frame(k) for s in streams]
            for i, (e, imu) in enumerate(zip(ests, imus)):
                t = frames[i][0]
                if t_prev[i] is not None:
                    dt = (t - t_prev[i]) / imu_per_frame
                    for s in range(1, imu_per_frame + 1):
                        acc, gyr = imu.sample(t_prev[i] + s * dt)
                        e.processIMU(dt, acc, gyr)
                else:
                    acc, gyr = imu.sample(t); e.processIMU(0.0, acc, gyr)
            gray = [np.ascontiguousarray(f[1]) for f in frames]
            depth = [np.ascontiguousarray(f[2]) if f[2] is not None else None for f in frames]
            step_boxes = [boxes[i][k] for i in range(K)] if boxes is not None else None
            if detector is not None:
                step_boxes = [r[0] for r in detector.detect_batch([np.ascontiguousarray(s.color(k)[..., ::-1]) for s in streams])]
            tg.submit([f[0] for f in frames], [g.ctypes.data for g in gray], [d.ctypes.data if d is not None else 0 for d in depth],
                      boxes=step_boxes)
            tg.wait()
            for i, (e, imu) in enumerate(zip(ests, imus)):
                if not e.nonlinear:                     # initialisation is out of scope: ground-truth states while the window fills
                    R_wb, P = imu.pose_t(frames[i][0])
                    e.set_state(e.frame_count, R_wb, P, imu.velocity(frames[i][0]))
            fcs = [e.frame_count for e in ests]
            for sl, fc in zip(slots, fcs):
                sl[fc] = k
            margins = wg.addFramesFromTrackerGroup(tg, fcs, [e.td for e in ests])
            for e, m in zip(ests, margins):
                e.margin_old = m
            t_prev = [f[0] for f in frames]
            full = [e.frame_added() for e in ests]
            assert len(set(full)) == 1, "the estimators of a group fill their windows in lockstep"
            if not full[0]:
                continue
            poses = [(e.Ps, e.Rs, e.tic, e.ric) for e in ests]
            wg.triangulateAll(fcs, poses)
            removed = [set() for _ in ests]
            if use_mcc:                                              # as processImage with USE_MCC
                removed = wg.movingConsistencyCheckW(poses)
                wg.removeOutliers(removed)
            pbs = [e.build_problem()[0] for e in ests]
            nfs = wg.fillProblems(pbs)
            before = [(e.Rs[0].copy(), e.Ps[0].copy()) for e in ests]
            sums, status = solve_multi(adjusters, pbs)
            if any(v < 0 for v in status):
                raise _lib.GfError("solve_multi: a window's IMU covariance is singular: %s" % status)
            xs = []
            for e, pb, nf, (R0, P0), sm in zip(ests, pbs, nfs, before, sums):
                e.last_summary = sm
                xs.append(e.adopt_solution(pb, nf, R0, P0))
            wg.setDepths(xs)
            priors, kept = marginalize_multi(adjusters, pbs, [_lib.MARGIN_OLD if e.margin_old else _lib.MARGIN_SECOND_NEW for e in ests])
            if any(v < 0 for v in kept):
                raise _lib.GfError("marginalize_multi: a window's IMU covariance is singular: %s" % kept)
            for e, pr in zip(ests, priors):
                e.adopt_prior(pr)
            poses = [(e.Ps, e.Rs, e.tic, e.ric) for e in ests]
            if not use_mcc:                                          # as after_optimization without USE_MCC
                wg.removeOutliers(wg.movingConsistencyCheckW(poses))
            if feedback:                                             # the set the tracker is told about is empty without USE_MCC
                preds = wg.predictPtsInNextFrame([e.frame_count for e in ests], poses)
                for e, tr, pred, rm in zip(ests, trackers, preds, removed):
                    tr.removeOutliers(rm)
                    tr.setPrediction(pred)
                    e.n_removed += len(rm); e.n_predicted += len(pred)
            shifts = [e.slide_states() for e in ests]
            wg.remove([_lib.FM_REMOVE_BACK_SHIFT_DEPTH if sh is not None else _lib.FM_REMOVE_FRONT for sh in shifts],
                      [e.frame_count for e in ests], shifts)
            wg.removeFailures()
            for sl, e in zip(slots, ests):
                slide_slots(sl, e.margin_old)
            if dg is not None:
                add_group_keyframes(dg, gg, streams, ests, slots, last_P)
            for i, (e, imu) in enumerate(zip(ests, imus)):
                R_wb, P = imu.pose_t(frames[i][0])
                r = rec[i]
                r["t"].append(frames[i][0]); r["P"].append(e.Ps[WINDOW_SIZE].copy()); r["R"].append(e.Rs[WINDOW_SIZE].copy())
                r["gP"].append(P); r["gR"].append(R_wb); r["it"].append(e.last_summary["iterations"])
    finally:
        for grp in (gg, dg, wg, tg):
            if grp is not None:
                grp.close()
    out = []
    for i, (e, r) in enumerate(zip(ests, rec)):
        P_est, P_gt = np.array(r["P"]), np.array(r["gP"])
        ate = float(np.sqrt(np.mean(np.sum((P_est - P_gt) ** 2, axis=1)))) if len(P_est) else float("nan")
        out.append({"t": np.array(r["t"]), "P_est": P_est, "P_gt": P_gt, "R_est": np.array(r["R"]), "R_gt": np.array(r["gR"]), "ate_m": ate,
                    "n_margin_old": e.n_old, "n_margin_second_new": e.n_second_new, "iterations": r["it"],
                    "n_removed": e.n_removed, "n_predicted": e.n_predicted})
        if dense_maps is not None:
            out[-1]["dense_map"] = dense_maps[i]
        if grid_maps is not None:
            out[-1]["grid_map"] = grid_maps[i]
    return out


def add_group_keyframes(dg, gg, streams, ests, slots, last_P):
    """The keyframes of one replay_group step: one dense-map group call for the members keyframe_members picks, each with the
    pose of window frame WINDOW_SIZE - 2 and the colour and depth of the stream frame in that slot; then, with a grid group gg,
    one call feeding each of those grids its dense map's new keyframe on the device.  A member's failure raises, as replay()'s
    single call does.  Returns the members fed."""
    from . import _lib
    req = keyframe_members(ests, last_P)
    if not req:
        return req
    W2 = WINDOW_SIZE - 2
    Rs = [ests[i].Rs[W2].copy() for i in req]
    Ps = [ests[i].Ps[W2].copy() for i in req]
    for i, P in zip(req, Ps):
        last_P[i] = P
    fr = [slots[i][W2] for i in req]
    _, st = dg.addKeyFrames(req, Rs, Ps, [streams[i].color(j) for i, j in zip(req, fr)], [streams[i].frame(j)[2] for i, j in zip(req, fr)])
    if np.any(st):
        raise _lib.GfError("dense map group: member status %s" % dict(zip(req, (int(v) for v in st))))
    if gg is not None:
        st = gg.addDenseKeyFrames(dg, req, Rs, Ps)
        if np.any(st):
            raise _lib.GfError("grid map group: member status %s" % dict(zip(req, (int(v) for v in st))))
    return req
