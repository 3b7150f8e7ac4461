"""ctypes binding of libgf_b200.so (the C ABI declared in include/gf_b200.h).

There is no CPU fallback: if the shared library is missing or no CUDA device is visible every entry
point raises.  The library is built in-tree by `make` / `__graft_entry__.build()`.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GF_B200_LIB") or os.path.join(_HERE, "libgf_b200.so")   # GF_B200_LIB: a -DGF_PROFILE build (tools/)
_LIB = None


class GfError(RuntimeError):
    pass


class TrackerCfg(ctypes.Structure):
    _fields_ = [("max_cnt", ctypes.c_int), ("min_dist", ctypes.c_int), ("flow_back", ctypes.c_int),
                ("depth_cam", ctypes.c_int), ("pinhole", ctypes.c_double * 8)]


class DenseMapCfg(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("pinhole", ctypes.c_double * 8), ("depth_dist", ctypes.c_int),
                ("depth_boundary", ctypes.c_int), ("ric", ctypes.c_double * 9), ("tic", ctypes.c_double * 3), ("max_points", ctypes.c_int),
                ("max_keyframes", ctypes.c_int)]


DENSE_MAP_CLOUD, DENSE_MAP_FILTERED = 0, 1      # gf_dense_map_read's `which`
MAP_GROUP_MAX = 64                              # GF_DENSE_MAP_GROUP_MAX = GF_GRID_MAP_GROUP_MAX


class GridMapCfg(ctypes.Structure):
    _fields_ = [("size_x", ctypes.c_int), ("size_y", ctypes.c_int), ("init_x", ctypes.c_int), ("init_y", ctypes.c_int),
                ("cell_size", ctypes.c_double), ("p_occ", ctypes.c_double), ("p_free", ctypes.c_double), ("p_prior", ctypes.c_double),
                ("ric", ctypes.c_double * 9), ("tic", ctypes.c_double * 3), ("max_points", ctypes.c_int), ("max_keyframes", ctypes.c_int),
                ("max_records", ctypes.c_int)]


GRID_MAP_BEL, GRID_MAP_IMAGE, GRID_MAP_OCCUPANCY = 0, 1, 2      # gf_grid_map_read's `which`


class FmWindowCfg(ctypes.Structure):
    _fields_ = [("max_features", ctypes.c_int), ("window_size", ctypes.c_int), ("min_parallax", ctypes.c_double),
                ("depth_threshold", ctypes.c_double), ("init_depth", ctypes.c_double)]


FM_WINDOW_ROWS, FM_WINDOW_ROW_DOUBLES = 11, 9
FM_OUTLIERS_REPROJECTION, FM_OUTLIERS_MOVING = 0, 1            # gf_fm_window_outliers' `mode`
FM_WINDOW_GROUP_MAX = 64                                       # GF_FM_WINDOW_GROUP_MAX
FM_REMOVE_NONE, FM_REMOVE_BACK_SHIFT_DEPTH, FM_REMOVE_BACK, FM_REMOVE_FRONT = 0, 1, 2, 3   # gf_fm_window_group_remove's ops


GF_MAX_BOXES = 100                                             # darknet_ros publishes at most 100 boxes
GF_DETECTOR_BATCH_MAX = 64                                     # frames per gf_detector_detect_batch call


class Obs(ctypes.Structure):
    _fields_ = [("id", ctypes.c_int32), ("track_cnt", ctypes.c_int32), ("v", ctypes.c_double * 8)]


OBS_DTYPE = np.dtype([("id", np.int32), ("track_cnt", np.int32), ("v", np.float64, (8,))])
assert OBS_DTYPE.itemsize == ctypes.sizeof(Obs) == 72


class TrackInfo(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("n_prev", "n_tracked", "n_kept", "n_new", "n_candidates",
                                                "nms_rounds", "eig_fixups", "lk_iterations")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ }


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise GfError("libgf_b200.so not built (%s): run `make` or __graft_entry__.build(); "
                          "there is no CPU fallback" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        vp, i, d, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_size_t
        L.gf_last_error.restype = ctypes.c_char_p
        L.gf_version.restype = ctypes.c_char_p
        L.gf_kernel_launch_count.restype = ctypes.c_uint64
        L.gf_tracker_create.argtypes = [ctypes.POINTER(vp), i, i, i, ctypes.POINTER(TrackerCfg)]
        L.gf_tracker_destroy.argtypes = [vp]
        L.gf_tracker_destroy.restype = None
        L.gf_tracker_host_buffers.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp)]
        L.gf_tracker_track.argtypes = [vp, d, vp, sz, vp, sz, i, vp, i, vp, ctypes.POINTER(i), vp, vp, ctypes.POINTER(TrackInfo)]
        L.gf_tracker_submit.argtypes = [vp, d, vp, sz, vp, sz, i, vp, i]
        L.gf_tracker_wait.argtypes = [vp, vp, ctypes.POINTER(i), vp, vp, ctypes.POINTER(TrackInfo)]
        L.gf_tracker_track_batch.argtypes = [vp, i, vp, vp, sz, vp, sz, i, vp, vp, vp, vp, vp, vp, vp]
        L.gf_tracker_track_batch_multi.argtypes = [vp, i, i, vp, vp, sz, vp, sz, i, vp, vp, vp, vp, vp, vp, vp]
        L.gf_tracker_timer_start.argtypes = [vp]
        L.gf_tracker_timer_stop.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
        L.gf_tracker_group_create.argtypes = [ctypes.POINTER(vp), vp, i]
        L.gf_tracker_group_destroy.argtypes = [vp]
        L.gf_tracker_group_destroy.restype = None
        L.gf_tracker_group_submit.argtypes = [vp, vp, vp, sz, vp, sz, i, vp, vp]
        L.gf_tracker_group_wait.argtypes = [vp, vp, vp, vp, vp, vp]
        L.gf_tracker_group_track_batch.argtypes = [vp, i, vp, vp, sz, vp, sz, i, vp, vp, vp, vp, vp, vp, vp]
        L.gf_stage_in_boxes.argtypes = [i, vp, i, vp, i, vp]
        L.gf_tracker_set_prediction.argtypes = [vp, vp, vp, i]
        L.gf_tracker_set_equalize.argtypes = [vp, d, i, i]
        L.gf_tracker_remove_ids.argtypes = [vp, vp, i]
        L.gf_tracker_last_device_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
        L.gf_tracker_set_profiling.argtypes = [vp, i]
        L.gf_tracker_last_stage_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
        L.gf_tracker_debug_read.argtypes = [vp, ctypes.POINTER(ctypes.c_longlong), ctypes.c_int]
        L.gf_stage_pyr_down.argtypes = [i, vp, i, i, vp]
        L.gf_stage_clahe.argtypes = [i, vp, sz, i, i, d, i, i, vp]
        L.gf_stage_min_eig.argtypes = [i, vp, i, i, vp, ctypes.POINTER(i)]
        L.gf_stage_lk.argtypes = [i, vp, vp, i, i, vp, vp, i, i, i, vp, i]
        L.gf_stage_gftt.argtypes = [i, vp, i, i, vp, i, i, i, vp, ctypes.POINTER(i), ctypes.POINTER(TrackInfo)]
        L.gf_stage_setmask_order.argtypes = [i, vp, i, vp]
        L.gf_dense_map_create.argtypes = [ctypes.POINTER(vp), i, ctypes.POINTER(DenseMapCfg)]
        L.gf_dense_map_destroy.argtypes = [vp]
        L.gf_dense_map_destroy.restype = None
        L.gf_dense_map_add_keyframe.argtypes = [vp, vp, vp, vp, sz, vp, sz, i, ctypes.POINTER(i)]
        L.gf_dense_map_update_poses.argtypes = [vp, i, vp, vp]
        L.gf_dense_map_size.argtypes = [vp, ctypes.POINTER(i), ctypes.POINTER(i), ctypes.POINTER(i)]
        L.gf_dense_map_read.argtypes = [vp, i, vp, vp, vp]
        L.gf_dense_map_keyframe_points.argtypes = [vp, i, vp, ctypes.POINTER(i)]
        L.gf_stage_radius_filter.argtypes = [i, vp, i, d, i, vp]
        L.gf_grid_map_create.argtypes = [ctypes.POINTER(vp), i, ctypes.POINTER(GridMapCfg)]
        L.gf_grid_map_destroy.argtypes = [vp]
        L.gf_grid_map_destroy.restype = None
        L.gf_grid_map_add_keyframe.argtypes = [vp, vp, vp, vp, i, i, i]
        L.gf_grid_map_update_poses.argtypes = [vp, i, vp, vp]
        L.gf_grid_map_read.argtypes = [vp, i, vp]
        L.gf_grid_map_size.argtypes = [vp] + [ctypes.POINTER(i)] * 4
        L.gf_grid_map_stats.argtypes = [vp, vp]
        L.gf_dense_map_group_create.argtypes = [ctypes.POINTER(vp), vp, i]
        L.gf_dense_map_group_destroy.argtypes = [vp]
        L.gf_dense_map_group_destroy.restype = None
        L.gf_dense_map_group_size.argtypes = [vp, ctypes.POINTER(i)]
        L.gf_dense_map_group_add_keyframes.argtypes = [vp, vp, i, vp, vp, vp, vp, vp, vp, i, vp, vp]
        L.gf_grid_map_group_create.argtypes = [ctypes.POINTER(vp), vp, i]
        L.gf_grid_map_group_destroy.argtypes = [vp]
        L.gf_grid_map_group_destroy.restype = None
        L.gf_grid_map_group_size.argtypes = [vp, ctypes.POINTER(i)]
        L.gf_grid_map_group_add_keyframes.argtypes = [vp, vp, i, vp, vp, vp, vp, vp, i, vp]
        L.gf_grid_map_group_add_dense_keyframes.argtypes = [vp, vp, vp, i, vp, vp, vp]
        ip, dp = ctypes.POINTER(i), ctypes.POINTER(d)
        L.gf_fm_window_create.argtypes = [ctypes.POINTER(vp), i, ctypes.POINTER(FmWindowCfg)]
        L.gf_fm_window_destroy.argtypes = [vp]
        L.gf_fm_window_destroy.restype = None
        L.gf_fm_window_clear.argtypes = [vp]
        L.gf_fm_window_add_frame.argtypes = [vp, i, vp, i, vp, d, ip, vp, dp]
        L.gf_fm_window_add_frame_from_tracker.argtypes = [vp, vp, i, d, ip, vp, dp]
        L.gf_fm_window_triangulate.argtypes = [vp, i, vp, vp, vp, vp]
        L.gf_fm_window_fill_problem.argtypes = [vp, vp, i, ip, vp, vp, ip]
        L.gf_fm_window_set_depth.argtypes = [vp, vp, i]
        L.gf_fm_window_remove_failures.argtypes = [vp]
        L.gf_fm_window_clear_depth.argtypes = [vp]
        L.gf_fm_window_remove_ids.argtypes = [vp, vp, i]
        L.gf_fm_window_remove_back_shift_depth.argtypes = [vp, vp, vp, vp, vp]
        L.gf_fm_window_remove_back.argtypes = [vp]
        L.gf_fm_window_remove_front.argtypes = [vp, i]
        L.gf_fm_window_outliers.argtypes = [vp, vp, vp, vp, vp, i, vp, ip]
        L.gf_fm_window_predict_next.argtypes = [vp, i, vp, vp, vp, vp, vp, vp, ip]
        L.gf_fm_window_read.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, i, ip]
        L.gf_fm_window_size.argtypes = [vp, ip]
        L.gf_fm_window_last_device_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
        L.gf_fm_window_group_create.argtypes = [ctypes.POINTER(vp), vp, i]
        L.gf_fm_window_group_destroy.argtypes = [vp]
        L.gf_fm_window_group_destroy.restype = None
        L.gf_fm_window_group_size.argtypes = [vp, ip]
        L.gf_fm_window_group_add_frame.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        L.gf_fm_window_group_add_frame_from_tracker_group.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
        L.gf_fm_window_group_triangulate.argtypes = [vp, vp, vp, vp, vp, vp]
        L.gf_fm_window_group_fill_problem.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
        L.gf_fm_window_group_set_depth.argtypes = [vp, vp, vp]
        L.gf_fm_window_group_remove.argtypes = [vp, vp, vp, vp]
        L.gf_fm_window_group_remove_failures.argtypes = [vp]
        L.gf_fm_window_group_clear_depth.argtypes = [vp]
        L.gf_fm_window_group_remove_ids.argtypes = [vp, vp, vp]
        L.gf_fm_window_group_outliers.argtypes = [vp, vp, vp, vp, vp, i, vp, vp]
        L.gf_fm_window_group_predict_next.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp]
        L.gf_fm_window_group_last_device_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
        _LIB = L
    return _LIB


YOLO_LIB_PATH = os.path.join(_HERE, "libgf_yolo.so")
_YOLO = None


def yolo_lib():
    """libgf_yolo.so: the YOLO detector's C ABI (gf_detector_*, gf_stage_letterbox, gf_stage_yolo_conv), built next to
    libgf_b200.so."""
    global _YOLO
    if _YOLO is None:
        if not os.path.exists(YOLO_LIB_PATH):
            raise GfError("libgf_yolo.so not built (%s): run `make` or __graft_entry__.build(); "
                          "there is no CPU fallback" % YOLO_LIB_PATH)
        L = ctypes.CDLL(YOLO_LIB_PATH)
        vp, i, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
        ip = ctypes.POINTER(i)
        L.gf_detector_last_error.restype = ctypes.c_char_p
        L.gf_detector_create.argtypes = [ctypes.POINTER(vp), i, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_float]
        L.gf_detector_destroy.argtypes = [vp]
        L.gf_detector_destroy.restype = None
        L.gf_detector_info.argtypes = [vp, vp, ip, ip]
        L.gf_detector_detect.argtypes = [vp, vp, sz, i, i, i, vp, vp, vp, i, ip]
        L.gf_detector_last_device_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
        L.gf_detector_layer_shape.argtypes = [vp, i, vp]
        L.gf_detector_layer_output.argtypes = [vp, i, vp, sz]
        L.gf_detector_layer_times.argtypes = [vp, i, vp]
        L.gf_stage_letterbox.argtypes = [i, vp, sz, i, i, i, i, i, vp]
        L.gf_detector_set_precision.argtypes = [vp, i]
        L.gf_detector_get_precision.argtypes = [vp, ip]
        L.gf_stage_yolo_conv.argtypes = [i, i, vp, vp, vp, vp, vp, vp, vp, vp]
        L.gf_detector_set_max_batch.argtypes = [vp, i]
        L.gf_detector_detect_batch.argtypes = [vp, i, vp, vp, vp, vp, i, vp, vp, vp, i, vp]
        L.gf_detector_member_layer_output.argtypes = [vp, i, i, vp, sz]
        _YOLO = L
    return _YOLO


def check_yolo(rc):
    if rc != 0:
        raise GfError("libgf_yolo error %d: %s" % (rc, yolo_lib().gf_detector_last_error().decode()))


def check(rc):
    if rc != 0:
        raise GfError("libgf_b200 error %d: %s" % (rc, lib().gf_last_error().decode()))


# ---------------------------------------------------------------------------------------------------
# back end (gf_ba_*): ctypes mirrors of the structs in include/gf_b200.h
# ---------------------------------------------------------------------------------------------------
_d = ctypes.c_double
_i = ctypes.c_int32
_dp = ctypes.POINTER(ctypes.c_double)


class BaVisualFactor(ctypes.Structure):
    _fields_ = [("imu_i", _i), ("imu_j", _i), ("feature", _i), ("reserved", _i), ("pts_i", _d * 3), ("pts_j", _d * 3),
                ("vel_i", _d * 2), ("vel_j", _d * 2), ("td_i", _d), ("td_j", _d)]


class BaImuFactor(ctypes.Structure):
    _fields_ = [("i", _i), ("j", _i), ("sum_dt", _d), ("delta_p", _d * 3), ("delta_q", _d * 4), ("delta_v", _d * 3),
                ("linearized_ba", _d * 3), ("linearized_bg", _d * 3), ("jacobian", _d * 225), ("covariance", _d * 225)]


class BaWheelFactor(ctypes.Structure):
    _fields_ = [("i", _i), ("j", _i), ("sum_dt", _d), ("delta_p", _d * 3), ("delta_q", _d * 4), ("jacobian", _d * 18),
                ("covariance", _d * 36), ("linearized_sx", _d), ("linearized_sy", _d), ("linearized_sw", _d), ("linearized_td", _d),
                ("linearized_vel", _d * 3), ("linearized_gyr", _d * 3), ("vel_1", _d * 3), ("gyr_1", _d * 3)]


class BaPrior(ctypes.Structure):
    _fields_ = [("n", _i), ("n_blocks", _i), ("block_kind", _i * 64), ("block_index", _i * 64), ("block_idx", _i * 64),
                ("x0", _dp), ("linearized_jacobians", _dp), ("linearized_residuals", _dp)]


class BaProblem(ctypes.Structure):
    _fields_ = [("n_frames", _i), ("n_features", _i), ("n_visual", _i), ("n_imu", _i), ("n_wheel", _i), ("max_num_iterations", _i),
                ("para_pose", _dp), ("para_speed_bias", _dp), ("para_ex_pose", _dp), ("para_feature", _dp), ("para_td", _dp),
                ("para_ex_wheel", _dp), ("para_ix_wheel", _dp), ("para_td_wheel", _dp),
                ("feature_const", ctypes.POINTER(ctypes.c_uint8)), ("frames_const", _i), ("pose0_const", _i), ("ex_pose_const", _i),
                ("td_const", _i), ("ex_wheel_const", _i), ("ix_wheel_const", _i), ("td_wheel_const", _i),
                ("visual", ctypes.POINTER(BaVisualFactor)), ("imu", ctypes.POINTER(BaImuFactor)), ("wheel", ctypes.POINTER(BaWheelFactor)),
                ("prior", ctypes.POINTER(BaPrior)), ("gravity", _d * 3), ("visual_sqrt_info", _d), ("ex_wheel_subset_mask", _i),
                ("n_plane", _i), ("plane_frames", ctypes.POINTER(_i)), ("para_plane_R", _dp), ("para_plane_Z", _dp), ("plane_const", _i),
                ("plane_r_subset_mask", _i), ("plane_sqrt_info", _d * 3)]


class BaSummary(ctypes.Structure):
    _fields_ = [("iterations", _i), ("num_successful_steps", _i), ("termination", _i), ("reduced_dim", _i), ("n_free_landmarks", _i),
                ("n_residuals", _i), ("initial_cost", _d), ("final_cost", _d), ("cost", _d * 17), ("radius", _d * 17), ("device_ms", _d)]

    def as_dict(self):
        n = self.iterations
        return {"iterations": n, "num_successful_steps": self.num_successful_steps, "termination": self.termination,
                "reduced_dim": self.reduced_dim, "n_free_landmarks": self.n_free_landmarks, "n_residuals": self.n_residuals,
                "initial_cost": self.initial_cost, "final_cost": self.final_cost, "cost": list(self.cost)[:n + 1],
                "radius": list(self.radius)[:n + 1], "device_ms": self.device_ms}


_MAXF = 11          # GF_BA_MAX_FRAMES


class BaStepCapture(ctypes.Structure):
    """gf_ba_step_capture: what the solve computes inside its first iteration (gf_ba_first_step)."""
    ARRAYS = ("imu_sqrt", "H", "Hp", "g", "W", "hll", "scale", "D", "gs", "e_l", "S", "gn", "delta", "Xc")
    _fields_ = ([(n, _i) for n in ("nc", "L", "n", "spill")] + [("col_pose", _i * _MAXF), ("col_sb", _i * _MAXF)]
                + [(n, _i) for n in ("col_ex", "col_td", "col_exw")] + [("col_ix", _i * 3)] + [(n, _i) for n in ("col_tdw", "col_pr", "col_pz")]
                + [(n, _i) for n in ("solver_failed", "step_valid", "done", "termination", "iterations")]
                + [(n, _d) for n in ("initial_cost", "cauchy_num", "cauchy_den", "alpha", "dogleg_a", "dogleg_b", "dogleg_norm",
                                     "model_change", "step_norm", "grad_max", "x_norm", "mu", "radius")]
                + [("col_feat", ctypes.POINTER(_i))] + [(n, _dp) for n in ARRAYS])


BLOCK_POSE, BLOCK_SPEEDBIAS, BLOCK_EX_POSE, BLOCK_TD = 0, 1, 2, 3
BLOCK_EX_WHEEL, BLOCK_SX, BLOCK_SY, BLOCK_SW, BLOCK_TD_WHEEL = 4, 5, 6, 7, 8
BLOCK_PLANE_R, BLOCK_PLANE_Z = 10, 11
# GF_MARG_PATH_* bits (which way a marginalisation went)
MARG_PATH_GENERIC, MARG_PATH_WIDE, MARG_PATH_NOT_PD, MARG_PATH_FORCED, MARG_PATH_REDUCED_JACOBI = 1, 2, 4, 8, 16
# GF_BA_MARGIN_* (gf_ba_marginalize_multi's modes; Estimator::marginalization_flag)
MARGIN_OLD, MARGIN_SECOND_NEW = 0, 1
