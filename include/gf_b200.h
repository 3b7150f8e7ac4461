/*
 * gf_b200.h -- C ABI of libgf_b200.so, the H100 (sm_90a) implementation of Ground-Fusion's two
 * data-parallel hot paths.  Plain pointers and sizes only; no exceptions cross this boundary.
 * Every entry point returns 0 on success or a negative gf_status.  Handles are thread-compatible:
 * one host thread per handle at a time (the reference runs FE on sync_thread and BA on processThread).
 *
 * Reference interfaces replaced (paths relative to /root/reference):
 *   gf_tracker_*   <- class FeatureTracker, vins_estimator/src/featureTracker/feature_tracker.h:43-99
 *   gf_ba_*        <- Estimator::optimization(), vins_estimator/src/estimator/estimator.h:147
 *                     (estimator.cpp:2890-3636) and MarginalizationInfo (factor/marginalization_factor.h)
 */
#ifndef GF_B200_H
#define GF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)   /* the library is built with -fvisibility=hidden */
#endif

typedef enum gf_status {
    GF_OK = 0,
    GF_ERR_INVALID_ARG = -1,
    GF_ERR_CUDA = -2,         /* a CUDA call failed; gf_last_error() has the text */
    GF_ERR_NO_DEVICE = -3,    /* no CUDA device: there is NO CPU fallback */
    GF_ERR_CAPACITY = -4,
    GF_ERR_UNSUPPORTED = -5
} gf_status;

/* Text of the last error raised on the calling thread (never NULL). */
const char* gf_last_error(void);
/* Library version string, e.g. "gf_b200 0.1 sm_90a". */
const char* gf_version(void);
/* Number of kernel launches issued by this library since load (all handles). */
uint64_t gf_kernel_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Front end: FeatureTracker (feature_tracker.h:43-99)
 * ---------------------------------------------------------------------------------------------- */
typedef struct gf_tracker gf_tracker; /* opaque: one per camera stream, bound to one GPU */

typedef struct gf_tracker_cfg {
    int max_cnt;        /* MAX_CNT   (parameters.h:130; groundchallenge.yaml:101)            */
    int min_dist;       /* MIN_DIST  (parameters.h:131; groundchallenge.yaml:102)            */
    int flow_back;      /* FLOW_BACK (parameters.h:134; groundchallenge.yaml:106)            */
    int depth_cam;      /* readIntrinsicParameter(calib, depth): RGB-D mode (feature_tracker.cpp:757-758) */
    double pinhole[8];  /* fx fy cx cy k1 k2 p1 p2 (camodocal PINHOLE; config/realsense/idc_cam.yaml) */
} gf_tracker_cfg;

/* One entry of the map trackImage returns (feature_tracker.cpp:344-366):
 * v = [x_n, y_n, 1, u, v, vx_n, vy_n, depth_m]; camera id is always 0 on this path. */
typedef struct gf_obs {
    int32_t id;
    int32_t track_cnt;
    double v[8];
} gf_obs;

/* Per-call diagnostics the parity tests compare with the oracle ("inlier masks"). */
typedef struct gf_track_info {
    int32_t n_prev;     /* points that entered LK                                           */
    int32_t n_tracked;  /* points that survived status/reverse/border/saturation             */
    int32_t n_kept;     /* ... and survived setMask                                          */
    int32_t n_new;      /* corners added by goodFeaturesToTrack                              */
    int32_t n_candidates; /* GFTT local-maximum candidates before the min-distance pass      */
    int32_t nms_rounds; /* parallel min-distance rounds used                                 */
    int32_t eig_fixups; /* always 0 (kept for ABI stability: the box-filter sums are no longer speculated) */
    int32_t lk_iterations; /* total LK Newton iterations of this frame (all points, levels, both passes) */
} gf_track_info;

/* FeatureTracker::FeatureTracker + readIntrinsicParameter (feature_tracker.cpp:48-54, 745-759). */
int gf_tracker_create(gf_tracker** out, int device, int width, int height, const gf_tracker_cfg* cfg);
void gf_tracker_destroy(gf_tracker* t);

/* Pinned host staging buffers owned by the tracker (width*height u8, width*height u16).  A caller
 * that renders/decodes straight into them avoids one host memcpy; any other pointer is also accepted
 * by gf_tracker_track and is copied into these buffers first. */
int gf_tracker_host_buffers(gf_tracker* t, uint8_t** gray, uint16_t** depth);

/* FeatureTracker::trackImage(t, img, depth) (feature_tracker.cpp:103-372).
 *   gray: H x W u8, row pitch gray_pitch bytes; only read during the call (as cv::Mat in the reference)
 *   depth: H x W u16 millimetres or NULL (then v[7] = -2.4 as feature_tracker.cpp:338)
 *   out: caller-allocated, capacity >= cfg.max_cnt; entries are in the tracker's internal order
 *        (the reference's std::map iterates by id: sort by id on the caller side if needed)
 *   status_out (nullable, capacity >= max_cnt): combined status of the n_prev points that entered LK
 *        (LK status & reverse check & inBorder & grey<=250), i.e. the reference's `status` vector at
 *        feature_tracker.cpp:170 */
int gf_tracker_track(gf_tracker* t, double time, const uint8_t* gray, size_t gray_pitch,
                     const uint16_t* depth, size_t depth_pitch, gf_obs* out, int* n_out,
                     uint8_t* status_out, gf_track_info* info);

/* Asynchronous split of gf_tracker_track.  _submit enqueues the copies and kernels of one frame and returns;
 * _wait blocks for the result of the OLDEST frame not yet collected.  Up to two frames may be in flight
 * (submit t, submit t+1, wait t, submit t+2, wait t+1, ...): the upload, pyramid and min-eig map of frame t+1 then
 * overlap the tracking of frame t, which is how a recorded sequence (rosbag replay) or a camera with one frame of
 * buffering is processed at the rate of the dependent chain alone.  Results are identical to the blocking call.
 * Pinned caller buffers passed to _submit must stay unchanged until that frame has been collected.
 * gf_tracker_set_prediction / gf_tracker_remove_ids act on the state after the last collected frame and are
 * therefore only accepted with no frame in flight, exactly as the reference calls them between trackImage calls. */
int gf_tracker_submit(gf_tracker* t, double time, const uint8_t* gray, size_t gray_pitch,
                      const uint16_t* depth, size_t depth_pitch);
int gf_tracker_wait(gf_tracker* t, gf_obs* out, int* n_out, uint8_t* status_out, gf_track_info* info);

/* Device-resident variant used by bench.py's kernel-only `value`: the frame is already in HBM
 * (device pointers, tightly packed W x H), nothing is copied from the host. */
int gf_tracker_track_device(gf_tracker* t, double time, const void* d_gray, const void* d_depth,
                            gf_obs* out, int* n_out, uint8_t* status_out, gf_track_info* info);
/* Asynchronous form of gf_tracker_track_device (collect with gf_tracker_wait; same two-frame rule as _submit). */
int gf_tracker_submit_device(gf_tracker* t, double time, const void* d_gray, const void* d_depth);

/* A recorded run of n consecutive frames (rosbag replay, one call per batch): the same submit / wait pipeline as above,
 * two frames in flight, driven from inside the library so that the host costs one call per batch instead of ~10 driver
 * calls per frame.  Frame k = (times[k], gray[k], depth[k] or NULL / depth == NULL); on_device != 0: the pointers are
 * device pointers to tightly packed frames (pitches ignored), else host pointers with the given row pitches (pinned
 * buffers make the uploads asynchronous).  Results of frame k land at out + k*max_cnt, n_out[k],
 * status_out + k*max_cnt, info[k] (each nullable).  Identical to n calls of gf_tracker_track. */
int gf_tracker_track_batch(gf_tracker* t, int n, const double* times, const void* const* gray, size_t gray_pitch,
                           const void* const* depth, size_t depth_pitch, int on_device,
                           gf_obs* out, int* n_out, uint8_t* status_out, gf_track_info* info);
/* The same for several independent camera streams at once (a multi-camera rig, several robots served by one GPU): stream i
 * is trackers[i] with frames times / gray / depth [i*n + k] and results at out + (i*n + k)*max_cnt, n_out / info [i*n + k],
 * status_out + (i*n + k)*max_cnt.  One host thread feeds all streams round-robin (frame k of every stream is enqueued before
 * frame k-1 of any stream is collected), so a server does not need one thread per camera: measured on one H100 SXM at 700 W,
 * 8 streams reach 26.6-27.0 k frames/s this way and 20.6-26.9 k with 8 threads calling gf_tracker_track_batch.  Results are identical to calling
 * gf_tracker_track_batch per stream. */
int gf_tracker_track_batch_multi(gf_tracker* const* trackers, int n_trackers, int n, const double* times, const void* const* gray,
                                 size_t gray_pitch, const void* const* depth, size_t depth_pitch, int on_device,
                                 gf_obs* out, int* n_out, uint8_t* status_out, gf_track_info* info);

/* FeatureTracker::setPrediction (feature_tracker.cpp:1006-1027): xyz are camera-frame 3-D points. */
int gf_tracker_set_prediction(gf_tracker* t, const int32_t* ids, const double* xyz, int n);
/* FeatureTracker::removeOutliers (feature_tracker.cpp:1029-1045). */
int gf_tracker_remove_ids(gf_tracker* t, const int32_t* ids, int n);

/* Device time (ms, CUDA events) from the first copy to the result copy of the last collected frame (its latency;
 * with two frames in flight consecutive latencies overlap). */
int gf_tracker_last_device_ms(gf_tracker* t, float* ms);
/* Device-side stopwatch over a run of frames: _start records a CUDA event ahead of the next frame's first copy,
 * _stop one behind the last frame's result copy and returns the elapsed ms.  Both need no frame in flight. */
int gf_tracker_timer_start(gf_tracker* t);
int gf_tracker_timer_stop(gf_tracker* t, float* ms);
/* Optional per-stage CUDA-event timing (adds event records, no synchronisation).  Stage order:
 * 0 upload, 1 pyramid, 2 lk (k_track), 3 setmask, 4 gftt select (mask..nms), 5 finalize, 6 download,
 * 7 min-eig (runs on the upload/pyramid stream, overlaps 2-3).  Profiling mode runs one frame at a time. */
#define GF_FE_STAGES 8
int gf_tracker_set_profiling(gf_tracker* t, int enable);
int gf_tracker_last_stage_ms(gf_tracker* t, float* ms /* GF_FE_STAGES */);
/* Development aid: clock64 phase counters of the single-CTA kernels ([0..63]) and per-feature LK cycles/iterations
 * ([64 + 8*i], [64 + 8*i + 1]).  n <= 64 + 8*1024. */
int gf_tracker_debug_read(gf_tracker* t, long long* out, int n);

/* ------------------------------------------------------------------------------------------------
 * Stage-level entry points (same kernels as the tracker; used by the parity tests, which read like
 * tests of the three OpenCV calls the reference makes).  All pointers are HOST pointers.
 * ---------------------------------------------------------------------------------------------- */
/* cv::pyrDown on u8 (LK pyramid level). dst is ((w+1)/2) x ((h+1)/2), tightly packed. */
int gf_stage_pyr_down(int device, const uint8_t* src, int w, int h, uint8_t* dst);
/* cv::cornerMinEigenVal(img, blockSize=3, ksize=3) as used by goodFeaturesToTrack. */
int gf_stage_min_eig(int device, const uint8_t* img, int w, int h, float* eig, int* n_fixups);
/* cv::calcOpticalFlowPyrLK(prev, next, prev_pts, next_pts, status, err, Size(21,21), max_level,
 * TermCriteria(COUNT+EPS,30,0.01), use_initial_flow ? OPTFLOW_USE_INITIAL_FLOW : 0). */
int gf_stage_lk(int device, const uint8_t* prev, const uint8_t* next, int w, int h,
                const float* prev_pts, float* next_pts, int n, int max_level, int use_initial_flow,
                uint8_t* status);
/* cv::goodFeaturesToTrack(img, max_corners, 0.01, min_dist, mask) where mask = 255 everywhere except
 * the integer disks d^2 <= min_dist^2 around cvRound(kept_pts[i]) (setMask, feature_tracker.cpp:56-83).
 * Returns the corners in OpenCV's output order. */
int gf_stage_gftt(int device, const uint8_t* img, int w, int h, const float* kept_pts, int n_kept,
                  int max_corners, int min_dist, float* corners, int* n_corners, gf_track_info* info);
/* The permutation libstdc++'s std::sort produces for setMask's comparator (device replica). */
int gf_stage_setmask_order(int device, const int32_t* track_cnt, int n, int32_t* perm);

/* The back end's dense linear solver on its own (same device code as gf_ba_solve: 8x8-tile left-looking Cholesky with FP64
 * tensor-core MMAs + back substitution; replaces Ceres' dense Cholesky of the reduced camera system, call site
 * estimator.cpp:3303-3318): x = A^-1 b for a symmetric positive definite A (n x n row-major, lower triangle read),
 * 1 <= n <= 383.  tile_cap < 0: default number of factor tiles kept in shared memory; smaller values force the L2 spill
 * path (tests). */
int gf_stage_spd_solve(int device, const double* A, const double* b, int n, double* x, int tile_cap);

/* Measured FP64 rates of the whole device (GFLOP/s, 2 flops per FMA): plain DFMA and tensor-core DMMA.8x8x4.  bench.py
 * quotes the back end's roofline fraction against these (MEASURED_PEAKS.json holds no FP64 figure). */
int gf_probe_fp64(int device, double* dfma_gflops, double* dmma_gflops);

/* ------------------------------------------------------------------------------------------------
 * Back end: Estimator::optimization() (estimator.cpp:2890-3636).  The caller (the Estimator adaptor)
 * fills one gf_ba_problem per call from its members exactly where the reference builds the
 * ceres::Problem (estimator.cpp:2895-3300); the library replaces ceres::Solve (DENSE_SCHUR + DOGLEG,
 * estimator.cpp:3303-3318) and writes the optimised parameter blocks back in place.
 * All doubles; quaternions are stored x,y,z,w as in para_Pose (estimator.cpp:2276-2353).
 * ---------------------------------------------------------------------------------------------- */
#define GF_BA_MAX_FRAMES 11          /* WINDOW_SIZE + 1 (parameters.h:24) */
#define GF_BA_MAX_ITERATIONS 16

/* ProjectionTwoFrameOneCamFactor (factor/projectionTwoFrameOneCamFactor.h:21, .cpp:43-151) */
typedef struct gf_ba_visual_factor {
    int32_t imu_i, imu_j;     /* para_Pose[imu_i], para_Pose[imu_j]                      */
    int32_t feature;          /* para_Feature[feature]                                     */
    int32_t reserved;
    double pts_i[3], pts_j[3];
    double vel_i[2], vel_j[2];
    double td_i, td_j;
} gf_ba_visual_factor;

/* IMUFactor (factor/imu_factor.h:20-191) with the IntegrationBase members Evaluate reads
 * (factor/integration_base.h:169-195): delta_{p,q,v}, jacobian, covariance, linearized biases. */
typedef struct gf_ba_imu_factor {
    int32_t i, j;             /* para_Pose[i], para_SpeedBias[i], para_Pose[j], para_SpeedBias[j] */
    double sum_dt;
    double delta_p[3], delta_q[4], delta_v[3];
    double linearized_ba[3], linearized_bg[3];
    double jacobian[225];     /* 15x15 row-major, order O_P O_R O_V O_BA O_BG               */
    double covariance[225];
} gf_ba_imu_factor;

/* WheelFactor (factor/wheel_factor.h:20-247) with the WheelIntegrationBase members it reads. */
typedef struct gf_ba_wheel_factor {
    int32_t i, j;
    double sum_dt;
    double delta_p[3], delta_q[4];
    double jacobian[18];      /* 6x3 row-major: d(p,q)/d(sx,sy,sw)                           */
    double covariance[36];
    double linearized_sx, linearized_sy, linearized_sw, linearized_td;
    double linearized_vel[3], linearized_gyr[3], vel_1[3], gyr_1[3];
} gf_ba_wheel_factor;

typedef enum gf_ba_block_kind {
    GF_BA_BLOCK_POSE = 0, GF_BA_BLOCK_SPEEDBIAS = 1, GF_BA_BLOCK_EX_POSE = 2, GF_BA_BLOCK_TD = 3,
    GF_BA_BLOCK_EX_WHEEL = 4, GF_BA_BLOCK_SX = 5, GF_BA_BLOCK_SY = 6, GF_BA_BLOCK_SW = 7,
    GF_BA_BLOCK_TD_WHEEL = 8, GF_BA_BLOCK_FEATURE = 9, GF_BA_BLOCK_PLANE_R = 10, GF_BA_BLOCK_PLANE_Z = 11
} gf_ba_block_kind;

/* MarginalizationInfo as consumed by MarginalizationFactor::Evaluate
 * (factor/marginalization_factor.cpp:332-392): r = r0 + J0 * dx(x, x0). */
typedef struct gf_ba_prior {
    int32_t n;                        /* rows = columns = kept local dimension (0: no prior)     */
    int32_t n_blocks;                 /* keep_block_size.size()                                   */
    int32_t block_kind[64];           /* gf_ba_block_kind of every kept block                     */
    int32_t block_index[64];          /* frame index for POSE / SPEEDBIAS, 0 otherwise            */
    int32_t block_idx[64];            /* keep_block_idx - m: first column of the block            */
    const double* x0;                 /* keep_block_data, concatenated in block order (global sizes) */
    const double* linearized_jacobians; /* n x n, row-major                                       */
    const double* linearized_residuals; /* n                                                      */
} gf_ba_prior;

typedef struct gf_ba_problem {
    int32_t n_frames;                 /* frame_count + 1, <= GF_BA_MAX_FRAMES                     */
    int32_t n_features;               /* entries of para_feature                                  */
    int32_t n_visual, n_imu, n_wheel;
    int32_t max_num_iterations;       /* NUM_ITERATIONS (estimator.cpp:3308)                      */
    /* parameter blocks, updated in place by gf_ba_solve */
    double* para_pose;                /* [n_frames][7]                                            */
    double* para_speed_bias;          /* [n_frames][9]                                            */
    double* para_ex_pose;             /* [7]  para_Ex_Pose[0]                                     */
    double* para_feature;             /* [n_features] inverse depths                              */
    double* para_td;                  /* [1]                                                      */
    double* para_ex_wheel;            /* [7]  para_Ex_Pose_wheel[0]  (read only if n_wheel > 0)   */
    double* para_ix_wheel;            /* [3]  sx sy sw                                            */
    double* para_td_wheel;            /* [1]                                                      */
    /* SetParameterBlockConstant decisions (estimator.cpp:2960-3100, 3233-3246, 3291-3292) */
    const uint8_t* feature_const;     /* [n_features] 1 = depth from the depth image, held fixed  */
    int32_t frames_const;             /* systemstationary && stationary_detect                    */
    int32_t pose0_const;              /* !USE_IMU                                                 */
    int32_t ex_pose_const, td_const, ex_wheel_const, ix_wheel_const, td_wheel_const;
    const gf_ba_visual_factor* visual;
    const gf_ba_imu_factor* imu;
    const gf_ba_wheel_factor* wheel;
    const gf_ba_prior* prior;         /* nullable                                                 */
    double gravity[3];                /* global G (parameters.cpp:74)                             */
    double visual_sqrt_info;          /* FOCAL_LENGTH / 1.5 (estimator.cpp:193)                   */
    int32_t ex_wheel_subset_mask;     /* PoseSubsetParameterization of para_Ex_Pose_wheel (estimator.cpp:3008-3027):
                                       * bit k set = local component k (0-2 translation, 3-5 rotation) is zeroed in Plus;
                                       * 0 = PoseLocalParameterization                              */
    /* PlaneFactor (factor/plane_factor.h:20-118, USE_PLANE): one factor per listed frame on (para_Pose[i],
     * para_Ex_Pose_wheel, para_plane_R, para_plane_Z).  para_ex_wheel must then be given even without wheel factors. */
    int32_t n_plane;
    const int32_t* plane_frames;      /* [n_plane] frame index of every PlaneFactor (estimator.cpp:3152-3166)     */
    double* para_plane_R;             /* [4] x y z w, updated in place                                            */
    double* para_plane_Z;             /* [1]                                                                      */
    int32_t plane_const;              /* both plane blocks constant (estimator.cpp:3064-3074)                     */
    int32_t plane_r_subset_mask;      /* OrientationSubsetParameterization: bit k = local component k zeroed in
                                       * Plus; the reference uses {2} -> 0b100                                    */
    double plane_sqrt_info[3];        /* PITCH_N_INV, ROLL_N_INV, ZPW_N_INV                                       */
} gf_ba_problem;

typedef enum gf_ba_termination {
    GF_BA_NO_CONVERGENCE = 0,         /* max_num_iterations reached                               */
    GF_BA_CONVERGENCE_FUNCTION = 1, GF_BA_CONVERGENCE_PARAMETER = 2, GF_BA_CONVERGENCE_GRADIENT = 3,
    GF_BA_FAILURE = 4
} gf_ba_termination;

typedef struct gf_ba_summary {
    int32_t iterations;               /* iterations run (successful or not), excluding iteration 0 */
    int32_t num_successful_steps;
    int32_t termination;              /* gf_ba_termination                                        */
    int32_t reduced_dim, n_free_landmarks, n_residuals;
    double initial_cost, final_cost;
    double cost[GF_BA_MAX_ITERATIONS + 1];    /* cost after iteration k (k = 0: initial)          */
    double radius[GF_BA_MAX_ITERATIONS + 1];  /* trust-region radius after iteration k            */
    double device_ms;                 /* CUDA-event time of the solve (0 for the CPU oracle)      */
} gf_ba_summary;

typedef struct gf_ba gf_ba;           /* opaque solver workspace bound to one GPU */
int gf_ba_create(gf_ba** out, int device);
void gf_ba_destroy(gf_ba* s);
/* ceres::Solve + double2vector's input: optimises the blocks of `p` in place. */
int gf_ba_solve(gf_ba* s, const gf_ba_problem* p, gf_ba_summary* summary);
/* Counters of the last solve (32 slots).  [30] = SM cycles (clock64) spent inside the k_ba_step launches that took a
 * trust-region step, [31] = their number: bench.py derives the step kernel's achieved FP64 rate from them.  Slots 0..15 are
 * per-phase cycles and only filled in a -DGF_PROFILE build. */
int gf_ba_debug_profile(gf_ba* s, long long* out32);

/* MARGIN_OLD: the marginalisation at the end of Estimator::optimization() (estimator.cpp:3334-3535) with
 * MarginalizationInfo::{preMarginalize, marginalize} (factor/marginalization_factor.cpp:115-308) on the GPU.
 * Input: the window as it stands after the solve (same descriptor as gf_ba_solve; the constancy flags are ignored, as
 * the reference's MarginalizationInfo ignores SetParameterBlockConstant).  Factors: the last prior, IMUFactor(0->1),
 * WheelFactor(0->1) (when the window has wheel factors), PlaneFactor on frame 0 (when plane_frames lists frame 0) and every
 * visual factor whose landmark starts in frame 0.  Output: the prior for the NEXT window -- kept blocks ordered pose[1..],
 * speedbias[1..], ex_pose, td, wheel extrinsic, sx, sy, sw, wheel time offset, plane rotation (4 columns: MarginalizationInfo
 * only knows the 7 -> 6 local size), plane height, with frame indices already shifted by one, their linearisation points,
 * J0 = sqrt(S) V^T (n x n row-major) and r0 = sqrt(S^-1) V^T b.
 *   out_x0 / out_J / out_r: caller buffers of 16*n_frames+24, n*n, n doubles (n <= 16*n_frames+22); `out` points into them.
 *   device_ms: nullable, CUDA-event time.
 * Returns n > 0, or a negative gf error code.  GNSS factors are not implemented (gnss_comm is not vendored). */
int gf_ba_marginalize_old(gf_ba* s, const gf_ba_problem* p, gf_ba_prior* out, double* out_x0, double* out_J, double* out_r,
                          float* device_ms);

/* MARGIN_SECOND_NEW (estimator.cpp:3536-3631): the only factor is the last prior evaluated at the current state; para_Pose
 * [WINDOW_SIZE - 1] (frame n_frames - 2 of the descriptor) is marginalised by the same eigen-truncated Schur complement
 * (preMarginalize + marginalize) and frame n_frames - 1 takes its index (addr_shift, estimator.cpp:3583-3621).  Same buffers
 * as gf_ba_marginalize_old.  Returns n > 0, 0 when the prior does not hold that pose (the reference then keeps the prior
 * unchanged: estimator.cpp:3538-3539), or a negative error code. */
int gf_ba_marginalize_second_new(gf_ba* s, const gf_ba_problem* p, gf_ba_prior* out, double* out_x0, double* out_J, double* out_r,
                                 float* device_ms);

/* Estimator::double2vector (estimator.cpp:2440-2494), the state part: host-only glue that maps the solved para_* arrays
 * back to Rs / Ps / Vs, rotating the window about z and shifting it so that frame 0 keeps the yaw and position it had
 * before the solve (Euler-singularity branch included).
 *   R0_before: Rs[0] before the solve, 3x3 row-major; P0_before: Ps[0]; use_imu: USE_IMU (0: plain copy)
 *   Rs [n_frames][9] row-major, Ps [n_frames][3], Vs [n_frames][3] (nullable) */
int gf_ba_double2vector(const gf_ba_problem* p, const double* R0_before, const double* P0_before, int use_imu,
                        double* Rs, double* Ps, double* Vs);

/* ------------------------------------------------------------------------------------------------
 * FeatureManager kernels (vins_estimator/src/estimator/feature_manager.cpp): the per-landmark work either side of
 * Estimator::optimization().  The observation lists (std::list<FeaturePerId>) stay with the caller and are passed flattened:
 * landmark i has n_obs[i] consecutive observations from frame start_frame[i] on, stored at obs_offset[i] in points
 * (FeaturePerFrame::point, xyz) / depths (FeaturePerFrame::depth).  All pointers are HOST pointers.
 * ---------------------------------------------------------------------------------------------- */
/* FeatureManager::triangulateWithDepth (:726-799) followed by FeatureManager::triangulate (:668-723), as processImage calls
 * them (estimator.cpp:1090-1102): landmarks with >= 4 observations and estimated_depth <= 0 get a depth -- the mean of the
 * RGB-D depths (0.1 .. depth_threshold) that re-project within 10/460 into another frame (estimate_flag 1), else the DLT
 * depth over all observations (flag 2); results < 0.1 become init_depth (flag 0).  Ps [n_frames][3], Rs [n_frames][9] row-major. */
int gf_fm_triangulate(int device, int n_features, const int32_t* start_frame, const int32_t* n_obs, const int32_t* obs_offset, int n_obs_total,
                      const double* points, const double* depths, double* estimated_depth, int32_t* estimate_flag,
                      int n_frames, const double* Ps, const double* Rs, const double* tic, const double* ric, double depth_threshold, double init_depth);
/* Sum of FeatureManager::compensatedParallax2 (:977-1011) over n landmarks: pts_i / pts_j are their points (xyz) in frames
 * frame_count-2 / frame_count-1 (addFeatureCheckParallax :96-104 divides by n and compares with MIN_PARALLAX). */
int gf_fm_parallax(int device, int n, const double* pts_i, const double* pts_j, double* parallax_sum);
/* The depth transfer of FeatureManager::removeBackShiftDepth (:838-849) for n landmarks that start in the marginalised frame:
 * uv_i = their first observation (xyz), estimated_depth updated in place (<= 0 after the transfer -> init_depth). */
int gf_fm_back_shift_depth(int device, int n, const double* uv_i, double* estimated_depth, const double* marg_R, const double* marg_P,
                           const double* new_R, const double* new_P, double init_depth);

/* The per-landmark loops of the estimator that run after optimization() and feed the front end back (single-threaded mode,
 * estimator.cpp:1115-1140).  Same flattened observation lists as gf_fm_triangulate.
 * Estimator::outliersRejection (:3909-3966) and Estimator::movingConsistencyCheckW (:3968-4011) both average, per landmark, the
 * reprojection error of its first observation into every later one (reprojectionError :3888-3898, reprojectionError3D
 * :3900-3907): err2d_sum[i], err3d_sum[i] = the sums, count[i] = the number of later observations.  The thresholds stay with
 * the caller (outliersRejection: n_obs >= 4 and FOCAL_LENGTH * err2d / count > 3; movingConsistencyCheckW: n_obs >= 2,
 * start_frame < WINDOW_SIZE - 2, depth >= 0 and FOCAL_LENGTH * err2d / count > 10 or err3d / count > 2). */
int gf_fm_reprojection_errors(int device, int n_features, const int32_t* start_frame, const int32_t* n_obs, const int32_t* obs_offset, int n_obs_total,
                              const double* points, const double* estimated_depth, int n_frames, const double* Ps, const double* Rs, const double* tic,
                              const double* ric, double* err2d_sum, double* err3d_sum, int32_t* count);
/* Estimator::predictPtsInNextFrame (:3853-3886): n landmarks (estimated_depth > 0, >= 2 observations, seen in frame frame_count:
 * the caller's selection) given by their first frame, first observation (xyz) and depth, carried into the camera of the next
 * frame predicted by constant-velocity motion nextT = curT (prevT^-1 curT).  pts_cam [n][3] is what FeatureTracker::setPrediction
 * (gf_tracker_set_prediction) takes. */
int gf_fm_predict_next(int device, int n, const int32_t* first_frame, const double* uv_first, const double* estimated_depth, int n_frames, int frame_count,
                       const double* Ps, const double* Rs, const double* tic, const double* ric, double* pts_cam);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* GF_B200_H */
