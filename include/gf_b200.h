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

/* Pinned host staging buffers owned by the tracker (width*height u8, width*height u16).  A caller that renders/decodes
 * straight into them and submits them gets truly asynchronous uploads; any other host pointer is also accepted (see
 * gf_tracker_submit). */
int gf_tracker_host_buffers(gf_tracker* t, uint8_t** gray, uint16_t** depth);

/* The config key `use_yolo` (parameters.cpp:159): FeatureTracker::trackImagebox (feature_tracker.cpp:374-678), which
 * Estimator::inputImagebox (estimator.cpp:244-273) calls on every frame whose detection message has the frame's timestamp.  It is
 * trackImage with one difference: a feature strictly inside a detected box, pointPolygonTest(contour of the box, pt, true) > 0, is
 * left out of featureFrame.  It stays in the tracker (cur_pts / ids / track_cnt / velocity history): it is tracked on the next
 * frame and counts against max_cnt.  The boxes are the fields of darknet_ros_msgs/BoundingBox; the reference copies them into
 * `int`, and so does the library (a modular wrap of values outside int32).  darknet_ros publishes at most GF_MAX_BOXES boxes
 * per frame (YoloObjectDetector.cpp:559). */
#define GF_MAX_BOXES 100
typedef struct gf_box { int64_t xmin, ymin, xmax, ymax; } gf_box;

/* FeatureTracker::trackImage(t, img, depth) (feature_tracker.cpp:103-372), and trackImagebox(t, img, depth, boxes) when
 * n_boxes > 0.  Blocking: gf_tracker_submit followed by gf_tracker_wait; no frame may be in flight.
 *   gray: H x W u8; depth: H x W u16 millimetres or NULL (then v[7] = -2.4 as feature_tracker.cpp:338).  on_device == 0: host
 *        pointers with row pitches gray_pitch / depth_pitch bytes, only read during the call (as cv::Mat in the reference).
 *        on_device != 0: device pointers to tightly packed frames already in HBM, nothing is copied from the host (the pitches
 *        are ignored); bench.py's kernel-only `value` runs this way.
 *   boxes: the frame's n_boxes detections; boxes == NULL, n_boxes == 0 is trackImage.  n_boxes > GF_MAX_BOXES: GF_ERR_CAPACITY;
 *        n_boxes < 0 or boxes == NULL with n_boxes > 0: GF_ERR_INVALID_ARG; in both cases no frame is consumed.
 *   out: caller-allocated, capacity >= cfg.max_cnt; entries are in the tracker's internal order
 *        (the reference's std::map iterates by id: sort by id on the caller side if needed)
 *   in_box (nullable, capacity >= max_cnt): in_box[i] = 1 for the entries of out that trackImagebox leaves out of featureFrame,
 *        0 otherwise (all 0 for a frame without boxes).  out / n_out / status_out / info are exactly what trackImage returns.
 *   status_out (nullable, capacity >= max_cnt): combined status of the n_prev points that entered LK
 *        (LK status & reverse check & inBorder & grey<=250), i.e. the reference's `status` vector at
 *        feature_tracker.cpp:170
 * The box test runs on the device, inside the last kernel of the frame; without boxes the same kernels run. */
int gf_tracker_track(gf_tracker* t, double time, const void* gray, size_t gray_pitch, const void* depth, size_t depth_pitch,
                     int on_device, const gf_box* boxes, int n_boxes, gf_obs* out, int* n_out, uint8_t* in_box,
                     uint8_t* status_out, gf_track_info* info);

/* Asynchronous split of gf_tracker_track, with its arguments.  _submit enqueues the copies and kernels of one frame and
 * returns (the boxes are copied before it returns); _wait blocks for the result of the OLDEST frame not yet collected, whatever
 * intake it came through.  Up to two frames may be in flight (submit t, submit t+1, wait t, submit t+2, wait t+1, ...): the
 * upload, pyramid and min-eig map of frame t+1 then overlap the tracking of frame t, which is how a recorded sequence (rosbag
 * replay) or a camera with one frame of buffering is processed at the rate of the dependent chain alone.  Results are
 * identical to the blocking call.  _submit reads host frames with the copy engine after it returns: truly asynchronous from
 * pinned memory (gf_tracker_host_buffers, cudaHostAlloc, cudaHostRegister), which must stay unchanged until that frame has
 * been collected; pageable memory is staged by CUDA before the call returns.
 * gf_tracker_set_prediction / gf_tracker_remove_ids act on the state after the last collected frame and are
 * therefore only accepted with no frame in flight, exactly as the reference calls them between trackImage calls. */
int gf_tracker_submit(gf_tracker* t, double time, const void* gray, size_t gray_pitch, const void* depth, size_t depth_pitch,
                      int on_device, const gf_box* boxes, int n_boxes);
int gf_tracker_wait(gf_tracker* t, gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info);

/* A recorded run of n consecutive frames (rosbag replay, one call per batch): the same submit / wait pipeline as above,
 * two frames in flight, driven from inside the library so that the host costs one call per batch instead of ~10 driver
 * calls per frame.  Frame k = (times[k], gray[k], depth[k] or NULL / depth == NULL), on_device and the pitches as for
 * gf_tracker_track (pinned host buffers make the uploads asynchronous); its boxes are boxes[box_start[k] .. box_start[k + 1])
 * (n + 1 offsets; box_start NULL: no boxes).  Every box list is checked before the first frame is submitted.  Results of
 * frame k land at out + k*max_cnt, n_out[k], in_box + k*max_cnt, status_out + k*max_cnt, info[k] (each nullable).
 * Identical to n calls of gf_tracker_track. */
int gf_tracker_track_batch(gf_tracker* t, int n, const double* times, const void* const* gray, size_t gray_pitch,
                           const void* const* depth, size_t depth_pitch, int on_device, const gf_box* boxes, const int* box_start,
                           gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info);
/* The same for several independent camera streams at once (a multi-camera rig, several robots served by one GPU): stream i
 * is trackers[i] with frame j = i*n + k at times / gray / depth [j], boxes[box_start[j] .. box_start[j + 1]) (n_trackers*n + 1
 * offsets) and results at out + j*max_cnt, n_out[j], in_box + j*max_cnt, status_out + j*max_cnt, info[j].  One host thread
 * feeds all streams round-robin (frame k of every stream is enqueued before frame k-1 of any stream is collected), so a server
 * does not need one thread per camera: measured on one H100 SXM at 700 W, 8 streams reach 26.6-27.0 k frames/s this way and
 * 20.6-26.9 k with 8 threads calling gf_tracker_track_batch.  Results are identical to calling gf_tracker_track_batch per
 * stream. */
int gf_tracker_track_batch_multi(gf_tracker* const* trackers, int n_trackers, int n, const double* times, const void* const* gray,
                                 size_t gray_pitch, const void* const* depth, size_t depth_pitch, int on_device,
                                 const gf_box* boxes, const int* box_start, gf_obs* out, int* n_out, uint8_t* in_box,
                                 uint8_t* status_out, gf_track_info* info);

/* The config key `equalize` (parameters.h:33): cv::createCLAHE(clip_limit, Size(tiles_x, tiles_y))->apply on every gray frame
 * before it is tracked, as getImageFromMsg does (rosNodeTest.cpp:256-261; the reference's call is createCLAHE() with its
 * defaults, clip_limit 40 and an 8 x 8 grid).  LK on both pyramids, goodFeaturesToTrack and the grey > 250 test then all see
 * the equalised image, bit-exact with OpenCV 4.13.  Off by default; tiles_x = 0 turns it off.  1 <= tiles_x, tiles_y <= 16;
 * clip_limit <= 0: no clipping.  Accepted only before the first frame is submitted (GF_ERR_INVALID_ARG afterwards).
 * Covers every intake path: host and device frames, _track / _submit and the batch calls. */
int gf_tracker_set_equalize(gf_tracker* t, double clip_limit, int tiles_x, int tiles_y);

/* A tracker group: n existing trackers (members) that track frame k of their streams in lockstep, one step at a time, with
 * ONE set of launches per step: every kernel of the frame runs once for the whole group (member = a grid dimension), so the
 * launch count and the driver calls per step do not grow with n.  Member i's results and its state afterwards are exactly
 * what gf_tracker_track_batch on that member alone would give (same kernels, same arithmetic).  A step ends with its slowest
 * member: the group trades per-camera latency for throughput (gf_tracker_track_batch_multi keeps the streams independent).
 *   _create: 1 <= n <= GF_TRACKER_GROUP_MAX (more: GF_ERR_CAPACITY).  The members must be distinct, bound to the same device,
 *       with the same width, height, max_cnt, min_dist, flow_back and depth_cam, and the same equalize setting and CLAHE
 *       geometry (pinhole may differ); none may have a frame in flight or be in profiling mode.  Any other violation is
 *       GF_ERR_INVALID_ARG, with gf_last_error() starting "member k: " for the member at fault.
 *   State stays in the members: a step reads and advances each member's features, frame counter, time of the last frame,
 *       pending prediction and depth flags.  Between steps (no step in flight) a member may be used directly
 *       (gf_tracker_set_prediction, _remove_ids, _track, batches); the next step continues from there.  A step in flight
 *       counts as a frame in flight on every member, so direct calls (the _submit calls included) are refused
 *       until it is collected by gf_tracker_group_wait (gf_tracker_wait on a member refuses to collect it).  A member whose
 *       equalize setting was changed after the group was created makes _submit fail ("member k: ...").
 *   _destroy: the members stay usable (a step still in flight is completed and dropped).  Destroying a member that belongs to
 *       a live group is a caller error.
 *   _submit: one step, two steps in flight at most (as gf_tracker_submit): member i tracks times[i], gray[i], depth[i] (depth
 *       nullable, and NULL entries: no depth image); on_device and the pitches as gf_tracker_submit; boxes / box_start:
 *       member i's detections are boxes[box_start[i] .. box_start[i + 1]) (n + 1 offsets; box_start NULL: no boxes).  Every
 *       member's pointers and box list are checked before anything is enqueued: an argument error consumes no frame.
 *   _wait: collects the oldest step: member i's results at out + i*max_cnt, n_out[i], in_box + i*max_cnt,
 *       status_out + i*max_cnt, info[i] (each nullable), as gf_tracker_wait returns them.
 *   _track_batch: n_steps steps in one call, two in flight, with the arguments and layout of
 *       gf_tracker_track_batch_multi (member i = stream i: frame k at [i*n_steps + k]).
 * gf_tracker_last_device_ms of a member reports the device time of the last collected step. */
typedef struct gf_tracker_group gf_tracker_group;
#define GF_TRACKER_GROUP_MAX 64
int gf_tracker_group_create(gf_tracker_group** out, gf_tracker* const* members, int n);
void gf_tracker_group_destroy(gf_tracker_group* g);
int gf_tracker_group_submit(gf_tracker_group* g, const double* times, const void* const* gray, size_t gray_pitch,
                            const void* const* depth, size_t depth_pitch, int on_device, const gf_box* boxes, const int* box_start);
int gf_tracker_group_wait(gf_tracker_group* g, gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info);
int gf_tracker_group_track_batch(gf_tracker_group* g, int n_steps, const double* times, const void* const* gray, size_t gray_pitch,
                                 const void* const* depth, size_t depth_pitch, int on_device, const gf_box* boxes, const int* box_start,
                                 gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info);

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
 * ([64 + 8*i], [64 + 8*i + 1]); of those iterations, the ones whose mismatch vector came from exact integer sums and
 * the ones that ran the sequential float chains ([64 + 8*i + 2], [64 + 8*i + 3]); the LK form of the frame's k_track
 * ([64 + 8*i + 4]: 2 = two warp roles, the tracker alone on its device; 1 = single role).  Rows past the frame's n_prev
 * are stale.  n <= 64 + 8*1024. */
int gf_tracker_debug_read(gf_tracker* t, long long* out, int n);

/* ------------------------------------------------------------------------------------------------
 * Stage-level entry points (same kernels as the tracker; used by the parity tests, which read like
 * tests of the three OpenCV calls the reference makes).  All pointers are HOST pointers.
 * ---------------------------------------------------------------------------------------------- */
/* cv::pyrDown on u8 (LK pyramid level). dst is ((w+1)/2) x ((h+1)/2), tightly packed. */
int gf_stage_pyr_down(int device, const uint8_t* src, int w, int h, uint8_t* dst);
/* cv::createCLAHE(clip_limit, Size(tiles_x, tiles_y))->apply(src, dst) on u8 with the tracker's kernels (gf_tracker_set_equalize).
 * src rows are src_pitch bytes apart; dst is w x h, tightly packed.  Same limits as the tracker's image and tile grid. */
int gf_stage_clahe(int device, const uint8_t* src, size_t src_pitch, int w, int h, double clip_limit, int tiles_x, int tiles_y,
                   uint8_t* dst);
/* trackImagebox's box test on its own (the device function of gf_tracker_submit with boxes): in_box[i] = 1 when point i
 * (pts: n x,y float pairs) lies strictly inside one of the n_boxes boxes, as pointPolygonTest(contour, pt, true) > 0 decides. */
int gf_stage_in_boxes(int device, const float* pts, int n, const gf_box* boxes, int n_boxes, uint8_t* in_box);
/* cv::cornerMinEigenVal(img, blockSize=3, ksize=3) as used by goodFeaturesToTrack. */
int gf_stage_min_eig(int device, const uint8_t* img, int w, int h, float* eig, int* n_fixups);
/* cv::calcOpticalFlowPyrLK(prev, next, prev_pts, next_pts, status, err, Size(21,21), max_level,
 * TermCriteria(COUNT+EPS,30,0.01), use_initial_flow ? OPTFLOW_USE_INITIAL_FLOW : 0).  roles selects the LK form of the
 * tracker's kernels: 1 = two warp roles (a tracker alone on its device), 0 = single role (several trackers, groups).
 * Both give the same bits. */
int gf_stage_lk(int device, const uint8_t* prev, const uint8_t* next, int w, int h,
                const float* prev_pts, float* next_pts, int n, int max_level, int use_initial_flow,
                uint8_t* status, int roles);
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
 * path (tests).  A non-finite entry of b or of A's lower triangle is GF_ERR_INVALID_ARG, and so is a pivot of the
 * factorisation that is not a positive normal number ("not positive definite"; x is then left unchanged). */
int gf_stage_spd_solve(int device, const double* A, const double* b, int n, double* x, int tile_cap);

/* The marginalisation's symmetric eigensolvers on their own (A n x n row-major, lower triangle read; w[n], V n x n row-major
 * with the eigenvectors in its columns, unsorted).  method 0: tridiagonalisation + implicit QL (k_sym_eig_ql, the reduced
 * system when n <= 128), 1 <= n <= 128; method 1: parallel cyclic Jacobi in global memory (k_jacobi_eig, Amm of the literal
 * path and reduced systems with n > 128), 1 <= n <= 2304.  sweeps: nullable, Jacobi's sweep count (cap 60; 0 for QL). */
int gf_stage_sym_eig(int device, const double* A, int n, int method, double* w, double* V, int* sweeps);

/* Which way a marginalisation went (bits of path[0] below and of gf_ba_last_marg_info). */
#define GF_MARG_PATH_GENERIC 1         /* literal path: eigen-truncated inverse of the whole Amm (Jacobi); else structured fast path */
#define GF_MARG_PATH_WIDE 2            /* ... because n > 127 (the fast path's c x (n + 1) buffer) */
#define GF_MARG_PATH_NOT_PD 4          /* ... because Amm - 1e-8 I is not positive definite */
#define GF_MARG_PATH_FORCED 8          /* ... because the caller asked for it */
#define GF_MARG_PATH_REDUCED_JACOBI 16 /* reduced system decomposed by Jacobi (n > 128); else by QL */

/* MarginalizationInfo::marginalize (marginalization_factor.cpp:272-302) on a given dense system, with the device code of
 * gf_ba_marginalize_old: A (N x N row-major), b (N) in the column layout [c dense | L landmarks | n = N - c - L kept],
 * 1 <= c <= 15, L >= 0, m = c + L <= 2304 (Jacobi size of the literal path), 1 <= n <= 16 * GF_BA_MAX_FRAMES + 22; the
 * L x L landmark block must be diagonal (GF_ERR_INVALID_ARG otherwise).  force_generic: take the literal path even when the
 * fast path applies.
 * Out: J0 (n x n row-major) = sqrt(S) V^T, r0 (n) = sqrt(S^-1) V^T b; path[3] = GF_MARG_PATH_* bits, Jacobi sweeps on Amm
 * (0 on the fast path), Jacobi sweeps on the reduced system (0 for QL). */
int gf_stage_marginalize(int device, const double* A, const double* b, int N, int c, int L, int force_generic,
                         double* J0, double* r0, int* path);

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
/* Free landmarks (entries of para_feature that are not constant and have a visual factor) one gf_ba_solve accepts; more is
 * GF_ERR_CAPACITY before anything is enqueued.  The Schur kernel stages 8 * (L + 2 nc + 2) bytes per CTA in shared memory
 * (nc <= 383 reduced unknowns): 71 KB at this bound. */
#define GF_BA_MAX_FREE_LANDMARKS 8192

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
/* The sliding windows of several estimators in one call (several robots or camera rigs served by one GPU): one window cannot
 * fill the device (its trust-region loop is a chain of small latency-bound launches), a batch runs every kernel of that chain
 * once for all windows (window = blockIdx.y), so the launch count does not grow with n.  Window k is problems[k], solved with
 * solvers[k]'s workspace and tile cap; its blocks are updated in place and summaries[k] filled exactly as
 * gf_ba_solve(solvers[k], &problems[k], &summaries[k]) would (same kernels, same arithmetic; like two gf_ba_solve calls of one
 * window, results may differ in the last bits because the Hessian is summed with atomics).  The exception is device_ms: the
 * CUDA-event time of the whole batch, the same in every summary.  max_num_iterations may differ between windows.
 *   1 <= n <= GF_BA_MAX_MULTI (more: GF_ERR_CAPACITY); the handles must be distinct and bound to the same device.  Every
 *   window is checked as gf_ba_solve checks it before anything is enqueued; on an argument error nothing is modified and
 *   gf_last_error() starts with "window k: ".
 *   status (nullable, n): 0, or GF_ERR_INVALID_ARG for a window whose IMU covariance turned out singular on the device: its
 *   blocks and summary are left untouched (summary zeroed), the other windows are written back, and the call returns
 *   GF_ERR_INVALID_ARG.
 * All work runs on solvers[0]'s stream, driven by the calling thread; no handle of the batch may be used by another thread
 * during the call. */
#define GF_BA_MAX_MULTI 256
int gf_ba_solve_multi(gf_ba* const* solvers, int n, const gf_ba_problem* problems, gf_ba_summary* summaries, int32_t* status);

/* What the solve computes inside its first iteration, for testing the kernels stage by stage (gf_ba_first_step).  Columns
 * follow the solve's layout: nc camera columns (col_* below, -1 = constant or absent), then the L free landmarks (col_feat).
 * The int / double scalars are filled by the call; every pointer is a caller buffer sized from gf_ba_step_dims, or NULL to
 * skip that array. */
typedef struct gf_ba_step_capture {
    int32_t nc, L, n, spill;          /* reduced dimension, free landmarks, nc + L; 1 = the factor spilled out of shared memory */
    int32_t col_pose[GF_BA_MAX_FRAMES], col_sb[GF_BA_MAX_FRAMES], col_ex, col_td, col_exw, col_ix[3], col_tdw, col_pr, col_pz;
    int32_t solver_failed, step_valid, done, termination, iterations;   /* BaState after the step (done: stopped before stepping) */
    double initial_cost;              /* cost at x                                                                           */
    double cauchy_num, cauchy_den, alpha;   /* |gs|^2, v^T H' v (v = gs / D), alpha = num / den                              */
    double dogleg_a, dogleg_b;        /* the D-space step dogleg_a * gs + dogleg_b * gn                                        */
    double dogleg_norm, model_change, step_norm, grad_max, x_norm;
    double mu, radius;                /* mu after k_ba_step (larger than the given one only if the Cholesky had to be retried) */
    int32_t* col_feat;                /* [n_features] column of each landmark, -1 = constant or unobserved                   */
    double* imu_sqrt;                 /* [n_imu][15][15] sqrt-information LLT(cov^-1).L^T of every IMU factor                */
    double* H;                        /* [nc][nc] camera block of J^T J without the prior                                    */
    double* Hp;                       /* [nc][nc] J0^T J0 of the marginalisation prior                                       */
    double* g;                        /* [n] J^T r (prior included)                                                          */
    double* W;                        /* [L][nc] landmark-camera block of J^T J                                              */
    double* hll;                      /* [L] landmark diagonal of J^T J                                                      */
    double *scale, *D, *gs;           /* [n] Jacobi scale, D = sqrt(clamp(diag(H') , 1e-6, 1e32)), gs = g' / D               */
    double* e_l;                      /* [L] 1 / (h'_ll + mu D_l^2)                                                          */
    double* S;                        /* [nc+1][nc+1] reduced system (H' + mu D^2 with the landmarks eliminated), lower
                                       * triangle; row nc holds the right-hand side, S[nc][nc] = 1                             */
    double* gn;                       /* [n] Gauss-Newton step in D-space                                                    */
    double* delta;                    /* [n] ambient step (dogleg_a gs + dogleg_b gn) / D * scale                            */
    double* Xc;                       /* [16 n_frames + 24 + n_features] candidate x (+) delta: pose[7F] | speed-bias[9F] | ex
                                       * pose[7] | td | wheel extrinsic[7] | sx sy sw | wheel td | plane R[4] | plane Z | features */
} gf_ba_step_capture;
/* dims3 = {nc, L, n} of the window as gf_ba_solve would lay it out; argument errors as gf_ba_solve. */
int gf_ba_step_dims(gf_ba* s, const gf_ba_problem* p, int* dims3);
/* The chain of gf_ba_solve_multi (same layout, packing, kernels, grids and launch attributes), started from the trust-region
 * radius `radius` and LM damping `mu` and stopped after the first k_ba_step: the initial linearisation, the reduced system, the
 * dogleg step and the candidate point of every window go to out[k].  No parameter block is written.  radius must be > 0 and mu
 * in (0, 1) (GF_ERR_INVALID_ARG).  A window whose IMU covariance is singular or indefinite fails the call with
 * GF_ERR_INVALID_ARG (error text "window k: ..." when n > 1). */
int gf_ba_first_step(gf_ba* const* solvers, int n, const gf_ba_problem* problems, double radius, double mu, gf_ba_step_capture* out);
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

/* The marginalisations of several estimators in one call, as gf_ba_solve_multi batches their solves.  Window k is problems[k]
 * on solvers[k]'s workspace, marginalised as modes[k] says; the result is exactly what gf_ba_marginalize_old /
 * gf_ba_marginalize_second_new(solvers[k], &problems[k], &outs[k], out_x0[k], out_J[k], out_r[k], ...) would give (same kernels,
 * same arithmetic; J0 may differ from a single call in the last bits, as between two single calls, because the Hessian is summed
 * with atomics), with the buffers of those calls.  Every kernel runs once for all windows that take its path (window =
 * blockIdx.y, or one CTA per window for the eigensolvers and k_marg_c_elim): the launch count depends on which paths occur
 * (fast path, literal path, QL or Jacobi on the reduced system), not on n, and the host synchronises at most once mid-batch, to
 * read every window's fast-path flag together.
 *   kept[k] (n entries): what the single call returns -- n_k > 0; 0 for MARGIN_SECOND_NEW when the prior does not hold the pose
 *   (outs[k] and its buffers untouched); GF_ERR_INVALID_ARG when the window's IMU covariance is singular on the device (outs[k]
 *   untouched; the other windows are written and the call returns GF_ERR_INVALID_ARG).
 *   1 <= n <= GF_BA_MAX_MULTI (more: GF_ERR_CAPACITY); the handles must be distinct and bound to the same device.  Every window
 *   is checked as the single call checks it, and modes[k] must be GF_BA_MARGIN_OLD or GF_BA_MARGIN_SECOND_NEW, before anything is
 *   enqueued; on an argument error nothing is written and gf_last_error() starts with "window k: ".
 *   gf_ba_last_marg_info(solvers[k]) reports window k.  device_ms (nullable): the CUDA-event time of the whole batch.
 * All work runs on the stream of the first window with work, driven by the calling thread; no handle of the batch may be used
 * by another thread during the call. */
#define GF_BA_MARGIN_OLD 0          /* estimator.cpp:3334-3535 */
#define GF_BA_MARGIN_SECOND_NEW 1   /* estimator.cpp:3536-3631 */
int gf_ba_marginalize_multi(gf_ba* const* solvers, int n, const gf_ba_problem* problems, const int32_t* modes, gf_ba_prior* outs,
                            double* const* out_x0, double* const* out_J, double* const* out_r, int32_t* kept, float* device_ms);
/* The last marginalisation of this handle: info[0] = GF_MARG_PATH_* bits, info[1] = Jacobi sweeps on Amm (0 on the fast
 * path), info[2] = Jacobi sweeps on the reduced system (0 for QL). */
int gf_ba_last_marg_info(gf_ba* s, int* info3);

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
 * depth over all observations (flag 2); results < 0.1, NaN or inf (a window without translation) become init_depth (flag 0).
 * Ps [n_frames][3], Rs [n_frames][9] row-major. */
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

/* ------------------------------------------------------------------------------------------------
 * gf_fm_window: one FeatureManager (feature_manager.h:90-150) whose landmark table -- the reference's std::list<FeaturePerId> --
 * stays on the GPU between frames, on the handle's own stream, with no allocation after creation.  It runs the arithmetic of
 * the stateless gf_fm_* calls above on the resident table (the results are bit-equal), takes the tracker's observations where
 * gf_tracker left them on the device, and emits the visual factors of gf_ba_problem.
 *
 * Per landmark, in LIST ORDER: feature_id, start_frame, n_obs, estimated_depth, estimate_flag, solve_flag and up to
 * GF_FM_WINDOW_ROWS observation rows [x y z u v vx vy depth td].  The list order is the reference's: the new landmarks of a
 * frame are appended in increasing id, every removal keeps the order of the rest.  It is not sorted by id.
 *
 * Every call checks its arguments before it changes anything; after an error the table is as it was.  Poses are Ps [11][3],
 * Rs [11][9] row-major, tic [3], ric [9]; a non-finite pose or a frame_count outside 0..WINDOW_SIZE is GF_ERR_INVALID_ARG.
 * Calls that return nothing (triangulate, set_depth, clear_depth, the removals, clear) only enqueue work; the others
 * synchronise the handle's stream once.  All pointers are HOST pointers.  A handle is used from one thread at a time.
 * ---------------------------------------------------------------------------------------------- */
typedef struct gf_fm_window gf_fm_window; /* opaque: one FeatureManager, bound to one GPU and one stream */
#define GF_FM_WINDOW_ROWS 11           /* WINDOW_SIZE + 1 observations per landmark */
#define GF_FM_WINDOW_ROW_DOUBLES 9
#define GF_FM_WINDOW_MAX_FRAME_OBS 2048 /* observations one add_frame takes */

typedef struct gf_fm_window_cfg {
    int max_features;        /* capacity of the table in landmarks, <= 8192; 0: 2048 */
    int window_size;         /* WINDOW_SIZE: 10 (or 0 for it); anything else is GF_ERR_UNSUPPORTED */
    double min_parallax;     /* MIN_PARALLAX, already divided by FOCAL_LENGTH (parameters.cpp:345-346) */
    double depth_threshold;  /* parameters.cpp:172 */
    double init_depth;       /* INIT_DEPTH (parameters.cpp:478) */
} gf_fm_window_cfg;

int gf_fm_window_create(gf_fm_window** out, int device, const gf_fm_window_cfg* cfg);
void gf_fm_window_destroy(gf_fm_window* w);
/* FeatureManager::clearState: the empty table */
int gf_fm_window_clear(gf_fm_window* w);
/* FeatureManager::addFeatureCheckParallax (:57-116) with the n observations of one frame (ids distinct and >= 0), without those
 * whose in_box[i] is set (nullable: none).  An observation of a known landmark is appended to its list, whether or not the
 * landmark was seen in the previous frame, as the reference does; the others start new landmarks.  *margin_old = the keyframe
 * decision (1: MARGIN_OLD); counters4 = last_track_num, new_feature_num, long_track_num, landmarks in the table afterwards;
 * *last_average_parallax in pixels at FOCAL_LENGTH (0 when the parallax test was not reached).  The parallax is summed in a
 * fixed order: two runs give the same bits.  More new landmarks than fit: GF_ERR_CAPACITY.  A landmark holds WINDOW_SIZE + 1
 * observation rows, one per window frame, so an observation of a landmark with start_frame + n_obs > WINDOW_SIZE (the frame at
 * WINDOW_SIZE added a second time without a slide in between) is GF_ERR_INVALID_ARG; the reference's list would grow. */
int gf_fm_window_add_frame(gf_fm_window* w, int frame_count, const gf_obs* obs, int n, const uint8_t* in_box, double td, int* margin_old,
                           int32_t* counters4, double* last_average_parallax);
/* The same with the frame `tracker` last returned through gf_tracker_wait (or a call built on it), read where the tracker left it
 * on the device (its observations and its in_box flags), ordered after the tracker's download of that frame.  The tracker is
 * only read.  With the pipelined calls the tracker has two result slots: the returned frame k stays on the device while frame
 * k + 1 is in flight (submit k + 1, wait k, add_frame_from_tracker is fine), and is gone once frame k + 2 has been submitted.
 * GF_ERR_INVALID_ARG if the tracker has returned no frame, returned its last one as a step of a gf_tracker_group, has had a
 * later frame submitted into that frame's result slot, or is bound to another device; the table is unchanged. */
int gf_fm_window_add_frame_from_tracker(gf_fm_window* w, const gf_tracker* tracker, int frame_count, double td, int* margin_old, int32_t* counters4,
                                        double* last_average_parallax);
/* triangulateWithDepth followed by triangulate (gf_fm_triangulate) over the table */
int gf_fm_window_triangulate(gf_fm_window* w, int frame_count, const double* Ps, const double* Rs, const double* tic, const double* ric);
/* The visual part of a gf_ba_problem (estimator.cpp:3268-3297, getDepthVector): the landmarks with n_obs >= 4 in list order are
 * features 0 .. *n_features - 1 with para_feature[k] = 1 / estimated_depth and feature_const[k] = (estimate_flag == 1); each
 * contributes one factor per observation after its first, (start_frame, start_frame + a, k), in that order.  visual_out
 * (nullable: only the feature arrays) holds cap rows, fewer than needed is GF_ERR_CAPACITY; para_feature and feature_const
 * (nullable) hold max_features entries. */
int gf_fm_window_fill_problem(gf_fm_window* w, gf_ba_visual_factor* visual_out, int cap, int* n_visual, double* para_feature, uint8_t* feature_const,
                              int* n_features);
/* FeatureManager::setDepth (:249-267) with the solved para_feature: n must be the n_features the last fill_problem returned,
 * with no frame added and no landmark removed since (GF_ERR_INVALID_ARG otherwise). */
int gf_fm_window_set_depth(gf_fm_window* w, const double* para_feature, int n);
/* removeFailures (solve_flag == 2), clearDepth (every estimated_depth = -1), removeOutlier (ids not in the table are ignored) */
int gf_fm_window_remove_failures(gf_fm_window* w);
int gf_fm_window_clear_depth(gf_fm_window* w);
int gf_fm_window_remove_ids(gf_fm_window* w, const int32_t* ids, int n);
/* removeBackShiftDepth (:818-856; marg / new: the camera poses R [9], P [3] of the marginalised and the new first frame; a
 * landmark left with fewer than two observations goes), removeBack and removeFront (frame_count must be WINDOW_SIZE; a landmark
 * left without observations goes) */
int gf_fm_window_remove_back_shift_depth(gf_fm_window* w, const double* marg_R, const double* marg_P, const double* new_R, const double* new_P);
int gf_fm_window_remove_back(gf_fm_window* w);
int gf_fm_window_remove_front(gf_fm_window* w, int frame_count);
/* Estimator::outliersRejection (mode GF_FM_OUTLIERS_REPROJECTION: n_obs >= 4, mean reprojection error over 3 px at FOCAL_LENGTH)
 * and movingConsistencyCheckW (GF_FM_OUTLIERS_MOVING: n_obs >= 2, start_frame < WINDOW_SIZE - 2, depth >= 0, mean error over
 * 10 px or mean 3-D error over 2): the ids in list order; ids_out holds max_features entries. */
#define GF_FM_OUTLIERS_REPROJECTION 0
#define GF_FM_OUTLIERS_MOVING 1
int gf_fm_window_outliers(gf_fm_window* w, const double* Ps, const double* Rs, const double* tic, const double* ric, int mode, int32_t* ids_out, int* n);
/* Estimator::predictPtsInNextFrame: ids_out / xyz_out [n][3] (max_features entries each, list order) are the arguments of
 * gf_tracker_set_prediction; *n = 0 when frame_count < 2. */
int gf_fm_window_predict_next(gf_fm_window* w, int frame_count, const double* Ps, const double* Rs, const double* tic, const double* ric, int32_t* ids_out,
                              double* xyz_out, int* n);
/* The table in list order: every array (nullable) holds cap entries, obs cap * GF_FM_WINDOW_ROWS * GF_FM_WINDOW_ROW_DOUBLES
 * doubles (landmark i's row a at (i * GF_FM_WINDOW_ROWS + a) * GF_FM_WINDOW_ROW_DOUBLES, rows from n_obs[i] on unspecified).
 * *n = the number of landmarks; more than cap is GF_ERR_CAPACITY with *n set. */
int gf_fm_window_read(gf_fm_window* w, int32_t* feature_id, int32_t* start_frame, int32_t* n_obs, double* estimated_depth, int32_t* estimate_flag,
                      int32_t* solve_flag, double* obs, int cap, int* n);
int gf_fm_window_size(gf_fm_window* w, int* n);
/* Device time of the last call's work on the handle's stream, from CUDA events (waits for that work) */
int gf_fm_window_last_device_ms(gf_fm_window* w, float* ms);

/* A window group: n existing gf_fm_windows (members, one per estimator) whose FeatureManager calls run with ONE set of launches
 * per call: every kernel runs once for the whole group (member = a grid dimension), so the number of launches and driver calls
 * of a group call does not grow with n, and a call that returns something synchronises once for the group.  Member i's table,
 * results and host-side state afterwards are exactly what the same single-window call on it would give (same kernels, same
 * arithmetic, same bits); a single-window call is the group of one.
 *   _create: 1 <= n <= GF_FM_WINDOW_GROUP_MAX; the windows must be distinct and bound to one device; capacities may differ.
 *       Any violation is GF_ERR_INVALID_ARG, with gf_last_error() starting "member k: " for the member at fault.  The group
 *       owns its stream and its ring of pinned input slots (descriptors, observations, depths, ids); it allocates nothing
 *       after creation.  Destroy the group before its members.
 *   State stays in the members.  Between group calls a member may be used directly, and the next group call continues from
 *   there: work is ordered between a member's stream and the group's in both directions, with no wait while every member
 *   stays on one of them.  A group is used from one thread at a time, and its members are not used by another thread during
 *   a group call.
 *   Per-member arguments are arrays of n (poses: Ps [n][11][3], Rs [n][11][9], tic [n][3], ric [n][9]; CSR lists: n + 1
 *   offsets from 0).  Every member's arguments are checked as the single call checks them before anything is enqueued: an
 *   argument error changes no member, and gf_last_error() starts "member k: ".
 *   Failures found on the device are per member: status[k] (nullable) is 0 or the single call's error code for member k,
 *   whose table and outputs are then left as they were; the other members are applied, and the call returns the code of the
 *   first member that failed.
 * gf_fm_window_group_last_device_ms reports the device time of the last group call. */
typedef struct gf_fm_window_group gf_fm_window_group;
#define GF_FM_WINDOW_GROUP_MAX 64      /* = GF_TRACKER_GROUP_MAX: a tracker group maps one to one onto a window group */
#define GF_FM_REMOVE_NONE 0
#define GF_FM_REMOVE_BACK_SHIFT_DEPTH 1
#define GF_FM_REMOVE_BACK 2
#define GF_FM_REMOVE_FRONT 3
int gf_fm_window_group_create(gf_fm_window_group** out, gf_fm_window* const* windows, int n);
void gf_fm_window_group_destroy(gf_fm_window_group* g);
int gf_fm_window_group_size(gf_fm_window_group* g, int* n);
/* add_frame for every member: member i's observations are obs[obs_start[i] .. obs_start[i + 1]), its box flags in_box at the
 * same indices (nullable: none); margin_old [n], counters4 [n][4], last_average_parallax [n] (each nullable).  A member that does
 * not fit (GF_ERR_CAPACITY) or would take a twelfth observation (GF_ERR_INVALID_ARG) reports it in status and is unchanged. */
int gf_fm_window_group_add_frame(gf_fm_window_group* g, const int32_t* frame_counts, const gf_obs* obs, const int32_t* obs_start, const uint8_t* in_box,
                                 const double* tds, int32_t* margin_old, int32_t* counters4, double* last_average_parallax, int32_t* status);
/* The same with member i of the tracker group tg's last collected step (gf_tracker_group_wait / _track_batch), read where tg left
 * it on the device, ordered after tg's download of that step; the count is gf_tracker_group_wait's.  tg is only read.  With
 * two steps in flight the collected step stays readable while the next one runs (submit k + 1, wait k, ingest).
 * GF_ERR_INVALID_ARG, every table unchanged, if tg has collected no step, has had a later step submitted into that step's
 * slot, has another number of members, or is bound to another device. */
int gf_fm_window_group_add_frame_from_tracker_group(gf_fm_window_group* g, const gf_tracker_group* tg, const int32_t* frame_counts, const double* tds,
                                                    int32_t* margin_old, int32_t* counters4, double* last_average_parallax, int32_t* status);
int gf_fm_window_group_triangulate(gf_fm_window_group* g, const int32_t* frame_counts, const double* Ps, const double* Rs, const double* tic, const double* ric);
/* fill_problem per member: visual_out[i] holds caps[i] rows (visual_out NULL, or an entry NULL: only the feature arrays of that
 * member); n_visual, n_features [n]; para_feature[i], feature_const[i] (nullable arrays and entries).  A member whose rows do not
 * fit reports GF_ERR_CAPACITY in status. */
int gf_fm_window_group_fill_problem(gf_fm_window_group* g, gf_ba_visual_factor* const* visual_out, const int32_t* caps, int32_t* n_visual,
                                    double* const* para_feature, uint8_t* const* feature_const, int32_t* n_features, int32_t* status);
int gf_fm_window_group_set_depth(gf_fm_window_group* g, const double* const* para_feature, const int32_t* n);
/* One removal per member, chosen per member (members decide MARGIN_OLD or MARGIN_SECOND_NEW independently): ops[i] is
 * GF_FM_REMOVE_NONE, _BACK_SHIFT_DEPTH (shift[i] = marg_R [9], marg_P [3], new_R [9], new_P [3], as
 * gf_fm_window_remove_back_shift_depth; shift may be NULL when no member takes it), _BACK or _FRONT (frame_counts[i] must be
 * WINDOW_SIZE, as gf_fm_window_remove_front requires). */
int gf_fm_window_group_remove(gf_fm_window_group* g, const int32_t* ops, const int32_t* frame_counts, const double* shift);
int gf_fm_window_group_remove_failures(gf_fm_window_group* g);
int gf_fm_window_group_clear_depth(gf_fm_window_group* g);
/* removeOutlier per member: ids[id_start[i] .. id_start[i + 1]) */
int gf_fm_window_group_remove_ids(gf_fm_window_group* g, const int32_t* ids, const int32_t* id_start);
/* outliers / predict_next per member: ids_out[i] (and xyz_out[i]) hold member i's max_features entries; n [n] */
int gf_fm_window_group_outliers(gf_fm_window_group* g, const double* Ps, const double* Rs, const double* tic, const double* ric, int mode,
                                int32_t* const* ids_out, int32_t* n);
int gf_fm_window_group_predict_next(gf_fm_window_group* g, const int32_t* frame_counts, const double* Ps, const double* Rs, const double* tic,
                                    const double* ric, int32_t* const* ids_out, double* const* xyz_out, int32_t* n);
int gf_fm_window_group_last_device_ms(gf_fm_window_group* g, float* ms);

/* ------------------------------------------------------------------------------------------------
 * Dense colour map (dense_map/src/pose_graph.cpp, pose_graph_node.cpp): the keyframe point sampling of the mapping node,
 * PoseGraph's voxel-density insertion (OctreePointCloudDensity, 0.01 m voxels), its RadiusOutlierRemoval (0.8 m, 10
 * neighbours) and updatePath's rebuild after a pose-graph correction.  Loop detection and the pose-graph optimisation stay
 * with the caller, which passes the corrected keyframe poses.  DESIGN.md "Dense colour map" has the semantics.
 * ---------------------------------------------------------------------------------------------- */
typedef struct gf_dense_map gf_dense_map; /* opaque: one map, bound to one GPU and one stream */

typedef struct gf_dense_map_cfg {
    int width, height;       /* image size (COL, ROW) */
    double pinhole[8];       /* fx fy cx cy k1 k2 p1 p2, as gf_tracker_cfg (cam0_calib) */
    int depth_dist;          /* DEPTH_DIST: sample every depth_dist-th pixel, >= 1 */
    int depth_boundary;      /* DEPTH_BOUNDARY: samples in [b, COL - b) x [b, ROW - b); 2 b < width and height */
    double ric[9];           /* qic (row-major) and tic: camera to body */
    double tic[3];
    int max_points;          /* capacity: points kept by all keyframes together (the cloud never holds more) */
    int max_keyframes;       /* capacity: keyframes */
} gf_dense_map_cfg;

enum { GF_DENSE_MAP_CLOUD = 0, GF_DENSE_MAP_FILTERED = 1 };

int gf_dense_map_create(gf_dense_map** map, int device, const gf_dense_map_cfg* cfg);
void gf_dense_map_destroy(gf_dense_map* map);
/* One keyframe: sample (pose_graph_node.cpp:598-623), insert with pose (R row-major, P) under the z band and the density gate
 * < 3 (pose_graph.cpp:191-221), then filter (:228-239).  rgb: RGB8 rows of rgb_pitch bytes; depth: uint16 millimetres, rows of
 * depth_pitch bytes; both HOST pointers, or device pointers when on_device != 0.  n_inserted (nullable): points added.
 * GF_ERR_CAPACITY (max_keyframes, max_points) and GF_ERR_INVALID_ARG (a point outside the octree's box) leave the map unchanged. */
int gf_dense_map_add_keyframe(gf_dense_map* map, const double* R, const double* P, const uint8_t* rgb, size_t rgb_pitch,
                              const uint16_t* depth, size_t depth_pitch, int on_device, int* n_inserted);
/* PoseGraph::updatePath's rebuild (:997-1058): a fresh octree over the wider box, every keyframe's kept points re-inserted in
 * keyframe order with its new pose (R [n][9], P [n][3]) under the gate < 5 and no z band, then a full filter.  n_keyframes must
 * equal the number of keyframes added (GF_ERR_INVALID_ARG otherwise, map unchanged). */
int gf_dense_map_update_poses(gf_dense_map* map, int n_keyframes, const double* R, const double* P);
int gf_dense_map_size(gf_dense_map* map, int* n_cloud, int* n_filtered, int* n_keyframes);
/* Host copies in cloud order of the whole cloud (which = GF_DENSE_MAP_CLOUD) or of the points the filter keeps
 * (GF_DENSE_MAP_FILTERED): xyz [n][3], rgb [n][3], idx [n] = each point's index in the cloud.  Each output is nullable. */
int gf_dense_map_read(gf_dense_map* map, int which, float* xyz, uint8_t* rgb, int32_t* idx);
/* Keyframe k's kept points (KeyFrame::point_rgbd after insertion): out6 [n][6] = camera-frame x y z and r g b; *n = their number
 * (out6 NULL: only the number). */
int gf_dense_map_keyframe_points(gf_dense_map* map, int k, float* out6, int* n);
/* The map's radius filter over n host points: keep[i] = 1 iff more than min_pts points (itself included) lie at float squared
 * distance < float(radius^2). */
int gf_stage_radius_filter(int device, const float* xyz, int n, double radius, int min_pts, uint8_t* keep);

/* A dense-map group: n existing gf_dense_maps (members, e.g. one per estimator) that take one keyframe each with ONE launch chain
 * per call and ONE host synchronisation, where n single calls make ten launches and two synchronisations each.  Member k's
 * cloud, keyframe lists, voxel counts, filter result and n_filtered afterwards are bit-equal to what
 * gf_dense_map_add_keyframe on it alone would give.  DESIGN.md "Groups of maps" has the layout and the order argument.
 *   _create: 1 <= n <= GF_DENSE_MAP_GROUP_MAX; the maps must be distinct, bound to one device and share width, height,
 *       depth_dist and depth_boundary (so the samples per keyframe); capacities, intrinsics and extrinsics may differ.  Any
 *       violation is GF_ERR_INVALID_ARG with gf_last_error() starting "member k: ".  The group borrows the maps (destroy it
 *       first) and allocates its scratch once: about 100 bytes per point of the members' max_points together.
 *   Between group calls a member may be used directly (add_keyframe, update_poses, read, keyframe_points): work is ordered
 *   between a member's stream and the group's in both directions.  A group is used from one thread at a time.
 * _add_keyframes: one keyframe for each of m distinct members, members[j] in [0, n) any subset; member members[j] takes pose
 * R [j][9], P [j][3] and the frame rgb[j] (rows of rgb_pitch[j] bytes), depth[j] (rows of depth_pitch[j] bytes), all HOST
 * pointers or all device pointers (on_device).  Argument errors (a member listed twice or out of range, a null frame, a pitch)
 * change nothing; gf_last_error() starts "member j: " for entry j.  A member that would fail the single call (max_keyframes,
 * max_points, a point outside the octree's box) reports that code in status[j] (nullable) and stays unchanged; the others are
 * applied, and the call returns the first failing entry's code.  n_inserted [m] (nullable): points added. */
typedef struct gf_dense_map_group gf_dense_map_group;
#define GF_DENSE_MAP_GROUP_MAX 64
int gf_dense_map_group_create(gf_dense_map_group** out, gf_dense_map* const* maps, int n);
void gf_dense_map_group_destroy(gf_dense_map_group* g);
int gf_dense_map_group_size(gf_dense_map_group* g, int* n);
int gf_dense_map_group_add_keyframes(gf_dense_map_group* g, const int32_t* members, int m, const double* R, const double* P,
                                     const uint8_t* const* rgb, const size_t* rgb_pitch, const uint16_t* const* depth, const size_t* depth_pitch,
                                     int on_device, int32_t* n_inserted, int32_t* status);

/* ------------------------------------------------------------------------------------------------
 * Occupancy grid (support_files/grid_mapping: main.cpp, grid_mapper.cpp, grid_map.cpp): the 2-D log-odds grid the reference
 * builds offline from every keyframe's point_rgbd and corrected pose, here built online.  Keyframe points whose world height
 * lies in [0.1, 0.5] m cast a ray from the body position in steps of one cell; every cell on the way gets the inverse sensor
 * model's free / occupied / prior update.  After any sequence of calls bel equals the tool's over the same keyframes in the
 * same order with the poses last passed, with the tool's log / exp replaced by the shared double-double ones of
 * csrc/gm_math.h.  DESIGN.md "Occupancy grid" has the semantics.
 * ---------------------------------------------------------------------------------------------- */
typedef struct gf_grid_map gf_grid_map; /* opaque: one grid, bound to one GPU and one stream */

typedef struct gf_grid_map_cfg {
    int size_x, size_y;      /* cells (1500 x 500 in the tool); size_x * size_y < 2^30 */
    int init_x, init_y;      /* the cell of world (0, 0) (750, 250) */
    double cell_size;        /* metres (0.05), > 0 */
    double p_occ, p_free, p_prior; /* inverse sensor model (0.6, 0.4, 0.5), each in (0, 1) */
    double ric[9];           /* qic (row-major) and tic: camera to body */
    double tic[3];
    int max_points;          /* capacity: points of all keyframes together */
    int max_keyframes;       /* capacity: keyframes */
    int max_records;         /* ray steps sorted at once; a call with more is processed in chunks of this many */
} gf_grid_map_cfg;

enum { GF_GRID_MAP_BEL = 0, GF_GRID_MAP_IMAGE = 1, GF_GRID_MAP_OCCUPANCY = 2 };

int gf_grid_map_create(gf_grid_map** map, int device, const gf_grid_map_cfg* cfg);
void gf_grid_map_destroy(gf_grid_map* map);
/* One keyframe with body pose (R row-major, P) applied on top of the grid: n camera-frame points, rows of stride_floats floats
 * (x y z first; 6 takes gf_dense_map_keyframe_points' rows as they are), a HOST pointer or a device pointer when on_device != 0.
 * GF_ERR_INVALID_ARG (a non-finite pose or point) and GF_ERR_CAPACITY (max_keyframes, max_points, a ray of more than 2^24 steps)
 * leave the grid unchanged. */
int gf_grid_map_add_keyframe(gf_grid_map* map, const double* R, const double* P, const float* pts, int n, int stride_floats, int on_device);
/* The rebuild after a pose correction: the grid back to 0.5, then every keyframe applied again in order with its new pose
 * (R [n][9], P [n][3]).  n_keyframes must equal the number of keyframes added (GF_ERR_INVALID_ARG otherwise, grid unchanged). */
int gf_grid_map_update_poses(gf_grid_map* map, int n_keyframes, const double* R, const double* P);
/* Host copy of GF_GRID_MAP_BEL: double [size_x * size_y], bel(x, y) at x + size_x * y (Eigen's column-major order);
 * GF_GRID_MAP_IMAGE: uint8 [size_x][size_y], the pixels GridMap::saveMap writes to map.png; GF_GRID_MAP_OCCUPANCY: int8
 * [size_x * size_y], the nav_msgs/OccupancyGrid data the mapping node publishes from that image (-1 unknown, else 0..100). */
int gf_grid_map_read(gf_grid_map* map, int which, void* out);
int gf_grid_map_size(gf_grid_map* map, int* size_x, int* size_y, int* n_keyframes, int* n_points);
/* Of the last add_keyframe / update_poses: out4 = ray steps (records), updates applied, updates the exact shortcuts skipped
 * (a repeated no-op update, a cell at 0 or 1) and the longest per-cell run within one chunk. */
int gf_grid_map_stats(gf_grid_map* map, int64_t* out4);

/* A grid group: n existing gf_grid_maps whose keyframes are applied with one launch chain per call (count, scan, emit, sort and
 * apply run once over every member's rays).  Member k's bel (so its image and occupancy) afterwards is bit-equal to what
 * gf_grid_map_add_keyframe on it alone would give; its stats are those of its own records.
 *   _create: 1 <= n <= GF_GRID_MAP_GROUP_MAX grids, distinct and bound to one device; sizes, sensor models and capacities may
 *       differ.  The group sorts at most min(max_records) of its members' records at once (more are chunked, in order) and
 *       allocates 16 bytes per point of the members' max_points together and 16 per record.  Member use between group calls
 *       and errors are as for the dense-map group.
 * _add_keyframes: member members[j] takes pose R [j][9], P [j][3] and n_pts[j] points, rows of stride_floats[j] floats at
 * pts[j], all host or all device pointers (on_device).  Per-member failures (a non-finite pose or point, max_keyframes,
 * max_points, a ray of more than 2^24 steps) go to status[j] with the member unchanged.
 * _add_dense_keyframes: the same, each grid member's points being, read on the device, the keyframe that member of the dense-map
 * group dg with the SAME index added last (grid member k pairs with dense member k); no host copy. */
typedef struct gf_grid_map_group gf_grid_map_group;
#define GF_GRID_MAP_GROUP_MAX 64
int gf_grid_map_group_create(gf_grid_map_group** out, gf_grid_map* const* grids, int n);
void gf_grid_map_group_destroy(gf_grid_map_group* g);
int gf_grid_map_group_size(gf_grid_map_group* g, int* n);
int gf_grid_map_group_add_keyframes(gf_grid_map_group* g, const int32_t* members, int m, const double* R, const double* P, const float* const* pts,
                                    const int32_t* n_pts, const int32_t* stride_floats, int on_device, int32_t* status);
int gf_grid_map_group_add_dense_keyframes(gf_grid_map_group* g, gf_dense_map_group* dg, const int32_t* members, int m, const double* R,
                                          const double* P, int32_t* status);

/* ---- YOLO detector (the use_yolo front end's darknet_ros node, YoloObjectDetector.cpp, on the GPU) ------------------------
 * darknet's inference forward pass for the networks the reference ships (vins_estimator/yolo_network_config/cfg: [net],
 * [convolutional], [maxpool], [route], [reorg], [shortcut], [upsample], [region], [yolo]; activations leaky and linear),
 * bit-exact with darknet's CPU build, followed by the node's decoding (get_network_boxes with hier 0.5, do_nms_obj 0.4) and box
 * extraction.  The boxes feed the tracker's boxes argument (trackImagebox).
 * The detector is implemented in its own library, libgf_yolo.so, built next to libgf_b200.so: libgf_b200.so exports these
 * entry points as forwarders that open it on the first call, so it carries none of the detector's device code and a process
 * that never detects never loads it.  A failing call sets gf_last_error() as usual; gf_detector_last_error() is the same
 * text as libgf_yolo.so holds it. */
typedef struct gf_detector gf_detector;
/* Text of the last error raised by a gf_detector_* / gf_stage_letterbox call on the calling thread (never NULL). */
const char* gf_detector_last_error(void);
/* The network is read from a darknet cfg and .weights file.  A layer type, activation or key value outside the set above:
 * GF_ERR_UNSUPPORTED with the reason in gf_last_error(); a missing or short weights file: GF_ERR_INVALID_ARG.  thresh in [0, 1)
 * is darknet_ros's detection threshold.  Every parameter goes to device memory here, once. */
int gf_detector_create(gf_detector** det, int device, const char* cfg_path, const char* weights_path, float thresh);
void gf_detector_destroy(gf_detector* det);
/* net_wh[2] = the [net] width and height; n_layers excludes [net]; classes of the last layer.  All three nullable. */
int gf_detector_info(gf_detector* det, int* net_wh, int* n_layers, int* classes);
/* One frame: BGR8, w x h pixels, rows `pitch` bytes apart, a host pointer or a device pointer when on_device != 0.  Writes the
 * boxes darknet_ros would publish, grouped by class in class order, with their class ids and probabilities (both nullable), and
 * their count in *n_out: 0 when there are none or more than GF_MAX_BOXES.  cap < *n_out: GF_ERR_CAPACITY (nothing past cap
 * written).  Synchronous: the boxes belong to this frame. */
int gf_detector_detect(gf_detector* det, const void* bgr, size_t pitch, int w, int h, int on_device, gf_box* boxes, int* class_ids,
                       float* probs, int cap, int* n_out);
/* Batches of frames: one handle runs the forward pass of up to max_batch frames (of any sizes) in one graph launch, one set of
 * weights for all.  Each frame's result is bit-equal to gf_detector_detect on that frame alone, in both precisions: a
 * convolution's summation order (the TF32 split-K plan included) is a function of the layer's per-image shape, never of the
 * batch or of a frame's position in it.  gf_detector_detect is the batch of one, through the same code.
 *   _set_max_batch  sizes the per-image buffers (every layer's output, the letterboxed inputs, the pinned head copies, the TF32
 *       split-K workspace) for max_batch frames; a handle starts at 1.  Per image at 416 x 416, from the layer shapes: layer
 *       outputs of about 28 MiB for yolov2-tiny, 75 MiB for yolov2 and 217 MiB for yolov3, plus 2 MiB of letterboxed input and,
 *       once TF32 is set, 8 MiB of split-K workspace.  The weights (236 MiB FP32 for yolov3, as much again once TF32 is set)
 *       are not per image.  max_batch outside [1, GF_DETECTOR_BATCH_MAX]:
 *       GF_ERR_INVALID_ARG; a failed allocation: GF_ERR_CUDA with the handle unchanged.  Drops the graphs and the last call's
 *       layer outputs.
 *   _detect_batch  frames bgr[i] (w[i] x h[i], rows pitch[i] bytes apart; all host or all device pointers as on_device says).
 *       Frame i's boxes, class ids and probabilities are boxes[box_start[i] .. box_start[i + 1]) (n + 1 offsets: the layout
 *       gf_tracker_group_submit takes), each range what gf_detector_detect writes for that frame.  1 <= n <= max_batch (more:
 *       GF_ERR_CAPACITY).  box_start[n] > cap: GF_ERR_CAPACITY with box_start filled and nothing written at or past cap.  Every
 *       argument is checked before any work, so an argument error changes nothing.  Synchronous.  The graph of each n is captured
 *       on its first use and kept; gf_detector_set_precision re-captures every one kept.
 *   _member_layer_output  as gf_detector_layer_output for frame `member` of the last call; gf_detector_layer_output is member 0.
 * gf_detector_last_device_ms and gf_detector_layer_times cover the whole last call. */
#define GF_DETECTOR_BATCH_MAX 64      /* = GF_TRACKER_GROUP_MAX: a tracker group maps one to one onto a batch */
int gf_detector_set_max_batch(gf_detector* det, int max_batch);
int gf_detector_detect_batch(gf_detector* det, int n, const void* const* bgr, const size_t* pitch, const int* w, const int* h,
                             int on_device, gf_box* boxes, int* class_ids, float* probs, int cap, int* box_start);
int gf_detector_member_layer_output(gf_detector* det, int member, int layer, float* out, size_t n);
/* Device time of the last detect (letterbox + network, at the precision in use), from CUDA events. */
int gf_detector_last_device_ms(gf_detector* det, float* ms);
/* whc[3] = output width, height and channels of layer `layer` (0-based, [net] excluded), or of the letterboxed input for -1. */
int gf_detector_layer_shape(gf_detector* det, int layer, int* whc);
/* Host copy of layer `layer`'s output after the last detect, planar [c][h][w] float; -1: the letterboxed input.  n is the
 * capacity of out in floats. */
int gf_detector_layer_output(gf_detector* det, int layer, float* out, size_t n);
/* Mean device time of each layer's kernels over `reps` launches on the last frame's data, into ms[n_layers] (profiling). */
int gf_detector_layer_times(gf_detector* det, int reps, float* ms);
/* Stage: darknet's letterbox of a BGR8 frame at net_w x net_h into out [3][net_h][net_w] (host), as gf_detector_detect does it. */
int gf_stage_letterbox(int device, const void* bgr, size_t pitch, int w, int h, int on_device, int net_w, int net_h, float* out);

/* The arithmetic of the detector's convolutions, per detector.  Everything else (letterbox, pooling, route, reorg, upsample,
 * shortcut, the heads, decoding, NMS, extraction) is the same in both.
 *   GF_DETECTOR_EXACT  the default: bit-exact with darknet's CPU build (sequential FMUL + FADD chains, no tensor cores).
 *   GF_DETECTOR_TF32   tensor cores (wgmma): weights and every convolution input rounded to TF32 by round-to-nearest, ties
 *                      away from zero (10 explicit mantissa bits), products summed in FP32 in a fixed order, so the same input
 *                      always gives the same bits.  Not equal to darknet's CPU or GPU build; DESIGN.md has the error bound. */
#define GF_DETECTOR_EXACT 0
#define GF_DETECTOR_TF32 1
/* Selects the precision of every later detect.  The first switch to TF32 allocates a TF32-rounded copy of every convolution's
 * weights beside the FP32 ones (about 250 MB for yolov3), so the handle can switch back.  Re-captures the network's graph.
 * Another value: GF_ERR_INVALID_ARG. */
int gf_detector_set_precision(gf_detector* det, int precision);
int gf_detector_get_precision(gf_detector* det, int* precision);
/* Stage: one convolutional layer at `precision` with host arrays, through the kernels and tile choice the detector uses for
 * that shape.  shape = C H W M size stride pad bn act (act 1 = leaky, 0 = linear); in [C][H][W], w [M][C size size], bias [M],
 * and with bn: scale, mean, var [M] (nullable without bn); out [M][OH][OW], OH = (H + 2 pad - size) / stride + 1. */
int gf_stage_yolo_conv(int device, int precision, const int* shape, const float* in, const float* w, const float* bias,
                       const float* scale, const float* mean, const float* var, float* out);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* GF_B200_H */
