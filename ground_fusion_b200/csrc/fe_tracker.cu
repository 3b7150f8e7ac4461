// fe_tracker.cu -- gf_tracker_* and gf_stage_* (C ABI), the host side of the front end.
//
// Mirrors FeatureTracker::trackImage (reference vins_estimator/src/featureTracker/feature_tracker.cpp:103-372).
// One frame = fixed sequences of copies and kernels on three streams (no host round trip inside the frame; the only
// synchronisation is the wait for the result).  Up to two frames are in flight: everything that does not depend on
// the previous frame's result (upload, pyramid, min-eig map) runs ahead on their own streams while s_main is still tracking the
// previous frame, so in steady state the frame period is the dependent chain alone.
//
//   s_up  : H2D gray/depth (ev_up)                  -- the copy of frame t+2 overlaps the pyramid / min-eig kernels of t+1
//   s_pyr : (ev_up) pyrDown x3 (ev_pyr)
//   s_eig : (ev_up) k_cov_rows -> k_box_chain -> k_eig_from_box (ev_eig)
//   s_main: (ev_pyr) [prediction LK] -> k_track (fwd LK 3 lvls + bwd LK 1 lvl + status rules) -> k_compact_setmask
//           -> (ev_eig) masked max -> candidates -> k_select_finalize (min-distance rounds, top-K, addPoints,
//           undistort, velocity, depth; trackImagebox's in-box flags from the boxes in FrameParams)  (ev_dep)
//   s_out : (ev_dep) D2H of the result block
//
// Buffers touched by more than one frame in flight are rotated: 3 pyramids (prev/cur/next), 2 depth images, 2 eig
// maps, 2 frame-parameter blocks, 2 result blocks.  All feature state (prev_pts, ids, track_cnt, undistorted points,
// n_id) lives in HBM between frames and is only touched on s_main.
#include <stdlib.h>
#include <new>
#include <vector>

#include "fe_clahe.cuh"
#include "fe_eig.cuh"
#include "fe_lk.cuh"
#include "fe_lk_single.cuh"
#include "fe_select.cuh"

namespace gf {

thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};


struct FrameParams {
    double dt; int has_pred; int depth_valid;
    BoxSet boxes;            // trackImagebox's detections (n = 0: trackImage)
};

// The reference copies the int64 fields of darknet_ros_msgs/BoundingBox into `int` (a modular wrap) and those into the float
// contour; the bounds of the open rectangle are kept ordered so that inverted boxes test as the contour does.
static void put_boxes(BoxSet& s, const gf_box* b, int n)
{
    s.n = n;
    for (int k = 0; k < n; k++) {
        const float x0 = (float)(int32_t)(uint32_t)(uint64_t)b[k].xmin, y0 = (float)(int32_t)(uint32_t)(uint64_t)b[k].ymin;
        const float x1 = (float)(int32_t)(uint32_t)(uint64_t)b[k].xmax, y1 = (float)(int32_t)(uint32_t)(uint64_t)b[k].ymax;
        s.b[k] = make_float4(fminf(x0, x1), fmaxf(x0, x1), fminf(y0, y1), fmaxf(y0, y1));
    }
}
static int check_boxes(const gf_box* b, int n)
{
    if (n < 0 || (n > 0 && !b)) return set_err(GF_ERR_INVALID_ARG, "bad box list");
    if (n > GF_MAX_BOXES) return set_err(GF_ERR_CAPACITY, "more than GF_MAX_BOXES boxes in one frame");
    return GF_OK;
}
// The box lists boxes[box_start[k] .. box_start[k + 1]) of frames k < count; *bad is the first bad frame.
static int check_box_lists(const gf_box* boxes, const int* box_start, long long count, long long* bad)
{
    for (long long k = 0; k < count; k++) {
        *bad = k;
        if (box_start[k] < 0) return set_err(GF_ERR_INVALID_ARG, "bad box offsets");
        int rc = check_boxes(boxes ? boxes + box_start[k] : nullptr, box_start[k + 1] - box_start[k]);
        if (rc) return rc;
    }
    return GF_OK;
}
// Host frames may have row pitches larger than the row; device frames are tightly packed (their pitches are ignored).
static int check_pitches(int w, bool on_device, size_t gray_pitch, bool has_depth, size_t depth_pitch)
{
    if (on_device) return GF_OK;
    if (gray_pitch < (size_t)w) return set_err(GF_ERR_INVALID_ARG, "gray_pitch smaller than width");
    if (has_depth && depth_pitch < (size_t)w * 2) return set_err(GF_ERR_INVALID_ARG, "depth_pitch smaller than width*2");
    return GF_OK;
}

// gf_stage_in_boxes: the test k_select_finalize applies to its outputs, on its own
__global__ void __launch_bounds__(256) k_in_boxes_stage(const float2* pts, int n, const BoxSet* boxes, uint8_t* in_box)
{
    __shared__ float4 s_box[GF_BOX_CAP];
    const int nb = boxes->n;
    if ((int)threadIdx.x < nb) s_box[threadIdx.x] = boxes->b[threadIdx.x];
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) in_box[i] = in_any_box(s_box, nb, pts[i]) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// kernels that need the LK device code
// ------------------------------------------------------------------------------------------------
// The LK form of a tracker kernel: ROLES = the two warp roles (fe_lk.cuh), which shorten each feature's chain, when one
// tracker has the GPU to itself; otherwise the single-role form (fe_lk_single.cuh), which measured faster when several
// trackers share it (DESIGN.md §1.3).  Both give the same bits.
template <bool ROLES> struct LKForm { using Smem = LKSmem; using Tma = LKTma; };
template <> struct LKForm<false> { using Smem = lk1::LKSmem; using Tma = lk1::LKTma; };
template <class Tma>
__device__ __forceinline__ Tma lk_tma_of(const LKMapSet& M)
{
    Tma T{};                    // phases 0
    T.mi = M.prevI; T.mj = M.curJ; T.on = M.enabled != 0;
    return T;
}

// gf_stage_lk: one CTA per point, in the LK form ROLES selects (LKForm above)
template <bool ROLES>
__global__ void __launch_bounds__(LK_THREADS) k_lk_stage(const __grid_constant__ Pyramid I, const __grid_constant__ Pyramid J, const float2* prev_pts, float2* next_pts,
                                                         int n, int max_level, int use_init, uint8_t* status, const __grid_constant__ LKMapSet M)
{
    __shared__ typename LKForm<ROLES>::Smem sm;
    const int tid = threadIdx.x, i = blockIdx.x;
    if (i >= n) return;
    lk_tma_init(sm, tid);
    auto T = lk_tma_of<typename LKForm<ROLES>::Tma>(M);
    float2 p = prev_pts[i], init = use_init ? next_pts[i] : p, out;
    int st, iters = 0, fallbacks = 0;
    long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    lk_track_point(sm, tid, I, J, p, init, use_init != 0, max_level, out, st, iters, fallbacks, pc, T);
    if (tid == 0) { next_pts[i] = out; status[i] = (uint8_t)st; }
}

// Prediction pass (feature_tracker.cpp:118-124): maxLevel 1 seeded with predict_pts; counts successes.  Feature blockIdx.x < n_prev.
template <int V, bool ROLES>
__device__ __forceinline__ void lk_pred_point(const Pyramid& prev, const Pyramid& cur, TrackScalars* sc, const FeatArrays& fa, const LKMapSet& M)
{
    __shared__ typename LKForm<ROLES>::Smem sm;
    const int tid = threadIdx.x, i = blockIdx.x;
    lk_tma_init(sm, tid);
    auto T = lk_tma_of<typename LKForm<ROLES>::Tma>(M);
    float2 out;
    int st, iters = 0, fallbacks = 0;
    long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    lk_track_point(sm, tid, prev, cur, fa.prev_pts[i], fa.pred_pts[i], true, 1, out, st, iters, fallbacks, pc, T);
    if (tid == 0) { fa.cur_pts[i] = out; fa.status[i] = (uint8_t)st; if (st) atomicAdd(&sc->pred_succ, 1); atomicAdd(&sc->lk_iters, iters); }
}
template <bool ROLES>
__global__ void __launch_bounds__(LK_THREADS) k_lk_pred(const __grid_constant__ Pyramid prev, const __grid_constant__ Pyramid cur, TrackScalars* sc, FeatArrays fa, const __grid_constant__ LKMapSet M)
{
    if ((int)blockIdx.x >= sc->n_prev) return;
    lk_pred_point<0, ROLES>(prev, cur, sc, fa, M);
}

// Forward LK (3 levels) + reverse check (1 level, USE_INITIAL_FLOW) + inBorder + grey<=250
// (feature_tracker.cpp:118-168).  One CTA of 4 warps per feature.
#ifndef GF_TRACK_MIN_CTAS
#define GF_TRACK_MIN_CTAS 3          // 80 registers: three features per SM when several streams share the GPU (2: 110 registers)
#endif
template <int V, bool ROLES>
__device__ __forceinline__ void track_point(const Pyramid& prev, const Pyramid& cur, TrackScalars* sc, const FeatArrays& fa,
                                            const FrameParams* fp, int flow_back, const LKMapSet& M)
{
    __shared__ typename LKForm<ROLES>::Smem sm;
    const int tid = threadIdx.x, i = blockIdx.x;
    lk_tma_init(sm, tid);
    auto T = lk_tma_of<typename LKForm<ROLES>::Tma>(M);
    const float2 p = fa.prev_pts[i];
    const long long t0 = gf_clock();
    float2 q;
    int st, iters = 0, fallbacks = 0;
    long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (fp->has_pred && sc->pred_succ >= 10) { q = fa.cur_pts[i]; st = fa.status[i]; }
    else lk_track_point(sm, tid, prev, cur, p, p, false, 3, q, st, iters, fallbacks, pc, T);
    if (flow_back) {
        float2 r;
        int rst;
        T.mi = M.curI; T.mj = M.prevJ;          // roles swap for the reverse check
        lk_track_point(sm, tid, cur, prev, q, p, true, 1, r, rst, iters, fallbacks, pc, T);
        double dx = (double)(p.x - r.x), dy = (double)(p.y - r.y);
        st = (st && rst && sqrt(dx * dx + dy * dy) <= 0.5) ? 1 : 0;
    }
    const int col = cur.lv[0].w, row = cur.lv[0].h;
    if (st) {   // inBorder (feature_tracker.cpp:14-20)
        int ix = __float2int_rn(q.x), iy = __float2int_rn(q.y);
        if (!(1 <= ix && ix < col - 1 && 1 <= iy && iy < row - 1)) st = 0;
    }
    if (st) {   // cur_img.at<uchar>((int)x, (int)y): row = x, col = y (sic); out of bounds => not saturated
        int p_u = __float2int_rz(q.x), p_v = __float2int_rz(q.y);
        int grey = (p_u >= 0 && p_u < row && p_v >= 0 && p_v < col) ? cur.lv[0].ptr[(size_t)p_u * cur.lv[0].pitch + p_v] : 0;
        if (grey > 250) st = 0;
    }
    if (tid == 0) {
        fa.cur_pts[i] = q; fa.status[i] = (uint8_t)st; atomicAdd(&sc->lk_iters, iters);
        if (fa.dbg && i < 4) for (int k = 0; k < 8; k++) fa.dbg[32 + 8 * i + k] = pc[k];
        if (fa.dbg) {   // cycles, LK iterations, of which b sums from the integer partials / from the sequential chains,
                        // and the LK form that ran: 2 = two warp roles, 1 = single role
            fa.dbg[64 + 8 * i] = gf_clock() - t0; fa.dbg[64 + 8 * i + 1] = iters;
            fa.dbg[64 + 8 * i + 2] = iters - fallbacks; fa.dbg[64 + 8 * i + 3] = fallbacks;
            fa.dbg[64 + 8 * i + 4] = ROLES ? 2 : 1;
        }
    }
}
template <bool ROLES>
__global__ void __launch_bounds__(LK_THREADS, GF_TRACK_MIN_CTAS) k_track(const __grid_constant__ Pyramid prev, const __grid_constant__ Pyramid cur,
                                                      TrackScalars* sc, FeatArrays fa, const FrameParams* fp, int flow_back, const __grid_constant__ LKMapSet M)
{
    if ((int)blockIdx.x >= sc->n_prev) return;
    track_point<0, ROLES>(prev, cur, sc, fa, fp, flow_back, M);
}

// setPrediction (feature_tracker.cpp:1006-1027)
__global__ void k_set_prediction(TrackScalars* sc, FeatArrays fa, const int* ids, const double* xyz, int n, CamParams cam)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sc->n_prev) return;
    int id = fa.ids[i];
    float2 pp = fa.prev_pts[i];
    for (int k = 0; k < n; k++)
        if (ids[k] == id) {
            double u, v;
            cam_project(cam, xyz[3 * k], xyz[3 * k + 1], xyz[3 * k + 2], u, v);
            pp = make_float2((float)u, (float)v);
            break;
        }
    fa.pred_pts[i] = pp;
    if (i == 0) sc->pred_succ = 0;
}

// removeOutliers (feature_tracker.cpp:1029-1045): stable removal from prev_pts / ids / track_cnt
__global__ void __launch_bounds__(FE_CAP) k_remove_ids(TrackScalars* sc, FeatArrays fa, const int* ids, int n)
{
    __shared__ int warp_sums[32];
    __shared__ int s_m;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int np = sc->n_prev;
    int keep = 0;
    float2 p, un; int id = 0, cnt = 0;
    if (tid < np) {
        id = fa.ids[tid]; p = fa.prev_pts[tid]; un = fa.prev_un[tid]; cnt = fa.track_cnt[tid];
        keep = 1;
        for (int k = 0; k < n; k++) if (ids[k] == id) { keep = 0; break; }
    }
    unsigned bal = __ballot_sync(0xffffffffu, keep);
    int pre = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_sums[wid] = __popc(bal);
    __syncthreads();
    if (wid == 0) {
        int v = warp_sums[lane], incl = v;
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        warp_sums[lane] = incl - v;
        if (lane == 31) s_m = incl;
    }
    __syncthreads();
    if (keep) {
        int d = warp_sums[wid] + pre;
        fa.prev_pts[d] = p; fa.ids[d] = id; fa.track_cnt[d] = cnt; fa.prev_un[d] = un;
    }
    if (tid == 0) sc->n_prev = s_m;
}

// ------------------------------------------------------------------------------------------------
// gf_tracker_group: the kernels of one frame, run once for every member of the group.  Member m's buffers for the step are
// row m of a table packed on the host and copied to the device with the frame; each kernel takes m from the grid dimension
// its single-tracker form does not use (z for 2-D grids, y for 1-D ones, y for the single-CTA kernels) and runs the body the
// single-tracker kernel runs.
// ------------------------------------------------------------------------------------------------
struct GroupMember {
    Pyramid prev, cur;                 // the member's pyramid slots of this step (cur level 0 holds the frame)
    const LKMapSet* maps;              // its tensor maps for these slots, in global memory (see lk_maps_acquire)
    TrackScalars* sc;
    FeatArrays fa;
    NmsGrid grid;
    CamParams cam;
    float* eig; double* cov; float* box;
    const uint16_t* depth;
    const uint8_t* raw; uint8_t* lut;  // equalize: the raw frame and the CLAHE LUTs
    OutHeader* hdr; gf_obs* obs; uint8_t* status; uint32_t* in_box;    // the member's result block of the step
    FrameParams fp;
};

// The 16 maps of a member cannot all be __grid_constant__ parameters of a launch that covers up to GF_TRACKER_GROUP_MAX
// members, so they are read from global memory.  They are written by a host copy when the group is created, long before any
// launch that reads them; the tensormap-proxy acquire fence orders that write before the TMA unit's reads, as the PTX memory
// model requires for a tensor map that is not a kernel parameter.  Threads 0 and 32 are the ones that issue the window loads.
__device__ __forceinline__ void lk_maps_acquire(const LKMapSet* M, int tid)
{
    if ((tid == 0 || tid == 32) && M->enabled) {
        const CUtensorMap* m = M->prevI;       // prevI, curJ, curI, prevJ are contiguous
        for (int k = 0; k < 4 * LK_MAXLEV; k++)
            asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(m + k) : "memory");
    }
}

__global__ void __launch_bounds__(PD_TX* PD_TY) k_pyr_down_g(const GroupMember* __restrict__ tab, int l)
{
    const GroupMember& G = tab[blockIdx.z];
    const Level& d = G.cur.lv[l];
    pyr_down_tile<1>(G.cur.lv[l - 1], const_cast<uint8_t*>(d.ptr), d.w, d.h, d.pitch);
}
__global__ void __launch_bounds__(EIG_TX) k_cov_rows_g(const GroupMember* __restrict__ tab)
{
    const GroupMember& G = tab[blockIdx.z];
    cov_rows_tile<1>(G.cur.lv[0], G.cov);
}
__global__ void __launch_bounds__(96) k_box_chain_g(const GroupMember* __restrict__ tab, int bp, int w, int h)
{
    const GroupMember& G = tab[blockIdx.y];
    box_chain_block<1>(G.cov, G.box, bp, w, h);
}
__global__ void __launch_bounds__(256) k_eig_from_box_g(const GroupMember* __restrict__ tab, int bp, int epitch, int w, int h)
{
    const GroupMember& G = tab[blockIdx.z];
    eig_from_box_tile<1>(G.box, bp, G.eig, epitch, w, h);
}
__global__ void __launch_bounds__(CLAHE_LUT_THREADS) k_clahe_lut_g(const GroupMember* __restrict__ tab, long long pitch, ClaheGeom g)
{
    const GroupMember& G = tab[blockIdx.y];
    clahe_lut_tile<1>(G.raw, pitch, g, G.lut);
}
__global__ void __launch_bounds__(CLAHE_APPLY_THREADS) k_clahe_apply_g(const GroupMember* __restrict__ tab, long long pitch, ClaheGeom g)
{
    const GroupMember& G = tab[blockIdx.y];
    clahe_apply_rows<1>(G.raw, pitch, g, G.lut, const_cast<uint8_t*>(G.cur.lv[0].ptr), G.cur.lv[0].pitch);
}
__global__ void __launch_bounds__(LK_THREADS) k_lk_pred_g(const GroupMember* __restrict__ tab)
{
    const GroupMember& G = tab[blockIdx.y];
    if (!G.fp.has_pred || (int)blockIdx.x >= G.sc->n_prev) return;
    lk_maps_acquire(G.maps, threadIdx.x);
    lk_pred_point<1, false>(G.prev, G.cur, G.sc, G.fa, *G.maps);     // a group is several cameras: the single-role form
}
__global__ void __launch_bounds__(LK_THREADS, GF_TRACK_MIN_CTAS) k_track_g(const GroupMember* __restrict__ tab, int flow_back)
{
    const GroupMember& G = tab[blockIdx.y];
    if ((int)blockIdx.x >= G.sc->n_prev) return;
    lk_maps_acquire(G.maps, threadIdx.x);
    track_point<1, false>(G.prev, G.cur, G.sc, G.fa, &G.fp, flow_back, *G.maps);
}
__global__ void __launch_bounds__(FE_CAP) k_compact_setmask_g(const GroupMember* __restrict__ tab, int min_dist)
{
    const GroupMember& G = tab[blockIdx.y];
    compact_setmask<1>(G.sc, G.fa, min_dist);
}
__global__ void __launch_bounds__(256) k_eig_max_g(const GroupMember* __restrict__ tab, int epitch, int w, int h, int r)
{
    const GroupMember& G = tab[blockIdx.z];
    eig_max_tile<1>(G.sc, G.fa.kept_pts, G.eig, epitch, w, h, r);
}
__global__ void __launch_bounds__(256) k_candidates_g(const GroupMember* __restrict__ tab, int epitch, int w, int h, int r)
{
    const GroupMember& G = tab[blockIdx.z];
    candidates_tile<1>(G.sc, G.fa.kept_pts, G.eig, epitch, w, h, r, G.grid);
}
__global__ void __launch_bounds__(1024) k_select_finalize_g(const GroupMember* __restrict__ tab, int w, int h, int max_cnt, int min_dist,
                                                            int dpitch, int depth_cam_cfg)
{
    const GroupMember& G = tab[blockIdx.y];
    select_finalize<1>(G.sc, G.fa, G.grid, w, max_cnt, min_dist, G.cam, &G.fp.dt, G.depth, dpitch, depth_cam_cfg, &G.fp.depth_valid, h,
                    G.hdr, G.obs, G.status, &G.fp.boxes, G.in_box);
}

}  // namespace gf

using namespace gf;

// ------------------------------------------------------------------------------------------------
constexpr int GF_PIPE = 2;           // frames in flight
struct OutBlock { OutHeader hdr; uint8_t status[FE_CAP]; uint32_t in_box[FE_CAP / 32]; gf_obs obs[FE_CAP]; };   // one D2H copy per frame
static_assert(GF_BOX_CAP == GF_MAX_BOXES, "BoxSet holds GF_MAX_BOXES boxes");

struct gf_tracker {
    int device, w, h;
    gf_tracker_cfg cfg;
    CamParams cam;
    cudaStream_t s_up, s_pyr, s_eig, s_main, s_out;
    cudaEvent_t ev_up[2], ev_pyr[2], ev_eig[2], ev_dep[2], ev_t0[2], ev_out[2];
    cudaEvent_t ev_st[GF_FE_STAGES + 2];   // stage boundaries (profiling mode)
    cudaEvent_t ev_span0, ev_span1;        // gf_tracker_timer_start / _stop
    bool profiling;
    float stage_ms[GF_FE_STAGES];
    // CUDA graphs keyed by frame number mod 6 (= pyramid slot mod 3 x two-slot buffers)
    cudaGraphExec_t g_pyr[6], g_eig[6], g_dep1[6][2][2], g_dep2[6];     // g_dep1[frame][prediction][LK roles]
    int gk_pyr[6], gk_eig[6], gk_dep1[6][2][2], gk_dep2[6];
    bool counted;                                                          // in g_live_trackers
    bool use_graph;
    // gf_tracker_set_equalize: CLAHE of every gray frame into pyramid level 0.  Frames land in d_raw first; the copy and both
    // CLAHE kernels (a graph keyed by pyramid slot) run in order on s_up, so one raw buffer and one LUT block serve every frame
    // in flight.
    bool equalize;
    ClaheGeom clahe;
    cudaGraphExec_t g_clahe[3]; int gk_clahe[3];
    uint8_t* d_raw; int raw_pitch;
    uint8_t* d_lut;
    uint8_t* d_pyr[3][4];
    LKMapSet lk_maps[3];                   // [cur slot]: previous pyramid = slot (cur + 2) % 3
    int lw[4], lh[4], lp[4];
    uint16_t* d_depth[2]; int depth_pitch_el;
    float* d_eig[2]; int epitch;
    double* d_cov; float* d_box;          // min-eig intermediates (fe_eig.cuh), only live inside one frame's s_eig work
    NmsGrid grid; size_t grid_cells;
    TrackScalars* d_sc;
    FeatArrays fa;
    OutBlock* d_out[2];
    FrameParams* d_fp[2];
    int* d_tmp_ids; double* d_tmp_xyz;
    // pinned host
    uint8_t* h_gray; uint16_t* h_depth; OutBlock* h_out[2]; FrameParams* h_fp[2];
    int* h_tmp_ids; double* h_tmp_xyz;
    long long n_submitted, n_waited;     // frame counters; n_submitted - n_waited frames are in flight
    int group_steps;                     // of those, steps of a gf_tracker_group (collected by gf_tracker_group_wait only)
    double prev_time;
    bool has_pred, depth_valid[2];
    float last_ms;
    long long out_frame1;                // 1 + the index of the frame gf_tracker_wait last returned (its results are in slot index % 2 until
                                         // frame index + GF_PIPE is submitted); 0: none, or a group step
};

static inline int in_flight(const gf_tracker* t) { return (int)(t->n_submitted - t->n_waited); }

// The number of features a result block returns.  Reference quirk: depth_cam with an empty depth image produces an empty
// featureFrame (feature_tracker.cpp:342).
static int out_count(const gf_tracker* t, const OutBlock* ob, bool depth_valid)
{
    return (t->cfg.depth_cam && !depth_valid) ? 0 : ob->hdr.n_out;
}

// Copies the host copy of a result block (an OutBlock prefix up to obs[max_cnt]) into the caller's arrays, each nullable.
static void decode_out(const gf_tracker* t, const OutBlock* ob, bool depth_valid, gf_obs* out, int* n_out, uint8_t* in_box,
                       uint8_t* status_out, gf_track_info* info)
{
    const OutHeader& hd = ob->hdr;
    const int n = out_count(t, ob, depth_valid);
    if (n_out) *n_out = n;
    if (out && n > 0) memcpy(out, ob->obs, (size_t)n * sizeof(gf_obs));
    if (in_box) for (int i = 0; i < n; i++) in_box[i] = (uint8_t)((ob->in_box[i >> 5] >> (i & 31)) & 1u);
    if (status_out && hd.n_prev > 0) memcpy(status_out, ob->status, hd.n_prev);
    if (info) {
        info->n_prev = hd.n_prev; info->n_tracked = hd.n_tracked; info->n_kept = hd.n_kept; info->n_new = hd.n_new;
        info->n_candidates = hd.n_cand; info->nms_rounds = hd.nms_rounds; info->eig_fixups = hd.eig_fixups; info->lk_iterations = hd.lk_iters;
    }
}

// Trackers alive per device (gf_tracker_create .. gf_tracker_destroy).  A tracker alone on its device runs k_track in the
// two-role LK form, which shortens the slowest feature's chain; while other trackers share the device, the throughput of
// all of them counts and the single-role form is faster (DESIGN.md §1.3).  The choice is made per frame; each form has
// its own captured graph.
constexpr int GF_LIVE_DEVICES = 64;
static std::atomic<int> g_live_trackers[GF_LIVE_DEVICES];
static inline bool lk_roles(const gf_tracker* t)
{
    return t->device >= GF_LIVE_DEVICES || g_live_trackers[t->device].load() <= 1;
}

static Pyramid make_pyr(const gf_tracker* t, int slot)
{
    Pyramid P;
    for (int l = 0; l < 4; l++) { P.lv[l].ptr = t->d_pyr[slot][l]; P.lv[l].w = t->lw[l]; P.lv[l].h = t->lh[l]; P.lv[l].pitch = t->lp[l]; }
    return P;
}

// ---- tensor maps of the LK windows (fe_lk.cuh) ----
typedef CUresult (*gf_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                       const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static int encode_u8_box(CUtensorMap* m, const Level& L, int box_w, int box_h)
{
    static gf_encode_tiled_fn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
        if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) return set_err(GF_ERR_CUDA, "cuTensorMapEncodeTiled is not available in this driver");
        fn = (gf_encode_tiled_fn)p;
    }
    if (((uintptr_t)L.ptr & 15) || (L.pitch & 15)) return set_err(GF_ERR_UNSUPPORTED, "pyramid level not addressable by a tensor map");
    const cuuint64_t dims[2] = {(cuuint64_t)L.w, (cuuint64_t)L.h}, strides[1] = {(cuuint64_t)L.pitch};
    const cuuint32_t box[2] = {(cuuint32_t)box_w, (cuuint32_t)box_h}, estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void*)L.ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { snprintf(g_err, sizeof(g_err), "cuTensorMapEncodeTiled failed (%d) for a %dx%d level", (int)r, L.w, L.h); return GF_ERR_CUDA; }
    return GF_OK;
}
// Window maps for LK from `prev` to `cur` and back.  GF_LK_NO_TMA=1 keeps the per-thread loads (A/B measurements).
static int make_lk_maps(LKMapSet* M, const Pyramid& prev, const Pyramid& cur, int levels = LK_MAXLEV)
{
    memset(M, 0, sizeof(*M));
    if (getenv("GF_LK_NO_TMA")) return GF_OK;
    for (int l = 0; l < LK_MAXLEV; l++) {
        const int k = l < levels ? l : levels - 1;
        // a level narrower than the search box (images below 640 px wide at level 3) keeps the per-thread loads for the whole set:
        // boxes wider than the tensor are not something this code has been run with
        const bool fits = prev.lv[k].w >= LK_JPITCH && cur.lv[k].w >= LK_JPITCH && prev.lv[k].h >= LK_JR && cur.lv[k].h >= LK_JR;
        if (!fits ||
            encode_u8_box(&M->prevI[l], prev.lv[k], LK_IPITCH, LK_IREG) || encode_u8_box(&M->curJ[l], cur.lv[k], LK_JPITCH, LK_JR) ||
            encode_u8_box(&M->curI[l], cur.lv[k], LK_IPITCH, LK_IREG) || encode_u8_box(&M->prevJ[l], prev.lv[k], LK_JPITCH, LK_JR)) {
            memset(M, 0, sizeof(*M));          // enabled = 0: the kernels stage the windows with ordinary loads
            return GF_OK;
        }
    }
    M->enabled = 1;
    return GF_OK;
}

static int select_device(int device)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        snprintf(g_err, sizeof(g_err), "no CUDA device visible (%s); libgf_b200 has no CPU fallback", cudaGetErrorString(e));
        return GF_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= n) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    return GF_OK;
}

static int alloc_nms_grid(NmsGrid& g, int w, int h, int min_dist, size_t* smem_bytes)
{
    g.cs = min_dist > 16 ? min_dist : 16;      // any cell size >= min_dist is exact; larger cells only cost rounds
    while (nms_smem_bytes((w + g.cs - 1) / g.cs, (h + g.cs - 1) / g.cs) > 160 * 1024) g.cs++;
    g.gw = (w + g.cs - 1) / g.cs;
    g.gh = (h + g.cs - 1) / g.cs;
    g.acc_cap = w * h / 16 + 64;
    GF_CUDA(cudaMalloc(&g.cand_key, (size_t)w * h * sizeof(unsigned long long)));
    GF_CUDA(cudaMalloc(&g.acc_key, (size_t)g.acc_cap * sizeof(unsigned long long)));
    size_t bytes = nms_smem_bytes(g.gw, g.gh);
    if (bytes > 160 * 1024) return set_err(GF_ERR_UNSUPPORTED, "image too large for the min-distance cell grid");
    GF_CUDA(cudaMalloc(&g.dead, (size_t)w * h));
    GF_CUDA(cudaFuncSetAttribute(k_select_finalize, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    if (smem_bytes) *smem_bytes = bytes;
    return GF_OK;
}
static void free_nms_grid(NmsGrid& g)
{
    cudaFree(g.cand_key); cudaFree(g.acc_key); cudaFree(g.dead);
}

// GFTT tail shared by the tracker and gf_stage_gftt: mask -> max -> candidates -> NMS rounds
static int enqueue_gftt_select(cudaStream_t s, TrackScalars* d_sc, const float2* kept_pts, const float* d_eig, int epitch, int w, int h,
                               int min_dist, NmsGrid& grid)
{
    dim3 tg((w + MASK_TX - 1) / MASK_TX, (h + MASK_TY - 1) / MASK_TY);
    k_eig_max<<<tg, 256, 0, s>>>(d_sc, kept_pts, d_eig, epitch, w, h, min_dist); GF_LAUNCHED();
    k_candidates<<<tg, 256, 0, s>>>(d_sc, kept_pts, d_eig, epitch, w, h, min_dist, grid); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

// cov: cov_rows_elems(w, h) doubles (zero-initialised once: the padding columns of the last block are streamed too);
// box: box_elems(w, h) floats
static int enqueue_min_eig(cudaStream_t s, const Level& img, float* d_eig, int epitch, double* d_cov, float* d_box)
{
    static bool attr_done[64] = {};     // per device
    int dev = 0;
    GF_CUDA(cudaGetDevice(&dev));
    if (!attr_done[dev & 63]) {
        GF_CUDA(cudaFuncSetAttribute(k_box_chain, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BC_SMEM));
        attr_done[dev & 63] = true;
    }
    dim3 g((img.w + EIG_TX - 1) / EIG_TX, (img.h + EIG_BAND - 1) / EIG_BAND);
    k_cov_rows<<<g, EIG_TX, 0, s>>>(img, d_cov); GF_LAUNCHED();
    const int bp = (img.w + 31) / 32 * 32;
    k_box_chain<<<(img.w + 31) / 32, 96, BC_SMEM, s>>>(d_cov, d_box, bp, img.w, img.h); GF_LAUNCHED();
    dim3 g3((img.w + 63) / 64, (img.h + 15) / 16);
    k_eig_from_box<<<g3, 256, 0, s>>>(d_box, bp, d_eig, epitch, img.w, img.h); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

static int enqueue_pyramid(cudaStream_t s, const gf_tracker* t, int slot)
{
    for (int l = 1; l < 4; l++) {
        Level src{t->d_pyr[slot][l - 1], t->lw[l - 1], t->lh[l - 1], t->lp[l - 1]};
        dim3 g((t->lw[l] + PD_TX - 1) / PD_TX, (t->lh[l] + PD_TY - 1) / PD_TY), b(PD_TX, PD_TY);
        k_pyr_down<<<g, b, 0, s>>>(src, t->d_pyr[slot][l], t->lw[l], t->lh[l], t->lp[l]); GF_LAUNCHED();
    }
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

extern "C" {

const char* gf_last_error(void) { return g_err; }
const char* gf_version(void) { return "gf_b200 0.1 sm_90a"; }
uint64_t gf_kernel_launch_count(void) { return g_launches.load(); }

static int tracker_init(gf_tracker* t, int width, int height, const gf_tracker_cfg* cfg);

int gf_tracker_create(gf_tracker** out, int device, int width, int height, const gf_tracker_cfg* cfg)
{
    if (!out || !cfg) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    if (cfg->max_cnt < 1 || cfg->max_cnt > FE_CAP) return set_err(GF_ERR_CAPACITY, "max_cnt must be in [1, 1024]");
    if (cfg->min_dist < 5 || cfg->min_dist > 255) return set_err(GF_ERR_INVALID_ARG, "min_dist must be in [5, 255]");
    // the 4-level pyramid needs every level larger than the 21x21 window plus the cached-region reach
    if (((width + 7) / 8) < 48 || ((height + 7) / 8) < 48 || width > 8192 || height > 8192)
        return set_err(GF_ERR_UNSUPPORTED, "image must be at least 377x377 and at most 8192x8192");
    int rc = select_device(device);
    if (rc) return rc;
    gf_tracker* t = new (std::nothrow) gf_tracker();
    if (!t) return set_err(GF_ERR_CUDA, "out of host memory");
    memset(t, 0, sizeof(*t));
    t->device = device; t->w = width; t->h = height; t->cfg = *cfg; t->cam = make_cam(cfg->pinhole);
    rc = tracker_init(t, width, height, cfg);
    if (rc) {                       // release whatever was created before the failure; keep the error text of the failure
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        gf_tracker_destroy(t);
        cudaGetLastError();
        memcpy(g_err, keep, sizeof(keep));
        return rc;
    }
    if (device < GF_LIVE_DEVICES) { g_live_trackers[device]++; t->counted = true; }
    *out = t;
    return GF_OK;
}

static int tracker_init(gf_tracker* t, int width, int height, const gf_tracker_cfg* cfg)
{
    int rc;
    GF_CUDA(cudaStreamCreateWithFlags(&t->s_up, cudaStreamNonBlocking));
    GF_CUDA(cudaStreamCreateWithFlags(&t->s_pyr, cudaStreamNonBlocking));
    GF_CUDA(cudaStreamCreateWithFlags(&t->s_eig, cudaStreamNonBlocking));
    GF_CUDA(cudaStreamCreateWithFlags(&t->s_main, cudaStreamNonBlocking));
    GF_CUDA(cudaStreamCreateWithFlags(&t->s_out, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) {
        GF_CUDA(cudaEventCreateWithFlags(&t->ev_up[i], cudaEventDisableTiming));
        GF_CUDA(cudaEventCreateWithFlags(&t->ev_pyr[i], cudaEventDisableTiming));
        GF_CUDA(cudaEventCreateWithFlags(&t->ev_eig[i], cudaEventDisableTiming));
        GF_CUDA(cudaEventCreateWithFlags(&t->ev_dep[i], cudaEventDisableTiming));
        GF_CUDA(cudaEventCreate(&t->ev_t0[i]));
        GF_CUDA(cudaEventCreate(&t->ev_out[i]));
    }
    for (int i = 0; i < GF_FE_STAGES + 2; i++) GF_CUDA(cudaEventCreate(&t->ev_st[i]));
    GF_CUDA(cudaEventCreate(&t->ev_span0)); GF_CUDA(cudaEventCreate(&t->ev_span1));
    int lw = width, lh = height;
    for (int l = 0; l < 4; l++) {
        t->lw[l] = lw; t->lh[l] = lh; t->lp[l] = align_up(lw, 16);
        for (int s = 0; s < 3; s++) {
            GF_CUDA(cudaMalloc(&t->d_pyr[s][l], (size_t)t->lp[l] * lh + 16));   // +16: aligned window loads may overrun the last row by <4 B
            GF_CUDA(cudaMemset(t->d_pyr[s][l], 0, (size_t)t->lp[l] * lh + 16));
        }
        lw = (lw + 1) / 2; lh = (lh + 1) / 2;
    }
    for (int c = 0; c < 3; c++) {
        rc = make_lk_maps(&t->lk_maps[c], make_pyr(t, (c + 2) % 3), make_pyr(t, c));
        if (rc) return rc;
    }
    t->depth_pitch_el = align_up(width, 8);
    t->epitch = align_up(width, 4);
    for (int i = 0; i < 2; i++) {
        GF_CUDA(cudaMalloc(&t->d_depth[i], (size_t)t->depth_pitch_el * height * sizeof(uint16_t)));
        GF_CUDA(cudaMalloc(&t->d_eig[i], (size_t)t->epitch * height * sizeof(float)));
        GF_CUDA(cudaMalloc(&t->d_out[i], sizeof(OutBlock)));
        GF_CUDA(cudaMalloc(&t->d_fp[i], sizeof(FrameParams)));
        GF_CUDA(cudaHostAlloc(&t->h_out[i], sizeof(OutBlock), cudaHostAllocDefault));
        GF_CUDA(cudaHostAlloc(&t->h_fp[i], sizeof(FrameParams), cudaHostAllocDefault));
    }
    GF_CUDA(cudaMalloc(&t->d_cov, cov_rows_elems(width, height) * sizeof(double)));
    GF_CUDA(cudaMemset(t->d_cov, 0, cov_rows_elems(width, height) * sizeof(double)));
    GF_CUDA(cudaMalloc(&t->d_box, box_elems(width, height) * sizeof(float)));
    rc = alloc_nms_grid(t->grid, width, height, cfg->min_dist, &t->grid_cells);
    if (rc) return rc;
    GF_CUDA(cudaMalloc(&t->d_sc, sizeof(TrackScalars)));
    GF_CUDA(cudaMemset(t->d_sc, 0, sizeof(TrackScalars)));
    FeatArrays& fa = t->fa;
    GF_CUDA(cudaMalloc(&fa.prev_pts, FE_CAP * sizeof(float2))); GF_CUDA(cudaMalloc(&fa.ids, FE_CAP * sizeof(int)));
    GF_CUDA(cudaMalloc(&fa.track_cnt, FE_CAP * sizeof(int))); GF_CUDA(cudaMalloc(&fa.prev_un, FE_CAP * sizeof(float2)));
    GF_CUDA(cudaMalloc(&fa.cur_pts, FE_CAP * sizeof(float2))); GF_CUDA(cudaMalloc(&fa.status, FE_CAP));
    GF_CUDA(cudaMalloc(&fa.kept_pts, FE_CAP * sizeof(float2))); GF_CUDA(cudaMalloc(&fa.kept_ids, FE_CAP * sizeof(int)));
    GF_CUDA(cudaMalloc(&fa.kept_cnt, FE_CAP * sizeof(int))); GF_CUDA(cudaMalloc(&fa.kept_un, FE_CAP * sizeof(float2)));
    GF_CUDA(cudaMalloc(&fa.pred_pts, FE_CAP * sizeof(float2)));
    GF_CUDA(cudaMalloc(&fa.dbg, FE_DBG_N * sizeof(long long))); GF_CUDA(cudaMemset(fa.dbg, 0, FE_DBG_N * sizeof(long long)));
    GF_CUDA(cudaMemset(fa.status, 0, FE_CAP));
    GF_CUDA(cudaMalloc(&t->d_tmp_ids, FE_CAP * sizeof(int)));
    GF_CUDA(cudaMalloc(&t->d_tmp_xyz, FE_CAP * 3 * sizeof(double)));
    GF_CUDA(cudaHostAlloc(&t->h_gray, (size_t)width * height, cudaHostAllocDefault));
    GF_CUDA(cudaHostAlloc(&t->h_depth, (size_t)width * height * sizeof(uint16_t), cudaHostAllocDefault));
    GF_CUDA(cudaHostAlloc(&t->h_tmp_ids, FE_CAP * sizeof(int), cudaHostAllocDefault));
    GF_CUDA(cudaHostAlloc(&t->h_tmp_xyz, FE_CAP * 3 * sizeof(double), cudaHostAllocDefault));
    t->use_graph = getenv("GF_NO_GRAPH") == nullptr;
    GF_CUDA(cudaDeviceSynchronize());
    return GF_OK;
}

void gf_tracker_destroy(gf_tracker* t)
{
    if (!t) return;
    if (t->counted) g_live_trackers[t->device]--;
    cudaSetDevice(t->device);
    cudaDeviceSynchronize();        // (a partially built tracker may lack some of its streams)
    for (int k = 0; k < 6; k++) {
        if (t->g_pyr[k]) cudaGraphExecDestroy(t->g_pyr[k]);
        if (t->g_eig[k]) cudaGraphExecDestroy(t->g_eig[k]);
        if (t->g_dep2[k]) cudaGraphExecDestroy(t->g_dep2[k]);
        for (int p = 0; p < 4; p++) if (t->g_dep1[k][p / 2][p % 2]) cudaGraphExecDestroy(t->g_dep1[k][p / 2][p % 2]);
    }
    for (int k = 0; k < 3; k++) if (t->g_clahe[k]) cudaGraphExecDestroy(t->g_clahe[k]);
    for (int s = 0; s < 3; s++) for (int l = 0; l < 4; l++) cudaFree(t->d_pyr[s][l]);
    for (int i = 0; i < 2; i++) {
        cudaFree(t->d_depth[i]); cudaFree(t->d_eig[i]); cudaFree(t->d_out[i]); cudaFree(t->d_fp[i]);
        cudaFreeHost(t->h_out[i]); cudaFreeHost(t->h_fp[i]);
        for (cudaEvent_t e : {t->ev_up[i], t->ev_pyr[i], t->ev_eig[i], t->ev_dep[i], t->ev_t0[i], t->ev_out[i]}) if (e) cudaEventDestroy(e);
    }
    cudaFree(t->d_cov); cudaFree(t->d_box);
    cudaFree(t->d_raw); cudaFree(t->d_lut);
    free_nms_grid(t->grid);
    cudaFree(t->d_sc);
    FeatArrays& fa = t->fa;
    cudaFree(fa.prev_pts); cudaFree(fa.ids); cudaFree(fa.track_cnt); cudaFree(fa.prev_un); cudaFree(fa.cur_pts); cudaFree(fa.status);
    cudaFree(fa.kept_pts); cudaFree(fa.kept_ids); cudaFree(fa.kept_cnt); cudaFree(fa.kept_un); cudaFree(fa.pred_pts); cudaFree(fa.dbg);
    cudaFree(t->d_tmp_ids); cudaFree(t->d_tmp_xyz);
    cudaFreeHost(t->h_gray); cudaFreeHost(t->h_depth); cudaFreeHost(t->h_tmp_ids); cudaFreeHost(t->h_tmp_xyz);
    for (cudaStream_t st_ : {t->s_up, t->s_pyr, t->s_eig, t->s_main, t->s_out}) if (st_) cudaStreamDestroy(st_);
    for (int i = 0; i < GF_FE_STAGES + 2; i++) if (t->ev_st[i]) cudaEventDestroy(t->ev_st[i]);
    if (t->ev_span0) cudaEventDestroy(t->ev_span0);
    if (t->ev_span1) cudaEventDestroy(t->ev_span1);
    cudaGetLastError();
    delete t;
}

int gf_tracker_set_equalize(gf_tracker* t, double clip_limit, int tiles_x, int tiles_y)
{
    if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
    // accepted before the first frame only: no captured graph ever has to change
    if (t->n_submitted > 0) return set_err(GF_ERR_INVALID_ARG, "gf_tracker_set_equalize must be called before the first frame");
    if (tiles_x == 0) { t->equalize = false; return GF_OK; }
    ClaheGeom g;
    int rc = clahe_geometry(g, t->w, t->h, clip_limit, tiles_x, tiles_y);
    if (rc) return rc;
    GF_CUDA(cudaSetDevice(t->device));
    rc = clahe_prepare(); if (rc) return rc;
    if (!t->d_raw) {
        t->raw_pitch = align_up(t->w, 16);
        GF_CUDA(cudaMalloc(&t->d_raw, (size_t)t->raw_pitch * t->h));
    }
    if (!t->d_lut) GF_CUDA(cudaMalloc(&t->d_lut, (size_t)CLAHE_MAX_TILES * CLAHE_MAX_TILES * 256));
    t->clahe = g;
    t->equalize = true;
    return GF_OK;
}

int gf_tracker_host_buffers(gf_tracker* t, uint8_t** gray, uint16_t** depth)
{
    if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
    if (gray) *gray = t->h_gray;
    if (depth) *depth = t->h_depth;
    return GF_OK;
}

}  // extern "C"

// ---- the four capturable pieces of a frame (fixed addresses for a given frame number mod 6) ----
#define GF_MARK(k, s) do { if (t->profiling) GF_CUDA(cudaEventRecord(t->ev_st[k], s)); } while (0)

static int body_pyr(gf_tracker* t, long long f)
{
    const int es = (int)(f % 2);
    GF_CUDA(cudaMemcpyAsync(t->d_fp[es], t->h_fp[es], sizeof(FrameParams), cudaMemcpyHostToDevice, t->s_pyr));
    return enqueue_pyramid(t->s_pyr, t, (int)(f % 3));
}

static int body_eig(gf_tracker* t, long long f)
{
    Pyramid Pc = make_pyr(t, (int)(f % 3));
    return enqueue_min_eig(t->s_eig, Pc.lv[0], t->d_eig[f % 2], t->epitch, t->d_cov, t->d_box);
}

static int body_dep1(gf_tracker* t, long long f, bool has_pred, bool roles)
{
    cudaStream_t s = t->s_main;
    Pyramid Pc = make_pyr(t, (int)(f % 3)), Pp = make_pyr(t, (int)((f + 2) % 3));
    const int lk_grid = t->cfg.max_cnt;
    const LKMapSet& M = t->lk_maps[f % 3];
    if (roles) {
        if (has_pred) { k_lk_pred<true><<<lk_grid, LK_THREADS, 0, s>>>(Pp, Pc, t->d_sc, t->fa, M); GF_LAUNCHED(); }
        k_track<true><<<lk_grid, LK_THREADS, 0, s>>>(Pp, Pc, t->d_sc, t->fa, t->d_fp[f % 2], t->cfg.flow_back, M); GF_LAUNCHED();
    } else {
        if (has_pred) { k_lk_pred<false><<<lk_grid, LK_THREADS, 0, s>>>(Pp, Pc, t->d_sc, t->fa, M); GF_LAUNCHED(); }
        k_track<false><<<lk_grid, LK_THREADS, 0, s>>>(Pp, Pc, t->d_sc, t->fa, t->d_fp[f % 2], t->cfg.flow_back, M); GF_LAUNCHED();
    }
    GF_MARK(2, s);
    k_compact_setmask<<<1, FE_CAP, 0, s>>>(t->d_sc, t->fa, t->cfg.min_dist); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_MARK(3, s);
    return GF_OK;
}

static int body_dep2(gf_tracker* t, long long f)
{
    cudaStream_t s = t->s_main;
    const int es = (int)(f % 2);
    int rc = enqueue_gftt_select(s, t->d_sc, t->fa.kept_pts, t->d_eig[es], t->epitch, t->w, t->h, t->cfg.min_dist, t->grid);
    if (rc) return rc;
    GF_MARK(4, s);
    // reference quirk: depth_cam with an empty depth image produces an empty featureFrame (feature_tracker.cpp:342)
    const int depth_mode = t->cfg.depth_cam ? 1 : 0;
    OutBlock* ob = t->d_out[es];
    k_select_finalize<<<1, 1024, t->grid_cells, s>>>(t->d_sc, t->fa, t->grid, t->w, t->cfg.max_cnt, t->cfg.min_dist, t->cam, &t->d_fp[es]->dt,
                                                     t->d_depth[es], t->depth_pitch_el, depth_mode, &t->d_fp[es]->depth_valid, t->h,
                                                     &ob->hdr, ob->obs, ob->status, &t->d_fp[es]->boxes, ob->in_box); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_MARK(5, s);
    return GF_OK;
}

// Runs one piece: replays its CUDA graph (captured on first use) or, when `direct` (profiling / GF_NO_GRAPH mode), launches it
// directly.
template <class Body>
static int run_piece(bool direct, cudaStream_t s, cudaGraphExec_t* exec, int* nk, Body body)
{
    if (direct) return body();
    if (!*exec) {
        const uint64_t l0 = g_launches.load();
        cudaGraph_t g = nullptr;
        GF_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        int rc = body();
        cudaError_t e = cudaStreamEndCapture(s, &g);
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        if (e != cudaSuccess) { snprintf(g_err, sizeof(g_err), "graph capture failed: %s", cudaGetErrorString(e)); return GF_ERR_CUDA; }
        GF_CUDA(cudaGraphInstantiate(exec, g, 0));
        cudaGraphDestroy(g);
        *nk = (int)(g_launches.load() - l0);
        g_launches.fetch_sub(*nk);      // capture did not launch anything
    }
    GF_CUDA(cudaGraphLaunch(*exec, s));
    g_launches.fetch_add(*nk);
    return GF_OK;
}

// Enqueues on s the copies of tracker t's next frame: gray into d_raw (equalisation) or pyramid level 0, depth (nullable)
// into the frame's depth slot.
static int enqueue_upload(cudaStream_t s, const gf_tracker* t, const void* gray, size_t gray_pitch, const void* depth, size_t depth_pitch,
                          bool on_device)
{
    const long long f = t->n_submitted;
    const int w = t->w, h = t->h;
    if (on_device) { gray_pitch = w; depth_pitch = (size_t)w * 2; }
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (t->equalize) GF_CUDA(cudaMemcpy2DAsync(t->d_raw, t->raw_pitch, gray, gray_pitch, w, h, kind, s));
    else GF_CUDA(cudaMemcpy2DAsync(t->d_pyr[f % 3][0], t->lp[0], gray, gray_pitch, w, h, kind, s));
    if (depth)
        GF_CUDA(cudaMemcpy2DAsync(t->d_depth[f % 2], (size_t)t->depth_pitch_el * 2, depth, depth_pitch, (size_t)w * 2, h, kind, s));
    return GF_OK;
}

// The parameters of tracker t's next frame, taken at `time`.
static void frame_params(FrameParams* fp, const gf_tracker* t, double time, bool depth_valid, const gf_box* boxes, int n_boxes)
{
    fp->dt = time - t->prev_time;
    fp->has_pred = t->has_pred ? 1 : 0;
    fp->depth_valid = depth_valid ? 1 : 0;
    put_boxes(fp->boxes, boxes, n_boxes);
}

// Advances tracker t's host state past its next frame, once that frame has been enqueued.
static void frame_enqueued(gf_tracker* t, double time, bool depth_valid)
{
    t->prev_time = time;
    t->has_pred = false;
    t->depth_valid[t->n_submitted % 2] = depth_valid;
    t->n_submitted++;
}

// Everything after the H2D (or D2D) copies of frame f have been enqueued on s_up.  With equalisation the gray frame is in
// d_raw and CLAHE writes pyramid level 0 on s_up, ahead of ev_up (profiling: part of stage 1).
static int enqueue_frame(gf_tracker* t, long long f, double time, bool depth_valid, const gf_box* boxes, int n_boxes)
{
    const int es = (int)(f % 2), key = (int)(f % 6), hp = t->has_pred ? 1 : 0;
    const bool direct = !t->use_graph || t->profiling;
    frame_params(t->h_fp[es], t, time, depth_valid, boxes, n_boxes);
    GF_MARK(0, t->s_up);   // end of upload
    if (t->equalize) {
        const int slot = (int)(f % 3);
        int rc = run_piece(direct, t->s_up, &t->g_clahe[slot], &t->gk_clahe[slot], [&] {
            return enqueue_clahe(t->s_up, t->d_raw, t->raw_pitch, t->clahe, t->d_lut, t->d_pyr[slot][0], t->lp[0]);
        });
        if (rc) return rc;
    }
    GF_CUDA(cudaEventRecord(t->ev_up[es], t->s_up));
    GF_CUDA(cudaStreamWaitEvent(t->s_pyr, t->ev_up[es], 0));
    GF_CUDA(cudaStreamWaitEvent(t->s_eig, t->ev_up[es], 0));
    int rc = run_piece(direct, t->s_pyr, &t->g_pyr[key], &t->gk_pyr[key], [&] { return body_pyr(t, f); });
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_pyr[es], t->s_pyr));
    GF_MARK(1, t->s_pyr);
    GF_MARK(7, t->s_eig);
    rc = run_piece(direct, t->s_eig, &t->g_eig[key], &t->gk_eig[key], [&] { return body_eig(t, f); });
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_eig[es], t->s_eig));
    GF_MARK(8, t->s_eig);
    GF_CUDA(cudaStreamWaitEvent(t->s_main, t->ev_pyr[es], 0));
    const int ro = lk_roles(t) ? 1 : 0;
    rc = run_piece(direct, t->s_main, &t->g_dep1[key][hp][ro], &t->gk_dep1[key][hp][ro], [&] { return body_dep1(t, f, hp != 0, ro != 0); });
    if (rc) return rc;
    GF_CUDA(cudaStreamWaitEvent(t->s_main, t->ev_eig[es], 0));
    rc = run_piece(direct, t->s_main, &t->g_dep2[key], &t->gk_dep2[key], [&] { return body_dep2(t, f); });
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_dep[es], t->s_main));
    GF_CUDA(cudaStreamWaitEvent(t->s_out, t->ev_dep[es], 0));
    GF_CUDA(cudaMemcpyAsync(t->h_out[es], t->d_out[es], offsetof(OutBlock, obs) + (size_t)t->cfg.max_cnt * sizeof(gf_obs),
                            cudaMemcpyDeviceToHost, t->s_out));
    GF_CUDA(cudaEventRecord(t->ev_out[es], t->s_out));
    frame_enqueued(t, time, depth_valid);
    return GF_OK;
}

extern "C" {

static int check_submit(gf_tracker* t)
{
    if (in_flight(t) >= GF_PIPE) return set_err(GF_ERR_INVALID_ARG, "two frames in flight: call gf_tracker_wait first");
    // a group step works on this tracker's buffers and state from the group's streams: no direct frame may overlap it
    if (t->group_steps > 0) return set_err(GF_ERR_INVALID_ARG, "a group step is in flight: collect it with gf_tracker_group_wait first");
    if (t->profiling && in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "profiling mode runs one frame at a time");
    return GF_OK;
}

// Frame intake.  The caller's host buffers are read by the copy engine directly: truly asynchronous when they are pinned
// (gf_tracker_host_buffers or any cudaHostAlloc/cudaHostRegister memory: keep them unchanged until the frame has been
// collected); for pageable memory CUDA stages the data before cudaMemcpy2DAsync returns.
int gf_tracker_submit(gf_tracker* t, double time, const void* gray, size_t gray_pitch, const void* depth, size_t depth_pitch, int on_device,
                      const gf_box* boxes, int n_boxes)
{
    int rc = check_boxes(boxes, n_boxes);
    if (rc) return rc;
    if (!t || !gray) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if ((rc = check_submit(t))) return rc;
    GF_CUDA(cudaSetDevice(t->device));
    if ((rc = check_pitches(t->w, on_device != 0, gray_pitch, depth != nullptr, depth_pitch))) return rc;
    const long long f = t->n_submitted;
    GF_CUDA(cudaEventRecord(t->ev_t0[f % 2], t->s_up));
    if ((rc = enqueue_upload(t->s_up, t, gray, gray_pitch, depth, depth_pitch, on_device != 0))) return rc;
    return enqueue_frame(t, f, time, depth != nullptr, boxes, n_boxes);
}

int gf_tracker_wait(gf_tracker* t, gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info)
{
    if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
    if (in_flight(t) == 0) return set_err(GF_ERR_INVALID_ARG, "no frame in flight");
    if (t->group_steps > 0) return set_err(GF_ERR_INVALID_ARG, "the frame in flight is a group step: collect it with gf_tracker_group_wait");
    GF_CUDA(cudaSetDevice(t->device));
    const int es = (int)(t->n_waited % 2);
    GF_CUDA(cudaEventSynchronize(t->ev_out[es]));
    t->n_waited++;
    t->out_frame1 = t->n_waited;         // n_waited was just advanced: 1 + this frame's index
    GF_CUDA(cudaEventElapsedTime(&t->last_ms, t->ev_t0[es], t->ev_out[es]));
    if (t->profiling) {
        cudaEvent_t b[8] = {t->ev_t0[es], t->ev_st[0], t->ev_st[1], t->ev_st[2], t->ev_st[3], t->ev_st[4], t->ev_st[5], t->ev_out[es]};
        for (int i = 0; i < 7; i++) GF_CUDA(cudaEventElapsedTime(&t->stage_ms[i], b[i], b[i + 1]));
        GF_CUDA(cudaEventElapsedTime(&t->stage_ms[7], t->ev_st[7], t->ev_st[8]));
    }
    decode_out(t, t->h_out[es], t->depth_valid[es], out, n_out, in_box, status_out, info);
    return GF_OK;
}

int gf_tracker_track(gf_tracker* t, double time, const void* gray, size_t gray_pitch, const void* depth, size_t depth_pitch, int on_device,
                     const gf_box* boxes, int n_boxes, gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info)
{
    if (t && in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "previous frame not collected: call gf_tracker_wait first");
    int rc = gf_tracker_submit(t, time, gray, gray_pitch, depth, depth_pitch, on_device, boxes, n_boxes);
    if (rc) return rc;
    return gf_tracker_wait(t, out, n_out, in_box, status_out, info);
}

// One camera stream of a batch call: its frames, where its results go, and how far it has got.
struct BatchLane {
    gf_tracker* t;
    const double* times; const void* const* gray; const void* const* depth;
    gf_obs* out; int* n_out; uint8_t* status_out; gf_track_info* info;
    const gf_box* boxes; const int* box_start; uint8_t* in_box;     // frame k: boxes[box_start[k] .. box_start[k + 1]); nullable
    int collected;
    const gf_box* frame_boxes(int k) const { return box_start ? boxes + box_start[k] : nullptr; }
    int n_boxes(int k) const { return box_start ? box_start[k + 1] - box_start[k] : 0; }
};

static int lane_collect(BatchLane& L)
{
    const int k = L.collected++;
    const size_t cap = (size_t)L.t->cfg.max_cnt;
    return gf_tracker_wait(L.t, L.out ? L.out + (size_t)k * cap : nullptr, L.n_out ? L.n_out + k : nullptr,
                           L.in_box ? L.in_box + (size_t)k * cap : nullptr, L.status_out ? L.status_out + (size_t)k * cap : nullptr,
                           L.info ? L.info + k : nullptr);
}

int gf_tracker_track_batch_multi(gf_tracker* const* trackers, int n_trackers, int n, const double* times, const void* const* gray,
                                 size_t gray_pitch, const void* const* depth, size_t depth_pitch, int on_device,
                                 const gf_box* boxes, const int* box_start, gf_obs* out, int* n_out, uint8_t* in_box,
                                 uint8_t* status_out, gf_track_info* info)
{
    if (!trackers || n_trackers < 1 || n < 0 || (n > 0 && (!times || !gray))) return set_err(GF_ERR_INVALID_ARG, "null argument");
    int rc;
    long long bad;
    // every frame's list is checked before the first frame is submitted
    if (box_start && (rc = check_box_lists(boxes, box_start, (long long)n_trackers * n, &bad))) return rc;
    std::vector<BatchLane> lanes((size_t)n_trackers);
    for (int i = 0; i < n_trackers; i++) {
        gf_tracker* t = trackers[i];
        if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
        for (int j = 0; j < i; j++) if (trackers[j] == t) return set_err(GF_ERR_INVALID_ARG, "the same tracker listed twice");
        if (in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "previous frame not collected");
        if (t->profiling) return set_err(GF_ERR_INVALID_ARG, "profiling mode runs one frame at a time");
        if ((rc = check_pitches(t->w, on_device != 0, gray_pitch, depth != nullptr, depth_pitch))) return rc;
        const size_t cap = (size_t)t->cfg.max_cnt, o = (size_t)i * n;
        BatchLane& L = lanes[i];
        L.t = t; L.times = times + o; L.gray = gray + o; L.depth = depth ? depth + o : nullptr;
        L.out = out ? out + o * cap : nullptr; L.n_out = n_out ? n_out + o : nullptr;
        L.status_out = status_out ? status_out + o * cap : nullptr; L.info = info ? info + o : nullptr;
        L.boxes = boxes; L.box_start = box_start ? box_start + o : nullptr; L.in_box = in_box ? in_box + o * cap : nullptr;
        L.collected = 0;
        for (int k = 0; k < n; k++) if (!L.gray[k]) return set_err(GF_ERR_INVALID_ARG, "null frame pointer");
    }
    if (n == 0) return GF_OK;
    // Every lane goes frame by frame through the five-stream submit / wait pipeline of gf_tracker_submit, lanes interleaved:
    // one host thread keeps up to two frames in flight on each tracker.
    for (int k = 0; k < n; k++) {
        for (BatchLane& L : lanes) {
            rc = gf_tracker_submit(L.t, L.times[k], L.gray[k], gray_pitch, L.depth ? L.depth[k] : nullptr, depth_pitch, on_device,
                                   L.frame_boxes(k), L.n_boxes(k));
            if (rc) return rc;
        }
        for (BatchLane& L : lanes) if (in_flight(L.t) == GF_PIPE && (rc = lane_collect(L))) return rc;
    }
    for (BatchLane& L : lanes) while (in_flight(L.t) > 0) if ((rc = lane_collect(L))) return rc;
    return GF_OK;
}

int gf_tracker_track_batch(gf_tracker* t, int n, const double* times, const void* const* gray, size_t gray_pitch,
                           const void* const* depth, size_t depth_pitch, int on_device, const gf_box* boxes, const int* box_start,
                           gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info)
{
    return gf_tracker_track_batch_multi(&t, 1, n, times, gray, gray_pitch, depth, depth_pitch, on_device, boxes, box_start,
                                        out, n_out, in_box, status_out, info);
}

int gf_tracker_set_prediction(gf_tracker* t, const int32_t* ids, const double* xyz, int n)
{
    if (!t || (n > 0 && (!ids || !xyz))) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (n < 0 || n > FE_CAP) return set_err(GF_ERR_CAPACITY, "too many predictions");
    if (in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "frame in flight");
    GF_CUDA(cudaSetDevice(t->device));
    cudaStream_t s = t->s_main;
    if (n > 0) {
        memcpy(t->h_tmp_ids, ids, (size_t)n * sizeof(int));
        memcpy(t->h_tmp_xyz, xyz, (size_t)n * 3 * sizeof(double));
        GF_CUDA(cudaMemcpyAsync(t->d_tmp_ids, t->h_tmp_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
        GF_CUDA(cudaMemcpyAsync(t->d_tmp_xyz, t->h_tmp_xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, s));
    }
    k_set_prediction<<<(FE_CAP + 255) / 256, 256, 0, s>>>(t->d_sc, t->fa, t->d_tmp_ids, t->d_tmp_xyz, n, t->cam); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaStreamSynchronize(s));
    t->has_pred = true;
    return GF_OK;
}

int gf_tracker_remove_ids(gf_tracker* t, const int32_t* ids, int n)
{
    if (!t || (n > 0 && !ids)) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (n < 0 || n > FE_CAP) return set_err(GF_ERR_CAPACITY, "too many ids");
    if (in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "frame in flight");
    if (n == 0) return GF_OK;
    GF_CUDA(cudaSetDevice(t->device));
    cudaStream_t s = t->s_main;
    memcpy(t->h_tmp_ids, ids, (size_t)n * sizeof(int));
    GF_CUDA(cudaMemcpyAsync(t->d_tmp_ids, t->h_tmp_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    k_remove_ids<<<1, FE_CAP, 0, s>>>(t->d_sc, t->fa, t->d_tmp_ids, n); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaStreamSynchronize(s));
    return GF_OK;
}

int gf_tracker_set_profiling(gf_tracker* t, int enable)
{
    if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
    if (in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "frame in flight");
    t->profiling = enable != 0;
    return GF_OK;
}

int gf_tracker_last_stage_ms(gf_tracker* t, float* ms)
{
    if (!t || !ms) return set_err(GF_ERR_INVALID_ARG, "null argument");
    memcpy(ms, t->stage_ms, sizeof(t->stage_ms));
    return GF_OK;
}

int gf_tracker_debug_read(gf_tracker* t, long long* out, int n)
{
    if (!t || !out || n < 0 || n > FE_DBG_N) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    GF_CUDA(cudaSetDevice(t->device));
    GF_CUDA(cudaStreamSynchronize(t->s_main));
    GF_CUDA(cudaMemcpy(out, t->fa.dbg, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_tracker_timer_start(gf_tracker* t)
{
    if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
    if (in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "frame in flight");
    GF_CUDA(cudaSetDevice(t->device));
    GF_CUDA(cudaEventRecord(t->ev_span0, t->s_up));      // the first operation of the next frame follows on this stream
    return GF_OK;
}

int gf_tracker_timer_stop(gf_tracker* t, float* ms)
{
    if (!t || !ms) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "frame in flight");
    GF_CUDA(cudaSetDevice(t->device));
    GF_CUDA(cudaEventRecord(t->ev_span1, t->s_out));     // after the last result copy
    GF_CUDA(cudaEventSynchronize(t->ev_span1));
    GF_CUDA(cudaEventElapsedTime(ms, t->ev_span0, t->ev_span1));
    return GF_OK;
}

int gf_tracker_last_device_ms(gf_tracker* t, float* ms)
{
    if (!t || !ms) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *ms = t->last_ms;
    return GF_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// gf_tracker_group: the frame of every member tracked by one set of launches per step.  The orchestration is the tracker's
// (upload -> pyramid || min-eig map -> dependent chain -> download on five streams, two steps in flight, so step t+1's
// pyramids and min-eig maps overlap step t's chain); the buffers are the members' own, named per step in a table
// (GroupMember), so the graphs only alternate with the table and result buffers.
// ------------------------------------------------------------------------------------------------
struct gf_tracker_group {
    int n, device;
    std::vector<gf_tracker*> m;
    cudaStream_t s_up, s_pyr, s_eig, s_main, s_out;
    cudaEvent_t ev_up[2], ev_pyr[2], ev_eig[2], ev_dep[2], ev_t0[2], ev_out[2];
    // CUDA graphs keyed by step parity and, for the first piece of the chain, by whether any member has a prediction
    cudaGraphExec_t g_clahe[2], g_pyr[2], g_eig[2], g_dep1[2][2], g_dep2[2];
    int gk_clahe[2], gk_pyr[2], gk_eig[2], gk_dep1[2][2], gk_dep2[2];
    bool use_graph, equalize;
    ClaheGeom clahe;                        // the members' equalize setting when the group was created (see group_submit)
    LKMapSet* d_maps;                       // [n][3]: the members' lk_maps, read by the LK kernels from global memory
    GroupMember* d_tab[2]; GroupMember* h_tab[2];
    // member i's result block of a step is the OutBlock prefix up to obs[max_cnt] at i * out_stride: one D2H copy per step
    uint8_t* d_out[2]; uint8_t* h_out[2]; size_t out_stride;
    std::vector<uint8_t> depth_valid[2];    // per step in flight: which members had a depth image
    long long n_submitted, n_waited;
};

static inline int group_in_flight(const gf_tracker_group* g) { return (int)(g->n_submitted - g->n_waited); }
// Member i's result block in a step's d_out or h_out
static inline OutBlock* group_block(uint8_t* out, const gf_tracker_group* g, int i)
{
    return reinterpret_cast<OutBlock*>(out + (size_t)i * g->out_stride);
}

static int member_err(int code, int k, const char* what)
{
    snprintf(g_err, sizeof(g_err), "member %d: %s", k, what);
    return code;
}
static int member_prefix(int rc, int k)         // an error text raised for one member's arguments, naming the member
{
    char keep[sizeof(g_err)];
    memcpy(keep, g_err, sizeof(keep));
    snprintf(g_err, sizeof(g_err), "member %d: %s", k, keep);
    return rc;
}

// What the members of a group share: every kernel of a step is launched once with this geometry and configuration.
static const char* group_mismatch(const gf_tracker* a, const gf_tracker* t)
{
    if (t->device != a->device) return "bound to another device";
    if (t->w != a->w || t->h != a->h) return "image size differs from member 0";
    if (t->cfg.max_cnt != a->cfg.max_cnt) return "max_cnt differs from member 0";
    if (t->cfg.min_dist != a->cfg.min_dist) return "min_dist differs from member 0";
    if (t->cfg.flow_back != a->cfg.flow_back) return "flow_back differs from member 0";
    if (t->cfg.depth_cam != a->cfg.depth_cam) return "depth_cam differs from member 0";
    if (t->equalize != a->equalize || (t->equalize && memcmp(&t->clahe, &a->clahe, sizeof(ClaheGeom)) != 0))
        return "equalize setting differs from member 0";
    return nullptr;
}

static int group_init(gf_tracker_group* g)
{
    const gf_tracker* a = g->m[0];
    GF_CUDA(cudaStreamCreateWithFlags(&g->s_up, cudaStreamNonBlocking));
    GF_CUDA(cudaStreamCreateWithFlags(&g->s_pyr, cudaStreamNonBlocking));
    GF_CUDA(cudaStreamCreateWithFlags(&g->s_eig, cudaStreamNonBlocking));
    GF_CUDA(cudaStreamCreateWithFlags(&g->s_main, cudaStreamNonBlocking));
    GF_CUDA(cudaStreamCreateWithFlags(&g->s_out, cudaStreamNonBlocking));
    g->out_stride = align_up((int)(offsetof(OutBlock, obs) + (size_t)a->cfg.max_cnt * sizeof(gf_obs)), 16);
    for (int i = 0; i < 2; i++) {
        GF_CUDA(cudaEventCreateWithFlags(&g->ev_up[i], cudaEventDisableTiming));
        GF_CUDA(cudaEventCreateWithFlags(&g->ev_pyr[i], cudaEventDisableTiming));
        GF_CUDA(cudaEventCreateWithFlags(&g->ev_eig[i], cudaEventDisableTiming));
        GF_CUDA(cudaEventCreateWithFlags(&g->ev_dep[i], cudaEventDisableTiming));
        GF_CUDA(cudaEventCreate(&g->ev_t0[i]));
        GF_CUDA(cudaEventCreate(&g->ev_out[i]));
        GF_CUDA(cudaMalloc(&g->d_tab[i], (size_t)g->n * sizeof(GroupMember)));
        GF_CUDA(cudaHostAlloc(&g->h_tab[i], (size_t)g->n * sizeof(GroupMember), cudaHostAllocDefault));
        memset(g->h_tab[i], 0, (size_t)g->n * sizeof(GroupMember));
        GF_CUDA(cudaMalloc(&g->d_out[i], (size_t)g->n * g->out_stride));
        GF_CUDA(cudaHostAlloc(&g->h_out[i], (size_t)g->n * g->out_stride, cudaHostAllocDefault));
        g->depth_valid[i].assign((size_t)g->n, 0);
    }
    GF_CUDA(cudaMalloc(&g->d_maps, (size_t)g->n * 3 * sizeof(LKMapSet)));
    for (int k = 0; k < g->n; k++)
        GF_CUDA(cudaMemcpy(g->d_maps + 3 * k, g->m[k]->lk_maps, 3 * sizeof(LKMapSet), cudaMemcpyHostToDevice));
    GF_CUDA(cudaFuncSetAttribute(k_box_chain_g, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BC_SMEM));
    GF_CUDA(cudaFuncSetAttribute(k_select_finalize_g, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    GF_CUDA(cudaFuncSetAttribute(k_clahe_apply_g, cudaFuncAttributeMaxDynamicSharedMemorySize, CLAHE_MAX_TILES * CLAHE_MAX_TILES * 256));
    g->equalize = a->equalize;
    g->clahe = a->clahe;
    g->use_graph = getenv("GF_NO_GRAPH") == nullptr;
    return GF_OK;
}

// ---- the four capturable pieces of a step (and CLAHE), every kernel once for all members ----
static int group_body_clahe(gf_tracker_group* g, int gs)
{
    const gf_tracker* a = g->m[0];
    const ClaheGeom& c = g->clahe;
    k_clahe_lut_g<<<dim3(c.tiles_x * c.tiles_y, g->n), CLAHE_LUT_THREADS, 0, g->s_up>>>(g->d_tab[gs], a->raw_pitch, c); GF_LAUNCHED();
    k_clahe_apply_g<<<dim3((c.h + CLAHE_APPLY_ROWS - 1) / CLAHE_APPLY_ROWS, g->n), CLAHE_APPLY_THREADS, clahe_lut_bytes(c), g->s_up>>>(
        g->d_tab[gs], a->raw_pitch, c); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

static int group_body_pyr(gf_tracker_group* g, int gs)
{
    const gf_tracker* a = g->m[0];
    for (int l = 1; l < 4; l++) {
        dim3 grid((a->lw[l] + PD_TX - 1) / PD_TX, (a->lh[l] + PD_TY - 1) / PD_TY, g->n), b(PD_TX, PD_TY);
        k_pyr_down_g<<<grid, b, 0, g->s_pyr>>>(g->d_tab[gs], l); GF_LAUNCHED();
    }
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

static int group_body_eig(gf_tracker_group* g, int gs)
{
    const gf_tracker* a = g->m[0];
    const int w = a->w, h = a->h, bp = (w + 31) / 32 * 32;
    cudaStream_t s = g->s_eig;
    k_cov_rows_g<<<dim3((w + EIG_TX - 1) / EIG_TX, (h + EIG_BAND - 1) / EIG_BAND, g->n), EIG_TX, 0, s>>>(g->d_tab[gs]); GF_LAUNCHED();
    k_box_chain_g<<<dim3((w + 31) / 32, g->n), 96, BC_SMEM, s>>>(g->d_tab[gs], bp, w, h); GF_LAUNCHED();
    k_eig_from_box_g<<<dim3((w + 63) / 64, (h + 15) / 16, g->n), 256, 0, s>>>(g->d_tab[gs], bp, a->epitch, w, h); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

static int group_body_dep1(gf_tracker_group* g, int gs, bool any_pred)
{
    const gf_tracker* a = g->m[0];
    cudaStream_t s = g->s_main;
    const dim3 lk(a->cfg.max_cnt, g->n);
    if (any_pred) { k_lk_pred_g<<<lk, LK_THREADS, 0, s>>>(g->d_tab[gs]); GF_LAUNCHED(); }
    k_track_g<<<lk, LK_THREADS, 0, s>>>(g->d_tab[gs], a->cfg.flow_back); GF_LAUNCHED();
    k_compact_setmask_g<<<dim3(1, g->n), FE_CAP, 0, s>>>(g->d_tab[gs], a->cfg.min_dist); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

static int group_body_dep2(gf_tracker_group* g, int gs)
{
    const gf_tracker* a = g->m[0];
    const int w = a->w, h = a->h, md = a->cfg.min_dist;
    cudaStream_t s = g->s_main;
    const dim3 tg((w + MASK_TX - 1) / MASK_TX, (h + MASK_TY - 1) / MASK_TY, g->n);
    k_eig_max_g<<<tg, 256, 0, s>>>(g->d_tab[gs], a->epitch, w, h, md); GF_LAUNCHED();
    k_candidates_g<<<tg, 256, 0, s>>>(g->d_tab[gs], a->epitch, w, h, md); GF_LAUNCHED();
    k_select_finalize_g<<<dim3(1, g->n), 1024, a->grid_cells, s>>>(g->d_tab[gs], w, h, a->cfg.max_cnt, md, a->depth_pitch_el,
                                                                  a->cfg.depth_cam ? 1 : 0); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

// One step: member i tracks (times[i], gray[i], depth[i]) with the boxes bx[i][0 .. nb[i]) (box lists already checked).
static int group_submit(gf_tracker_group* g, const double* times, const void* const* gray, size_t gray_pitch, const void* const* depth,
                        size_t depth_pitch, bool on_device, const gf_box* const* bx, const int* nb)
{
    if (group_in_flight(g) >= GF_PIPE) return set_err(GF_ERR_INVALID_ARG, "two steps in flight: call gf_tracker_group_wait first");
    int rc = check_pitches(g->m[0]->w, on_device, gray_pitch, depth != nullptr, depth_pitch);
    if (rc) return rc;
    for (int i = 0; i < g->n; i++) {
        const gf_tracker* t = g->m[i];
        if (!gray[i]) return member_err(GF_ERR_INVALID_ARG, i, "null frame pointer");
        if (in_flight(t) != group_in_flight(g)) return member_err(GF_ERR_INVALID_ARG, i, "has a frame in flight outside this group");
        if (t->profiling) return member_err(GF_ERR_INVALID_ARG, i, "is in profiling mode");
        // gf_tracker_set_equalize is still accepted on a member that has tracked no frame; the graphs and the frame intake
        // of the group follow the setting the members had when the group was created
        if (t->equalize != g->equalize || (g->equalize && memcmp(&t->clahe, &g->clahe, sizeof(ClaheGeom)) != 0))
            return member_err(GF_ERR_INVALID_ARG, i, "equalize setting changed since the group was created");
    }
    GF_CUDA(cudaSetDevice(g->device));
    const int gs = (int)(g->n_submitted % 2);
    bool any_pred = false;
    for (int i = 0; i < g->n; i++) {
        gf_tracker* t = g->m[i];
        const long long f = t->n_submitted;
        const int es = (int)(f % 2), slot = (int)(f % 3);
        GroupMember& G = g->h_tab[gs][i];
        G.prev = make_pyr(t, (slot + 2) % 3); G.cur = make_pyr(t, slot);
        G.maps = g->d_maps + 3 * i + slot;
        G.sc = t->d_sc; G.fa = t->fa; G.grid = t->grid; G.cam = t->cam;
        G.eig = t->d_eig[es]; G.cov = t->d_cov; G.box = t->d_box;
        G.depth = t->d_depth[es]; G.raw = t->d_raw; G.lut = t->d_lut;
        OutBlock* ob = group_block(g->d_out[gs], g, i);
        G.hdr = &ob->hdr; G.obs = ob->obs; G.status = ob->status; G.in_box = ob->in_box;
        frame_params(&G.fp, t, times[i], depth && depth[i], bx[i], nb[i]);
        any_pred |= t->has_pred;
    }
    cudaStream_t s = g->s_up;
    GF_CUDA(cudaEventRecord(g->ev_t0[gs], s));
    GF_CUDA(cudaMemcpyAsync(g->d_tab[gs], g->h_tab[gs], (size_t)g->n * sizeof(GroupMember), cudaMemcpyHostToDevice, s));
    for (int i = 0; i < g->n; i++)
        if ((rc = enqueue_upload(s, g->m[i], gray[i], gray_pitch, depth ? depth[i] : nullptr, depth_pitch, on_device))) return rc;
    const bool direct = !g->use_graph;
    const int hp = any_pred ? 1 : 0;
    if (g->equalize && (rc = run_piece(direct, s, &g->g_clahe[gs], &g->gk_clahe[gs], [&] { return group_body_clahe(g, gs); }))) return rc;
    GF_CUDA(cudaEventRecord(g->ev_up[gs], s));
    GF_CUDA(cudaStreamWaitEvent(g->s_pyr, g->ev_up[gs], 0));
    GF_CUDA(cudaStreamWaitEvent(g->s_eig, g->ev_up[gs], 0));
    if ((rc = run_piece(direct, g->s_pyr, &g->g_pyr[gs], &g->gk_pyr[gs], [&] { return group_body_pyr(g, gs); }))) return rc;
    GF_CUDA(cudaEventRecord(g->ev_pyr[gs], g->s_pyr));
    if ((rc = run_piece(direct, g->s_eig, &g->g_eig[gs], &g->gk_eig[gs], [&] { return group_body_eig(g, gs); }))) return rc;
    GF_CUDA(cudaEventRecord(g->ev_eig[gs], g->s_eig));
    GF_CUDA(cudaStreamWaitEvent(g->s_main, g->ev_pyr[gs], 0));
    if ((rc = run_piece(direct, g->s_main, &g->g_dep1[gs][hp], &g->gk_dep1[gs][hp], [&] { return group_body_dep1(g, gs, any_pred); }))) return rc;
    GF_CUDA(cudaStreamWaitEvent(g->s_main, g->ev_eig[gs], 0));
    if ((rc = run_piece(direct, g->s_main, &g->g_dep2[gs], &g->gk_dep2[gs], [&] { return group_body_dep2(g, gs); }))) return rc;
    GF_CUDA(cudaEventRecord(g->ev_dep[gs], g->s_main));
    GF_CUDA(cudaStreamWaitEvent(g->s_out, g->ev_dep[gs], 0));
    GF_CUDA(cudaMemcpyAsync(g->h_out[gs], g->d_out[gs], (size_t)g->n * g->out_stride, cudaMemcpyDeviceToHost, g->s_out));
    GF_CUDA(cudaEventRecord(g->ev_out[gs], g->s_out));
    for (int i = 0; i < g->n; i++) {
        const bool dv = depth && depth[i];
        frame_enqueued(g->m[i], times[i], dv);
        g->m[i]->group_steps++;
        g->depth_valid[gs][i] = dv ? 1 : 0;
    }
    g->n_submitted++;
    return GF_OK;
}

int gf::tracker_last_out(const gf_tracker* t, TrackerOut* o)
{
    if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
    if (t->out_frame1 == 0) return set_err(GF_ERR_INVALID_ARG, "the tracker has returned no frame of its own yet");
    const long long f = t->out_frame1 - 1;
    // frame f + GF_PIPE runs in frame f's result slot: once it is submitted the slot, its header and its event belong to that frame
    if (t->n_submitted - f > GF_PIPE)
        return set_err(GF_ERR_INVALID_ARG, "the frame the tracker last returned is no longer on the device: a later frame was submitted into its result slot");
    const int es = (int)(f % GF_PIPE);
    o->device = t->device;
    o->n = out_count(t, t->h_out[es], t->depth_valid[es]);
    o->obs = t->d_out[es]->obs; o->in_box = t->d_out[es]->in_box;
    o->downloaded = t->ev_out[es];
    return GF_OK;
}

// The step the group collected last, where the group left it on the device: member i's observations and in_box bits at
// d_out[slot] + i * out_stride, counted as group_collect counts them.  It stays readable while the next step runs and is gone
// once the step after that has been submitted into its slot.
int gf::tracker_group_last_out(const gf_tracker_group* g, int n, TrackerOut* o, cudaEvent_t* downloaded)
{
    if (!g) return set_err(GF_ERR_INVALID_ARG, "null tracker group");
    if (g->n != n) return set_err(GF_ERR_INVALID_ARG, "the tracker group and the window group differ in their number of members");
    if (g->n_waited == 0) return set_err(GF_ERR_INVALID_ARG, "the tracker group has collected no step yet");
    const long long s = g->n_waited - 1;
    if (g->n_submitted - s > GF_PIPE)
        return set_err(GF_ERR_INVALID_ARG, "the step the tracker group last collected is no longer on the device: a later step was submitted into its slot");
    const int gs = (int)(s % 2);
    for (int i = 0; i < n; i++) {
        const OutBlock* db = group_block(g->d_out[gs], g, i);
        o[i].device = g->device;
        o[i].n = out_count(g->m[i], group_block(g->h_out[gs], g, i), g->depth_valid[gs][i]);
        o[i].obs = db->obs;
        o[i].in_box = db->in_box;
        o[i].downloaded = g->ev_out[gs];
    }
    *downloaded = g->ev_out[gs];
    return GF_OK;
}

// Collects the oldest step: member i's results at out + i*out_stride, in_box / status_out likewise, n_out[i*n_stride],
// info[i*n_stride].
static int group_collect(gf_tracker_group* g, gf_obs* out, size_t out_stride, int* n_out, size_t n_stride, uint8_t* in_box,
                         uint8_t* status_out, gf_track_info* info)
{
    if (group_in_flight(g) == 0) return set_err(GF_ERR_INVALID_ARG, "no step in flight");
    GF_CUDA(cudaSetDevice(g->device));
    const int gs = (int)(g->n_waited % 2);
    GF_CUDA(cudaEventSynchronize(g->ev_out[gs]));
    float ms = 0.f;
    GF_CUDA(cudaEventElapsedTime(&ms, g->ev_t0[gs], g->ev_out[gs]));
    g->n_waited++;
    for (int i = 0; i < g->n; i++) {
        gf_tracker* t = g->m[i];
        t->n_waited++;
        t->group_steps--;
        t->out_frame1 = 0;
        t->last_ms = ms;
        const size_t o = (size_t)i * out_stride, q = (size_t)i * n_stride;
        decode_out(t, group_block(g->h_out[gs], g, i), g->depth_valid[gs][i], out ? out + o : nullptr, n_out ? n_out + q : nullptr,
                   in_box ? in_box + o : nullptr, status_out ? status_out + o : nullptr, info ? info + q : nullptr);
    }
    return GF_OK;
}

extern "C" {

void gf_tracker_group_destroy(gf_tracker_group* g)
{
    if (!g) return;
    cudaSetDevice(g->device);
    cudaDeviceSynchronize();
    for (; g->n_waited < g->n_submitted; g->n_waited++)       // steps still in flight are complete: the members move on
        for (gf_tracker* t : g->m) { t->n_waited++; t->group_steps--; }
    for (int k = 0; k < 2; k++) {
        for (cudaGraphExec_t e : {g->g_clahe[k], g->g_pyr[k], g->g_eig[k], g->g_dep1[k][0], g->g_dep1[k][1], g->g_dep2[k]})
            if (e) cudaGraphExecDestroy(e);
        cudaFree(g->d_tab[k]); cudaFreeHost(g->h_tab[k]); cudaFree(g->d_out[k]); cudaFreeHost(g->h_out[k]);
        for (cudaEvent_t e : {g->ev_up[k], g->ev_pyr[k], g->ev_eig[k], g->ev_dep[k], g->ev_t0[k], g->ev_out[k]}) if (e) cudaEventDestroy(e);
    }
    cudaFree(g->d_maps);
    for (cudaStream_t s : {g->s_up, g->s_pyr, g->s_eig, g->s_main, g->s_out}) if (s) cudaStreamDestroy(s);
    cudaGetLastError();
    delete g;
}

int gf_tracker_group_create(gf_tracker_group** out, gf_tracker* const* members, int n)
{
    if (!out) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    if (n > GF_TRACKER_GROUP_MAX) return set_err(GF_ERR_CAPACITY, "more than GF_TRACKER_GROUP_MAX members");
    if (n < 1 || !members) return set_err(GF_ERR_INVALID_ARG, "a group needs at least one member");
    for (int k = 0; k < n; k++) {
        const gf_tracker* t = members[k];
        if (!t) return member_err(GF_ERR_INVALID_ARG, k, "null tracker");
        for (int j = 0; j < k; j++) if (members[j] == t) return member_err(GF_ERR_INVALID_ARG, k, "the same tracker listed twice");
        const char* why = group_mismatch(members[0], t);
        if (why) return member_err(GF_ERR_INVALID_ARG, k, why);
        if (in_flight(t) > 0) return member_err(GF_ERR_INVALID_ARG, k, "has a frame in flight");
        if (t->profiling) return member_err(GF_ERR_INVALID_ARG, k, "is in profiling mode");
    }
    GF_CUDA(cudaSetDevice(members[0]->device));
    gf_tracker_group* g = new (std::nothrow) gf_tracker_group();
    if (!g) return set_err(GF_ERR_CUDA, "out of host memory");
    g->n = n; g->device = members[0]->device;
    g->m.assign(members, members + n);
    int rc = group_init(g);
    if (rc) {
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        gf_tracker_group_destroy(g);
        memcpy(g_err, keep, sizeof(keep));
        return rc;
    }
    *out = g;
    return GF_OK;
}

int gf_tracker_group_submit(gf_tracker_group* g, const double* times, const void* const* gray, size_t gray_pitch,
                            const void* const* depth, size_t depth_pitch, int on_device, const gf_box* boxes, const int* box_start)
{
    if (!g || !times || !gray) return set_err(GF_ERR_INVALID_ARG, "null argument");
    long long bad;
    int rc = box_start ? check_box_lists(boxes, box_start, g->n, &bad) : GF_OK;
    if (rc) return member_prefix(rc, (int)bad);
    std::vector<const gf_box*> bx((size_t)g->n, nullptr);
    std::vector<int> nb((size_t)g->n, 0);
    for (int i = 0; box_start && i < g->n; i++) { bx[i] = boxes ? boxes + box_start[i] : nullptr; nb[i] = box_start[i + 1] - box_start[i]; }
    return group_submit(g, times, gray, gray_pitch, depth, depth_pitch, on_device != 0, bx.data(), nb.data());
}

int gf_tracker_group_wait(gf_tracker_group* g, gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info)
{
    if (!g) return set_err(GF_ERR_INVALID_ARG, "null group");
    return group_collect(g, out, (size_t)g->m[0]->cfg.max_cnt, n_out, 1, in_box, status_out, info);
}

int gf_tracker_group_track_batch(gf_tracker_group* g, int n_steps, const double* times, const void* const* gray, size_t gray_pitch,
                                 const void* const* depth, size_t depth_pitch, int on_device, const gf_box* boxes, const int* box_start,
                                 gf_obs* out, int* n_out, uint8_t* in_box, uint8_t* status_out, gf_track_info* info)
{
    if (!g || n_steps < 0 || (n_steps > 0 && (!times || !gray))) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (group_in_flight(g) > 0) return set_err(GF_ERR_INVALID_ARG, "a step in flight: call gf_tracker_group_wait first");
    const int K = g->n, n = n_steps;
    // every box list and frame pointer is checked before the first step is submitted
    long long bad;
    int rc = box_start ? check_box_lists(boxes, box_start, (long long)K * n, &bad) : GF_OK;
    if (rc) return member_prefix(rc, (int)(bad / n));
    for (long long j = 0; j < (long long)K * n; j++)
        if (!gray[j]) return member_err(GF_ERR_INVALID_ARG, (int)(j / n), "null frame pointer");
    std::vector<double> ts((size_t)K);
    std::vector<const void*> gp((size_t)K), dp((size_t)K);
    std::vector<const gf_box*> bx((size_t)K, nullptr);
    std::vector<int> nb((size_t)K, 0);
    const size_t cap = (size_t)g->m[0]->cfg.max_cnt;
    int collected = 0;
    auto collect = [&]() {
        const size_t j = (size_t)collected++;
        return group_collect(g, out ? out + j * cap : nullptr, (size_t)n * cap, n_out ? n_out + j : nullptr, (size_t)n,
                             in_box ? in_box + j * cap : nullptr, status_out ? status_out + j * cap : nullptr, info ? info + j : nullptr);
    };
    for (int k = 0; k < n; k++) {
        for (int i = 0; i < K; i++) {
            const size_t j = (size_t)i * n + k;
            ts[i] = times[j]; gp[i] = gray[j]; dp[i] = depth ? depth[j] : nullptr;
            if (box_start) { bx[i] = boxes ? boxes + box_start[j] : nullptr; nb[i] = box_start[j + 1] - box_start[j]; }
        }
        if ((rc = group_submit(g, ts.data(), gp.data(), gray_pitch, depth ? dp.data() : nullptr, depth_pitch, on_device != 0, bx.data(), nb.data())))
            return rc;
        if (group_in_flight(g) == GF_PIPE && (rc = collect())) return rc;
    }
    while (group_in_flight(g) > 0) if ((rc = collect())) return rc;
    return GF_OK;
}

// ------------------------------------------------------------------------------------------------
// stage-level entry points (tests)
// ------------------------------------------------------------------------------------------------
}  // extern "C"

struct DevBuf {
    void* p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    int alloc(size_t n) { GF_CUDA(cudaMalloc(&p, n ? n : 1)); return GF_OK; }
    template <class T> T* as() { return (T*)p; }
};

static int upload_image(const uint8_t* src, int w, int h, DevBuf& d, int& pitch)
{
    pitch = align_up(w, 16);
    int rc = d.alloc((size_t)pitch * h + 16);
    if (rc) return rc;
    GF_CUDA(cudaMemcpy2D(d.p, pitch, src, w, w, h, cudaMemcpyHostToDevice));
    return GF_OK;
}

extern "C" {

int gf_stage_pyr_down(int device, const uint8_t* src, int w, int h, uint8_t* dst)
{
    if (!src || !dst || w < 3 || h < 3) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    int rc = select_device(device); if (rc) return rc;
    DevBuf ds, dd; int sp;
    rc = upload_image(src, w, h, ds, sp); if (rc) return rc;
    int dw = (w + 1) / 2, dh = (h + 1) / 2, dp = align_up(dw, 16);
    rc = dd.alloc((size_t)dp * dh); if (rc) return rc;
    Level L{ds.as<uint8_t>(), w, h, sp};
    dim3 g((dw + PD_TX - 1) / PD_TX, (dh + PD_TY - 1) / PD_TY), b(PD_TX, PD_TY);
    k_pyr_down<<<g, b>>>(L, dd.as<uint8_t>(), dw, dh, dp); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy2D(dst, dw, dd.p, dp, dw, dh, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_stage_clahe(int device, const uint8_t* src, size_t src_pitch, int w, int h, double clip_limit, int tiles_x, int tiles_y, uint8_t* dst)
{
    if (!src || !dst || src_pitch < (size_t)w) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (((w + 7) / 8) < 48 || ((h + 7) / 8) < 48 || w > 8192 || h > 8192)
        return set_err(GF_ERR_UNSUPPORTED, "image must be at least 377x377 and at most 8192x8192");
    ClaheGeom g;
    int rc = clahe_geometry(g, w, h, clip_limit, tiles_x, tiles_y); if (rc) return rc;
    rc = select_device(device); if (rc) return rc;
    rc = clahe_prepare(); if (rc) return rc;
    DevBuf ds, dd, dl;
    const int pitch = align_up(w, 16);
    if ((rc = ds.alloc((size_t)pitch * h)) || (rc = dd.alloc((size_t)pitch * h)) || (rc = dl.alloc(clahe_lut_bytes(g)))) return rc;
    GF_CUDA(cudaMemcpy2D(ds.p, pitch, src, src_pitch, w, h, cudaMemcpyHostToDevice));
    rc = enqueue_clahe(0, ds.as<uint8_t>(), pitch, g, dl.as<uint8_t>(), dd.as<uint8_t>(), pitch); if (rc) return rc;
    GF_CUDA(cudaMemcpy2D(dst, w, dd.p, pitch, w, h, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_stage_in_boxes(int device, const float* pts, int n, const gf_box* boxes, int n_boxes, uint8_t* in_box)
{
    if (n < 0 || (n > 0 && (!pts || !in_box))) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    int rc = check_boxes(boxes, n_boxes); if (rc) return rc;
    rc = select_device(device); if (rc) return rc;
    if (n == 0) return GF_OK;
    BoxSet bs;
    put_boxes(bs, boxes, n_boxes);
    DevBuf dp, db, dr;
    if ((rc = dp.alloc((size_t)n * 8)) || (rc = db.alloc(sizeof(BoxSet))) || (rc = dr.alloc(n))) return rc;
    GF_CUDA(cudaMemcpy(dp.p, pts, (size_t)n * 8, cudaMemcpyHostToDevice));
    GF_CUDA(cudaMemcpy(db.p, &bs, sizeof(BoxSet), cudaMemcpyHostToDevice));
    k_in_boxes_stage<<<(n + 255) / 256, 256>>>(dp.as<float2>(), n, db.as<BoxSet>(), dr.as<uint8_t>()); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy(in_box, dr.p, n, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_stage_min_eig(int device, const uint8_t* img, int w, int h, float* eig, int* n_fixups)
{
    if (!img || !eig || w < 4 || h < 4) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    int rc = select_device(device); if (rc) return rc;
    DevBuf di, de, s0, s1, fx; int ip;
    rc = upload_image(img, w, h, di, ip); if (rc) return rc;
    int ep = align_up(w, 4);
    if ((rc = de.alloc((size_t)ep * h * 4)) || (rc = s0.alloc(cov_rows_elems(w, h) * 8)) || (rc = s1.alloc(box_elems(w, h) * 4))) return rc;
    GF_CUDA(cudaMemset(s0.p, 0, cov_rows_elems(w, h) * 8));
    Level L{di.as<uint8_t>(), w, h, ip};
    rc = enqueue_min_eig(0, L, de.as<float>(), ep, s0.as<double>(), s1.as<float>()); if (rc) return rc;
    GF_CUDA(cudaMemcpy2D(eig, (size_t)w * 4, de.p, (size_t)ep * 4, (size_t)w * 4, h, cudaMemcpyDeviceToHost));
    if (n_fixups) *n_fixups = 0;     // the running sums are no longer speculated
    return GF_OK;
}

int gf_stage_lk(int device, const uint8_t* prev, const uint8_t* next, int w, int h, const float* prev_pts, float* next_pts, int n,
                int max_level, int use_initial_flow, uint8_t* status, int roles)
{
    if (!prev || !next || !prev_pts || !next_pts || !status || n < 0 || max_level < 0 || max_level > 3) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if ((w >> max_level) < 48 || (h >> max_level) < 48) return set_err(GF_ERR_UNSUPPORTED, "coarsest pyramid level must be at least 48x48");
    int rc = select_device(device); if (rc) return rc;
    if (n == 0) return GF_OK;
    DevBuf lv[2][4], dp, dq, dst;
    Pyramid P[2];
    for (int k = 0; k < 2; k++) {
        int lw = w, lh = h;
        for (int l = 0; l <= max_level; l++) {
            int pitch = align_up(lw, 16);
            if (l == 0) { rc = upload_image(k ? next : prev, w, h, lv[k][0], pitch); if (rc) return rc; }
            else {
                rc = lv[k][l].alloc((size_t)pitch * lh + 16); if (rc) return rc;
                dim3 g((lw + PD_TX - 1) / PD_TX, (lh + PD_TY - 1) / PD_TY), b(PD_TX, PD_TY);
                k_pyr_down<<<g, b>>>(P[k].lv[l - 1], lv[k][l].as<uint8_t>(), lw, lh, pitch); GF_LAUNCHED();
            }
            P[k].lv[l] = Level{lv[k][l].as<uint8_t>(), lw, lh, pitch};
            lw = (lw + 1) / 2; lh = (lh + 1) / 2;
        }
        for (int l = max_level + 1; l < 4; l++) P[k].lv[l] = P[k].lv[max_level];
    }
    if ((rc = dp.alloc((size_t)n * 8)) || (rc = dq.alloc((size_t)n * 8)) || (rc = dst.alloc(n))) return rc;
    GF_CUDA(cudaMemcpy(dp.p, prev_pts, (size_t)n * 8, cudaMemcpyHostToDevice));
    GF_CUDA(cudaMemcpy(dq.p, next_pts, (size_t)n * 8, cudaMemcpyHostToDevice));
    LKMapSet M;
    rc = make_lk_maps(&M, P[0], P[1], max_level + 1); if (rc) return rc;
    if (roles) k_lk_stage<true><<<n, LK_THREADS>>>(P[0], P[1], dp.as<float2>(), dq.as<float2>(), n, max_level, use_initial_flow, dst.as<uint8_t>(), M);
    else k_lk_stage<false><<<n, LK_THREADS>>>(P[0], P[1], dp.as<float2>(), dq.as<float2>(), n, max_level, use_initial_flow, dst.as<uint8_t>(), M);
    GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy(next_pts, dq.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
    GF_CUDA(cudaMemcpy(status, dst.p, n, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_stage_gftt(int device, const uint8_t* img, int w, int h, const float* kept_pts, int n_kept, int max_corners, int min_dist,
                  float* corners, int* n_corners, gf_track_info* info)
{
    if (!img || !corners || !n_corners || max_corners < 0 || n_kept < 0 || n_kept + max_corners > FE_CAP || min_dist < 5 || min_dist > 255)
        return set_err(GF_ERR_INVALID_ARG, "bad argument");
    int rc = select_device(device); if (rc) return rc;
    DevBuf di, de, s0, s1, dsc, dk, dhdr, dobs, dummy[8]; int ip;
    rc = upload_image(img, w, h, di, ip); if (rc) return rc;
    int ep = align_up(w, 4);
    if ((rc = de.alloc((size_t)ep * h * 4)) || (rc = s0.alloc(cov_rows_elems(w, h) * 8)) ||
        (rc = s1.alloc(box_elems(w, h) * 4)) || (rc = dsc.alloc(sizeof(TrackScalars))) || (rc = dk.alloc((size_t)FE_CAP * 8)) ||
        (rc = dhdr.alloc(sizeof(OutHeader))) || (rc = dobs.alloc(FE_CAP * sizeof(gf_obs))))
        return rc;
    for (int i = 0; i < 8; i++) if ((rc = dummy[i].alloc(FE_CAP * 8))) return rc;
    TrackScalars hs; memset(&hs, 0, sizeof(hs));
    hs.n_kept = n_kept;
    GF_CUDA(cudaMemcpy(dsc.p, &hs, sizeof(hs), cudaMemcpyHostToDevice));
    if (n_kept) GF_CUDA(cudaMemcpy(dk.p, kept_pts, (size_t)n_kept * 8, cudaMemcpyHostToDevice));
    NmsGrid grid; size_t cells;
    rc = alloc_nms_grid(grid, w, h, min_dist, &cells); if (rc) return rc;
    Level L{di.as<uint8_t>(), w, h, ip};
    TrackScalars* sc = dsc.as<TrackScalars>();
    GF_CUDA(cudaMemset(s0.p, 0, cov_rows_elems(w, h) * 8));
    rc = enqueue_min_eig(0, L, de.as<float>(), ep, s0.as<double>(), s1.as<float>());
    if (!rc) rc = enqueue_gftt_select(0, sc, dk.as<float2>(), de.as<float>(), ep, w, h, min_dist, grid);
    if (!rc) {
        FeatArrays fa;
        fa.prev_pts = dummy[0].as<float2>(); fa.ids = dummy[1].as<int>(); fa.track_cnt = dummy[2].as<int>(); fa.prev_un = dummy[3].as<float2>();
        fa.cur_pts = nullptr; fa.status = nullptr; fa.pred_pts = nullptr; fa.dbg = nullptr;
        fa.kept_pts = dk.as<float2>(); fa.kept_ids = dummy[4].as<int>(); fa.kept_cnt = dummy[5].as<int>(); fa.kept_un = dummy[6].as<float2>();
        CamParams cam; memset(&cam, 0, sizeof(cam)); cam.fx = cam.fy = 1.0; cam.no_distortion = 1;
        // max_cnt such that exactly max_corners new corners are requested
        k_select_finalize<<<1, 1024, cells>>>(sc, fa, grid, w, n_kept + max_corners, min_dist, cam, nullptr, nullptr, 0, 0, nullptr, h, dhdr.as<OutHeader>(), dobs.as<gf_obs>(), nullptr, nullptr, nullptr); GF_LAUNCHED();
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { snprintf(g_err, sizeof(g_err), "k_select_finalize launch: %s", cudaGetErrorString(e)); rc = GF_ERR_CUDA; }
    }
    OutHeader hd; memset(&hd, 0, sizeof(hd));
    std::vector<gf_obs> obs(FE_CAP);
    if (!rc) {
        cudaError_t e = cudaMemcpy(&hd, dhdr.p, sizeof(hd), cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(obs.data(), dobs.p, FE_CAP * sizeof(gf_obs), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { snprintf(g_err, sizeof(g_err), "gftt stage: %s", cudaGetErrorString(e)); rc = GF_ERR_CUDA; }
    }
    free_nms_grid(grid);
    if (rc) return rc;
    *n_corners = hd.n_new;
    for (int i = 0; i < hd.n_new; i++) { corners[2 * i] = (float)obs[n_kept + i].v[3]; corners[2 * i + 1] = (float)obs[n_kept + i].v[4]; }
    if (info) { memset(info, 0, sizeof(*info)); info->n_kept = hd.n_kept; info->n_new = hd.n_new; info->n_candidates = hd.n_cand; info->nms_rounds = hd.nms_rounds; info->eig_fixups = hd.eig_fixups; }
    return GF_OK;
}

}  // extern "C"
__global__ void k_sort_stage(sort_elem* e, int n)
{
    __shared__ sort_elem v[FE_CAP];
    __shared__ SortWork W;
    for (int i = threadIdx.x; i < n; i += blockDim.x) v[i] = e[i];
    __syncthreads();
    setmask_sort_parallel(v, n, W);
    for (int i = threadIdx.x; i < n; i += blockDim.x) e[i] = v[i];
}
extern "C" {

int gf_stage_setmask_order(int device, const int32_t* track_cnt, int n, int32_t* perm)
{
    if (!track_cnt || !perm || n < 0 || n > FE_CAP) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    int rc = select_device(device); if (rc) return rc;
    if (n == 0) return GF_OK;
    std::vector<sort_elem> e(n);
    for (int i = 0; i < n; i++) e[i] = ((sort_elem)(unsigned)track_cnt[i] << 32) | (unsigned)i;
    DevBuf d; rc = d.alloc((size_t)n * 8); if (rc) return rc;
    GF_CUDA(cudaMemcpy(d.p, e.data(), (size_t)n * 8, cudaMemcpyHostToDevice));
    k_sort_stage<<<1, FE_CAP>>>(d.as<sort_elem>(), n); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy(e.data(), d.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; i++) perm[i] = (int32_t)(e[i] & 0xffffffffu);
    return GF_OK;
}

}  // extern "C"
