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
//           undistort, velocity, depth)  (ev_dep)
//   s_out : (ev_dep) D2H of the result block
//
// Buffers touched by more than one frame in flight are rotated: 3 pyramids (prev/cur/next), 2 depth images, 2 eig
// maps, 2 frame-parameter blocks, 2 result blocks.  All feature state (prev_pts, ids, track_cnt, undistorted points,
// n_id) lives in HBM between frames and is only touched on s_main.
#include <stdlib.h>
#include <new>
#include <vector>

#include "fe_eig.cuh"
#include "fe_lk.cuh"
#include "fe_select.cuh"

namespace gf {

thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};


struct FrameParams {
    double dt; int has_pred; int depth_valid;
    // batch pipeline only: where k_copy_in finds the frame (device pointers: the caller's, or the tracker's staging buffers)
    const uint8_t* src_gray; const uint16_t* src_depth; long long src_gray_pitch, src_depth_pitch;   // pitches in bytes
};

// Frame intake of the batch pipeline: copies the frame named by *fp into pyramid level 0 and the depth slot (16 B per thread when
// source and row pitch allow it).  A kernel instead of a memcpy node because the source address changes every frame while the
// graph stays fixed.
__global__ void __launch_bounds__(256) k_copy_in(const FrameParams* __restrict__ fp, uint8_t* __restrict__ dst_gray, int gray_pitch,
                                                 uint16_t* __restrict__ dst_depth, int depth_pitch_el, int w, int h)
{
    const uint8_t* sg = fp->src_gray;
    const uint8_t* sd = (const uint8_t*)fp->src_depth;
    const long long gp = fp->src_gray_pitch, dp = fp->src_depth_pitch;
    const int depth_rows = (fp->depth_valid && sd) ? h : 0;
    const int row = blockIdx.y;                       // rows 0..h-1: gray, h..2h-1: depth
    const bool is_depth = row >= h;
    if (is_depth && row - h >= depth_rows) return;
    const uint8_t* src = is_depth ? sd + (long long)(row - h) * dp : sg + (long long)row * gp;
    uint8_t* dst = is_depth ? (uint8_t*)(dst_depth + (size_t)(row - h) * depth_pitch_el) : dst_gray + (size_t)row * gray_pitch;
    const int nbytes = is_depth ? 2 * w : w;
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 16;
    if (x >= nbytes) return;
    if ((((uintptr_t)src | (uintptr_t)dst) & 15) == 0 && x + 16 <= nbytes) {
        *(uint4*)(dst + x) = __ldg((const uint4*)(src + x));
    } else {
        for (int k = x; k < min(x + 16, nbytes); k++) dst[k] = __ldg(src + k);
    }
}

// ------------------------------------------------------------------------------------------------
// kernels that need the LK device code
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LK_THREADS) k_lk_stage(Pyramid I, Pyramid J, const float2* prev_pts, float2* next_pts,
                                                         int n, int max_level, int use_init, uint8_t* status, const __grid_constant__ LKMapSet M)
{
    __shared__ LKSmem sm;
    const int tid = threadIdx.x, i = blockIdx.x;
    if (i >= n) return;
    lk_tma_init(sm, tid);
    LKTma T{M.prevI, M.curJ, 0u, M.enabled != 0};
    float2 p = prev_pts[i], init = use_init ? next_pts[i] : p, out;
    int st, iters = 0;
    long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    lk_track_point(sm, tid, I, J, p, init, use_init != 0, max_level, out, st, iters, pc, T);
    if (tid == 0) { next_pts[i] = out; status[i] = (uint8_t)st; }
}

// Prediction pass (feature_tracker.cpp:118-124): maxLevel 1 seeded with predict_pts; counts successes.
__global__ void __launch_bounds__(LK_THREADS) k_lk_pred(Pyramid prev, Pyramid cur, TrackScalars* sc, FeatArrays fa, const __grid_constant__ LKMapSet M)
{
    __shared__ LKSmem sm;
    const int tid = threadIdx.x, i = blockIdx.x;
    if (i >= sc->n_prev) return;
    lk_tma_init(sm, tid);
    LKTma T{M.prevI, M.curJ, 0u, M.enabled != 0};
    float2 out;
    int st, iters = 0;
    long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    lk_track_point(sm, tid, prev, cur, fa.prev_pts[i], fa.pred_pts[i], true, 1, out, st, iters, pc, T);
    if (tid == 0) { fa.cur_pts[i] = out; fa.status[i] = (uint8_t)st; if (st) atomicAdd(&sc->pred_succ, 1); atomicAdd(&sc->lk_iters, iters); }
}

// Forward LK (3 levels) + reverse check (1 level, USE_INITIAL_FLOW) + inBorder + grey<=250
// (feature_tracker.cpp:118-168).  One CTA of 4 warps per feature.
#ifndef GF_TRACK_MIN_CTAS
#define GF_TRACK_MIN_CTAS 3          // 80 registers: three features per SM when several streams share the GPU (2: 110 registers)
#endif
__global__ void __launch_bounds__(LK_THREADS, GF_TRACK_MIN_CTAS) k_track(Pyramid prev, Pyramid cur, TrackScalars* sc, FeatArrays fa,
                                                      const FrameParams* fp, int flow_back, const __grid_constant__ LKMapSet M)
{
    __shared__ LKSmem sm;
    const int tid = threadIdx.x, i = blockIdx.x;
    if (i >= sc->n_prev) return;
    gf_pdl_trigger();
    lk_tma_init(sm, tid);
    LKTma T{M.prevI, M.curJ, 0u, M.enabled != 0};
    const float2 p = fa.prev_pts[i];
    const long long t0 = gf_clock();
    float2 q;
    int st, iters = 0;
    long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (fp->has_pred && sc->pred_succ >= 10) { q = fa.cur_pts[i]; st = fa.status[i]; }
    else lk_track_point(sm, tid, prev, cur, p, p, false, 3, q, st, iters, pc, T);
    if (flow_back) {
        float2 r;
        int rst;
        T.mi = M.curI; T.mj = M.prevJ;          // roles swap for the reverse check
        lk_track_point(sm, tid, cur, prev, q, p, true, 1, r, rst, iters, pc, T);
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
        if (fa.dbg) { fa.dbg[64 + 8 * i] = gf_clock() - t0; fa.dbg[64 + 8 * i + 1] = iters; }
    }
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

}  // namespace gf

using namespace gf;

// ------------------------------------------------------------------------------------------------
constexpr int GF_PIPE = 2;           // frames in flight
struct OutBlock { OutHeader hdr; uint8_t status[FE_CAP]; gf_obs obs[FE_CAP]; };   // one D2H copy per frame

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
    cudaGraphExec_t g_pyr[6], g_eig[6], g_dep1[6][2], g_dep2[6];
    int gk_pyr[6], gk_eig[6], gk_dep1[6][2], gk_dep2[6];
    bool use_graph, use_pdl, pdl_single_cta, batch_pipeline;
    // batch pipeline (gf_tracker_track_batch): one graph launch per frame on s_main = {track + select of frame f} || {intake,
    // pyramid and min-eig map of frame f+1}; keyed by frame number mod 6 like the pieces above
    cudaGraphExec_t gb_prep[6], gb_dep[6], gb_both[6];
    int gbk_prep[6], gbk_dep[6], gbk_both[6];
    cudaEvent_t ev_fork, ev_fork2, ev_join[2];
    uint8_t* d_stage_gray[2]; uint16_t* d_stage_depth[2];   // H2D landing buffers of the batch pipeline (host frames)
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
    double prev_time;
    bool has_pred, depth_valid[2], t0_valid[2];
    float last_ms;
};

static inline int in_flight(const gf_tracker* t) { return (int)(t->n_submitted - t->n_waited); }

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

static CamParams make_cam(const double* p)
{
    CamParams c;
    c.fx = p[0]; c.fy = p[1]; c.cx = p[2]; c.cy = p[3]; c.k1 = p[4]; c.k2 = p[5]; c.p1 = p[6]; c.p2 = p[7];
    c.no_distortion = (p[4] == 0.0 && p[5] == 0.0 && p[6] == 0.0 && p[7] == 0.0);
    return c;
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

// Launch with (pdl) or without a programmatic dependency on the previous kernel of the stream (gf_pdl_wait / gf_pdl_trigger).
template <class... KArgs, class... Args>
static cudaError_t launch_k(void (*k)(KArgs...), dim3 g, dim3 b, size_t smem, cudaStream_t s, bool pdl, Args... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = g; cfg.blockDim = b; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, k, KArgs(args)...);
}

// GFTT tail shared by the tracker and gf_stage_gftt: mask -> max -> candidates -> NMS rounds
static int enqueue_gftt_select(cudaStream_t s, TrackScalars* d_sc, const float2* kept_pts, const float* d_eig, int epitch, int w, int h,
                               int min_dist, NmsGrid& grid, bool pdl = false)
{
    dim3 tg((w + MASK_TX - 1) / MASK_TX, (h + MASK_TY - 1) / MASK_TY);
    GF_CUDA(launch_k(k_eig_max, tg, dim3(256), 0, s, pdl, d_sc, kept_pts, d_eig, epitch, w, h, min_dist)); GF_LAUNCHED();
    GF_CUDA(launch_k(k_candidates, tg, dim3(256), 0, s, pdl, d_sc, kept_pts, d_eig, epitch, w, h, min_dist, grid)); GF_LAUNCHED();
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
    GF_CUDA(cudaEventCreateWithFlags(&t->ev_fork, cudaEventDisableTiming)); GF_CUDA(cudaEventCreateWithFlags(&t->ev_fork2, cudaEventDisableTiming));
    for (int i = 0; i < 2; i++) GF_CUDA(cudaEventCreateWithFlags(&t->ev_join[i], cudaEventDisableTiming));
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
        GF_CUDA(cudaMalloc(&t->d_stage_gray[i], (size_t)width * height));
        GF_CUDA(cudaMalloc(&t->d_stage_depth[i], (size_t)width * height * sizeof(uint16_t)));
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
    t->batch_pipeline = getenv("GF_BATCH_PIPELINE") != nullptr;   // one graph per frame for batches (see gf_tracker_track_batch_multi)
    t->pdl_single_cta = getenv("GF_FE_PDL1") != nullptr && !t->profiling;   // PDL only into the two single-CTA kernels
    t->use_pdl = getenv("GF_PDL") != nullptr;      // programmatic dependent launch inside dep(f): off by default (DESIGN 1.3)
    GF_CUDA(cudaDeviceSynchronize());
    return GF_OK;
}

void gf_tracker_destroy(gf_tracker* t)
{
    if (!t) return;
    cudaSetDevice(t->device);
    cudaDeviceSynchronize();        // (a partially built tracker may lack some of its streams)
    for (int k = 0; k < 6; k++) {
        if (t->g_pyr[k]) cudaGraphExecDestroy(t->g_pyr[k]);
        if (t->g_eig[k]) cudaGraphExecDestroy(t->g_eig[k]);
        if (t->g_dep2[k]) cudaGraphExecDestroy(t->g_dep2[k]);
        for (cudaGraphExec_t g : {t->gb_prep[k], t->gb_dep[k], t->gb_both[k]}) if (g) cudaGraphExecDestroy(g);
        for (int p = 0; p < 2; p++) if (t->g_dep1[k][p]) cudaGraphExecDestroy(t->g_dep1[k][p]);
    }
    for (int s = 0; s < 3; s++) for (int l = 0; l < 4; l++) cudaFree(t->d_pyr[s][l]);
    for (int i = 0; i < 2; i++) {
        cudaFree(t->d_depth[i]); cudaFree(t->d_eig[i]); cudaFree(t->d_out[i]); cudaFree(t->d_fp[i]);
        cudaFree(t->d_stage_gray[i]); cudaFree(t->d_stage_depth[i]);
        if (t->ev_join[i]) cudaEventDestroy(t->ev_join[i]);
        cudaFreeHost(t->h_out[i]); cudaFreeHost(t->h_fp[i]);
        for (cudaEvent_t e : {t->ev_up[i], t->ev_pyr[i], t->ev_eig[i], t->ev_dep[i], t->ev_t0[i], t->ev_out[i]}) if (e) cudaEventDestroy(e);
    }
    cudaFree(t->d_cov); cudaFree(t->d_box);
    free_nms_grid(t->grid);
    cudaFree(t->d_sc);
    FeatArrays& fa = t->fa;
    cudaFree(fa.prev_pts); cudaFree(fa.ids); cudaFree(fa.track_cnt); cudaFree(fa.prev_un); cudaFree(fa.cur_pts); cudaFree(fa.status);
    cudaFree(fa.kept_pts); cudaFree(fa.kept_ids); cudaFree(fa.kept_cnt); cudaFree(fa.kept_un); cudaFree(fa.pred_pts); cudaFree(fa.dbg);
    cudaFree(t->d_tmp_ids); cudaFree(t->d_tmp_xyz);
    cudaFreeHost(t->h_gray); cudaFreeHost(t->h_depth); cudaFreeHost(t->h_tmp_ids); cudaFreeHost(t->h_tmp_xyz);
    for (cudaStream_t st_ : {t->s_up, t->s_pyr, t->s_eig, t->s_main, t->s_out}) if (st_) cudaStreamDestroy(st_);
    for (int i = 0; i < GF_FE_STAGES + 2; i++) if (t->ev_st[i]) cudaEventDestroy(t->ev_st[i]);
    if (t->ev_fork) cudaEventDestroy(t->ev_fork);
    if (t->ev_fork2) cudaEventDestroy(t->ev_fork2);
    if (t->ev_span0) cudaEventDestroy(t->ev_span0);
    if (t->ev_span1) cudaEventDestroy(t->ev_span1);
    cudaGetLastError();
    delete t;
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

static int body_dep1(gf_tracker* t, long long f, bool has_pred, bool pdl = false)
{
    cudaStream_t s = t->s_main;
    Pyramid Pc = make_pyr(t, (int)(f % 3)), Pp = make_pyr(t, (int)((f + 2) % 3));
    const int lk_grid = t->cfg.max_cnt;
    const LKMapSet& M = t->lk_maps[f % 3];
    if (has_pred) { k_lk_pred<<<lk_grid, LK_THREADS, 0, s>>>(Pp, Pc, t->d_sc, t->fa, M); GF_LAUNCHED(); }
    k_track<<<lk_grid, LK_THREADS, 0, s>>>(Pp, Pc, t->d_sc, t->fa, t->d_fp[f % 2], t->cfg.flow_back, M); GF_LAUNCHED();
    GF_MARK(2, s);
    GF_CUDA(launch_k(k_compact_setmask, dim3(1), dim3(FE_CAP), 0, s, pdl || (t->pdl_single_cta && !t->profiling), t->d_sc, t->fa, t->cfg.min_dist)); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_MARK(3, s);
    return GF_OK;
}

static int body_dep2(gf_tracker* t, long long f, bool mirror = false)
{
    const bool pdl = mirror && t->use_pdl;
    cudaStream_t s = t->s_main;
    const int es = (int)(f % 2);
    int rc = enqueue_gftt_select(s, t->d_sc, t->fa.kept_pts, t->d_eig[es], t->epitch, t->w, t->h, t->cfg.min_dist, t->grid, pdl);
    if (rc) return rc;
    GF_MARK(4, s);
    // reference quirk: depth_cam with an empty depth image produces an empty featureFrame (feature_tracker.cpp:342)
    const int depth_mode = t->cfg.depth_cam ? 1 : 0;
    OutBlock* ob = t->d_out[es];
    GF_CUDA(launch_k(k_select_finalize, dim3(1), dim3(1024), t->grid_cells, s, pdl || (t->pdl_single_cta && !t->profiling), t->d_sc, t->fa, t->grid, t->w,
                     t->cfg.max_cnt, t->cfg.min_dist, t->cam, (const double*)&t->d_fp[es]->dt, (const uint16_t*)t->d_depth[es], t->depth_pitch_el, depth_mode,
                     (const int*)&t->d_fp[es]->depth_valid, t->h, &ob->hdr, ob->obs, ob->status,
                     mirror ? reinterpret_cast<uint4*>(t->h_out[es]) : (uint4*)nullptr, (int)offsetof(OutBlock, obs))); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_MARK(5, s);
    return GF_OK;
}

// Runs one piece: replays its CUDA graph (captured on first use) or, in profiling / GF_NO_GRAPH mode, launches it directly.
template <class Body>
static int run_piece(gf_tracker* t, cudaStream_t s, cudaGraphExec_t* exec, int* nk, Body body)
{
    if (!t->use_graph || t->profiling) return body();
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

// Everything after the H2D (or D2D) copies of frame f have been enqueued on s_up.
static int enqueue_frame(gf_tracker* t, long long f, double time, bool depth_valid)
{
    const int es = (int)(f % 2), key = (int)(f % 6), hp = t->has_pred ? 1 : 0;
    t->h_fp[es]->dt = time - t->prev_time;
    t->h_fp[es]->has_pred = hp;
    t->h_fp[es]->depth_valid = depth_valid ? 1 : 0;
    GF_MARK(0, t->s_up);   // end of upload
    GF_CUDA(cudaEventRecord(t->ev_up[es], t->s_up));
    GF_CUDA(cudaStreamWaitEvent(t->s_pyr, t->ev_up[es], 0));
    GF_CUDA(cudaStreamWaitEvent(t->s_eig, t->ev_up[es], 0));
    int rc = run_piece(t, t->s_pyr, &t->g_pyr[key], &t->gk_pyr[key], [&] { return body_pyr(t, f); });
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_pyr[es], t->s_pyr));
    GF_MARK(1, t->s_pyr);
    GF_MARK(7, t->s_eig);
    rc = run_piece(t, t->s_eig, &t->g_eig[key], &t->gk_eig[key], [&] { return body_eig(t, f); });
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_eig[es], t->s_eig));
    GF_MARK(8, t->s_eig);
    GF_CUDA(cudaStreamWaitEvent(t->s_main, t->ev_pyr[es], 0));
    rc = run_piece(t, t->s_main, &t->g_dep1[key][hp], &t->gk_dep1[key][hp], [&] { return body_dep1(t, f, hp != 0); });
    if (rc) return rc;
    GF_CUDA(cudaStreamWaitEvent(t->s_main, t->ev_eig[es], 0));
    rc = run_piece(t, t->s_main, &t->g_dep2[key], &t->gk_dep2[key], [&] { return body_dep2(t, f); });
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_dep[es], t->s_main));
    GF_CUDA(cudaStreamWaitEvent(t->s_out, t->ev_dep[es], 0));
    GF_CUDA(cudaMemcpyAsync(t->h_out[es], t->d_out[es], offsetof(OutBlock, obs) + (size_t)t->cfg.max_cnt * sizeof(gf_obs),
                            cudaMemcpyDeviceToHost, t->s_out));
    GF_CUDA(cudaEventRecord(t->ev_out[es], t->s_out));
    t->prev_time = time;
    t->has_pred = false;
    t->depth_valid[es] = depth_valid;
    t->n_submitted = f + 1;
    return GF_OK;
}

// ---- batch pipeline: the bodies of gb_prep / gb_dep / gb_both (see gf_tracker) ----
// Frame intake + pyramid + min-eig map of frame f, enqueued on m with the min-eig chain forked to s_eig and joined back.
static int body_prep_b(gf_tracker* t, long long f, cudaStream_t m)
{
    const int es = (int)(f % 2), slot = (int)(f % 3);
    GF_CUDA(cudaMemcpyAsync(t->d_fp[es], t->h_fp[es], sizeof(FrameParams), cudaMemcpyHostToDevice, m));
    dim3 g((2 * t->w + 16 * 256 - 1) / (16 * 256), 2 * t->h);
    k_copy_in<<<g, 256, 0, m>>>(t->d_fp[es], t->d_pyr[slot][0], t->lp[0], t->d_depth[es], t->depth_pitch_el, t->w, t->h); GF_LAUNCHED();
    GF_CUDA(cudaEventRecord(t->ev_fork2, m));
    GF_CUDA(cudaStreamWaitEvent(t->s_eig, t->ev_fork2, 0));
    int rc = enqueue_pyramid(m, t, slot);
    if (rc) return rc;
    Pyramid Pc = make_pyr(t, slot);
    rc = enqueue_min_eig(t->s_eig, Pc.lv[0], t->d_eig[es], t->epitch, t->d_cov, t->d_box);
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_join[1], t->s_eig));
    GF_CUDA(cudaStreamWaitEvent(m, t->ev_join[1], 0));
    return GF_OK;
}

// Track + setMask + corner selection + observations of frame f (result block mirrored to pinned host memory), on s_main.
static int body_dep_b(gf_tracker* t, long long f)
{
    int rc = body_dep1(t, f, false, t->use_pdl);
    if (rc) return rc;
    return body_dep2(t, f, true);      // the result block reaches the pinned host buffer from inside k_select_finalize
}

// dep(f) on s_main with prep(f + 1) as a parallel branch on s_pyr (+ s_eig): nothing in prep(f + 1) touches what dep(f) reads
// (pyramid slots f % 3 and (f - 1) % 3, eig / depth / params / out slots f % 2).
static int body_both_b(gf_tracker* t, long long f)
{
    GF_CUDA(cudaEventRecord(t->ev_fork, t->s_main));
    GF_CUDA(cudaStreamWaitEvent(t->s_pyr, t->ev_fork, 0));
    int rc = body_prep_b(t, f + 1, t->s_pyr);
    if (rc) return rc;
    rc = body_dep_b(t, f);
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_join[0], t->s_pyr));
    GF_CUDA(cudaStreamWaitEvent(t->s_main, t->ev_join[0], 0));
    return GF_OK;
}

extern "C" {

static int check_submit(gf_tracker* t)
{
    if (in_flight(t) >= GF_PIPE) return set_err(GF_ERR_INVALID_ARG, "two frames in flight: call gf_tracker_wait first");
    if (t->profiling && in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "profiling mode runs one frame at a time");
    return GF_OK;
}

int gf_tracker_submit(gf_tracker* t, double time, const uint8_t* gray, size_t gray_pitch, const uint16_t* depth, size_t depth_pitch)
{
    if (!t || !gray) return set_err(GF_ERR_INVALID_ARG, "null argument");
    int rc = check_submit(t);
    if (rc) return rc;
    GF_CUDA(cudaSetDevice(t->device));
    const int w = t->w, h = t->h;
    if (gray_pitch < (size_t)w) return set_err(GF_ERR_INVALID_ARG, "gray_pitch smaller than width");
    if (depth && depth_pitch < (size_t)w * 2) return set_err(GF_ERR_INVALID_ARG, "depth_pitch smaller than width*2");
    // The caller's buffers are read by the copy engine directly: truly asynchronous when they are pinned
    // (gf_tracker_host_buffers or any cudaHostAlloc/cudaHostRegister memory: keep them unchanged until the frame has
    // been collected); for pageable memory CUDA stages the data before cudaMemcpy2DAsync returns.
    const long long f = t->n_submitted;
    cudaStream_t s = t->s_up;
    GF_CUDA(cudaEventRecord(t->ev_t0[f % 2], s));
    t->t0_valid[f % 2] = true;
    GF_CUDA(cudaMemcpy2DAsync(t->d_pyr[f % 3][0], t->lp[0], gray, gray_pitch, w, h, cudaMemcpyHostToDevice, s));
    if (depth)
        GF_CUDA(cudaMemcpy2DAsync(t->d_depth[f % 2], (size_t)t->depth_pitch_el * 2, depth, depth_pitch, (size_t)w * 2, h, cudaMemcpyHostToDevice, s));
    return enqueue_frame(t, f, time, depth != nullptr);
}

int gf_tracker_submit_device(gf_tracker* t, double time, const void* d_gray, const void* d_depth)
{
    if (!t || !d_gray) return set_err(GF_ERR_INVALID_ARG, "null argument");
    int rc = check_submit(t);
    if (rc) return rc;
    GF_CUDA(cudaSetDevice(t->device));
    const int w = t->w, h = t->h;
    const long long f = t->n_submitted;
    cudaStream_t s = t->s_up;
    GF_CUDA(cudaEventRecord(t->ev_t0[f % 2], s));
    t->t0_valid[f % 2] = true;
    GF_CUDA(cudaMemcpy2DAsync(t->d_pyr[f % 3][0], t->lp[0], d_gray, w, w, h, cudaMemcpyDeviceToDevice, s));
    if (d_depth)
        GF_CUDA(cudaMemcpy2DAsync(t->d_depth[f % 2], (size_t)t->depth_pitch_el * 2, d_depth, (size_t)w * 2, (size_t)w * 2, h, cudaMemcpyDeviceToDevice, s));
    return enqueue_frame(t, f, time, d_depth != nullptr);
}

int gf_tracker_wait(gf_tracker* t, gf_obs* out, int* n_out, uint8_t* status_out, gf_track_info* info)
{
    if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
    if (in_flight(t) == 0) return set_err(GF_ERR_INVALID_ARG, "no frame in flight");
    GF_CUDA(cudaSetDevice(t->device));
    const int es = (int)(t->n_waited % 2);
    GF_CUDA(cudaEventSynchronize(t->ev_out[es]));
    t->n_waited++;
    if (t->t0_valid[es]) GF_CUDA(cudaEventElapsedTime(&t->last_ms, t->ev_t0[es], t->ev_out[es]));
    else t->last_ms = 0.f;          // batch pipeline: frames are not stamped individually
    if (t->profiling) {
        cudaEvent_t b[8] = {t->ev_t0[es], t->ev_st[0], t->ev_st[1], t->ev_st[2], t->ev_st[3], t->ev_st[4], t->ev_st[5], t->ev_out[es]};
        for (int i = 0; i < 7; i++) GF_CUDA(cudaEventElapsedTime(&t->stage_ms[i], b[i], b[i + 1]));
        GF_CUDA(cudaEventElapsedTime(&t->stage_ms[7], t->ev_st[7], t->ev_st[8]));
    }
    const OutBlock& ob = *t->h_out[es];
    const OutHeader& hd = ob.hdr;
    int n = hd.n_out;
    if (t->cfg.depth_cam && !t->depth_valid[es]) n = 0;   // see body_dep2
    if (n_out) *n_out = n;
    if (out && n > 0) memcpy(out, ob.obs, (size_t)n * sizeof(gf_obs));
    if (status_out && hd.n_prev > 0) memcpy(status_out, ob.status, hd.n_prev);
    if (info) {
        info->n_prev = hd.n_prev; info->n_tracked = hd.n_tracked; info->n_kept = hd.n_kept; info->n_new = hd.n_new;
        info->n_candidates = hd.n_cand; info->nms_rounds = hd.nms_rounds; info->eig_fixups = hd.eig_fixups; info->lk_iterations = hd.lk_iters;
    }
    return GF_OK;
}

int gf_tracker_track(gf_tracker* t, double time, const uint8_t* gray, size_t gray_pitch, const uint16_t* depth, size_t depth_pitch,
                     gf_obs* out, int* n_out, uint8_t* status_out, gf_track_info* info)
{
    if (t && in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "previous frame not collected: call gf_tracker_wait first");
    int rc = gf_tracker_submit(t, time, gray, gray_pitch, depth, depth_pitch);
    if (rc) return rc;
    return gf_tracker_wait(t, out, n_out, status_out, info);
}

int gf_tracker_track_device(gf_tracker* t, double time, const void* d_gray, const void* d_depth, gf_obs* out, int* n_out,
                            uint8_t* status_out, gf_track_info* info)
{
    if (t && in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "previous frame not collected");
    int rc = gf_tracker_submit_device(t, time, d_gray, d_depth);
    if (rc) return rc;
    return gf_tracker_wait(t, out, n_out, status_out, info);
}

// One camera stream of a batch call: its frames, where its results go, and how far it has got.
struct BatchLane {
    gf_tracker* t;
    const double* times; const void* const* gray; const void* const* depth;
    gf_obs* out; int* n_out; uint8_t* status_out; gf_track_info* info;
    int collected, k0;
};

static int lane_collect(BatchLane& L)
{
    const int k = L.collected++;
    const size_t cap = (size_t)L.t->cfg.max_cnt;
    return gf_tracker_wait(L.t, L.out ? L.out + (size_t)k * cap : nullptr, L.n_out ? L.n_out + k : nullptr,
                           L.status_out ? L.status_out + (size_t)k * cap : nullptr, L.info ? L.info + k : nullptr);
}
static int lane_submit_plain(BatchLane& L, int k, size_t gray_pitch, size_t depth_pitch, int on_device)
{
    const void* dk = L.depth ? L.depth[k] : nullptr;
    return on_device ? gf_tracker_submit_device(L.t, L.times[k], L.gray[k], dk)
                     : gf_tracker_submit(L.t, L.times[k], (const uint8_t*)L.gray[k], gray_pitch, (const uint16_t*)dk, depth_pitch);
}
// Makes frame k reachable by its intake kernel: fills the pinned FrameParams slot the graph uploads and, for host frames,
// copies them to the staging slot on s_up (s_main then waits for that copy before the graph that holds prep(k)).
static int lane_stage(BatchLane& L, int k, long long f, size_t gray_pitch, size_t depth_pitch, int on_device)
{
    gf_tracker* t = L.t;
    const int es = (int)(f % 2), w = t->w, h = t->h;
    const void* dk = L.depth ? L.depth[k] : nullptr;
    FrameParams* fp = t->h_fp[es];
    fp->dt = L.times[k] - (k > 0 ? L.times[k - 1] : t->prev_time);
    fp->has_pred = 0;
    fp->depth_valid = dk ? 1 : 0;
    if (on_device) {
        fp->src_gray = (const uint8_t*)L.gray[k]; fp->src_gray_pitch = w;
        fp->src_depth = (const uint16_t*)dk; fp->src_depth_pitch = 2ll * w;
    } else {
        GF_CUDA(cudaMemcpy2DAsync(t->d_stage_gray[es], w, L.gray[k], gray_pitch, w, h, cudaMemcpyHostToDevice, t->s_up));
        if (dk) GF_CUDA(cudaMemcpy2DAsync(t->d_stage_depth[es], (size_t)w * 2, dk, depth_pitch, (size_t)w * 2, h, cudaMemcpyHostToDevice, t->s_up));
        GF_CUDA(cudaEventRecord(t->ev_up[es], t->s_up));
        GF_CUDA(cudaStreamWaitEvent(t->s_main, t->ev_up[es], 0));
        fp->src_gray = t->d_stage_gray[es]; fp->src_gray_pitch = w;
        fp->src_depth = dk ? t->d_stage_depth[es] : nullptr; fp->src_depth_pitch = 2ll * w;
    }
    return GF_OK;
}
// Launches the graph of frame k of the lane: dep(k) || prep(k + 1), or dep(k) alone for the last frame.
static int lane_issue(BatchLane& L, int k, int n, size_t gray_pitch, size_t depth_pitch, int on_device)
{
    gf_tracker* t = L.t;
    GF_CUDA(cudaSetDevice(t->device));
    const long long f = t->n_submitted;
    const int es = (int)(f % 2), key = (int)(f % 6);
    int rc;
    if (k + 1 < n) {
        rc = lane_stage(L, k + 1, f + 1, gray_pitch, depth_pitch, on_device);
        if (rc) return rc;
        rc = run_piece(t, t->s_main, &t->gb_both[key], &t->gbk_both[key], [&] { return body_both_b(t, f); });
    } else {
        rc = run_piece(t, t->s_main, &t->gb_dep[key], &t->gbk_dep[key], [&] { return body_dep_b(t, f); });
    }
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(t->ev_out[es], t->s_main));
    t->prev_time = L.times[k];
    t->has_pred = false;
    t->depth_valid[es] = L.depth && L.depth[k];
    t->t0_valid[es] = false;
    t->n_submitted = f + 1;
    return GF_OK;
}

int gf_tracker_track_batch_multi(gf_tracker* const* trackers, int n_trackers, int n, const double* times, const void* const* gray, size_t gray_pitch,
                                 const void* const* depth, size_t depth_pitch, int on_device,
                                 gf_obs* out, int* n_out, uint8_t* status_out, gf_track_info* info)
{
    if (!trackers || n_trackers < 1 || n < 0 || (n > 0 && (!times || !gray))) return set_err(GF_ERR_INVALID_ARG, "null argument");
    std::vector<BatchLane> lanes((size_t)n_trackers);
    for (int i = 0; i < n_trackers; i++) {
        gf_tracker* t = trackers[i];
        if (!t) return set_err(GF_ERR_INVALID_ARG, "null tracker");
        for (int j = 0; j < i; j++) if (trackers[j] == t) return set_err(GF_ERR_INVALID_ARG, "the same tracker listed twice");
        if (in_flight(t) > 0) return set_err(GF_ERR_INVALID_ARG, "previous frame not collected");
        if (t->profiling) return set_err(GF_ERR_INVALID_ARG, "profiling mode runs one frame at a time");
        if (!on_device) {
            if (gray_pitch < (size_t)t->w) return set_err(GF_ERR_INVALID_ARG, "gray_pitch smaller than width");
            if (depth && depth_pitch < (size_t)t->w * 2) return set_err(GF_ERR_INVALID_ARG, "depth_pitch smaller than width*2");
        }
        const size_t cap = (size_t)t->cfg.max_cnt, o = (size_t)i * n;
        BatchLane& L = lanes[i];
        L.t = t; L.times = times + o; L.gray = gray + o; L.depth = depth ? depth + o : nullptr;
        L.out = out ? out + o * cap : nullptr; L.n_out = n_out ? n_out + o : nullptr;
        L.status_out = status_out ? status_out + o * cap : nullptr; L.info = info ? info + o : nullptr;
        L.collected = 0; L.k0 = 0;
        for (int k = 0; k < n; k++) if (!L.gray[k]) return set_err(GF_ERR_INVALID_ARG, "null frame pointer");
    }
    if (n == 0) return GF_OK;
    int rc;
    // Default: every lane goes frame by frame through the five-stream submit / wait pipeline of gf_tracker_submit, lanes interleaved.
    // GF_BATCH_PIPELINE=1 selects the one-graph-per-frame pipeline below instead; measured on one H100 SXM at 700 W (C2, same run):
    // single stream 10.0 k (default) vs 9.6 k frames/s, 8 streams 26.6 k vs 23.0 k -- joining prep(f+1) into the graph of
    // dep(f) costs more overlap than the saved driver calls give back (DESIGN 1.3).
    bool any_pipeline = false;
    for (BatchLane& L : lanes) any_pipeline = any_pipeline || (L.t->use_graph && L.t->batch_pipeline);
    if (!any_pipeline) {
        for (int k = 0; k < n; k++) {
            for (BatchLane& L : lanes) if ((rc = lane_submit_plain(L, k, gray_pitch, depth_pitch, on_device))) return rc;
            for (BatchLane& L : lanes) if (in_flight(L.t) == GF_PIPE && (rc = lane_collect(L))) return rc;
        }
        for (BatchLane& L : lanes) while (in_flight(L.t) > 0) if ((rc = lane_collect(L))) return rc;
        return GF_OK;
    }
    // lanes that cannot use the one-graph-per-frame pipeline for their first frame(s)
    for (BatchLane& L : lanes) {
        gf_tracker* t = L.t;
        if (!t->use_graph || !t->batch_pipeline) {
            for (int k = 0; k < n; k++) {
                if ((rc = lane_submit_plain(L, k, gray_pitch, depth_pitch, on_device))) return rc;
                if (in_flight(t) == GF_PIPE && (rc = lane_collect(L))) return rc;
            }
            while (in_flight(t) > 0) if ((rc = lane_collect(L))) return rc;
            L.k0 = n;
        } else if (t->has_pred) {                 // a pending setPrediction only concerns the first frame: it takes the other path
            if ((rc = lane_submit_plain(L, 0, gray_pitch, depth_pitch, on_device)) || (rc = lane_collect(L))) return rc;
            L.k0 = 1;
        }
    }
    // one host thread feeds every lane round-robin: prep of the first frame, then one graph launch per lane and frame
    // (tools/graph_rate_probe.cu: one thread replays small graphs into 8 streams at 114 k launches/s, 8 threads at 48-80 k)
    for (BatchLane& L : lanes) {
        if (L.k0 >= n) continue;
        gf_tracker* t = L.t;
        GF_CUDA(cudaSetDevice(t->device));
        const long long f = t->n_submitted;
        if ((rc = lane_stage(L, L.k0, f, gray_pitch, depth_pitch, on_device))) return rc;
        const int key = (int)(f % 6);
        if ((rc = run_piece(t, t->s_main, &t->gb_prep[key], &t->gbk_prep[key], [&] { return body_prep_b(t, f, t->s_main); }))) return rc;
    }
    for (int k = 0; k < n; k++) {
        for (BatchLane& L : lanes) if (k >= L.k0 && (rc = lane_issue(L, k, n, gray_pitch, depth_pitch, on_device))) return rc;
        for (BatchLane& L : lanes) if (in_flight(L.t) == GF_PIPE && (rc = lane_collect(L))) return rc;
    }
    for (BatchLane& L : lanes) while (in_flight(L.t) > 0) if ((rc = lane_collect(L))) return rc;
    return GF_OK;
}

int gf_tracker_track_batch(gf_tracker* t, int n, const double* times, const void* const* gray, size_t gray_pitch,
                           const void* const* depth, size_t depth_pitch, int on_device,
                           gf_obs* out, int* n_out, uint8_t* status_out, gf_track_info* info)
{
    return gf_tracker_track_batch_multi(&t, 1, n, times, gray, gray_pitch, depth, depth_pitch, on_device, out, n_out, status_out, info);
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
                int max_level, int use_initial_flow, uint8_t* status)
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
    k_lk_stage<<<n, LK_THREADS>>>(P[0], P[1], dp.as<float2>(), dq.as<float2>(), n, max_level, use_initial_flow, dst.as<uint8_t>(), M); GF_LAUNCHED();
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
        k_select_finalize<<<1, 1024, cells>>>(sc, fa, grid, w, n_kept + max_corners, min_dist, cam, nullptr, nullptr, 0, 0, nullptr, h, dhdr.as<OutHeader>(), dobs.as<gf_obs>(), nullptr); GF_LAUNCHED();
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
