// fm_window.cu -- gf_fm_window (C ABI): one FeatureManager whose landmark table (the reference's std::list<FeaturePerId>,
// vins_estimator/src/estimator/feature_manager.{h,cpp}) stays in HBM between frames, on the window's own stream, with no
// allocation after creation.  The per-landmark arithmetic is fm_device.cuh, the code the stateless gf_fm_* kernels run.
//
// Layout: structure of arrays over landmarks in LIST ORDER (the order the reference's list has: new landmarks appended in
// increasing id, every removal a stable compaction), plus [max_features][11][9] observation rows [x y z u v vx vy depth td].
// The number of landmarks lives on the device: calls that return nothing enqueue and return, so the host never learns it
// from them, and every kernel is sized by the capacity.  Two copies of the table alternate: a removal plans (keep flag, row to
// drop), scans, and scatters the survivors from one copy into the other.  Ids are found through an open-addressing hash
// (id -> slot) that the scatter rebuilds; the list is not sorted by id (a landmark removed by removeOutlier while the tracker
// still tracks it comes back at the end with a smaller id than its neighbours).
//
// Results travel through one block of mapped pinned memory that the kernels write directly; a call that returns something
// synchronises its stream once and then copies the counted part into the caller's arrays.  Arrays going in (set_depth,
// remove_ids, add_frame) pass through a small ring of pinned slots so that calls without a synchronisation never reuse a
// slot the copy engine may still be reading.
//
// Groups (gf_fm_window_group): every kernel takes its window from blockIdx.y and reads that window's state and the call's
// arguments from a descriptor (Win).  A call on K windows launches each kernel once with gridDim.y = K; its K descriptors
// (and poses) travel in the call's one upload, ahead of the members' input arrays.  A single window is the group of one
// through the same kernels and host code; its descriptor goes by value as a kernel parameter, so it uploads nothing more
// than before.
#include <algorithm>
#include <cmath>
#include <new>
#include <vector>

#include "fm_device.cuh"

using namespace gf;
using namespace gffm;

namespace gffw {

constexpr int W = 10;                   // WINDOW_SIZE
constexpr int NROW = W + 1;             // observation rows per landmark
constexpr int ROW = 9;                  // doubles per row
constexpr int LM = NROW * ROW;          // doubles per landmark
constexpr double FOCAL_LENGTH = 600.0;  // parameters.h:23
constexpr int MAX_FEATURES = 8192;      // the single-CTA scans hold at most 32 landmarks per thread at 256 threads
constexpr int RING = 4;
constexpr int GROUP_MAX = GF_FM_WINDOW_GROUP_MAX;
typedef unsigned long long u64;
constexpr u64 EMPTY = ~0ull;

struct Table { int* n; int *id, *start, *nobs, *eflag, *sflag; double* est; double* obs; };

// what the kernels report back, in mapped pinned memory
struct Result {
    int status, margin_old, last_track, new_feature, long_track, n, n_visual, n_features, n_ids;
    int pad;
    double avg_parallax;
};

enum PlanOp { OP_NONE, OP_FAILURES, OP_IDS, OP_BACK_SHIFT, OP_BACK, OP_FRONT };
struct ShiftT { double v[24]; };
struct NextT { double v[12]; };

// One window of a launch: its table, hash and scratch, and this call's arguments.  Device pointers throughout.
struct Win {
    Table T, D;                         // the current copy of the table; the other copy (a removal's destination)
    u64* hash; int hmask, cap;
    int *mark, *drop, *dst, *lm_of, *row0, *totals;
    Result* res;
    int op, fc, n_in, skip;             // op: PlanOp, or the outliers mode; n_in: observations / ids; skip: the window sits out
    double td, min_parallax, depth_threshold, init_depth;
    const gf_obs* obs; const uint32_t* in_box; const double* x; const int* ids;
    int* ids_out; double* xyz_out; double* feat_out; uint8_t* const_out; gf_ba_visual_factor* rows_out;
    union { ShiftT sh; NextT nt; };
};
// the kernel parameter: a group's descriptors on the device (tab), or one window's by value (tab == nullptr)
struct Args { const Win* tab; Win one; };
struct ArgsP { const Win* tab; const FmPoses* ps_tab; Win one; FmPoses ps_one; };

__device__ __forceinline__ const Win& win(const Args& a) { return a.tab ? a.tab[blockIdx.y] : a.one; }
__device__ __forceinline__ const Win& win(const ArgsP& a) { return a.tab ? a.tab[blockIdx.y] : a.one; }
__device__ __forceinline__ const FmPoses& poses(const ArgsP& a) { return a.tab ? a.ps_tab[blockIdx.y] : a.ps_one; }

__device__ __forceinline__ unsigned hash_id(int id) { return (unsigned)id * 2654435761u; }
__device__ __forceinline__ int hash_find(const u64* __restrict__ h, int mask, int id)
{
    for (unsigned k = hash_id(id) & mask;; k = (k + 1) & mask) {
        const u64 e = h[k];
        if (e == EMPTY) return -1;
        if ((int)(e >> 32) == id) return (int)(unsigned)e;
    }
}
__device__ __forceinline__ void hash_put(u64* h, int mask, int id, int slot)
{
    const u64 e = ((u64)(unsigned)id << 32) | (unsigned)slot;
    for (unsigned k = hash_id(id) & mask;; k = (k + 1) & mask)
        if (atomicCAS(&h[k], EMPTY, e) == EMPTY) return;
}

// exclusive prefix of v over the CTA's threads in thread order; *total = the sum.  BS threads, all must call.
template <int BS>
__device__ __forceinline__ int block_scan(int v, int* total)
{
    __shared__ int warp_sum[BS / 32];
    __shared__ int all;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    __syncthreads();                                            // a previous call's warp_sum / all are no longer read
    if (lane == 31) warp_sum[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int s = lane < BS / 32 ? warp_sum[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
        if (lane < BS / 32) warp_sum[lane] = s;
        if (lane == 31) all = s;
    }
    __syncthreads();
    *total = all;
    return x - v + (wid ? warp_sum[wid - 1] : 0);
}

// ---- addFeatureCheckParallax (:57-116) ----
// One CTA per window.  A: every incoming observation outside a box looks its id up; hits and misses are only counted, so that
// a frame that does not fit leaves the table as it was.  B: hits append at n_obs (without checking that frames are contiguous,
// as the reference: a landmark hidden by a box for a frame comes back with a short list); misses are ranked by id and appended
// to the list.  C: the keyframe test, its parallax summed per thread in index order and then by a fixed tree, so that two runs
// agree.
constexpr int INGEST_BS = 1024;
constexpr int MAX_FRAME_OBS = 2048;
constexpr size_t BOX_BYTES = MAX_FRAME_OBS / 8;
__global__ void __launch_bounds__(INGEST_BS) k_fmw_ingest(const __grid_constant__ Args a)
{
    const Win& w = win(a);
    const Table T = w.T;
    u64* __restrict__ hash = w.hash;
    const int hmask = w.hmask, cap = w.cap, n_in = w.n_in, fc = w.fc;
    const double td = w.td;
    const gf_obs* __restrict__ obs = w.obs;
    const uint32_t* __restrict__ in_box = w.in_box;
    Result* __restrict__ res = w.res;
    __shared__ int s_slot[MAX_FRAME_OBS], s_mid[MAX_FRAME_OBS], s_msrc[MAX_FRAME_OBS];
    __shared__ int s_m, s_bad, s_last, s_long, s_sel;
    __shared__ double s_sum[INGEST_BS];
    const int tid = threadIdx.x;
    if (tid == 0) { s_m = s_bad = s_last = s_long = s_sel = 0; }
    __syncthreads();
    const int n = *T.n;
    for (int i = tid; i < n_in; i += INGEST_BS) {
        int slot = -2;                                          // -2: in a box, -1: new
        if (!((in_box[i >> 5] >> (i & 31)) & 1u)) {
            const int id = obs[i].id;
            slot = hash_find(hash, hmask, id);
            if (slot < 0) { const int k = atomicAdd(&s_m, 1); s_mid[k] = id; s_msrc[k] = i; }
            else if (T.start[slot] + T.nobs[slot] > W) s_bad = 1;
        }
        s_slot[i] = slot;
    }
    __syncthreads();
    const int m = s_m;
    if (s_bad || n + m > cap) {
        if (tid == 0) { res->status = s_bad ? GF_ERR_INVALID_ARG : GF_ERR_CAPACITY; res->n = n; }
        return;
    }
    for (int i0 = 0; i0 < n_in; i0 += INGEST_BS) {
        const int i = i0 + tid;
        const int slot = i < n_in ? s_slot[i] : -2;
        bool lng = false;
        if (slot >= 0) {
            const int r = T.nobs[slot];
            double* row = T.obs + (size_t)slot * LM + r * ROW;
            for (int k = 0; k < 8; k++) row[k] = obs[i].v[k];
            row[8] = td;
            T.nobs[slot] = r + 1;
            lng = r + 1 >= 4;
        }
        const unsigned hits = __ballot_sync(0xffffffffu, slot >= 0), longs = __ballot_sync(0xffffffffu, lng);
        if ((tid & 31) == 0 && hits) { atomicAdd(&s_last, __popc(hits)); atomicAdd(&s_long, __popc(longs)); }
    }
    for (int k = tid; k < m; k += INGEST_BS) {
        const int id = s_mid[k];
        int rank = 0;
        for (int j = 0; j < m; j++) rank += s_mid[j] < id;
        const int slot = n + rank, i = s_msrc[k];
        T.id[slot] = id; T.start[slot] = fc; T.nobs[slot] = 1; T.est[slot] = -1.0; T.eflag[slot] = 0; T.sflag[slot] = 0;
        double* row = T.obs + (size_t)slot * LM;
        for (int c = 0; c < 8; c++) row[c] = obs[i].v[c];
        row[8] = td;
        hash_put(hash, hmask, id, slot);
    }
    __syncthreads();
    const int n1 = n + m, last = s_last, lng = s_long;
    double s = 0;
    const bool test = !(fc < 2 || last < 20 || lng < 40 || (double)m > 0.5 * (double)last);
    if (test) {
        int c = 0;
        for (int i = tid; i < n1; i += INGEST_BS) {
            const int st = T.start[i];
            if (st <= fc - 2 && st + T.nobs[i] - 1 >= fc - 1) {
                const double* r = T.obs + (size_t)i * LM + (fc - 2 - st) * ROW;
                s += fm_parallax_one(r, r + ROW);
                c++;
            }
        }
        if (c) atomicAdd(&s_sel, c);
        s_sum[tid] = s;
        __syncthreads();
        for (int o = INGEST_BS / 2; o > 0; o >>= 1) { if (tid < o) s_sum[tid] += s_sum[tid + o]; __syncthreads(); }
    }
    if (tid == 0) {
        *T.n = n1;
        res->status = GF_OK; res->n = n1; res->last_track = last; res->new_feature = m; res->long_track = lng;
        int margin = 1; double avg = 0.0;
        if (test && s_sel > 0) {
            const double mean = s_sum[0] / s_sel;
            avg = mean * FOCAL_LENGTH; margin = mean >= w.min_parallax;
        }
        res->margin_old = margin; res->avg_parallax = avg;
    }
}

// ---- triangulateWithDepth + triangulate ----
__global__ void __launch_bounds__(64) k_fmw_triangulate(const __grid_constant__ ArgsP a)
{
    const Win& w = win(a);
    const Table T = w.T;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *T.n) return;
    const double* p = T.obs + (size_t)i * LM;
    fm_triangulate_one(T.nobs[i], T.start[i], p, ROW, p + 7, ROW, T.est + i, T.eflag + i, poses(a), w.depth_threshold, w.init_depth);
}

__global__ void k_fmw_clear_depth(const __grid_constant__ Args a)
{
    const Table T = win(a).T;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < *T.n) T.est[i] = -1.0;
}

// ---- the factor loop of Estimator::optimization (estimator.cpp:3268-3297) and getDepthVector ----
// One CTA per window: landmark i with >= 4 observations is feature k (scan of the flags) and owns n_obs - 1 factor rows from
// row0[k] (scan of n_obs - 1).
constexpr int SCAN_BS = 1024;
__global__ void __launch_bounds__(SCAN_BS) k_fmw_fill_scan(const __grid_constant__ Args a)
{
    const Win& w = win(a);
    const Table T = w.T;
    int* __restrict__ lm_of = w.lm_of;
    int* __restrict__ row0 = w.row0;
    double* __restrict__ para_feature = w.feat_out;
    uint8_t* __restrict__ feature_const = w.const_out;
    const int n = *T.n, C = (n + SCAN_BS - 1) / SCAN_BS, b = threadIdx.x * C, e = min(n, b + C);
    int nf = 0, nr = 0;
    for (int i = b; i < e; i++) if (T.nobs[i] >= 4) { nf++; nr += T.nobs[i] - 1; }
    int tf, tr;
    int k = block_scan<SCAN_BS>(nf, &tf), r = block_scan<SCAN_BS>(nr, &tr);
    for (int i = b; i < e; i++) {
        const int m = T.nobs[i];
        if (m < 4) continue;
        lm_of[k] = i; row0[k] = r;
        para_feature[k] = 1.0 / T.est[i];
        feature_const[k] = T.eflag[i] == 1;                    // depth from the depth image: SetParameterBlockConstant (:3291-3292)
        k++; r += m - 1;
    }
    if (threadIdx.x == 0) {
        Result* res = w.res;
        w.totals[0] = tf; w.totals[1] = tr; res->n_features = tf; res->n_visual = tr; res->n = n; res->status = GF_OK;
    }
}
// one thread per factor: its landmark is the last k with row0[k] <= f.  A window without rows_out sits out.
__global__ void k_fmw_fill_rows(const __grid_constant__ Args a)
{
    const Win& w = win(a);
    gf_ba_visual_factor* __restrict__ out = w.rows_out;
    if (!out) return;
    const Table T = w.T;
    const int* __restrict__ lm_of = w.lm_of;
    const int* __restrict__ row0 = w.row0;
    const int* __restrict__ totals = w.totals;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= totals[1]) return;
    int lo = 0, hi = totals[0] - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (row0[mid] <= f) lo = mid; else hi = mid - 1; }
    const int i = lm_of[lo], ai = f - row0[lo] + 1, st = T.start[i];
    const double* r0 = T.obs + (size_t)i * LM;
    const double* ra = r0 + ai * ROW;
    gf_ba_visual_factor v;
    v.imu_i = st; v.imu_j = st + ai; v.feature = lo; v.reserved = 0;
    for (int c = 0; c < 3; c++) { v.pts_i[c] = r0[c]; v.pts_j[c] = ra[c]; }
    for (int c = 0; c < 2; c++) { v.vel_i[c] = r0[5 + c]; v.vel_j[c] = ra[5 + c]; }
    v.td_i = r0[8]; v.td_j = ra[8];
    out[f] = v;
}

// ---- setDepth (:249-267) ----  x[k] belongs to the k-th landmark with >= 4 observations
__global__ void __launch_bounds__(SCAN_BS) k_fmw_set_depth(const __grid_constant__ Args a)
{
    const Win& w = win(a);
    if (w.skip) return;
    const Table T = w.T;
    const double* __restrict__ x = w.x;
    const int n = *T.n, C = (n + SCAN_BS - 1) / SCAN_BS, b = threadIdx.x * C, e = min(n, b + C);
    int nf = 0, tf;
    for (int i = b; i < e; i++) nf += T.nobs[i] >= 4;
    int k = block_scan<SCAN_BS>(nf, &tf);
    for (int i = b; i < e; i++) {
        if (T.nobs[i] < 4) continue;
        const double d = 1.0 / x[k++];
        T.est[i] = d; T.sflag[i] = d < 0 ? 2 : 1;
    }
}

// ---- the removals ----
__global__ void k_fmw_mark_ids(const __grid_constant__ Args a)
{
    const Win& w = win(a);
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= w.n_in) return;
    const int slot = hash_find(w.hash, w.hmask, w.ids[k]);
    if (slot >= 0) w.mark[slot] = 1;
}
// One CTA per window: the hash is emptied for the scatter to rebuild; per landmark the keep flag, the observation row the
// removal deletes (drop, -1: none) and the new start frame and depth, which are written in place; then the scan of the keep
// flags gives every survivor its place dst[i] in the other copy of the table (-1: removed).  A window with OP_NONE sits out.
__global__ void __launch_bounds__(SCAN_BS) k_fmw_plan(const __grid_constant__ Args a)
{
    const Win& w = win(a);
    const int op = w.op;
    if (op == OP_NONE) return;
    const Table S = w.T;
    const int fc = w.fc;
    const double init_depth = w.init_depth;
    int* __restrict__ mark = w.mark;
    int* __restrict__ drop = w.drop;
    int* __restrict__ dst = w.dst;
    u64* __restrict__ hash = w.hash;
    for (int j = threadIdx.x; j <= w.hmask; j += SCAN_BS) hash[j] = EMPTY;
    const int n = *S.n, C = (n + SCAN_BS - 1) / SCAN_BS, b = threadIdx.x * C, e = min(n, b + C);
    unsigned keep = 0;
    for (int i = b; i < e; i++) {
        bool k = true;
        int dr = -1;
        const int st = S.start[i], m = S.nobs[i];
        if (op == OP_FAILURES) k = S.sflag[i] != 2;
        else if (op == OP_IDS) { k = !mark[i]; mark[i] = 0; }
        else if (op == OP_FRONT) {
            if (st == fc) S.start[i] = st - 1;
            else if (st + m - 1 >= fc - 1) { dr = W - 1 - st; k = m - 1 > 0; }
        } else if (st != 0) S.start[i] = st - 1;
        else {
            dr = 0;
            if (op == OP_BACK) k = m - 1 > 0;
            else {
                k = m - 1 >= 2;
                if (k) S.est[i] = fm_back_shift_one(S.obs + (size_t)i * LM, S.est[i], w.sh.v, init_depth);
            }
        }
        drop[i] = dr;
        keep |= (unsigned)k << (i - b);
    }
    int total;
    int k = block_scan<SCAN_BS>(__popc(keep), &total);
    for (int i = b; i < e; i++) dst[i] = ((keep >> (i - b)) & 1u) ? k++ : -1;
    if (threadIdx.x == 0) *w.D.n = total;
}
// one warp per landmark: the survivor's scalars and rows (without the dropped one) into the other copy, and its id into the hash
__global__ void k_fmw_scatter(const __grid_constant__ Args a)
{
    const Win& w = win(a);
    if (w.op == OP_NONE) return;
    const Table S = w.T, D = w.D;
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= *S.n) return;
    const int d = w.dst[i];
    if (d < 0) return;
    const int dr = w.drop[i], m = S.nobs[i];
    if (lane == 0) {
        D.id[d] = S.id[i]; D.start[d] = S.start[i]; D.nobs[d] = dr >= 0 ? m - 1 : m; D.est[d] = S.est[i]; D.eflag[d] = S.eflag[i]; D.sflag[d] = S.sflag[i];
        hash_put(w.hash, w.hmask, S.id[i], d);
    }
    const double* s = S.obs + (size_t)i * LM;
    double* o = D.obs + (size_t)d * LM;
    const int cut = dr >= 0 ? dr * ROW : m * ROW, len = dr >= 0 ? (m - 1) * ROW : m * ROW;
    for (int c = lane; c < len; c += 32) o[c] = s[c < cut ? c : c + ROW];
}

// ---- outliersRejection (estimator.cpp:3909-3966) / movingConsistencyCheckW (:3968-4011) ----
// One CTA per window; the ids leave in list order through a scan of the flags.
constexpr int MATH_BS = 256;
__global__ void __launch_bounds__(MATH_BS) k_fmw_outliers(const __grid_constant__ ArgsP a)
{
    const Win& w = win(a);
    const FmPoses& ps = poses(a);
    const Table T = w.T;
    const int mode = w.op;
    int* __restrict__ ids_out = w.ids_out;
    const int n = *T.n, C = (n + MATH_BS - 1) / MATH_BS, b = threadIdx.x * C, e = min(n, b + C);
    unsigned bad = 0;
    for (int i = b; i < e; i++) {
        const int m = T.nobs[i], st = T.start[i];
        const double d = T.est[i];
        if (mode == GF_FM_OUTLIERS_REPROJECTION ? m < 4 : (m < 2 || st >= W - 2 || d < 0)) continue;
        double e2, e3; int c;
        fm_reproj_one(st, m, T.obs + (size_t)i * LM, ROW, d, ps, &e2, &e3, &c);
        bool o;
        if (mode == GF_FM_OUTLIERS_REPROJECTION) o = (e2 / c) * FOCAL_LENGTH > 3;
        else o = c > 0 && ((FOCAL_LENGTH * e2) / c > 10 || e3 / c > 2.0);
        bad |= (unsigned)o << (i - b);
    }
    int total;
    int k = block_scan<MATH_BS>(__popc(bad), &total);
    for (int i = b; i < e; i++) if ((bad >> (i - b)) & 1u) ids_out[k++] = T.id[i];
    if (threadIdx.x == 0) { Result* res = w.res; res->n_ids = total; res->n = n; res->status = GF_OK; }
}

// ---- predictPtsInNextFrame (estimator.cpp:3853-3886) ----  a window with frame_count < 2 sits out
__global__ void __launch_bounds__(MATH_BS) k_fmw_predict(const __grid_constant__ ArgsP a)
{
    const Win& w = win(a);
    if (w.skip) return;
    const FmPoses& ps = poses(a);
    const Table T = w.T;
    const int fc = w.fc;
    int* __restrict__ ids_out = w.ids_out;
    double* __restrict__ xyz_out = w.xyz_out;
    const int n = *T.n, C = (n + MATH_BS - 1) / MATH_BS, b = threadIdx.x * C, e = min(n, b + C);
    unsigned sel = 0;
    for (int i = b; i < e; i++) sel |= (unsigned)(T.est[i] > 0 && T.nobs[i] >= 2 && T.start[i] + T.nobs[i] - 1 == fc) << (i - b);
    int total;
    int k = block_scan<MATH_BS>(__popc(sel), &total);
    for (int i = b; i < e; i++) {
        if (!((sel >> (i - b)) & 1u)) continue;
        ids_out[k] = T.id[i];
        fm_predict_one(T.start[i], T.obs + (size_t)i * LM, T.est[i], ps, w.nt.v, xyz_out + 3 * (size_t)k);
        k++;
    }
    if (threadIdx.x == 0) { Result* res = w.res; res->n_ids = total; res->n = n; res->status = GF_OK; }
}

__global__ void k_fmw_size(Table T, Result* __restrict__ res) { res->n = *T.n; res->status = GF_OK; }

}  // namespace gffw

using namespace gffw;

// Where a call's work runs: a window's own stream and input ring, or a group's.  ev1 is recorded at the end of every call, so
// another chain that takes over a window orders itself after the window's last work by waiting on it.
struct Chain {
    int device;
    bool group;                         // errors name the member at fault ("member k: ")
    cudaStream_t s;
    cudaEvent_t ev0, ev1;               // around the device work of the last call (last_device_ms)
    uint8_t* d_in;                      // what a ring slot carried in: descriptors, poses, then the members' arrays
    size_t in_bytes;
    uint8_t* h_ring[RING]; cudaEvent_t ring_ev[RING]; bool ring_used[RING]; int ring_k;
};

struct gf_fm_window {
    int device, cap, hcap;
    gf_fm_window_cfg cfg;
    Chain c;
    Chain* last;                        // the chain of the last call that enqueued work on this window
    Table t[2]; int cur;
    int* d_n;                           // [2]
    u64* hash;
    int *d_mark, *d_drop, *d_dst, *d_lm_of, *d_row0, *d_totals;
    // pinned
    uint8_t* h_out; uint8_t* d_out;     // mapped: Result, ids, xyz / para_feature, feature_const, factor rows
    size_t o_ids, o_xyz, o_feat, o_const, o_rows;
    uint8_t* h_read;                    // the table on its way out (gf_fm_window_read)
    int n_upper;                        // landmarks after the last add_frame: removals only lower the count, so read() copies this many
    bool depth_vector_valid; int depth_vector_n;   // n_features of the last fill_problem while the list is as it was then
};

struct gf_fm_window_group {
    int n, device;
    std::vector<gf_fm_window*> m;
    std::vector<size_t> seg;            // member k's input arrays start at seg[k] after the descriptors and poses
    Chain c;
};

namespace {

typedef gf_fm_window* Wp;

bool finite_all(const double* p, int n) { for (int i = 0; i < n; i++) if (!std::isfinite(p[i])) return false; return true; }
int load_poses(FmPoses* ps, const double* Ps, const double* Rs, const double* tic, const double* ric)
{
    if (!Ps || !Rs || !tic || !ric) return set_err(GF_ERR_INVALID_ARG, "null pose argument");
    if (!finite_all(Ps, 3 * NROW) || !finite_all(Rs, 9 * NROW) || !finite_all(tic, 3) || !finite_all(ric, 9))
        return set_err(GF_ERR_INVALID_ARG, "non-finite pose");
    memcpy(ps->P, Ps, sizeof(ps->P)); memcpy(ps->R, Rs, sizeof(ps->R)); memcpy(ps->tic, tic, 24); memcpy(ps->ric, ric, 72);
    return GF_OK;
}
int member_err(int rc, int k, bool named)           // an error raised for one member of a group call names the member
{
    if (!named) return rc;
    char keep[sizeof(g_err)];
    memcpy(keep, g_err, sizeof(keep));
    snprintf(g_err, sizeof(g_err), "member %d: %s", k, keep);
    return rc;
}
Result* result(gf_fm_window* w) { return reinterpret_cast<Result*>(w->h_out); }
template <class T> T* dev_out(gf_fm_window* w, size_t off) { return reinterpret_cast<T*>(w->d_out + off); }
template <class T> T* host_out(gf_fm_window* w, size_t off) { return reinterpret_cast<T*>(w->h_out + off); }
int blocks(int cap, int per_block) { return (cap + per_block - 1) / per_block; }
size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// a pinned slot the copy engine is not reading; the wait only happens when the device is RING uploads behind
int ring_acquire(Chain* c, uint8_t** p, int* k)
{
    *k = c->ring_k; c->ring_k = (c->ring_k + 1) % RING;
    if (c->ring_used[*k]) GF_CUDA(cudaEventSynchronize(c->ring_ev[*k]));
    *p = c->h_ring[*k];
    return GF_OK;
}
int ring_upload(Chain* c, int k, size_t bytes)
{
    GF_CUDA(cudaMemcpyAsync(c->d_in, c->h_ring[k], bytes, cudaMemcpyHostToDevice, c->s));
    GF_CUDA(cudaEventRecord(c->ring_ev[k], c->s));
    c->ring_used[k] = true;
    return GF_OK;
}
int begin(Chain* c) { GF_CUDA(cudaEventRecord(c->ev0, c->s)); return GF_OK; }
int end_async(Chain* c) { GF_CUDA(cudaGetLastError()); GF_CUDA(cudaEventRecord(c->ev1, c->s)); return GF_OK; }
int end_sync(Chain* c) { int rc = end_async(c); if (rc) return rc; GF_CUDA(cudaStreamSynchronize(c->s)); return GF_OK; }

int chain_init(Chain* c, int device, size_t in_bytes)
{
    c->device = device;
    GF_CUDA(cudaStreamCreateWithFlags(&c->s, cudaStreamNonBlocking));
    GF_CUDA(cudaEventCreate(&c->ev0)); GF_CUDA(cudaEventCreate(&c->ev1));
    c->in_bytes = in_bytes;
    GF_CUDA(cudaMalloc(&c->d_in, in_bytes));
    for (int k = 0; k < RING; k++) {
        GF_CUDA(cudaHostAlloc(&c->h_ring[k], in_bytes, cudaHostAllocDefault));
        GF_CUDA(cudaEventCreateWithFlags(&c->ring_ev[k], cudaEventDisableTiming));
    }
    GF_CUDA(cudaEventRecord(c->ev0, c->s));            // a chain that has run nothing can be waited on and timed (0 ms)
    GF_CUDA(cudaEventRecord(c->ev1, c->s));
    return GF_OK;
}
void chain_free(Chain* c)
{
    if (c->s) cudaStreamSynchronize(c->s);
    cudaFree(c->d_in);
    for (int k = 0; k < RING; k++) { if (c->h_ring[k]) cudaFreeHost(c->h_ring[k]); if (c->ring_ev[k]) cudaEventDestroy(c->ring_ev[k]); }
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->s) cudaStreamDestroy(c->s);
}

// What a window's input arrays take in a ring slot: one frame's box bits and observations, or a depth per landmark.
size_t window_in_bytes(int cap) { return std::max(BOX_BYTES + (size_t)MAX_FRAME_OBS * sizeof(gf_obs), 8 * (size_t)cap); }
// a group's ring slot: K descriptors, then either K poses (triangulate, outliers, predict) or the members' input arrays
size_t tab_bytes(int K) { return align256((size_t)K * sizeof(Win)); }

// ---- one call over K windows: the descriptors, one upload, the launches ----
struct Call {
    Chain* c; const Wp* w; int K;
    bool pose;                          // the kernels take poses (ArgsP)
    Win one; FmPoses one_ps;            // K == 1: the descriptor goes by value
    Win* win; FmPoses* ps;              // the K descriptors on the host
    uint8_t* slot; int ring_k; size_t used;
    const std::vector<size_t>* seg;     // K > 1: where member k's input arrays go in the slot
    cudaEvent_t after;                  // an event the work waits for, after the start event (nullable)
    bool named;                         // a group call: errors name the member
};

Win base_desc(gf_fm_window* w)
{
    Win d;
    memset(&d, 0, sizeof(d));
    d.T = w->t[w->cur]; d.D = w->t[w->cur ^ 1];
    d.hash = w->hash; d.hmask = w->hcap - 1; d.cap = w->cap;
    d.mark = w->d_mark; d.drop = w->d_drop; d.dst = w->d_dst; d.lm_of = w->d_lm_of; d.row0 = w->d_row0; d.totals = w->d_totals;
    d.res = dev_out<Result>(w, 0);
    d.min_parallax = w->cfg.min_parallax; d.depth_threshold = w->cfg.depth_threshold; d.init_depth = w->cfg.init_depth;
    return d;
}

// the host side of a call: descriptors filled from the windows' state; a ring slot when anything must be uploaded
int call_open(Call& a, Chain* c, const Wp* w, int K, bool pose, bool input, const std::vector<size_t>* seg)
{
    a.c = c; a.w = w; a.K = K; a.pose = pose; a.slot = nullptr; a.ring_k = 0; a.used = 0; a.seg = seg; a.after = nullptr; a.named = c->group;
    if (K > 1 || input) {
        int rc = ring_acquire(c, &a.slot, &a.ring_k);
        if (rc) return rc;
    }
    if (K > 1) {
        a.win = reinterpret_cast<Win*>(a.slot);
        a.ps = reinterpret_cast<FmPoses*>(a.slot + tab_bytes(K));
        a.used = tab_bytes(K) + (pose ? (size_t)K * sizeof(FmPoses) : 0);
    } else {
        a.win = &a.one; a.ps = &a.one_ps;
    }
    for (int i = 0; i < K; i++) a.win[i] = base_desc(w[i]);
    return GF_OK;
}
// member i's input arrays: host address in the slot, and the device address they will have after the upload
uint8_t* call_input(Call& a, int i, size_t bytes, const void** dev)
{
    const size_t off = a.K > 1 ? (*a.seg)[i] : 0;
    a.used = std::max(a.used, off + bytes);
    *dev = a.c->d_in + off;
    return a.slot + off;
}
// the windows' work on chain c is ordered after whatever another chain last enqueued on them: no wait while every window
// stays on one chain
int bind(Chain* c, const Wp* w, int K)
{
    for (int i = 0; i < K; i++) {
        if (w[i]->last != c) GF_CUDA(cudaStreamWaitEvent(c->s, w[i]->last->ev1, 0));
        w[i]->last = c;
    }
    return GF_OK;
}
// bind, the start event and the upload
int call_start(Call& a)
{
    int rc = bind(a.c, a.w, a.K);
    if (rc || (rc = begin(a.c))) return rc;
    if (a.after) GF_CUDA(cudaStreamWaitEvent(a.c->s, a.after, 0));
    if (a.slot) return ring_upload(a.c, a.ring_k, a.used);
    return GF_OK;
}
// a call with nothing to launch still orders itself and brackets its (empty) device time
int call_empty(Chain* c, const Wp* w, int K)
{
    int rc = bind(c, w, K);
    if (rc || (rc = begin(c))) return rc;
    return end_async(c);
}
Args args(const Call& a)
{
    Args g;
    g.tab = a.K > 1 ? reinterpret_cast<const Win*>(a.c->d_in) : nullptr;
    g.one = a.one;
    return g;
}
ArgsP args_p(const Call& a)
{
    ArgsP g;
    g.tab = a.K > 1 ? reinterpret_cast<const Win*>(a.c->d_in) : nullptr;
    g.ps_tab = a.K > 1 ? reinterpret_cast<const FmPoses*>(a.c->d_in + tab_bytes(a.K)) : nullptr;
    g.one = a.one; g.ps_one = a.one_ps;
    return g;
}
int max_cap(const Call& a) { int m = 0; for (int i = 0; i < a.K; i++) m = std::max(m, a.w[i]->cap); return m; }
dim3 grid(const Call& a, int per_block, int mult = 1) { return dim3((unsigned)(blocks(max_cap(a), per_block) * mult), (unsigned)a.K); }
dim3 one_cta(const Call& a) { return dim3(1, (unsigned)a.K); }

// the plan / scan / scatter of one removal per window whose op is not OP_NONE; those windows' copies then swap roles
int removal(Call& a)
{
    k_fmw_plan<<<one_cta(a), SCAN_BS, 0, a.c->s>>>(args(a));
    GF_LAUNCHED();
    k_fmw_scatter<<<grid(a, 8), 256, 0, a.c->s>>>(args(a));
    GF_LAUNCHED();
    for (int i = 0; i < a.K; i++) {
        if (a.win[i].op == OP_NONE) continue;
        a.w[i]->cur ^= 1;
        a.w[i]->depth_vector_valid = false;
    }
    return end_async(a.c);
}

// add_frame's arguments for member i (host side); the observations' ids must be distinct and >= 0
int check_frame(int frame_count, const gf_obs* obs, int n, double td)
{
    if (frame_count < 0 || frame_count > W) return set_err(GF_ERR_INVALID_ARG, "frame_count out of range");
    if (n < 0 || (n > 0 && !obs) || !std::isfinite(td)) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n > MAX_FRAME_OBS) return set_err(GF_ERR_CAPACITY, "a frame carries at most 2048 observations");
    // an id twice in one frame has no meaning (the reference's frame is a std::map)
    std::vector<int32_t> ids(n);
    for (int i = 0; i < n; i++) {
        if (obs[i].id < 0) return set_err(GF_ERR_INVALID_ARG, "negative feature id");
        ids[i] = obs[i].id;
    }
    std::sort(ids.begin(), ids.end());
    if (std::adjacent_find(ids.begin(), ids.end()) != ids.end()) return set_err(GF_ERR_INVALID_ARG, "feature id twice in one frame");
    return GF_OK;
}

// the ingest launch and its results; a member that failed on the device keeps its table and reports status
int ingest(Call& a, const int* frame_count, const double* td, int* margin_old, int32_t* counters4, double* parallax, int32_t* status)
{
    for (int i = 0; i < a.K; i++) { a.win[i].fc = frame_count[i]; a.win[i].td = td[i]; }
    int rc = call_start(a);
    if (rc) return rc;
    k_fmw_ingest<<<one_cta(a), INGEST_BS, 0, a.c->s>>>(args(a));
    GF_LAUNCHED();
    if ((rc = end_sync(a.c))) return rc;
    int first = -1;
    for (int i = 0; i < a.K; i++) {
        gf_fm_window* w = a.w[i];
        const Result* r = result(w);
        const int st = r->status == GF_OK ? GF_OK : r->status == GF_ERR_CAPACITY ? GF_ERR_CAPACITY : GF_ERR_INVALID_ARG;
        if (status) status[i] = st;
        if (st) { if (first < 0) first = i; continue; }
        w->depth_vector_valid = false;
        w->n_upper = r->n;
        if (margin_old) margin_old[i] = r->margin_old;
        if (counters4) { int32_t* c4 = counters4 + 4 * i; c4[0] = r->last_track; c4[1] = r->new_feature; c4[2] = r->long_track; c4[3] = r->n; }
        if (parallax) parallax[i] = r->avg_parallax;
    }
    if (first < 0) return GF_OK;
    if (result(a.w[first])->status == GF_ERR_CAPACITY)
        return member_err(set_err(GF_ERR_CAPACITY, "the frame's new landmarks do not fit max_features; the table is unchanged"), first, a.named);
    return member_err(set_err(GF_ERR_INVALID_ARG, "a landmark of the frame already has an observation in the last window frame; the table is unchanged"),
                      first, a.named);
}

// ---- the operations over K windows; the single-window entry points are K == 1 on the window's own chain ----
int op_add_frame(Chain* c, const Wp* w, int K, const std::vector<size_t>* seg, const int* frame_count, const gf_obs* obs, const int* start,
                 const uint8_t* in_box, const double* td, int* margin_old, int32_t* counters4, double* parallax, int32_t* status)
{
    int rc;
    for (int i = 0; i < K; i++)
        if ((rc = check_frame(frame_count[i], obs ? obs + start[i] : nullptr, start[i + 1] - start[i], td[i]))) return member_err(rc, i, c->group);
    Call a;
    if ((rc = call_open(a, c, w, K, false, true, seg))) return rc;
    for (int i = 0; i < K; i++) {
        const int n = start[i + 1] - start[i];
        const void* dev;
        uint8_t* p = call_input(a, i, BOX_BYTES + (size_t)n * sizeof(gf_obs), &dev);
        uint32_t* bits = reinterpret_cast<uint32_t*>(p);                 // box bits, then the observations
        memset(bits, 0, BOX_BYTES);
        if (in_box) for (int j = 0; j < n; j++) if (in_box[start[i] + j]) bits[j >> 5] |= 1u << (j & 31);
        if (n) memcpy(p + BOX_BYTES, obs + start[i], (size_t)n * sizeof(gf_obs));
        a.win[i].in_box = reinterpret_cast<const uint32_t*>(dev);
        a.win[i].obs = reinterpret_cast<const gf_obs*>(reinterpret_cast<const uint8_t*>(dev) + BOX_BYTES);
        a.win[i].n_in = n;
    }
    return ingest(a, frame_count, td, margin_old, counters4, parallax, status);
}

int op_triangulate(Chain* c, const Wp* w, int K, const int* frame_count, const double* Ps, const double* Rs, const double* tic, const double* ric)
{
    int rc;
    for (int i = 0; i < K; i++) {
        if (frame_count[i] < 0 || frame_count[i] > W) return member_err(set_err(GF_ERR_INVALID_ARG, "frame_count out of range"), i, c->group);
        FmPoses ps;
        if ((rc = load_poses(&ps, Ps ? Ps + 33 * i : nullptr, Rs ? Rs + 99 * i : nullptr, tic ? tic + 3 * i : nullptr, ric ? ric + 9 * i : nullptr)))
            return member_err(rc, i, c->group);
    }
    Call a;
    if ((rc = call_open(a, c, w, K, true, false, nullptr))) return rc;
    for (int i = 0; i < K; i++) load_poses(a.ps + i, Ps + 33 * i, Rs + 99 * i, tic + 3 * i, ric + 9 * i);
    if ((rc = call_start(a))) return rc;
    k_fmw_triangulate<<<grid(a, 64), 64, 0, c->s>>>(args_p(a));
    GF_LAUNCHED();
    return end_async(c);
}

int op_fill_problem(Chain* c, const Wp* w, int K, gf_ba_visual_factor* const* visual_out, const int* cap, int* n_visual, double* const* para_feature,
                    uint8_t* const* feature_const, int* n_features, int32_t* status)
{
    int rc;
    if (!n_features) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    bool rows = false;
    for (int i = 0; i < K; i++) {
        const int ci = visual_out ? cap[i] : 0;
        gf_ba_visual_factor* vo = visual_out ? visual_out[i] : nullptr;
        if (ci < 0 || (ci > 0 && !vo)) return member_err(set_err(GF_ERR_INVALID_ARG, "bad argument"), i, c->group);
        rows |= vo != nullptr;
    }
    Call a;
    if ((rc = call_open(a, c, w, K, false, false, nullptr))) return rc;
    for (int i = 0; i < K; i++) {
        a.win[i].feat_out = dev_out<double>(w[i], w[i]->o_feat); a.win[i].const_out = dev_out<uint8_t>(w[i], w[i]->o_const);
        a.win[i].rows_out = visual_out && visual_out[i] ? dev_out<gf_ba_visual_factor>(w[i], w[i]->o_rows) : nullptr;
    }
    if ((rc = call_start(a))) return rc;
    k_fmw_fill_scan<<<one_cta(a), SCAN_BS, 0, c->s>>>(args(a));
    GF_LAUNCHED();
    if (rows) {
        k_fmw_fill_rows<<<grid(a, 256, W), 256, 0, c->s>>>(args(a));
        GF_LAUNCHED();
    }
    if ((rc = end_sync(c))) return rc;
    int first = -1;
    for (int i = 0; i < K; i++) {
        gf_fm_window* wi = w[i];
        const Result* r = result(wi);
        gf_ba_visual_factor* vo = visual_out ? visual_out[i] : nullptr;
        const int st = vo && r->n_visual > cap[i] ? GF_ERR_CAPACITY : GF_OK;
        if (status) status[i] = st;
        if (st) { if (first < 0) first = i; continue; }
        n_features[i] = r->n_features;
        if (n_visual) n_visual[i] = r->n_visual;
        if (para_feature && para_feature[i]) memcpy(para_feature[i], host_out<double>(wi, wi->o_feat), 8 * (size_t)r->n_features);
        if (feature_const && feature_const[i]) memcpy(feature_const[i], host_out<uint8_t>(wi, wi->o_const), (size_t)r->n_features);
        if (vo) memcpy(vo, host_out<gf_ba_visual_factor>(wi, wi->o_rows), sizeof(gf_ba_visual_factor) * (size_t)r->n_visual);
        wi->depth_vector_valid = true; wi->depth_vector_n = r->n_features;
    }
    return first < 0 ? GF_OK : member_err(set_err(GF_ERR_CAPACITY, "visual_out is too small for the window's factors"), first, c->group);
}

int op_set_depth(Chain* c, const Wp* w, int K, const std::vector<size_t>* seg, const double* const* x, const int* n)
{
    int rc;
    bool any = false;
    for (int i = 0; i < K; i++) {
        if (n[i] < 0 || (n[i] > 0 && !x[i])) return member_err(set_err(GF_ERR_INVALID_ARG, "bad argument"), i, c->group);
        if (!w[i]->depth_vector_valid || n[i] != w[i]->depth_vector_n)
            return member_err(set_err(GF_ERR_INVALID_ARG, "set_depth takes the n_features values of the last fill_problem, with no frame added or landmark removed since"), i, c->group);
        any |= n[i] > 0;
    }
    if (!any) return call_empty(c, w, K);           // nothing to upload or launch
    Call a;
    if ((rc = call_open(a, c, w, K, false, true, seg))) return rc;
    for (int i = 0; i < K; i++) {
        if (n[i] == 0) { a.win[i].skip = 1; continue; }
        const void* dev;
        memcpy(call_input(a, i, 8 * (size_t)n[i], &dev), x[i], 8 * (size_t)n[i]);
        a.win[i].x = reinterpret_cast<const double*>(dev);
    }
    if ((rc = call_start(a))) return rc;
    k_fmw_set_depth<<<one_cta(a), SCAN_BS, 0, c->s>>>(args(a));
    GF_LAUNCHED();
    return end_async(c);
}

// removals without input arrays: op[i] (PlanOp) and, for OP_BACK_SHIFT, shift[i] (marg R, marg P, new R, new P); fc[i] is
// the frame count OP_FRONT works on
int op_remove(Chain* c, const Wp* w, int K, const int* op, const ShiftT* shift, const int* fc)
{
    Call a;
    int rc = call_open(a, c, w, K, false, false, nullptr);
    if (rc) return rc;
    for (int i = 0; i < K; i++) {
        a.win[i].op = op[i]; a.win[i].fc = fc ? fc[i] : 0;
        if (op[i] == OP_BACK_SHIFT) a.win[i].sh = shift[i];
    }
    if ((rc = call_start(a))) return rc;
    return removal(a);
}

int op_clear_depth(Chain* c, const Wp* w, int K)
{
    Call a;
    int rc = call_open(a, c, w, K, false, false, nullptr);
    if (rc || (rc = call_start(a))) return rc;
    k_fmw_clear_depth<<<grid(a, 256), 256, 0, c->s>>>(args(a));
    GF_LAUNCHED();
    return end_async(c);
}

// ids of member i: ids[start[i] .. start[i + 1]); more ids than a member's input arrays hold go in pieces (marks accumulate
// and one compaction follows).  A member without ids is left as it is.
int op_remove_ids(Chain* c, const Wp* w, int K, const std::vector<size_t>* seg, const int32_t* ids, const int* start)
{
    int rc;
    int rounds = 0;
    for (int i = 0; i < K; i++) {
        const int n = start[i + 1] - start[i];
        if (n < 0 || (n > 0 && !ids)) return member_err(set_err(GF_ERR_INVALID_ARG, "bad argument"), i, c->group);
        const int piece = (int)(window_in_bytes(w[i]->cap) / 4);
        rounds = std::max(rounds, (n + piece - 1) / piece);
    }
    if (rounds == 0) return call_empty(c, w, K);
    Call a;
    for (int r = 0; r < rounds; r++) {
        if ((rc = call_open(a, c, w, K, false, true, seg))) return rc;
        int most = 0;
        for (int i = 0; i < K; i++) {
            const int n = start[i + 1] - start[i], piece = (int)(window_in_bytes(w[i]->cap) / 4);
            const int o = r * piece, m = std::max(0, std::min(piece, n - o));
            a.win[i].op = n > 0 ? OP_IDS : OP_NONE;
            a.win[i].n_in = m;
            if (m) {
                const void* dev;
                memcpy(call_input(a, i, 4 * (size_t)m, &dev), ids + start[i] + o, 4 * (size_t)m);
                a.win[i].ids = reinterpret_cast<const int*>(dev);
            }
            most = std::max(most, m);
        }
        if (r == 0) { if ((rc = call_start(a))) return rc; }
        else if ((rc = ring_upload(c, a.ring_k, a.used))) return rc;
        k_fmw_mark_ids<<<dim3((unsigned)((most + 255) / 256), (unsigned)K), 256, 0, c->s>>>(args(a));
        GF_LAUNCHED();
    }
    return removal(a);                  // the last round's descriptors carry each member's op
}

int op_outliers(Chain* c, const Wp* w, int K, const double* Ps, const double* Rs, const double* tic, const double* ric, int mode, int32_t* const* ids_out,
                int* n)
{
    int rc;
    if (!ids_out || !n || (mode != GF_FM_OUTLIERS_REPROJECTION && mode != GF_FM_OUTLIERS_MOVING)) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    for (int i = 0; i < K; i++) {
        if (!ids_out[i]) return member_err(set_err(GF_ERR_INVALID_ARG, "bad argument"), i, c->group);
        FmPoses ps;
        if ((rc = load_poses(&ps, Ps ? Ps + 33 * i : nullptr, Rs ? Rs + 99 * i : nullptr, tic ? tic + 3 * i : nullptr, ric ? ric + 9 * i : nullptr)))
            return member_err(rc, i, c->group);
    }
    Call a;
    if ((rc = call_open(a, c, w, K, true, false, nullptr))) return rc;
    for (int i = 0; i < K; i++) {
        load_poses(a.ps + i, Ps + 33 * i, Rs + 99 * i, tic + 3 * i, ric + 9 * i);
        a.win[i].op = mode; a.win[i].ids_out = dev_out<int>(w[i], w[i]->o_ids);
    }
    if ((rc = call_start(a))) return rc;
    k_fmw_outliers<<<one_cta(a), MATH_BS, 0, c->s>>>(args_p(a));
    GF_LAUNCHED();
    if ((rc = end_sync(c))) return rc;
    for (int i = 0; i < K; i++) {
        n[i] = result(w[i])->n_ids;
        memcpy(ids_out[i], host_out<int>(w[i], w[i]->o_ids), 4 * (size_t)n[i]);
    }
    return GF_OK;
}

int op_predict(Chain* c, const Wp* w, int K, const int* frame_count, const double* Ps, const double* Rs, const double* tic, const double* ric,
               int32_t* const* ids_out, double* const* xyz_out, int* n)
{
    int rc;
    if (!ids_out || !xyz_out || !n) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    bool any = false;
    for (int i = 0; i < K; i++) {
        if (!ids_out[i] || !xyz_out[i]) return member_err(set_err(GF_ERR_INVALID_ARG, "bad argument"), i, c->group);
        if (frame_count[i] < 0 || frame_count[i] > W) return member_err(set_err(GF_ERR_INVALID_ARG, "frame_count out of range"), i, c->group);
        FmPoses ps;
        if ((rc = load_poses(&ps, Ps ? Ps + 33 * i : nullptr, Rs ? Rs + 99 * i : nullptr, tic ? tic + 3 * i : nullptr, ric ? ric + 9 * i : nullptr)))
            return member_err(rc, i, c->group);
        any |= frame_count[i] >= 2;
    }
    for (int i = 0; i < K; i++) n[i] = 0;
    if (!any) return GF_OK;                                              // estimator.cpp:3855
    Call a;
    if ((rc = call_open(a, c, w, K, true, false, nullptr))) return rc;
    for (int i = 0; i < K; i++) {
        load_poses(a.ps + i, Ps + 33 * i, Rs + 99 * i, tic + 3 * i, ric + 9 * i);
        Win& d = a.win[i];
        d.fc = frame_count[i]; d.skip = frame_count[i] < 2;
        if (!d.skip) fm_next_pose(Ps + 33 * i, Rs + 99 * i, frame_count[i], d.nt.v);
        d.ids_out = dev_out<int>(w[i], w[i]->o_ids); d.xyz_out = dev_out<double>(w[i], w[i]->o_xyz);
    }
    if ((rc = call_start(a))) return rc;
    k_fmw_predict<<<one_cta(a), MATH_BS, 0, c->s>>>(args_p(a));
    GF_LAUNCHED();
    if ((rc = end_sync(c))) return rc;
    for (int i = 0; i < K; i++) {
        if (frame_count[i] < 2) continue;
        n[i] = result(w[i])->n_ids;
        memcpy(ids_out[i], host_out<int>(w[i], w[i]->o_ids), 4 * (size_t)n[i]);
        memcpy(xyz_out[i], host_out<double>(w[i], w[i]->o_xyz), 24 * (size_t)n[i]);
    }
    return GF_OK;
}

// ---- a single window: its own chain, K == 1 ----
int use(gf_fm_window* w)
{
    if (!w) return set_err(GF_ERR_INVALID_ARG, "null window");
    GF_CUDA(cudaSetDevice(w->device));
    return GF_OK;
}
// a direct call that enqueues without going through a Call (clear, size, read) follows the window's last work too
int take(gf_fm_window* w) { return bind(&w->c, &w, 1); }

int alloc_table(Table* t, int* d_n, int cap)
{
    t->n = d_n;
    GF_CUDA(cudaMalloc(&t->id, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&t->start, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&t->nobs, 4 * (size_t)cap));
    GF_CUDA(cudaMalloc(&t->eflag, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&t->sflag, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&t->est, 8 * (size_t)cap));
    GF_CUDA(cudaMalloc(&t->obs, 8 * (size_t)cap * LM));
    return GF_OK;
}

int window_init(gf_fm_window* w)
{
    const int cap = w->cap;
    int rc;
    if ((rc = chain_init(&w->c, w->device, window_in_bytes(cap)))) return rc;
    w->last = &w->c;
    GF_CUDA(cudaMalloc(&w->d_n, 8));
    for (int i = 0; i < 2; i++) if ((rc = alloc_table(&w->t[i], w->d_n + i, cap))) return rc;
    GF_CUDA(cudaMalloc(&w->hash, 8 * (size_t)w->hcap));
    GF_CUDA(cudaMalloc(&w->d_mark, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&w->d_drop, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&w->d_dst, 4 * (size_t)cap));
    GF_CUDA(cudaMalloc(&w->d_lm_of, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&w->d_row0, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&w->d_totals, 8));
    // every array starts on 16 bytes, whatever the capacity (an odd one would leave the doubles misaligned)
    auto a16 = [](size_t b) { return (b + 15) / 16 * 16; };
    w->o_ids = 64; w->o_xyz = a16(w->o_ids + 4 * (size_t)cap); w->o_feat = a16(w->o_xyz + 24 * (size_t)cap); w->o_const = a16(w->o_feat + 8 * (size_t)cap);
    w->o_rows = a16(w->o_const + cap);
    static_assert(sizeof(Result) <= 64, "Result fits the head of the block");
    GF_CUDA(cudaHostAlloc(&w->h_out, w->o_rows + sizeof(gf_ba_visual_factor) * (size_t)cap * W, cudaHostAllocMapped));
    GF_CUDA(cudaHostGetDevicePointer(&w->d_out, w->h_out, 0));
    GF_CUDA(cudaHostAlloc(&w->h_read, (size_t)cap * (28 + 8 * LM), cudaHostAllocDefault));
    return gf_fm_window_clear(w);
}

// ---- a group ----
int group_use(gf_fm_window_group* g)
{
    if (!g) return set_err(GF_ERR_INVALID_ARG, "null group");
    GF_CUDA(cudaSetDevice(g->device));
    return GF_OK;
}

int group_init(gf_fm_window_group* g)
{
    size_t off = tab_bytes(g->n);
    g->seg.resize((size_t)g->n);
    for (int k = 0; k < g->n; k++) { g->seg[k] = off; off += align256(window_in_bytes(g->m[k]->cap)); }
    g->c.group = true;
    return chain_init(&g->c, g->device, std::max(off, tab_bytes(g->n) + (size_t)g->n * sizeof(FmPoses)));
}

}  // namespace

extern "C" {

int gf_fm_window_create(gf_fm_window** out, int device, const gf_fm_window_cfg* cfg)
{
    if (!out || !cfg) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    const int cap = cfg->max_features == 0 ? 2048 : cfg->max_features;
    if (cap < 1) return set_err(GF_ERR_INVALID_ARG, "max_features must be positive");
    if (cap > MAX_FEATURES) return set_err(GF_ERR_CAPACITY, "max_features must be at most 8192");
    if (cfg->window_size != 0 && cfg->window_size != W) return set_err(GF_ERR_UNSUPPORTED, "window_size must be 10");
    if (!std::isfinite(cfg->min_parallax) || !std::isfinite(cfg->depth_threshold) || !std::isfinite(cfg->init_depth) || cfg->init_depth <= 0)
        return set_err(GF_ERR_INVALID_ARG, "min_parallax, depth_threshold and init_depth must be finite, init_depth positive");
    int nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0) return set_err(GF_ERR_NO_DEVICE, "no CUDA device visible; libgf_b200 has no CPU fallback");
    if (device < 0 || device >= nd) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    gf_fm_window* w = new (std::nothrow) gf_fm_window();
    if (!w) return set_err(GF_ERR_CUDA, "out of host memory");
    memset(w, 0, sizeof(*w));
    w->device = device; w->cfg = *cfg; w->cfg.max_features = cap; w->cfg.window_size = W; w->cap = cap;
    w->hcap = 64;
    while (w->hcap < 2 * cap) w->hcap *= 2;
    int rc = window_init(w);
    if (rc) {
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        gf_fm_window_destroy(w);
        cudaGetLastError();
        memcpy(g_err, keep, sizeof(keep));
        return rc;
    }
    *out = w;
    return GF_OK;
}

void gf_fm_window_destroy(gf_fm_window* w)
{
    if (!w) return;
    cudaSetDevice(w->device);
    if (w->c.s) cudaStreamSynchronize(w->c.s);
    for (int i = 0; i < 2; i++) {
        Table& t = w->t[i];
        cudaFree(t.id); cudaFree(t.start); cudaFree(t.nobs); cudaFree(t.eflag); cudaFree(t.sflag); cudaFree(t.est); cudaFree(t.obs);
    }
    cudaFree(w->d_n); cudaFree(w->hash); cudaFree(w->d_mark); cudaFree(w->d_drop); cudaFree(w->d_dst); cudaFree(w->d_lm_of); cudaFree(w->d_row0);
    cudaFree(w->d_totals);
    if (w->h_out) cudaFreeHost(w->h_out);
    if (w->h_read) cudaFreeHost(w->h_read);
    chain_free(&w->c);
    delete w;
}

int gf_fm_window_clear(gf_fm_window* w)
{
    int rc = use(w);
    if (rc || (rc = take(w)) || (rc = begin(&w->c))) return rc;
    cudaStream_t s = w->c.s;
    GF_CUDA(cudaMemsetAsync(w->d_n, 0, 8, s));
    GF_CUDA(cudaMemsetAsync(w->d_mark, 0, 4 * (size_t)w->cap, s));
    GF_CUDA(cudaMemsetAsync(w->hash, 0xff, 8 * (size_t)w->hcap, s));
    w->depth_vector_valid = false;
    w->n_upper = 0;
    return end_async(&w->c);
}

int gf_fm_window_add_frame(gf_fm_window* w, int frame_count, const gf_obs* obs, int n, const uint8_t* in_box, double td, int* margin_old,
                           int32_t* counters4, double* last_average_parallax)
{
    int rc = use(w);
    if (rc) return rc;
    if (n < 0) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    const int start[2] = {0, n};
    int32_t c4[4];
    double par;
    int mo;
    if ((rc = op_add_frame(&w->c, &w, 1, nullptr, &frame_count, obs, start, in_box, &td, &mo, c4, &par, nullptr))) return rc;
    if (margin_old) *margin_old = mo;
    if (counters4) memcpy(counters4, c4, sizeof(c4));
    if (last_average_parallax) *last_average_parallax = par;
    return GF_OK;
}

int gf_fm_window_add_frame_from_tracker(gf_fm_window* w, const gf_tracker* tracker, int frame_count, double td, int* margin_old, int32_t* counters4,
                                        double* last_average_parallax)
{
    int rc = use(w);
    if (rc) return rc;
    if (frame_count < 0 || frame_count > W || !std::isfinite(td)) return set_err(GF_ERR_INVALID_ARG, "frame_count out of range or td not finite");
    TrackerOut o;
    if ((rc = tracker_last_out(tracker, &o))) return rc;
    if (o.device != w->device) return set_err(GF_ERR_INVALID_ARG, "the tracker is bound to another device");
    Call a;
    if ((rc = call_open(a, &w->c, &w, 1, false, false, nullptr))) return rc;
    a.win[0].obs = o.obs; a.win[0].in_box = o.in_box; a.win[0].n_in = o.n;
    a.after = o.downloaded;
    int32_t c4[4];
    double par;
    int mo;
    if ((rc = ingest(a, &frame_count, &td, &mo, c4, &par, nullptr))) return rc;
    if (margin_old) *margin_old = mo;
    if (counters4) memcpy(counters4, c4, sizeof(c4));
    if (last_average_parallax) *last_average_parallax = par;
    return GF_OK;
}

int gf_fm_window_triangulate(gf_fm_window* w, int frame_count, const double* Ps, const double* Rs, const double* tic, const double* ric)
{
    int rc = use(w);
    return rc ? rc : op_triangulate(&w->c, &w, 1, &frame_count, Ps, Rs, tic, ric);
}

int gf_fm_window_fill_problem(gf_fm_window* w, gf_ba_visual_factor* visual_out, int cap, int* n_visual, double* para_feature, uint8_t* feature_const,
                              int* n_features)
{
    int rc = use(w);
    if (rc) return rc;
    if (cap < 0 || (cap > 0 && !visual_out) || !n_features) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    return op_fill_problem(&w->c, &w, 1, visual_out ? &visual_out : nullptr, &cap, n_visual, &para_feature, &feature_const, n_features, nullptr);
}

int gf_fm_window_set_depth(gf_fm_window* w, const double* para_feature, int n)
{
    int rc = use(w);
    return rc ? rc : op_set_depth(&w->c, &w, 1, nullptr, &para_feature, &n);
}

int gf_fm_window_clear_depth(gf_fm_window* w)
{
    int rc = use(w);
    return rc ? rc : op_clear_depth(&w->c, &w, 1);
}

int gf_fm_window_remove_failures(gf_fm_window* w)
{
    int rc = use(w);
    const int op = OP_FAILURES;
    return rc ? rc : op_remove(&w->c, &w, 1, &op, nullptr, nullptr);
}

int gf_fm_window_remove_ids(gf_fm_window* w, const int32_t* ids, int n)
{
    int rc = use(w);
    if (rc) return rc;
    if (n < 0) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    const int start[2] = {0, n};
    return op_remove_ids(&w->c, &w, 1, nullptr, ids, start);
}

int gf_fm_window_remove_back_shift_depth(gf_fm_window* w, const double* marg_R, const double* marg_P, const double* new_R, const double* new_P)
{
    int rc = use(w);
    if (rc) return rc;
    if (!marg_R || !marg_P || !new_R || !new_P) return set_err(GF_ERR_INVALID_ARG, "null pose argument");
    if (!finite_all(marg_R, 9) || !finite_all(marg_P, 3) || !finite_all(new_R, 9) || !finite_all(new_P, 3)) return set_err(GF_ERR_INVALID_ARG, "non-finite pose");
    ShiftT sh;
    memcpy(sh.v, marg_R, 72); memcpy(sh.v + 9, marg_P, 24); memcpy(sh.v + 12, new_R, 72); memcpy(sh.v + 21, new_P, 24);
    const int op = OP_BACK_SHIFT;
    return op_remove(&w->c, &w, 1, &op, &sh, nullptr);
}

int gf_fm_window_remove_back(gf_fm_window* w)
{
    int rc = use(w);
    const int op = OP_BACK;
    return rc ? rc : op_remove(&w->c, &w, 1, &op, nullptr, nullptr);
}

int gf_fm_window_remove_front(gf_fm_window* w, int frame_count)
{
    int rc = use(w);
    if (rc) return rc;
    // slideWindowNew runs on a full window only; row WINDOW_SIZE - 1 - start_frame is then the second newest frame's
    if (frame_count != W) return set_err(GF_ERR_INVALID_ARG, "remove_front takes frame_count == WINDOW_SIZE");
    const int op = OP_FRONT;
    return op_remove(&w->c, &w, 1, &op, nullptr, &frame_count);
}

int gf_fm_window_outliers(gf_fm_window* w, const double* Ps, const double* Rs, const double* tic, const double* ric, int mode, int32_t* ids_out, int* n)
{
    int rc = use(w);
    if (rc) return rc;
    if (!ids_out || !n) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    return op_outliers(&w->c, &w, 1, Ps, Rs, tic, ric, mode, &ids_out, n);
}

int gf_fm_window_predict_next(gf_fm_window* w, int frame_count, const double* Ps, const double* Rs, const double* tic, const double* ric, int32_t* ids_out,
                              double* xyz_out, int* n)
{
    int rc = use(w);
    if (rc) return rc;
    if (!ids_out || !xyz_out || !n) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    return op_predict(&w->c, &w, 1, &frame_count, Ps, Rs, tic, ric, &ids_out, &xyz_out, n);
}

int gf_fm_window_size(gf_fm_window* w, int* n)
{
    int rc = use(w);
    if (rc) return rc;
    if (!n) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if ((rc = take(w)) || (rc = begin(&w->c))) return rc;
    k_fmw_size<<<1, 1, 0, w->c.s>>>(w->t[w->cur], dev_out<Result>(w, 0));
    GF_LAUNCHED();
    if ((rc = end_sync(&w->c))) return rc;
    *n = result(w)->n;
    return GF_OK;
}

int gf_fm_window_read(gf_fm_window* w, int32_t* feature_id, int32_t* start_frame, int32_t* n_obs, double* estimated_depth, int32_t* estimate_flag,
                      int32_t* solve_flag, double* obs, int cap, int* n)
{
    int rc = use(w);
    if (rc) return rc;
    if (!n || cap < 0) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if ((rc = take(w)) || (rc = begin(&w->c))) return rc;
    const Table& T = w->t[w->cur];
    const size_t c = (size_t)w->n_upper;
    uint8_t* h = w->h_read;
    const void* src[7] = {T.id, T.start, T.nobs, T.eflag, T.sflag, T.est, T.obs};
    void* dst[7] = {feature_id, start_frame, n_obs, estimate_flag, solve_flag, estimated_depth, obs};
    const size_t el[7] = {4, 4, 4, 4, 4, 8, 8 * (size_t)LM};
    size_t off[8] = {0};
    for (int k = 0; k < 7; k++) {
        off[k + 1] = off[k] + el[k] * c;
        if (dst[k] && c) GF_CUDA(cudaMemcpyAsync(h + off[k], src[k], el[k] * c, cudaMemcpyDeviceToHost, w->c.s));
    }
    k_fmw_size<<<1, 1, 0, w->c.s>>>(T, dev_out<Result>(w, 0));
    GF_LAUNCHED();
    if ((rc = end_sync(&w->c))) return rc;
    const int m = result(w)->n;
    *n = m;
    if (m > cap) return set_err(GF_ERR_CAPACITY, "the table holds more landmarks than the arrays passed");
    for (int k = 0; k < 7; k++) if (dst[k]) memcpy(dst[k], h + off[k], el[k] * (size_t)m);
    return GF_OK;
}

int gf_fm_window_last_device_ms(gf_fm_window* w, float* ms)
{
    int rc = use(w);
    if (rc) return rc;
    if (!ms) return set_err(GF_ERR_INVALID_ARG, "null argument");
    GF_CUDA(cudaEventSynchronize(w->c.ev1));
    GF_CUDA(cudaEventElapsedTime(ms, w->c.ev0, w->c.ev1));
    return GF_OK;
}

// ---- gf_fm_window_group ----

int gf_fm_window_group_create(gf_fm_window_group** out, gf_fm_window* const* windows, int n)
{
    if (!out || !windows) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    if (n < 1) return set_err(GF_ERR_INVALID_ARG, "a group has at least one window");
    if (n > GROUP_MAX) return member_err(set_err(GF_ERR_INVALID_ARG, "a group has at most GF_FM_WINDOW_GROUP_MAX (64) windows"), GROUP_MAX, true);
    for (int k = 0; k < n; k++) {
        if (!windows[k]) return member_err(set_err(GF_ERR_INVALID_ARG, "null window"), k, true);
        for (int j = 0; j < k; j++) if (windows[j] == windows[k]) return member_err(set_err(GF_ERR_INVALID_ARG, "the window is listed twice"), k, true);
        if (windows[k]->device != windows[0]->device) return member_err(set_err(GF_ERR_INVALID_ARG, "bound to another device than member 0"), k, true);
    }
    GF_CUDA(cudaSetDevice(windows[0]->device));
    gf_fm_window_group* g = new (std::nothrow) gf_fm_window_group();
    if (!g) return set_err(GF_ERR_CUDA, "out of host memory");
    g->n = n; g->device = windows[0]->device;
    g->m.assign(windows, windows + n);
    memset(&g->c, 0, sizeof(g->c));
    int rc = group_init(g);
    if (rc) {
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        gf_fm_window_group_destroy(g);
        cudaGetLastError();
        memcpy(g_err, keep, sizeof(keep));
        return rc;
    }
    *out = g;
    return GF_OK;
}

void gf_fm_window_group_destroy(gf_fm_window_group* g)
{
    if (!g) return;
    cudaSetDevice(g->device);
    if (g->c.s) cudaStreamSynchronize(g->c.s);
    for (gf_fm_window* w : g->m) if (w->last == &g->c) w->last = &w->c;      // the group's work on it is complete
    chain_free(&g->c);
    delete g;
}

int gf_fm_window_group_size(gf_fm_window_group* g, int* n)
{
    if (!g || !n) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *n = g->n;
    return GF_OK;
}

int gf_fm_window_group_add_frame(gf_fm_window_group* g, const int32_t* frame_counts, const gf_obs* obs, const int32_t* obs_start, const uint8_t* in_box,
                                 const double* tds, int32_t* margin_old, int32_t* counters4, double* last_average_parallax, int32_t* status)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (!frame_counts || !obs_start || !tds) return set_err(GF_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < g->n; i++)
        if (obs_start[i + 1] < obs_start[i] || obs_start[0] != 0) return member_err(set_err(GF_ERR_INVALID_ARG, "obs_start is not non-decreasing from 0"), i, true);
    return op_add_frame(&g->c, g->m.data(), g->n, &g->seg, frame_counts, obs, obs_start, in_box, tds, margin_old, counters4, last_average_parallax, status);
}

int gf_fm_window_group_add_frame_from_tracker_group(gf_fm_window_group* g, const gf_tracker_group* tg, const int32_t* frame_counts, const double* tds,
                                                    int32_t* margin_old, int32_t* counters4, double* last_average_parallax, int32_t* status)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (!frame_counts || !tds) return set_err(GF_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < g->n; i++)
        if (frame_counts[i] < 0 || frame_counts[i] > W || !std::isfinite(tds[i]))
            return member_err(set_err(GF_ERR_INVALID_ARG, "frame_count out of range or td not finite"), i, true);
    TrackerOut o[GROUP_MAX];
    cudaEvent_t downloaded;
    if ((rc = tracker_group_last_out(tg, g->n, o, &downloaded))) return rc;
    if (o[0].device != g->device) return set_err(GF_ERR_INVALID_ARG, "the tracker group is bound to another device");
    Call a;
    if ((rc = call_open(a, &g->c, g->m.data(), g->n, false, false, &g->seg))) return rc;
    for (int i = 0; i < g->n; i++) { a.win[i].obs = o[i].obs; a.win[i].in_box = o[i].in_box; a.win[i].n_in = o[i].n; }
    a.after = downloaded;
    return ingest(a, frame_counts, tds, margin_old, counters4, last_average_parallax, status);
}

int gf_fm_window_group_triangulate(gf_fm_window_group* g, const int32_t* frame_counts, const double* Ps, const double* Rs, const double* tic, const double* ric)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (!frame_counts) return set_err(GF_ERR_INVALID_ARG, "null argument");
    return op_triangulate(&g->c, g->m.data(), g->n, frame_counts, Ps, Rs, tic, ric);
}

int gf_fm_window_group_fill_problem(gf_fm_window_group* g, gf_ba_visual_factor* const* visual_out, const int32_t* caps, int32_t* n_visual,
                                    double* const* para_feature, uint8_t* const* feature_const, int32_t* n_features, int32_t* status)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (visual_out && !caps) return set_err(GF_ERR_INVALID_ARG, "null argument");
    return op_fill_problem(&g->c, g->m.data(), g->n, visual_out, caps, n_visual, para_feature, feature_const, n_features, status);
}

int gf_fm_window_group_set_depth(gf_fm_window_group* g, const double* const* para_feature, const int32_t* n)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (!para_feature || !n) return set_err(GF_ERR_INVALID_ARG, "null argument");
    return op_set_depth(&g->c, g->m.data(), g->n, &g->seg, para_feature, n);
}

int gf_fm_window_group_remove(gf_fm_window_group* g, const int32_t* ops, const int32_t* frame_counts, const double* shift)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (!ops || !frame_counts) return set_err(GF_ERR_INVALID_ARG, "null argument");
    std::vector<int> op((size_t)g->n);
    std::vector<ShiftT> sh((size_t)g->n);
    for (int i = 0; i < g->n; i++) {
        switch (ops[i]) {
        case GF_FM_REMOVE_NONE: op[i] = OP_NONE; break;
        case GF_FM_REMOVE_BACK_SHIFT_DEPTH:
            if (!shift) return member_err(set_err(GF_ERR_INVALID_ARG, "null pose argument"), i, true);
            if (!finite_all(shift + 24 * i, 24)) return member_err(set_err(GF_ERR_INVALID_ARG, "non-finite pose"), i, true);
            op[i] = OP_BACK_SHIFT; memcpy(sh[i].v, shift + 24 * i, sizeof(ShiftT));
            break;
        case GF_FM_REMOVE_BACK: op[i] = OP_BACK; break;
        case GF_FM_REMOVE_FRONT:
            // slideWindowNew runs on a full window only, as gf_fm_window_remove_front requires
            if (frame_counts[i] != W) return member_err(set_err(GF_ERR_INVALID_ARG, "remove_front takes frame_count == WINDOW_SIZE"), i, true);
            op[i] = OP_FRONT;
            break;
        default: return member_err(set_err(GF_ERR_INVALID_ARG, "unknown removal"), i, true);
        }
    }
    return op_remove(&g->c, g->m.data(), g->n, op.data(), sh.data(), frame_counts);
}

int gf_fm_window_group_remove_failures(gf_fm_window_group* g)
{
    int rc = group_use(g);
    if (rc) return rc;
    std::vector<int> op((size_t)g->n, OP_FAILURES);
    return op_remove(&g->c, g->m.data(), g->n, op.data(), nullptr, nullptr);
}

int gf_fm_window_group_clear_depth(gf_fm_window_group* g)
{
    int rc = group_use(g);
    return rc ? rc : op_clear_depth(&g->c, g->m.data(), g->n);
}

int gf_fm_window_group_remove_ids(gf_fm_window_group* g, const int32_t* ids, const int32_t* id_start)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (!id_start) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (id_start[0] != 0) return set_err(GF_ERR_INVALID_ARG, "id_start[0] must be 0");
    return op_remove_ids(&g->c, g->m.data(), g->n, &g->seg, ids, id_start);
}

int gf_fm_window_group_outliers(gf_fm_window_group* g, const double* Ps, const double* Rs, const double* tic, const double* ric, int mode,
                                int32_t* const* ids_out, int32_t* n)
{
    int rc = group_use(g);
    return rc ? rc : op_outliers(&g->c, g->m.data(), g->n, Ps, Rs, tic, ric, mode, ids_out, n);
}

int gf_fm_window_group_predict_next(gf_fm_window_group* g, const int32_t* frame_counts, const double* Ps, const double* Rs, const double* tic,
                                    const double* ric, int32_t* const* ids_out, double* const* xyz_out, int32_t* n)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (!frame_counts) return set_err(GF_ERR_INVALID_ARG, "null argument");
    return op_predict(&g->c, g->m.data(), g->n, frame_counts, Ps, Rs, tic, ric, ids_out, xyz_out, n);
}

int gf_fm_window_group_last_device_ms(gf_fm_window_group* g, float* ms)
{
    int rc = group_use(g);
    if (rc) return rc;
    if (!ms) return set_err(GF_ERR_INVALID_ARG, "null argument");
    GF_CUDA(cudaEventSynchronize(g->c.ev1));
    GF_CUDA(cudaEventElapsedTime(ms, g->c.ev0, g->c.ev1));
    return GF_OK;
}

}  // extern "C"
