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
typedef unsigned long long u64;
constexpr u64 EMPTY = ~0ull;

struct Table { int* n; int *id, *start, *nobs, *eflag, *sflag; double* est; double* obs; };

// what the kernels report back, in mapped pinned memory
struct Result {
    int status, margin_old, last_track, new_feature, long_track, n, n_visual, n_features, n_ids;
    int pad;
    double avg_parallax;
};

enum PlanOp { OP_FAILURES, OP_IDS, OP_BACK_SHIFT, OP_BACK, OP_FRONT };
struct ShiftT { double v[24]; };
struct NextT { double v[12]; };

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
// One CTA.  A: every incoming observation outside a box looks its id up; hits and misses are only counted, so that a frame
// that does not fit leaves the table as it was.  B: hits append at n_obs (without checking that frames are contiguous, as the
// reference: a landmark hidden by a box for a frame comes back with a short list); misses are ranked by id and appended to the
// list.  C: the keyframe test, its parallax summed per thread in index order and then by a fixed tree, so that two runs agree.
constexpr int INGEST_BS = 1024;
constexpr int MAX_FRAME_OBS = 2048;
constexpr size_t BOX_BYTES = MAX_FRAME_OBS / 8;
__global__ void __launch_bounds__(INGEST_BS) k_fmw_ingest(Table T, u64* __restrict__ hash, int hmask, int cap, const gf_obs* __restrict__ obs,
                                                          const uint32_t* __restrict__ in_box, int n_in, int fc, double td, double min_parallax,
                                                          Result* __restrict__ res)
{
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
            avg = mean * FOCAL_LENGTH; margin = mean >= min_parallax;
        }
        res->margin_old = margin; res->avg_parallax = avg;
    }
}

// ---- triangulateWithDepth + triangulate ----
__global__ void __launch_bounds__(64) k_fmw_triangulate(Table T, FmPoses ps, double depth_threshold, double init_depth)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *T.n) return;
    const double* p = T.obs + (size_t)i * LM;
    fm_triangulate_one(T.nobs[i], T.start[i], p, ROW, p + 7, ROW, T.est + i, T.eflag + i, ps, depth_threshold, init_depth);
}

__global__ void k_fmw_clear_depth(Table T)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < *T.n) T.est[i] = -1.0;
}

// ---- the factor loop of Estimator::optimization (estimator.cpp:3268-3297) and getDepthVector ----
// One CTA: landmark i with >= 4 observations is feature k (scan of the flags) and owns n_obs - 1 factor rows from row0[k]
// (scan of n_obs - 1).
constexpr int SCAN_BS = 1024;
__global__ void __launch_bounds__(SCAN_BS) k_fmw_fill_scan(Table T, int* __restrict__ lm_of, int* __restrict__ row0, int* __restrict__ totals,
                                                           double* __restrict__ para_feature, uint8_t* __restrict__ feature_const,
                                                           Result* __restrict__ res)
{
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
    if (threadIdx.x == 0) { totals[0] = tf; totals[1] = tr; res->n_features = tf; res->n_visual = tr; res->n = n; res->status = GF_OK; }
}
// one thread per factor: its landmark is the last k with row0[k] <= f
__global__ void k_fmw_fill_rows(Table T, const int* __restrict__ lm_of, const int* __restrict__ row0, const int* __restrict__ totals,
                                gf_ba_visual_factor* __restrict__ out)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= totals[1]) return;
    int lo = 0, hi = totals[0] - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (row0[mid] <= f) lo = mid; else hi = mid - 1; }
    const int i = lm_of[lo], a = f - row0[lo] + 1, st = T.start[i];
    const double* r0 = T.obs + (size_t)i * LM;
    const double* ra = r0 + a * ROW;
    gf_ba_visual_factor v;
    v.imu_i = st; v.imu_j = st + a; v.feature = lo; v.reserved = 0;
    for (int c = 0; c < 3; c++) { v.pts_i[c] = r0[c]; v.pts_j[c] = ra[c]; }
    for (int c = 0; c < 2; c++) { v.vel_i[c] = r0[5 + c]; v.vel_j[c] = ra[5 + c]; }
    v.td_i = r0[8]; v.td_j = ra[8];
    out[f] = v;
}

// ---- setDepth (:249-267) ----  x[k] belongs to the k-th landmark with >= 4 observations
__global__ void __launch_bounds__(SCAN_BS) k_fmw_set_depth(Table T, const double* __restrict__ x)
{
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
__global__ void k_fmw_mark_ids(const u64* __restrict__ hash, int hmask, const int* __restrict__ ids, int n_ids, int* __restrict__ mark)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_ids) return;
    const int slot = hash_find(hash, hmask, ids[k]);
    if (slot >= 0) mark[slot] = 1;
}
// One CTA: per landmark the keep flag, the observation row the removal deletes (drop, -1: none) and the new start frame and
// depth, which are written in place; then the scan of the keep flags gives every survivor its place dst[i] in the other copy
// of the table (-1: removed).
__global__ void __launch_bounds__(SCAN_BS) k_fmw_plan(Table S, Table D, int op, int fc, ShiftT sh, double init_depth, int* __restrict__ mark,
                                                      int* __restrict__ drop, int* __restrict__ dst)
{
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
                if (k) S.est[i] = fm_back_shift_one(S.obs + (size_t)i * LM, S.est[i], sh.v, init_depth);
            }
        }
        drop[i] = dr;
        keep |= (unsigned)k << (i - b);
    }
    int total;
    int k = block_scan<SCAN_BS>(__popc(keep), &total);
    for (int i = b; i < e; i++) dst[i] = ((keep >> (i - b)) & 1u) ? k++ : -1;
    if (threadIdx.x == 0) *D.n = total;
}
// one warp per landmark: the survivor's scalars and rows (without the dropped one) into the other copy, and its id into the hash
__global__ void k_fmw_scatter(Table S, Table D, const int* __restrict__ drop, const int* __restrict__ dst, u64* __restrict__ hash, int hmask)
{
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= *S.n) return;
    const int d = dst[i];
    if (d < 0) return;
    const int dr = drop[i], m = S.nobs[i];
    if (lane == 0) {
        D.id[d] = S.id[i]; D.start[d] = S.start[i]; D.nobs[d] = dr >= 0 ? m - 1 : m; D.est[d] = S.est[i]; D.eflag[d] = S.eflag[i]; D.sflag[d] = S.sflag[i];
        hash_put(hash, hmask, S.id[i], d);
    }
    const double* s = S.obs + (size_t)i * LM;
    double* o = D.obs + (size_t)d * LM;
    const int cut = dr >= 0 ? dr * ROW : m * ROW, len = dr >= 0 ? (m - 1) * ROW : m * ROW;
    for (int c = lane; c < len; c += 32) o[c] = s[c < cut ? c : c + ROW];
}

// ---- outliersRejection (estimator.cpp:3909-3966) / movingConsistencyCheckW (:3968-4011) ----
// One CTA; the ids leave in list order through a scan of the flags.
constexpr int MATH_BS = 256;
__global__ void __launch_bounds__(MATH_BS) k_fmw_outliers(Table T, FmPoses ps, int mode, int* __restrict__ ids_out, Result* __restrict__ res)
{
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
    if (threadIdx.x == 0) { res->n_ids = total; res->n = n; res->status = GF_OK; }
}

// ---- predictPtsInNextFrame (estimator.cpp:3853-3886) ----
__global__ void __launch_bounds__(MATH_BS) k_fmw_predict(Table T, FmPoses ps, NextT nt, int fc, int* __restrict__ ids_out, double* __restrict__ xyz_out,
                                                         Result* __restrict__ res)
{
    const int n = *T.n, C = (n + MATH_BS - 1) / MATH_BS, b = threadIdx.x * C, e = min(n, b + C);
    unsigned sel = 0;
    for (int i = b; i < e; i++) sel |= (unsigned)(T.est[i] > 0 && T.nobs[i] >= 2 && T.start[i] + T.nobs[i] - 1 == fc) << (i - b);
    int total;
    int k = block_scan<MATH_BS>(__popc(sel), &total);
    for (int i = b; i < e; i++) {
        if (!((sel >> (i - b)) & 1u)) continue;
        ids_out[k] = T.id[i];
        fm_predict_one(T.start[i], T.obs + (size_t)i * LM, T.est[i], ps, nt.v, xyz_out + 3 * (size_t)k);
        k++;
    }
    if (threadIdx.x == 0) { res->n_ids = total; res->n = n; res->status = GF_OK; }
}

__global__ void k_fmw_size(Table T, Result* __restrict__ res) { res->n = *T.n; res->status = GF_OK; }

}  // namespace gffw

using namespace gffw;

struct gf_fm_window {
    int device, cap, hcap;
    gf_fm_window_cfg cfg;
    cudaStream_t s;
    cudaEvent_t ev0, ev1;               // around the device work of the last call (gf_fm_window_last_device_ms)
    Table t[2]; int cur;
    int* d_n;                           // [2]
    u64* hash;
    int *d_mark, *d_drop, *d_dst, *d_lm_of, *d_row0, *d_totals;
    uint8_t* d_in;                      // what a ring slot carried in: observations + box bits, depths, ids
    size_t in_bytes;
    // pinned
    uint8_t* h_ring[RING]; cudaEvent_t ring_ev[RING]; bool ring_used[RING]; int ring_k;
    uint8_t* h_out; uint8_t* d_out;     // mapped: Result, ids, xyz / para_feature, feature_const, factor rows
    size_t o_ids, o_xyz, o_feat, o_const, o_rows;
    uint8_t* h_read;                    // the table on its way out (gf_fm_window_read)
    int n_upper;                        // landmarks after the last add_frame: removals only lower the count, so read() copies this many
    bool depth_vector_valid; int depth_vector_n;   // n_features of the last fill_problem while the list is as it was then
};

namespace {

int use(gf_fm_window* w)
{
    if (!w) return set_err(GF_ERR_INVALID_ARG, "null window");
    GF_CUDA(cudaSetDevice(w->device));
    return GF_OK;
}
bool finite_all(const double* p, int n) { for (int i = 0; i < n; i++) if (!std::isfinite(p[i])) return false; return true; }
int load_poses(FmPoses* ps, const double* Ps, const double* Rs, const double* tic, const double* ric)
{
    if (!Ps || !Rs || !tic || !ric) return set_err(GF_ERR_INVALID_ARG, "null pose argument");
    if (!finite_all(Ps, 3 * NROW) || !finite_all(Rs, 9 * NROW) || !finite_all(tic, 3) || !finite_all(ric, 9))
        return set_err(GF_ERR_INVALID_ARG, "non-finite pose");
    memcpy(ps->P, Ps, sizeof(ps->P)); memcpy(ps->R, Rs, sizeof(ps->R)); memcpy(ps->tic, tic, 24); memcpy(ps->ric, ric, 72);
    return GF_OK;
}
Result* result(gf_fm_window* w) { return reinterpret_cast<Result*>(w->h_out); }
template <class T> T* dev_out(gf_fm_window* w, size_t off) { return reinterpret_cast<T*>(w->d_out + off); }
template <class T> T* host_out(gf_fm_window* w, size_t off) { return reinterpret_cast<T*>(w->h_out + off); }
int grid(const gf_fm_window* w, int per_block) { return (w->cap + per_block - 1) / per_block; }

// a pinned slot the copy engine is not reading; the wait only happens when the device is RING uploads behind
int ring_acquire(gf_fm_window* w, uint8_t** p, int* k)
{
    *k = w->ring_k; w->ring_k = (w->ring_k + 1) % RING;
    if (w->ring_used[*k]) GF_CUDA(cudaEventSynchronize(w->ring_ev[*k]));
    *p = w->h_ring[*k];
    return GF_OK;
}
int ring_upload(gf_fm_window* w, int k, size_t bytes)
{
    GF_CUDA(cudaMemcpyAsync(w->d_in, w->h_ring[k], bytes, cudaMemcpyHostToDevice, w->s));
    GF_CUDA(cudaEventRecord(w->ring_ev[k], w->s));
    w->ring_used[k] = true;
    return GF_OK;
}
int begin(gf_fm_window* w) { GF_CUDA(cudaEventRecord(w->ev0, w->s)); return GF_OK; }
int end_async(gf_fm_window* w) { GF_CUDA(cudaGetLastError()); GF_CUDA(cudaEventRecord(w->ev1, w->s)); return GF_OK; }
int end_sync(gf_fm_window* w) { int rc = end_async(w); if (rc) return rc; GF_CUDA(cudaStreamSynchronize(w->s)); return GF_OK; }

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
    GF_CUDA(cudaStreamCreateWithFlags(&w->s, cudaStreamNonBlocking));
    GF_CUDA(cudaEventCreate(&w->ev0)); GF_CUDA(cudaEventCreate(&w->ev1));
    GF_CUDA(cudaMalloc(&w->d_n, 8));
    int rc;
    for (int i = 0; i < 2; i++) if ((rc = alloc_table(&w->t[i], w->d_n + i, cap))) return rc;
    GF_CUDA(cudaMalloc(&w->hash, 8 * (size_t)w->hcap));
    GF_CUDA(cudaMalloc(&w->d_mark, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&w->d_drop, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&w->d_dst, 4 * (size_t)cap));
    GF_CUDA(cudaMalloc(&w->d_lm_of, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&w->d_row0, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&w->d_totals, 8));
    w->in_bytes = BOX_BYTES + (size_t)MAX_FRAME_OBS * sizeof(gf_obs);
    if (w->in_bytes < 8 * (size_t)cap) w->in_bytes = 8 * (size_t)cap;
    GF_CUDA(cudaMalloc(&w->d_in, w->in_bytes));
    for (int k = 0; k < RING; k++) {
        GF_CUDA(cudaHostAlloc(&w->h_ring[k], w->in_bytes, cudaHostAllocDefault));
        GF_CUDA(cudaEventCreateWithFlags(&w->ring_ev[k], cudaEventDisableTiming));
    }
    w->o_ids = 64; w->o_xyz = w->o_ids + 4 * (size_t)cap; w->o_feat = w->o_xyz + 24 * (size_t)cap; w->o_const = w->o_feat + 8 * (size_t)cap;
    w->o_rows = (w->o_const + cap + 15) / 16 * 16;
    static_assert(sizeof(Result) <= 64, "Result fits the head of the block");
    GF_CUDA(cudaHostAlloc(&w->h_out, w->o_rows + sizeof(gf_ba_visual_factor) * (size_t)cap * W, cudaHostAllocMapped));
    GF_CUDA(cudaHostGetDevicePointer(&w->d_out, w->h_out, 0));
    GF_CUDA(cudaHostAlloc(&w->h_read, (size_t)cap * (28 + 8 * LM), cudaHostAllocDefault));
    return gf_fm_window_clear(w);
}

// the plan / scan / scatter of one removal; the copies of the table then swap roles.  begun: the caller recorded the start
// event already (remove_ids, whose upload and marking belong to the call's device time)
int remove(gf_fm_window* w, int op, int fc, const ShiftT& sh, bool begun = false)
{
    int rc;
    if (!begun && (rc = begin(w))) return rc;
    Table S = w->t[w->cur], D = w->t[w->cur ^ 1];
    k_fmw_plan<<<1, SCAN_BS, 0, w->s>>>(S, D, op, fc, sh, w->cfg.init_depth, w->d_mark, w->d_drop, w->d_dst);
    GF_LAUNCHED();
    GF_CUDA(cudaMemsetAsync(w->hash, 0xff, 8 * (size_t)w->hcap, w->s));
    k_fmw_scatter<<<grid(w, 8), 256, 0, w->s>>>(S, D, w->d_drop, w->d_dst, w->hash, w->hcap - 1);
    GF_LAUNCHED();
    w->cur ^= 1;
    w->depth_vector_valid = false;
    return end_async(w);
}

int ingest(gf_fm_window* w, const gf_obs* d_obs, const uint32_t* d_in_box, int n, int frame_count, double td, int* margin_old, int32_t* counters4,
           double* last_average_parallax)
{
    Result* r = result(w);
    k_fmw_ingest<<<1, INGEST_BS, 0, w->s>>>(w->t[w->cur], w->hash, w->hcap - 1, w->cap, d_obs, d_in_box, n, frame_count, td, w->cfg.min_parallax,
                                            dev_out<Result>(w, 0));
    GF_LAUNCHED();
    int rc = end_sync(w);
    if (rc) return rc;
    if (r->status == GF_ERR_CAPACITY) return set_err(GF_ERR_CAPACITY, "the frame's new landmarks do not fit max_features; the table is unchanged");
    if (r->status) return set_err(GF_ERR_INVALID_ARG, "a landmark of the frame already has an observation in the last window frame; the table is unchanged");
    w->depth_vector_valid = false;
    w->n_upper = r->n;
    if (margin_old) *margin_old = r->margin_old;
    if (counters4) { counters4[0] = r->last_track; counters4[1] = r->new_feature; counters4[2] = r->long_track; counters4[3] = r->n; }
    if (last_average_parallax) *last_average_parallax = r->avg_parallax;
    return GF_OK;
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
    if (w->s) cudaStreamSynchronize(w->s);
    for (int i = 0; i < 2; i++) {
        Table& t = w->t[i];
        cudaFree(t.id); cudaFree(t.start); cudaFree(t.nobs); cudaFree(t.eflag); cudaFree(t.sflag); cudaFree(t.est); cudaFree(t.obs);
    }
    cudaFree(w->d_n); cudaFree(w->hash); cudaFree(w->d_mark); cudaFree(w->d_drop); cudaFree(w->d_dst); cudaFree(w->d_lm_of); cudaFree(w->d_row0);
    cudaFree(w->d_totals); cudaFree(w->d_in);
    for (int k = 0; k < RING; k++) { if (w->h_ring[k]) cudaFreeHost(w->h_ring[k]); if (w->ring_ev[k]) cudaEventDestroy(w->ring_ev[k]); }
    if (w->h_out) cudaFreeHost(w->h_out);
    if (w->h_read) cudaFreeHost(w->h_read);
    if (w->ev0) cudaEventDestroy(w->ev0);
    if (w->ev1) cudaEventDestroy(w->ev1);
    if (w->s) cudaStreamDestroy(w->s);
    delete w;
}

int gf_fm_window_clear(gf_fm_window* w)
{
    int rc = use(w);
    if (rc || (rc = begin(w))) return rc;
    GF_CUDA(cudaMemsetAsync(w->d_n, 0, 8, w->s));
    GF_CUDA(cudaMemsetAsync(w->d_mark, 0, 4 * (size_t)w->cap, w->s));
    GF_CUDA(cudaMemsetAsync(w->hash, 0xff, 8 * (size_t)w->hcap, w->s));
    w->depth_vector_valid = false;
    w->n_upper = 0;
    return end_async(w);
}

int gf_fm_window_add_frame(gf_fm_window* w, int frame_count, const gf_obs* obs, int n, const uint8_t* in_box, double td, int* margin_old,
                           int32_t* counters4, double* last_average_parallax)
{
    int rc = use(w);
    if (rc) return rc;
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
    uint8_t* slot; int k;
    if ((rc = ring_acquire(w, &slot, &k))) return rc;
    uint32_t* bits = reinterpret_cast<uint32_t*>(slot);               // slot: box bits, then the observations
    memset(bits, 0, BOX_BYTES);
    if (in_box) for (int i = 0; i < n; i++) if (in_box[i]) bits[i >> 5] |= 1u << (i & 31);
    if (n) memcpy(slot + BOX_BYTES, obs, (size_t)n * sizeof(gf_obs));
    if ((rc = begin(w)) || (rc = ring_upload(w, k, BOX_BYTES + (size_t)n * sizeof(gf_obs)))) return rc;
    return ingest(w, reinterpret_cast<const gf_obs*>(w->d_in + BOX_BYTES), reinterpret_cast<const uint32_t*>(w->d_in), n, frame_count, td, margin_old,
                  counters4, last_average_parallax);
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
    if ((rc = begin(w))) return rc;
    GF_CUDA(cudaStreamWaitEvent(w->s, o.downloaded, 0));
    return ingest(w, o.obs, o.in_box, o.n, frame_count, td, margin_old, counters4, last_average_parallax);
}

int gf_fm_window_triangulate(gf_fm_window* w, int frame_count, const double* Ps, const double* Rs, const double* tic, const double* ric)
{
    int rc = use(w);
    if (rc) return rc;
    if (frame_count < 0 || frame_count > W) return set_err(GF_ERR_INVALID_ARG, "frame_count out of range");
    FmPoses ps;
    if ((rc = load_poses(&ps, Ps, Rs, tic, ric)) || (rc = begin(w))) return rc;
    k_fmw_triangulate<<<grid(w, 64), 64, 0, w->s>>>(w->t[w->cur], ps, w->cfg.depth_threshold, w->cfg.init_depth);
    GF_LAUNCHED();
    return end_async(w);
}

int gf_fm_window_fill_problem(gf_fm_window* w, gf_ba_visual_factor* visual_out, int cap, int* n_visual, double* para_feature, uint8_t* feature_const,
                              int* n_features)
{
    int rc = use(w);
    if (rc) return rc;
    if (cap < 0 || (cap > 0 && !visual_out) || !n_features) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if ((rc = begin(w))) return rc;
    k_fmw_fill_scan<<<1, SCAN_BS, 0, w->s>>>(w->t[w->cur], w->d_lm_of, w->d_row0, w->d_totals, dev_out<double>(w, w->o_feat), dev_out<uint8_t>(w, w->o_const),
                                             dev_out<Result>(w, 0));
    GF_LAUNCHED();
    if (visual_out) {
        k_fmw_fill_rows<<<grid(w, 256) * W, 256, 0, w->s>>>(w->t[w->cur], w->d_lm_of, w->d_row0, w->d_totals, dev_out<gf_ba_visual_factor>(w, w->o_rows));
        GF_LAUNCHED();
    }
    if ((rc = end_sync(w))) return rc;
    const Result* r = result(w);
    if (visual_out && r->n_visual > cap) return set_err(GF_ERR_CAPACITY, "visual_out is too small for the window's factors");
    *n_features = r->n_features;
    if (n_visual) *n_visual = r->n_visual;
    if (para_feature) memcpy(para_feature, host_out<double>(w, w->o_feat), 8 * (size_t)r->n_features);
    if (feature_const) memcpy(feature_const, host_out<uint8_t>(w, w->o_const), (size_t)r->n_features);
    if (visual_out) memcpy(visual_out, host_out<gf_ba_visual_factor>(w, w->o_rows), sizeof(gf_ba_visual_factor) * (size_t)r->n_visual);
    w->depth_vector_valid = true; w->depth_vector_n = r->n_features;
    return GF_OK;
}

int gf_fm_window_set_depth(gf_fm_window* w, const double* para_feature, int n)
{
    int rc = use(w);
    if (rc) return rc;
    if (n < 0 || (n > 0 && !para_feature)) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (!w->depth_vector_valid || n != w->depth_vector_n)
        return set_err(GF_ERR_INVALID_ARG, "set_depth takes the n_features values of the last fill_problem, with no frame added or landmark removed since");
    if ((rc = begin(w))) return rc;
    if (n == 0) return end_async(w);
    uint8_t* slot; int k;
    if ((rc = ring_acquire(w, &slot, &k))) return rc;
    memcpy(slot, para_feature, 8 * (size_t)n);
    if ((rc = ring_upload(w, k, 8 * (size_t)n))) return rc;
    k_fmw_set_depth<<<1, SCAN_BS, 0, w->s>>>(w->t[w->cur], reinterpret_cast<const double*>(w->d_in));
    GF_LAUNCHED();
    return end_async(w);
}

int gf_fm_window_clear_depth(gf_fm_window* w)
{
    int rc = use(w);
    if (rc || (rc = begin(w))) return rc;
    k_fmw_clear_depth<<<grid(w, 256), 256, 0, w->s>>>(w->t[w->cur]);
    GF_LAUNCHED();
    return end_async(w);
}

int gf_fm_window_remove_failures(gf_fm_window* w)
{
    int rc = use(w);
    return rc ? rc : remove(w, OP_FAILURES, 0, ShiftT());
}

int gf_fm_window_remove_ids(gf_fm_window* w, const int32_t* ids, int n)
{
    int rc = use(w);
    if (rc) return rc;
    if (n < 0 || (n > 0 && !ids)) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if ((rc = begin(w))) return rc;
    if (n == 0) return end_async(w);
    uint8_t* slot = nullptr; int k = 0;
    // more ids than a slot holds go in pieces: marks accumulate and one compaction follows
    const int piece = (int)(w->in_bytes / 4);
    for (int o = 0; o < n; o += piece) {
        const int m = n - o < piece ? n - o : piece;
        if ((rc = ring_acquire(w, &slot, &k))) return rc;
        memcpy(slot, ids + o, 4 * (size_t)m);
        if ((rc = ring_upload(w, k, 4 * (size_t)m))) return rc;
        k_fmw_mark_ids<<<(m + 255) / 256, 256, 0, w->s>>>(w->hash, w->hcap - 1, reinterpret_cast<const int*>(w->d_in), m, w->d_mark);
        GF_LAUNCHED();
    }
    return remove(w, OP_IDS, 0, ShiftT(), true);
}

int gf_fm_window_remove_back_shift_depth(gf_fm_window* w, const double* marg_R, const double* marg_P, const double* new_R, const double* new_P)
{
    int rc = use(w);
    if (rc) return rc;
    if (!marg_R || !marg_P || !new_R || !new_P) return set_err(GF_ERR_INVALID_ARG, "null pose argument");
    if (!finite_all(marg_R, 9) || !finite_all(marg_P, 3) || !finite_all(new_R, 9) || !finite_all(new_P, 3)) return set_err(GF_ERR_INVALID_ARG, "non-finite pose");
    ShiftT sh;
    memcpy(sh.v, marg_R, 72); memcpy(sh.v + 9, marg_P, 24); memcpy(sh.v + 12, new_R, 72); memcpy(sh.v + 21, new_P, 24);
    return remove(w, OP_BACK_SHIFT, 0, sh);
}

int gf_fm_window_remove_back(gf_fm_window* w)
{
    int rc = use(w);
    return rc ? rc : remove(w, OP_BACK, 0, ShiftT());
}

int gf_fm_window_remove_front(gf_fm_window* w, int frame_count)
{
    int rc = use(w);
    if (rc) return rc;
    // slideWindowNew runs on a full window only; row WINDOW_SIZE - 1 - start_frame is then the second newest frame's
    if (frame_count != W) return set_err(GF_ERR_INVALID_ARG, "remove_front takes frame_count == WINDOW_SIZE");
    return remove(w, OP_FRONT, frame_count, ShiftT());
}

int gf_fm_window_outliers(gf_fm_window* w, const double* Ps, const double* Rs, const double* tic, const double* ric, int mode, int32_t* ids_out, int* n)
{
    int rc = use(w);
    if (rc) return rc;
    if (!ids_out || !n || (mode != GF_FM_OUTLIERS_REPROJECTION && mode != GF_FM_OUTLIERS_MOVING)) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    FmPoses ps;
    if ((rc = load_poses(&ps, Ps, Rs, tic, ric)) || (rc = begin(w))) return rc;
    k_fmw_outliers<<<1, MATH_BS, 0, w->s>>>(w->t[w->cur], ps, mode, dev_out<int>(w, w->o_ids), dev_out<Result>(w, 0));
    GF_LAUNCHED();
    if ((rc = end_sync(w))) return rc;
    *n = result(w)->n_ids;
    memcpy(ids_out, host_out<int>(w, w->o_ids), 4 * (size_t)*n);
    return GF_OK;
}

int gf_fm_window_predict_next(gf_fm_window* w, int frame_count, const double* Ps, const double* Rs, const double* tic, const double* ric, int32_t* ids_out,
                              double* xyz_out, int* n)
{
    int rc = use(w);
    if (rc) return rc;
    if (!ids_out || !xyz_out || !n) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (frame_count < 0 || frame_count > W) return set_err(GF_ERR_INVALID_ARG, "frame_count out of range");
    FmPoses ps;
    if ((rc = load_poses(&ps, Ps, Rs, tic, ric))) return rc;
    *n = 0;
    if (frame_count < 2) return GF_OK;                                  // estimator.cpp:3855
    NextT nt;
    fm_next_pose(Ps, Rs, frame_count, nt.v);
    if ((rc = begin(w))) return rc;
    k_fmw_predict<<<1, MATH_BS, 0, w->s>>>(w->t[w->cur], ps, nt, frame_count, dev_out<int>(w, w->o_ids), dev_out<double>(w, w->o_xyz), dev_out<Result>(w, 0));
    GF_LAUNCHED();
    if ((rc = end_sync(w))) return rc;
    *n = result(w)->n_ids;
    memcpy(ids_out, host_out<int>(w, w->o_ids), 4 * (size_t)*n);
    memcpy(xyz_out, host_out<double>(w, w->o_xyz), 24 * (size_t)*n);
    return GF_OK;
}

int gf_fm_window_size(gf_fm_window* w, int* n)
{
    int rc = use(w);
    if (rc) return rc;
    if (!n) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if ((rc = begin(w))) return rc;
    k_fmw_size<<<1, 1, 0, w->s>>>(w->t[w->cur], dev_out<Result>(w, 0));
    GF_LAUNCHED();
    if ((rc = end_sync(w))) return rc;
    *n = result(w)->n;
    return GF_OK;
}

int gf_fm_window_read(gf_fm_window* w, int32_t* feature_id, int32_t* start_frame, int32_t* n_obs, double* estimated_depth, int32_t* estimate_flag,
                      int32_t* solve_flag, double* obs, int cap, int* n)
{
    int rc = use(w);
    if (rc) return rc;
    if (!n || cap < 0) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if ((rc = begin(w))) return rc;
    const Table& T = w->t[w->cur];
    const size_t c = (size_t)w->n_upper;
    uint8_t* h = w->h_read;
    const void* src[7] = {T.id, T.start, T.nobs, T.eflag, T.sflag, T.est, T.obs};
    void* dst[7] = {feature_id, start_frame, n_obs, estimate_flag, solve_flag, estimated_depth, obs};
    const size_t el[7] = {4, 4, 4, 4, 4, 8, 8 * (size_t)LM};
    size_t off[8] = {0};
    for (int k = 0; k < 7; k++) {
        off[k + 1] = off[k] + el[k] * c;
        if (dst[k] && c) GF_CUDA(cudaMemcpyAsync(h + off[k], src[k], el[k] * c, cudaMemcpyDeviceToHost, w->s));
    }
    k_fmw_size<<<1, 1, 0, w->s>>>(T, dev_out<Result>(w, 0));
    GF_LAUNCHED();
    if ((rc = end_sync(w))) return rc;
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
    GF_CUDA(cudaEventSynchronize(w->ev1));
    GF_CUDA(cudaEventElapsedTime(ms, w->ev0, w->ev1));
    return GF_OK;
}

}  // extern "C"
