// fe_select.cuh -- the order-dependent part of the front end, kept on the device:
//   k_compact_setmask : reduceVector x4 + track_cnt++ + setMask   (feature_tracker.cpp:170-179, 56-83)
//   (mask)            : the mask goodFeaturesToTrack sees (cv::circle == integer disk d^2<=r^2 around the kept
//                       features) is never materialised: tiles test pixels against the kept features in reach
//   k_eig_max / k_candidates : minMaxLoc(masked) -> threshold -> 3x3 dilate -> local maxima
//   k_select_finalize : cv::goodFeaturesToTrack's greedy min-distance pass by cell-head rounds (the accepted set is
//                       exactly the sequential greedy's; the maxCorners cap = top-K of that set by rank; the rounds stop
//                       once the top K can no longer change), then
//                       addPoints, undistortedPts, ptsVelocity, depth and the state of the next frame
// Arithmetic and ordering follow oracle/fe_cv_restate.c and oracle/fe_oracle.py.
#pragma once
#include "fe_sort.cuh"
#include "gf_camera.cuh"
#include "gf_common.cuh"

namespace gf {

constexpr int FE_CAP = 1024;        // max max_cnt (one thread per feature in the single-CTA kernels)
constexpr int FE_SORT_CAP = 4096;   // accepted corners sorted in shared memory by k_finalize

struct TrackScalars {
    int n_prev;       // features entering LK this frame (= features at the end of the previous frame)
    int n_id;         // next feature id (FeatureTracker::n_id)
    int n_tracked;
    int n_kept;
    int n_new;
    int n_cand;
    int n_acc;
    unsigned int max_key;   // order-preserving encoding of the masked eig maximum (0 = no unmasked pixel)
    int eig_fixups;
    int pred_succ;    // successes of the prediction LK pass (feature_tracker.cpp:125-131)
    int n_out;
    int nms_rounds;
    int nms_remaining[16];
    int lk_iters;
};

struct FeatArrays {   // all device pointers, capacity FE_CAP
    float2* prev_pts; int* ids; int* track_cnt; float2* prev_un;      // persistent feature state
    float2* cur_pts; uint8_t* status;                                  // LK output for the n_prev features
    float2* kept_pts; int* kept_ids; int* kept_cnt; float2* kept_un;  // after setMask
    float2* pred_pts;
    long long* dbg;                                                    // clock64 phase counters (gf_tracker_debug_read); may be null
};
constexpr int FE_DBG_N = 64 + 8 * FE_CAP;
#define GF_DBG(slot, v) do { if (fa.dbg && threadIdx.x == 0 && blockIdx.x == 0) fa.dbg[slot] = (v); } while (0)

__device__ __forceinline__ unsigned int float_order_key(float v)
{
    unsigned int b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);   // monotone, never 0 for finite v
}
__device__ __forceinline__ float float_from_order_key(unsigned int k)
{
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// ------------------------------------------------------------------------------------------------
constexpr int SM_CF_MAX = 6;   // earlier features within min_dist remembered per feature (more: full rescans)
template <int V>
__device__ __forceinline__ void compact_setmask(TrackScalars* sc, const FeatArrays& fa, int min_dist)
{
    __shared__ sort_elem elems[FE_CAP];
    __shared__ float2 c_pt[FE_CAP];
    __shared__ short c_orig[FE_CAP];       // compacted position -> index before reduceVector
    __shared__ short2 rc[FE_CAP];          // rounded centres in sorted order
    __shared__ short cf[FE_CAP * SM_CF_MAX];
    __shared__ int ncf[FE_CAP];
    __shared__ uint8_t st[FE_CAP];
    __shared__ int warp_sums[32];
    __shared__ int s_m;
    __shared__ SortWork swork;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int n = sc->n_prev;
    const long long c0 = gf_clock();
    // ---- reduceVector (stable compaction by status) ----
    int keep = (tid < n) ? (fa.status[tid] != 0) : 0;
    unsigned bal = __ballot_sync(0xffffffffu, keep);
    int pre = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_sums[wid] = __popc(bal);
    ncf[tid] = 0;
    __syncthreads();
    if (wid == 0) {
        int v = warp_sums[lane];
        int incl = v;
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        warp_sums[lane] = incl - v;
        if (lane == 31) s_m = incl;
    }
    __syncthreads();
    const int m = s_m;
    if (keep) {
        int p = warp_sums[wid] + pre;
        c_pt[p] = fa.cur_pts[tid];
        c_orig[p] = (short)tid;
        int cnt = fa.track_cnt[tid] + 1;                     // for (auto &n : track_cnt) n++;
        elems[p] = ((sort_elem)(unsigned)cnt << 32) | (unsigned)p;
    }
    __syncthreads();
    const long long c1 = gf_clock();
    // ---- std::sort replica: same comparisons and moves as libstdc++, replayed in parallel (fe_sort.cuh) ----
    setmask_sort_parallel(elems, m, swork);
    const long long c2 = gf_clock();
    int src = 0;
    if (tid < m) {
        src = (int)(elems[tid] & 0xffffffffu);
        float2 p = c_pt[src];
        rc[tid] = make_short2((short)__float2int_rn(p.x), (short)__float2int_rn(p.y));
        st[tid] = 0;
    }
    __syncthreads();
    // ---- "if (mask.at(pt) == 255) keep, draw disk": feature j is kept iff no kept earlier feature i has
    //      d^2 <= r^2.  Pass 1 (all threads): the earlier features within range of each j.  Pass 2: rounds over those
    //      short lists (a feature decides once all of its listed predecessors have). ----
    const int r2 = min_dist * min_dist;
    {
        const int mp = (m + 31) & ~31;
        const int parts = mp ? max(1, FE_CAP / mp) : 1;
        const int j = mp ? tid % mp : 0, part = mp ? tid / mp : parts;
        if (j < m && part < parts) {
            const short2 c = rc[j];
            for (int i = part; i < j; i += parts) {
                int dx = c.x - rc[i].x, dy = c.y - rc[i].y;
                if (dx * dx + dy * dy <= r2) {
                    int k = atomicAdd(&ncf[j], 1);
                    if (k < SM_CF_MAX) cf[j * SM_CF_MAX + k] = (short)i;
                }
            }
        }
    }
    __syncthreads();
    int my = 0;  // 0 undecided, 1 kept, 2 rejected
    const int nc = (tid < m) ? ncf[tid] : 0;
    while (true) {
        int ns = my;
        if (tid < m && my == 0) {
            bool rej = false, blk = false;
            if (nc <= SM_CF_MAX) {
                for (int k = 0; k < nc; k++) {
                    int s = st[cf[tid * SM_CF_MAX + k]];
                    if (s == 1) rej = true;
                    if (s == 0) blk = true;
                }
            } else {
                short2 c = rc[tid];
                for (int i = 0; i < tid; i++) {
                    int dx = c.x - rc[i].x, dy = c.y - rc[i].y;
                    if (dx * dx + dy * dy <= r2) {
                        int s = st[i];
                        if (s == 1) { rej = true; break; }
                        if (s == 0) blk = true;
                    }
                }
            }
            ns = rej ? 2 : (blk ? 0 : 1);
        }
        __syncthreads();
        if (tid < m) { st[tid] = (uint8_t)ns; my = ns; }
        int undecided = __syncthreads_or((tid < m) && ns == 0);
        if (!undecided) break;
    }
    const long long c3 = gf_clock();
    // ---- emit kept features in sorted order ----
    int k = (tid < m) && (my == 1);
    bal = __ballot_sync(0xffffffffu, k);
    pre = __popc(bal & ((1u << lane) - 1));
    __syncthreads();
    if (lane == 0) warp_sums[wid] = __popc(bal);
    __syncthreads();
    if (wid == 0) {
        int v = warp_sums[lane];
        int incl = v;
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        warp_sums[lane] = incl - v;
        if (lane == 31) { sc->n_kept = incl; sc->n_tracked = m; }
    }
    __syncthreads();
    if (k) {
        int p = warp_sums[wid] + pre;
        const int o = c_orig[src];
        fa.kept_pts[p] = c_pt[src];
        fa.kept_un[p] = fa.prev_un[o];
        fa.kept_ids[p] = fa.ids[o];
        fa.kept_cnt[p] = (int)(elems[tid] >> 32);
    }
    if (tid == 0) {   // per-frame counters consumed downstream
        sc->n_cand = 0; sc->max_key = 0; sc->n_new = 0; sc->nms_rounds = 0;
        for (int i = 0; i < 16; i++) sc->nms_remaining[i] = 0;
    }
    GF_DBG(0, c1 - c0); GF_DBG(1, c2 - c1); GF_DBG(2, c3 - c2); GF_DBG(3, gf_clock() - c3);
}
__global__ void __launch_bounds__(FE_CAP) k_compact_setmask(TrackScalars* sc, FeatArrays fa, int min_dist)
{
    compact_setmask<0>(sc, fa, min_dist);
}

// ------------------------------------------------------------------------------------------------
// The mask goodFeaturesToTrack sees (setMask, feature_tracker.cpp:56-83) is 255 except inside the integer disks
// d^2 <= r^2 around the rounded centres of the kept features (cv::circle == integer disk, SURVEY A.5).  It is never
// materialised: every CTA collects the kept features that can touch its tile into shared memory and tests pixels
// against that short list.
constexpr int MASK_TX = 64, MASK_TY = 16, MASK_LIST = 64;
struct MaskTile { short2 pt[MASK_LIST]; int n; int overflow; };

__device__ __forceinline__ void mask_tile_load(MaskTile& M, const TrackScalars* sc, const float2* kept, int x0, int y0, int r)
{
    if (threadIdx.x == 0) { M.n = 0; M.overflow = 0; }
    __syncthreads();
    const int nk = sc->n_kept;
    for (int i = threadIdx.x; i < nk; i += blockDim.x) {
        float2 p = kept[i];
        int cx = __float2int_rn(p.x), cy = __float2int_rn(p.y);
        if (cx >= x0 - r && cx < x0 + MASK_TX + r && cy >= y0 - r && cy < y0 + MASK_TY + r) {
            int k = atomicAdd(&M.n, 1);
            if (k < MASK_LIST) M.pt[k] = make_short2((short)cx, (short)cy); else M.overflow = 1;
        }
    }
    __syncthreads();
}
__device__ __forceinline__ bool mask_open(const MaskTile& M, const TrackScalars* sc, const float2* kept, int x, int y, int r2)
{
    // More neighbours than the list holds: exact slow path.  Kept features are > r apart, but at r = 5 about 75 of them fit a
    // tile's 74x26 apron when packed on a lattice (gf_stage_gftt with such a kept list reaches this); the tracker's kept
    // features on textured scenes put at most ~16 there at max_cnt 1000, min_dist 5.
    if (M.overflow) {
        for (int i = 0; i < sc->n_kept; i++) {
            int dx = x - __float2int_rn(kept[i].x), dy = y - __float2int_rn(kept[i].y);
            if (dx * dx + dy * dy <= r2) return false;
        }
        return true;
    }
    const int n = M.n;
    for (int i = 0; i < n; i++) {
        int dx = x - M.pt[i].x, dy = y - M.pt[i].y;
        if (dx * dx + dy * dy <= r2) return false;
    }
    return true;
}

// masked maximum of the eig map (cv::minMaxLoc(eig, 0, &maxVal, 0, 0, mask)); one 64x16 tile per CTA of 256 threads
template <int V>
__device__ __forceinline__ void eig_max_tile(TrackScalars* sc, const float2* kept, const float* eig, int epitch, int w, int h, int r)
{
    __shared__ MaskTile M;
    __shared__ unsigned int wb[8];
    const int x0 = blockIdx.x * MASK_TX, y0 = blockIdx.y * MASK_TY;
    mask_tile_load(M, sc, kept, x0, y0, r);
    unsigned int best = 0;
    const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
    for (int yy = ty; yy < MASK_TY; yy += 4) {
        int x = x0 + tx, y = y0 + yy;
        if (x < w && y < h && mask_open(M, sc, kept, x, y, r * r)) best = max(best, float_order_key(eig[(size_t)y * epitch + x]));
    }
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((threadIdx.x & 31) == 0) wb[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < 8; i++) best = max(best, wb[i]);
        if (best) atomicMax(&sc->max_key, best);
    }
}
__global__ void __launch_bounds__(256) k_eig_max(TrackScalars* sc, const float2* kept, const float* eig, int epitch, int w, int h, int r)
{
    eig_max_tile<0>(sc, kept, eig, epitch, w, h, r);
}

// Candidate list + the cell grid used by the min-distance pass.  cell = max(min_dist, 16) so that a corner's
// r-neighbourhood is covered by the 3x3 cells around it.
struct NmsGrid {
    int cs, gw, gh;                 // cell size, grid dims
    unsigned long long* cand_key;   // [w*h] flat candidate list: (eig bits << 32 | y << 16 | x), any order; same order as (eig, address)
    unsigned long long* acc_key;    // [w*h / 16 + 64] accepted corners (any order), count in TrackScalars::n_acc
    int acc_cap;
    uint8_t* dead;                  // [w*h] slow path only (more than 65536 candidates)
};

// threshold(TOZERO, 0.01*max) -> dilate 3x3 -> val != 0 && val == dilated && mask, on the interior
template <int V>
__device__ __forceinline__ void candidates_tile(TrackScalars* sc, const float2* kept, const float* eig, int epitch, int w, int h, int r,
                                                const NmsGrid& g)
{
    __shared__ MaskTile M;
    const int x0 = blockIdx.x * MASK_TX, y0 = blockIdx.y * MASK_TY;
    mask_tile_load(M, sc, kept, x0, y0, r);
    const double maxVal = sc->max_key ? (double)float_from_order_key(sc->max_key) : 0.0;
    const float thr = (float)(maxVal * 0.01);
    const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
#pragma unroll 1
    for (int yy = ty; yy < MASK_TY; yy += 4) {
    const int x = x0 + tx, y = y0 + yy;
    bool is_cand = false;
    float v = 0.f;
    if (x >= 1 && x < w - 1 && y >= 1 && y < h - 1) {
        const float* e = eig + (size_t)y * epitch + x;
        v = __ldg(e);
        if (v > thr && v != 0.f && mask_open(M, sc, kept, x, y, r * r)) {
            float m = fmaxf(fmaxf(__ldg(e - 1), __ldg(e + 1)), fmaxf(__ldg(e - epitch), __ldg(e + epitch)));
            m = fmaxf(m, fmaxf(fmaxf(__ldg(e - epitch - 1), __ldg(e - epitch + 1)), fmaxf(__ldg(e + epitch - 1), __ldg(e + epitch + 1))));
            is_cand = !(m > v);   // a larger neighbour is itself > thr, so the dilated value would exceed v
        }
    }
    // warp-aggregated append
    unsigned bal = __ballot_sync(0xffffffffu, is_cand);
    if (bal) {
        int lane = threadIdx.x & 31, base = 0;
        if (lane == (__ffs(bal) - 1)) base = atomicAdd(&sc->n_cand, __popc(bal));
        base = __shfl_sync(0xffffffffu, base, __ffs(bal) - 1);
        if (is_cand) g.cand_key[base + __popc(bal & ((1u << lane) - 1))] = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned)((y << 16) | x);
    }
    }
}
__global__ void __launch_bounds__(256) k_candidates(TrackScalars* sc, const float2* kept, const float* eig, int epitch,
                                                    int w, int h, int r, NmsGrid g)
{
    candidates_tile<0>(sc, kept, eig, epitch, w, h, r, g);
}

// cv::goodFeaturesToTrack's greedy min-distance pass, exact, by rounds (single CTA, 1024 threads):
//   every alive candidate is killed if one of LAST round's accepted corners in its 3x3 cells is closer than r
//   (older accepted corners have already killed their neighbours), otherwise it bids for the head of its cell.
//   A head that outranks the heads of the 8 surrounding cells has no undecided higher-ranked candidate within r
//   (every candidate of a cell ranks below its head) and no accepted corner within r (else it would be dead), so the
//   sequential greedy would accept it too.  The globally best head can always decide, so the loop terminates;
//   measured 5-11 rounds at 640x480 to decide every candidate.  Only the first `want` accepted corners by rank are kept,
//   so the loop stops as soon as `want` corners accepted in earlier rounds outrank every cell head (see the early exit).
// The single SM is issue-bound on this, so the rounds are kept lean: the head election is two native 32-bit
// ATOMS.MAX (eig bits, then packed address among the ties; a 64-bit shared atomicMax is a CAS spin loop), a per-cell
// flag says whether any of the 3x3 cells accepted a corner last round (most candidates skip the distance tests),
// the first two candidates of a thread and their cells live in registers, and the per-round arrays are double-buffered
// so that a round needs three barriers.
// Dynamic shared memory: nms_smem_bytes(gw, gh).
constexpr int NMS_MAX_PER_THREAD = 64;
constexpr int NMS_CELL_BYTES = 32;   // per padded cell: head_hi[2] + head_lo[2] + acc[2] (4 B each) + flag[2] (1 B each) + index (2 B), rounded up
__device__ __forceinline__ int div_cell(int x, float rcp, int cs)
{   // x / cs for 0 <= x < 65536 without an integer division
    int q = (int)((float)x * rcp);
    if (q * cs > x) q--;
    else if ((q + 1) * cs <= x) q++;
    return q;
}
__host__ __device__ inline size_t nms_smem_bytes(int gw, int gh) { return (size_t)(gw + 2) * (gh + 2) * NMS_CELL_BYTES; }
template <int V>
__device__ __forceinline__ void nms_cells(TrackScalars* sc, const NmsGrid& g, int w, int min_dist, int want, unsigned char* smem_raw, long long* dbg)
{
    const int tid = threadIdx.x, nt = blockDim.x;
    // the grid is padded by one ring of empty cells: the 3x3 neighbourhoods below are nine unconditional loads
    const int gwp = g.gw + 2, ncp = gwp * (g.gh + 2), ncell = g.gw * g.gh;
    unsigned int* head_hi = reinterpret_cast<unsigned int*>(smem_raw);   // [2][ncp] eig bits of the cell's best alive candidate
    unsigned int* head_lo = head_hi + 2 * ncp;                            // [2][ncp] its packed address (y << 16 | x)
    int* acc = reinterpret_cast<int*>(head_lo + 2 * ncp);                 // [2][ncp] corner accepted by the cell in a round, or -1
    uint8_t* flag = reinterpret_cast<uint8_t*>(acc + 2 * ncp);            // [2][ncp] some 3x3 neighbour accepted a corner in that round
    unsigned short* pidx = reinterpret_cast<unsigned short*>(flag + 2 * ncp);   // [ncell] interior cell -> padded index
    const int n = sc->n_cand;
    const int r2 = min_dist * min_dist;
    const float rcp = 1.0f / (float)g.cs;
    unsigned long long alive = 0ull;                            // bit k <-> candidate tid + k*nt
    const int per = (n + nt - 1) / nt;
    for (int k = 0; k < per && k < NMS_MAX_PER_THREAD; k++) if (tid + k * nt < n) alive |= (1ull << k);
    // the first two candidates of a thread stay in registers (covers 2 * blockDim candidates without reloads)
    const unsigned long long key0 = (tid < n) ? __ldg(&g.cand_key[tid]) : 0ull, key1 = (tid + nt < n) ? __ldg(&g.cand_key[tid + nt]) : 0ull;
    auto cell_of = [&](unsigned long long key) {
        return (div_cell((int)((key >> 16) & 0xffffu), rcp, g.cs) + 1) * gwp + div_cell((int)(key & 0xffffu), rcp, g.cs) + 1;
    };
    const int cell0 = cell_of(key0), cell1 = cell_of(key1);
    for (int c = tid; c < 2 * ncp; c += nt) { head_hi[c] = 0u; head_lo[c] = 0u; acc[c] = -1; flag[c] = 0; }
    for (int i = tid; i < ncell; i += nt) { int cy = i / g.gw, cx = i - cy * g.gw; pidx[i] = (unsigned short)((cy + 1) * gwp + cx + 1); }
    __shared__ int s_nacc, s_above;
    __shared__ unsigned long long s_u;
    if (tid == 0) { s_nacc = 0; s_above = 0; s_u = 0ull; }
    int rounds = 0;
    long long tA = 0, tB = 0, tC = 0, tl = gf_clock();
    const long long tstart = tl;
    __syncthreads();
    while (true) {
        const int nacc_prev = s_nacc;                           // corners accepted by the earlier rounds
        const int p = rounds & 1;
        unsigned int* hh = head_hi + p * ncp;
        unsigned int* hl = head_lo + p * ncp;
        const int* acc_prev = acc + p * ncp;                    // written by the previous round as its "next"
        const uint8_t* flag_prev = flag + p * ncp;
        // phase A: kill by last round's accepted corners, bid the eig bits
        auto visit = [&](unsigned long long key, int c) -> bool {     // returns true if the candidate dies this round
            if (rounds > 0 && flag_prev[c]) {
                const int x = (int)(key & 0xffffu), y = (int)((key >> 16) & 0xffffu);
                bool dead = false;
#pragma unroll
                for (int dy = -1; dy <= 1; dy++)
#pragma unroll
                    for (int dx = -1; dx <= 1; dx++) {
                        const int q = acc_prev[c + dy * gwp + dx];
                        const int ex = x - (q & 0xffff), ey = y - (q >> 16);
                        dead |= (q >= 0) && (ex * ex + ey * ey < r2);
                    }
                if (dead) return true;
            }
            atomicMax(&hh[c], (unsigned)(key >> 32));
            return false;
        };
        if ((alive & 1ull) && visit(key0, cell0)) alive &= ~1ull;
        if ((alive & 2ull) && visit(key1, cell1)) alive &= ~2ull;
        {
            unsigned long long a = alive & ~3ull;
            while (a) {
                int k = __ffsll((long long)a) - 1;
                a &= a - 1;
                const unsigned long long key = __ldg(&g.cand_key[tid + k * nt]);
                if (visit(key, cell_of(key))) alive &= ~(1ull << k);
            }
        }
        for (int i = tid + NMS_MAX_PER_THREAD * nt; i < n; i += nt) {   // slow path: liveness in HBM
            if (rounds == 0) g.dead[i] = 0;
            if (!g.dead[i]) { const unsigned long long key = __ldg(&g.cand_key[i]); if (visit(key, cell_of(key))) g.dead[i] = 1; }
        }
        __syncthreads();
        { long long t_ = gf_clock(); tA += t_ - tl; tl = t_; }
        // phase B: among the candidates that carry the cell's best eig bits, the largest address wins
        auto visit2 = [&](unsigned long long key, int c) {
            if (hh[c] == (unsigned)(key >> 32)) atomicMax(&hl[c], (unsigned)(key & 0xffffffffu));
        };
        if (alive & 1ull) visit2(key0, cell0);
        if (alive & 2ull) visit2(key1, cell1);
        {
            unsigned long long a = alive & ~3ull;
            while (a) {
                int k = __ffsll((long long)a) - 1;
                a &= a - 1;
                const unsigned long long key = __ldg(&g.cand_key[tid + k * nt]);
                visit2(key, cell_of(key));
            }
        }
        for (int i = tid + NMS_MAX_PER_THREAD * nt; i < n; i += nt)
            if (!g.dead[i]) { const unsigned long long key = __ldg(&g.cand_key[i]); visit2(key, cell_of(key)); }
        // next round's election arrays and this round's "accepted nearby" flags start clean
        for (int c = tid; c < ncp; c += nt) { head_hi[(p ^ 1) * ncp + c] = 0u; head_lo[(p ^ 1) * ncp + c] = 0u; flag[(p ^ 1) * ncp + c] = 0; }
        __syncthreads();
        { long long t_ = gf_clock(); tB += t_ - tl; tl = t_; }
        // Early exit: every candidate still alive ranks at most U, the best cell head of this round, and so does every corner
        // a later round could accept.  Once `want` corners accepted earlier rank above U, the first `want` corners of the
        // accepted set by rank (the output) are fixed, and the rounds stop.
        if (nacc_prev >= want) {
            unsigned long long u = 0ull;
            for (int i = tid; i < ncell; i += nt) {
                const int c = pidx[i];
                const unsigned long long hk = ((unsigned long long)hh[c] << 32) | hl[c];
                u = hk > u ? hk : u;
            }
            for (int o = 16; o > 0; o >>= 1) { const unsigned long long t_ = __shfl_xor_sync(0xffffffffu, u, o); u = t_ > u ? t_ : u; }
            if ((tid & 31) == 0 && u) atomicMax(&s_u, u);
            __syncthreads();
            const unsigned long long U = s_u;
            int above = 0;
            for (int i = tid; i < min(nacc_prev, g.acc_cap); i += nt) above += g.acc_key[i] > U;
            above = __reduce_add_sync(0xffffffffu, above);
            if ((tid & 31) == 0 && above) atomicAdd(&s_above, above);
            __syncthreads();
            const bool done = s_above >= want;
            __syncthreads();                                    // s_u and s_above are read by everyone before they are reset
            if (tid == 0) { s_u = 0ull; s_above = 0; }
            if (done) break;
        }
        // phase C: a head that outranks its 8 neighbours is accepted
        int any = 0;
        int* acc_next = acc + (p ^ 1) * ncp;
        uint8_t* flag_next = flag + (p ^ 1) * ncp;
        for (int i = tid; i < ncell; i += nt) {
            const int c = pidx[i];
            const unsigned long long hk = ((unsigned long long)hh[c] << 32) | hl[c];
            int out = -1;
            if (hk) {
                any = 1;
                bool top = true;
#pragma unroll
                for (int dy = -1; dy <= 1; dy++)
#pragma unroll
                    for (int dx = -1; dx <= 1; dx++) {
                        const int o = c + dy * gwp + dx;
                        top &= !((((unsigned long long)hh[o] << 32) | hl[o]) > hk);
                    }
                if (top) {
                    out = (int)(hk & 0xffffffffu);          // (y << 16) | x
#pragma unroll
                    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
                        for (int dx = -1; dx <= 1; dx++) flag_next[c + dy * gwp + dx] = 1;
                    int q = atomicAdd(&s_nacc, 1);
                    if (q < g.acc_cap) g.acc_key[q] = hk;
                }
            }
            acc_next[c] = out;
        }
        rounds++;
        const int more = __syncthreads_or(any);
        { long long t_ = gf_clock(); tC += t_ - tl; tl = t_; }
        if (!more) break;
    }
    if (dbg && tid == 0) { dbg[13] = tA; dbg[14] = tB; dbg[15] = tC; dbg[17] = gf_clock() - tstart; }
    if (tid == 0) { sc->n_acc = min(s_nacc, g.acc_cap); sc->nms_rounds = rounds; }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------
struct OutHeader { int n_out, n_prev, n_tracked, n_kept, n_new, n_cand, nms_rounds, eig_fixups, lk_iters, pad; };

// The detections of one frame (trackImagebox, feature_tracker.cpp:374-678), converted on the host: box k is
// b[k] = (lo_x, hi_x, lo_y, hi_y) with the corners as the reference has them, (float)(int)xmin etc.
constexpr int GF_BOX_CAP = 100;      // GF_MAX_BOXES
struct BoxSet { int n; int pad[3]; float4 b[GF_BOX_CAP]; };

// pointPolygonTest(contour {xmin,ymin},{xmin,ymax},{xmax,ymax},{xmax,ymin}, pt, true) > 0 for any box: strictly inside.
// For this axis-aligned contour the signed distance is positive exactly on the open rectangle between the float corners
// (pinned against cv2 by tests/test_box_oracle.py), so the polygon test is four comparisons per box.
__device__ __forceinline__ bool in_any_box(const float4* b, int n, float2 p)
{
    bool in = false;
    for (int k = 0; k < n; k++) in |= (b[k].x < p.x) & (p.x < b[k].y) & (b[k].z < p.y) & (p.y < b[k].w);
    return in;
}

// min-distance rounds, then top-K of the accepted corners, addPoints, undistortedPts, ptsVelocity, depth,
// next-frame state.  Single CTA of 1024 threads; dynamic shared memory for the cell grid (see nms_cells).
template <int V>
__device__ __forceinline__ void select_finalize(TrackScalars* sc, const FeatArrays& fa, const NmsGrid& g, int w, int max_cnt, int min_dist,
                                                const CamParams& cam, const double* dt_ptr, const uint16_t* depth, int dpitch /*elements*/,
                                                int depth_cam_cfg, const int* depth_valid_ptr, int h, OutHeader* out_hdr, gf_obs* out_obs,
                                                uint8_t* out_status /* may be null: copy of the LK status of the n_prev input features */,
                                                const BoxSet* boxes /* the frame's detections, or null */,
                                                uint32_t* out_in_box /* FE_CAP bits: output i lies inside a box; may be null */)
{
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    __shared__ unsigned long long keys[FE_SORT_CAP];
    __shared__ float4 s_box[GF_BOX_CAP];
    const int tid = threadIdx.x;
    const int n_box = boxes ? boxes->n : 0;
    if (tid < n_box) s_box[tid] = boxes->b[tid];            // visible after the barriers of nms_cells
    const long long c0 = gf_clock();
    const int n_kept = sc->n_kept;
    const int want = max(max_cnt - n_kept, 0);
    nms_cells<V>(sc, g, w, min_dist, want, dyn_smem, fa.dbg);
    const long long c1 = gf_clock();
    const double dt = dt_ptr ? *dt_ptr : 1.0;
    const int depth_cam = depth_cam_cfg && depth_valid_ptr && *depth_valid_ptr;
    const int ncand = sc->n_cand;
    const int nacc = sc->n_acc;
    int n_new;
    if (nacc <= (int)blockDim.x) {
        // few accepted corners (the usual case): position = number of larger keys (keys are distinct)
        if (tid < nacc) keys[FE_SORT_CAP / 2 + tid] = g.acc_key[tid];
        __syncthreads();
        if (tid < nacc) {
            const unsigned long long mine = keys[FE_SORT_CAP / 2 + tid];
            int rank = 0;
            for (int j = 0; j < nacc; j++) rank += keys[FE_SORT_CAP / 2 + j] > mine;
            keys[rank] = mine;
        }
        __syncthreads();
        n_new = min(want, nacc);
    } else if (nacc <= FE_SORT_CAP) {
        int np2 = 1;
        while (np2 < nacc) np2 <<= 1;
        for (int i = tid; i < np2; i += blockDim.x) keys[i] = (i < nacc) ? g.acc_key[i] : 0ull;
        __syncthreads();
        for (int k = 2; k <= np2; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = tid; i < np2; i += blockDim.x) {
                    int ixj = i ^ j;
                    if (ixj > i) {
                        unsigned long long a = keys[i], b = keys[ixj];
                        bool desc = ((i & k) == 0);
                        if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
                    }
                }
                __syncthreads();
            }
        n_new = min(want, nacc);
    } else {
        // more accepted corners than the shared sort buffer (tiny min_dist): K selection passes over HBM
        __shared__ unsigned long long s_best[32];
        __shared__ unsigned long long s_prev;
        n_new = min(min(want, nacc), FE_SORT_CAP);
        if (tid == 0) s_prev = ~0ull;
        __syncthreads();
        for (int k = 0; k < n_new; k++) {
            unsigned long long lim = s_prev, best = 0ull;
            for (int i = tid; i < nacc; i += blockDim.x) { unsigned long long kk = g.acc_key[i]; if (kk < lim && kk > best) best = kk; }
            for (int o = 16; o > 0; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o); if (t > best) best = t; }
            if ((tid & 31) == 0) s_best[tid >> 5] = best;
            __syncthreads();
            if (tid == 0) { for (int i = 1; i < 32; i++) if (s_best[i] > best) best = s_best[i]; keys[k] = best; s_prev = best; }
            __syncthreads();
        }
    }
    const long long c2 = gf_clock();
    const int total = n_kept + n_new;
    const int n_id = sc->n_id;
    // addPoints + per-feature outputs; thread i <-> feature i of the new cur_pts order (kept..., new...)
    bool boxed = false;
    if (tid < total) {
        float2 p, un_prev = make_float2(0.f, 0.f);
        int id, cnt;
        bool has_prev = false;
        if (tid < n_kept) {
            p = fa.kept_pts[tid]; id = fa.kept_ids[tid]; cnt = fa.kept_cnt[tid]; un_prev = fa.kept_un[tid]; has_prev = true;
        } else {
            const unsigned addr = (unsigned)(keys[tid - n_kept] & 0xffffffffu);
            p = make_float2((float)(addr & 0xffffu), (float)(addr >> 16)); id = n_id + (tid - n_kept); cnt = 1;
        }
        double ux, uy;
        cam_lift(cam, (double)p.x, (double)p.y, ux, uy);
        float2 un = make_float2((float)(ux / 1.0), (float)(uy / 1.0));
        float2 vel = make_float2(0.f, 0.f);
        if (has_prev) {
            double vx = (double)(un.x - un_prev.x) / dt, vy = (double)(un.y - un_prev.y) / dt;
            vel = make_float2((float)vx, (float)vy);
        }
        double dval = -2.4;
        if (depth_cam) {
            int r = (int)round((double)p.y), c = (int)round((double)p.x);
            r = min(max(r, 0), h - 1); c = min(max(c, 0), w - 1);   // always in range after inBorder; belt and braces
            dval = (double)(int)depth[(size_t)r * dpitch + c] / 1000.0;
        }
        gf_obs o;
        o.id = id; o.track_cnt = cnt;
        o.v[0] = (double)un.x; o.v[1] = (double)un.y; o.v[2] = 1.0; o.v[3] = (double)p.x; o.v[4] = (double)p.y;
        o.v[5] = (double)vel.x; o.v[6] = (double)vel.y; o.v[7] = dval;
        out_obs[tid] = o;
        // state for the next frame (prev_pts = cur_pts; prev_un_pts_map = cur_un_pts_map)
        fa.prev_pts[tid] = p; fa.ids[tid] = id; fa.track_cnt[tid] = cnt; fa.prev_un[tid] = un;
        boxed = in_any_box(s_box, n_box, p);
    }
    if (out_in_box) {       // a boxed feature stays in the state above; only featureFrame leaves it out
        const unsigned bits = __ballot_sync(0xffffffffu, boxed);
        if ((tid & 31) == 0) out_in_box[tid >> 5] = bits;
    }
    if (out_status && tid < sc->n_prev) out_status[tid] = fa.status[tid];
    __syncthreads();
    if (tid == 0) {
        out_hdr->n_out = total; out_hdr->n_prev = sc->n_prev; out_hdr->n_tracked = sc->n_tracked;
        out_hdr->n_kept = n_kept; out_hdr->n_new = n_new; out_hdr->n_cand = ncand;
        out_hdr->nms_rounds = sc->nms_rounds; out_hdr->eig_fixups = sc->eig_fixups; out_hdr->lk_iters = sc->lk_iters; sc->lk_iters = 0;
        sc->n_new = n_new; sc->n_out = total;
        sc->n_prev = total; sc->n_id = n_id + n_new; sc->eig_fixups = 0;
    }
    GF_DBG(8, c1 - c0); GF_DBG(9, c2 - c1); GF_DBG(10, gf_clock() - c2); GF_DBG(11, nacc); GF_DBG(12, ncand);
}
__global__ void __launch_bounds__(1024) k_select_finalize(TrackScalars* sc, FeatArrays fa, NmsGrid g, int w, int max_cnt, int min_dist,
                                                          CamParams cam, const double* dt_ptr, const uint16_t* depth, int dpitch /*elements*/,
                                                          int depth_cam_cfg, const int* depth_valid_ptr, int h, OutHeader* out_hdr, gf_obs* out_obs,
                                                          uint8_t* out_status, const BoxSet* boxes = nullptr, uint32_t* out_in_box = nullptr)
{
    select_finalize<0>(sc, fa, g, w, max_cnt, min_dist, cam, dt_ptr, depth, dpitch, depth_cam_cfg, depth_valid_ptr, h, out_hdr, out_obs, out_status,
                    boxes, out_in_box);
}

}  // namespace gf
