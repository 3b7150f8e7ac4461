// fe_lk.cuh -- pyramidal Lucas-Kanade, one CTA of 8 warps per point, bit-exact with OpenCV 4.13's SSE path.
//
// Replaces the two cv::calcOpticalFlowPyrLK calls of FeatureTracker::trackImage
// (reference vins_estimator/src/featureTracker/feature_tracker.cpp:118-153).  The arithmetic follows
// oracle/fe_cv_restate.c (pinned bit-for-bit against cv2 4.13.0): fixed-point bilinear windows
// (W_BITS=14), Scharr derivatives computed on the fly from the staged u8 window (no derivative image
// ever touches HBM), float32 sums accumulated in OpenCV's SIMD lane order:
//   A11/A12/A22: 4 lane chains over columns 0..15 (lane l <- columns l, l+4, l+8, l+12, row-major)
//                + 1 scalar tail chain over columns 16..20, result = tail + ((l0+l2)+(l1+l3))
//   b1/b2:       4 chains of pmaddwd pairs (col k, col k+4 | k+8, k+12) + 1 tail chain,
//                result = tail + ((c0+c2) + (c1+c3))
// The order of the float additions is what makes the result bit-exact, and it is inherently sequential.
// Everything around it is organised to keep those chains short in instructions: the parallel phase (all 256 threads)
// produces the *terms* (exact integers converted to float, pair sums for the pmaddwd chains) already laid
// out in chain order in shared memory, so that the chain phase is one predicated LDS+FADD loop of 105 steps
// run by 15 (A) or 10 (b) lanes.  Compile with -fmad=false: every float op must round on its own.
//
// The b chains have an exact shortcut.  Every b term is an integer; when the positive terms of a chain sum to less
// than 2^24 and so do the magnitudes of its negative terms, every prefix sum in any order is an integer below 2^24,
// so each float add of the chain is exact and the chain's result is (float) of its integer sum.  The term phase
// therefore also reduces, per warp and chain, the positive and negative parts as integers (lk_bpart_write); after one
// barrier every warp sums the per-warp partials itself (lk_bsum_int).  When all ten chains are within the bound (99.5 %
// of the iterations of the C2 synthetic stream) that sum replaces the sequential chains.  Otherwise the threads store
// their terms in chain order and warp 0 runs lk_chain on them.
//
// The CTA has two warp roles (lk_track_point).  Consumer warps 0..3 run the iterations of level l; producer warps 4..7
// meanwhile build level l-1 -- Scharr, the template, the gradient-matrix terms and chains, minEig and D -- into the other
// of two level buffers.  A level's setup depends only on the point p and the staged template window, so only the
// coarsest level of a pass waits for its setup.  Each role synchronises on its own named barrier; the roles meet once
// per level at a 256-thread named barrier, whatever path the level took.  The producers also fetch each level's first
// search window, placed from the pass's initial guess, so a level restages only when its iterate leaves that window.
// fe_lk_single.cuh keeps the single-role form (all 8 warps set up a level, then iterate it), which fe_tracker.cu launches
// while several trackers share the GPU.
#pragma once
#include <cuda.h>          // CUtensorMap (types only: the encoder is fetched with cudaGetDriverEntryPoint, fe_tracker.cu)
#include "gf_common.cuh"
#include "fe_eig.cuh"      // smem_u32, mbar_* helpers

namespace gf {

constexpr int LK_WIN = 21;
constexpr int LK_NPIX = LK_WIN * LK_WIN;  // 441
constexpr int LK_IREG = 24;               // staged I window incl. Scharr apron + bilinear +1
constexpr int LK_IPITCH = 48;             // bytes per staged I row (24 + up to 15 bytes of alignment slack: TMA boxes start 16-byte aligned)
constexpr int LK_SCH = 22;                // integer positions needing a derivative
constexpr int LK_JR = 40;                 // cached J region (window 22 + 9 px drift each side)
constexpr int LK_JPITCH = 80;             // bytes per staged J row (40 + up to 15 bytes of alignment slack; 80 keeps four rows on distinct banks)
constexpr int LK_THREADS = 256;            // one CTA of 8 warps per feature (two warps per SM scheduler), ~one feature per SM
constexpr int LK_MAXLEV = 4;               // pyramid levels 0..3
constexpr int LK_CHAIN = 84, LK_TAIL = 105;        // terms per SIMD-lane chain / tail chain of the A sums
constexpr int LK_BCHAIN = 42;                       // pair terms per chain of the b sums
constexpr int LK_AT = 4 * LK_CHAIN + LK_TAIL;       // 441 terms per A quantity
constexpr int LK_BT = 4 * LK_BCHAIN + LK_TAIL;      // 273 terms per b component (168 pair units + 105 tail pixels)
constexpr int LK_Q = 5 * LK_TAIL;                   // slots per quantity: [step 0..104][chain 0..4], short chains padded with +0.0f
// Warp roles: consumer warps 0..LK_CWARPS-1 iterate, the others (producers) build the next level.
constexpr int LK_CWARPS = 4;
constexpr int LK_CTHREADS = 32 * LK_CWARPS;                 // 128
constexpr int LK_PTHREADS = LK_THREADS - LK_CTHREADS;       // 128
// Units of the b terms per consumer thread t (lk_iterate): pair unit t, and pair unit t + 128 (t < 40) or tail unit t - 40
// (t >= 40), plus tail unit t + 48 for 40 <= t < 57 -- at most four pixels per thread.  Pair units u and u + 128 belong to
// the same chain (u & 3), so every thread holds one pair chain and the tail chain.
constexpr int LK_PAIR2 = 4 * LK_BCHAIN - LK_CTHREADS;       // 40 threads hold a second pair unit
constexpr int LK_TAIL2 = LK_TAIL - (LK_CTHREADS - LK_PAIR2); // 17 threads hold a second tail unit
static_assert(LK_CTHREADS == 128 && LK_PAIR2 > 0 && LK_TAIL2 > 0 && LK_PAIR2 + LK_TAIL2 <= LK_CTHREADS, "unit map of lk_iterate");
constexpr int LK_BSLOTS = 5 * LK_CWARPS;    // per-warp partials: slot w*4 + k pair chain k of warp w, slot 4*LK_CWARPS + w its tail
// named barriers (0 is __syncthreads)
constexpr int LK_BAR_HANDOFF = 1, LK_BAR_CONS = 2, LK_BAR_PROD = 3;

// One built level: the gradient matrix, scaled, and whether the level is tracked at all (inside the image, minEig and
// the determinant above OpenCV's thresholds).
struct LKLevelA { float A11, A12, A22, D; int ok, pad_[3]; };

struct __align__(128) LKSmem {
    uint8_t ireg[LK_MAXLEV][LK_IREG * LK_IPITCH];   // per level: raw bytes, row r at r*32, first needed column at byte xoff
    uint8_t jreg[2][LK_JR * LK_JPITCH];             // search window of level l in [l & 1]; 128-byte aligned like ireg[l]: TMA box destinations
    int16_t sch[LK_SCH * LK_SCH * 2];               // producers only
    short4 tpl[2][LK_NPIX + 1];            // per level buffer: template patch per pixel (I*32, Ix, Iy, 0), one 8-byte load
    float aterms[3 * LK_Q];                // A terms [quantity][step][chain] (producers); slots beyond a chain's length hold +0.0f
    float bterms[2 * LK_Q];                // b terms of the sequential fallback (consumers), same layout
    LKLevelA lv[2];                        // per level buffer: the built gradient matrix
    float bsums[2];                        // fallback b chain results broadcast from warp 0
    float2 res;                            // result of the pass, broadcast from consumer thread 0
    int res_status;
    // [iteration parity][slot][x+, x-, y+, y-]: per-warp sums of the positive b terms and of the magnitudes of the negative
    // ones of one chain (slots as LK_BSLOTS)
    alignas(16) unsigned bpart[2][LK_BSLOTS][4];
    unsigned long long mbar_i;             // completion barrier of the template window loads (all threads wait)
    unsigned long long mbar_p[2];          // completion barriers of the producers' first search window of level l, [l & 1]
                                           // (consumers wait; level l+2 reuses a barrier only after level l's wait)
    unsigned long long mbar_j;             // completion barrier of the search windows restaged within a level (consumers wait)
};
static_assert((LK_IREG * LK_IPITCH) % 128 == 0 && (LK_MAXLEV * LK_IREG * LK_IPITCH) % 128 == 0 && (LK_JR * LK_JPITCH) % 128 == 0,
              "TMA destinations must be 128-byte aligned");

// ---- 2-D TMA staging of the LK windows --------------------------------------------------------------------------------
// A window that lies inside its pyramid level is one cp.async.bulk.tensor.2d box: LK_IPITCH x LK_IREG bytes for a template
// window, LK_JPITCH x LK_JR for a search region (the box is as wide as the staged row pitch, so the box IS the staging
// layout).  The innermost box coordinate is kept on a 16-byte boundary (an unaligned x has been seen to raise "illegal
// instruction" at the UTMALDG), so the box starts at x0 & ~15 and the first needed column sits at byte x0 & 15 of every
// staged row.  Tensor maps: u8, rank 2, {w, h}, row stride = level pitch, no swizzle;
// columns beyond the image width are zero-filled and never read.  Windows that touch the border keep the REFLECT_101 gathers.
struct LKMapSet {
    CUtensorMap prevI[LK_MAXLEV], curJ[LK_MAXLEV];   // forward pass: templates from the previous pyramid, search in the current one
    CUtensorMap curI[LK_MAXLEV], prevJ[LK_MAXLEV];   // reverse pass
    int enabled, pad_[15];
};
// phase_i: the template windows' barrier (every thread waits on it); phase_p (bit b: S.mbar_p[b]), phase_j: the search
// windows' barriers (only consumers wait, so only their copies advance)
struct LKTma { const CUtensorMap* mi; const CUtensorMap* mj; unsigned phase_i, phase_p, phase_j; bool on; };

__device__ __forceinline__ void lk_tma_box(void* dst, const CUtensorMap* map, int x, int y, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(x), "r"(y), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void lk_tma_wait(unsigned long long* bar, unsigned& phase)
{
    while (!mbar_try_wait(bar, phase)) { }
    phase ^= 1u;
}
// once per kernel, before the first lk_track_point.  Also zeroes the chain padding, which must read +0.0f: no pass writes a
// padding slot, and every pass rewrites each real slot before the chains read it.
__device__ __forceinline__ void lk_tma_init(LKSmem& S, int tid)
{
    for (int i = tid; i < 3 * LK_Q; i += LK_THREADS) S.aterms[i] = 0.f;
    for (int i = tid; i < 2 * LK_Q; i += LK_THREADS) S.bterms[i] = 0.f;
    if (tid == 0) {
        mbar_init(&S.mbar_i, 1);
        mbar_init(&S.mbar_p[0], 1);
        mbar_init(&S.mbar_p[1], 1);
        mbar_init(&S.mbar_j, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}
__device__ __forceinline__ void lk_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
template <int RW, int RH>
__device__ __forceinline__ bool lk_inside(const Level& L, int x0, int y0)
{
    return x0 >= 0 && y0 >= 0 && x0 + RW <= L.w && y0 + RH <= L.h;
}

__device__ __forceinline__ int lk_descale(int v, int n) { return (v + (1 << (n - 1))) >> n; }

__device__ __forceinline__ void lk_weights(float a, float b, int& w00, int& w01, int& w10, int& w11)
{
    w00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
    w01 = __float2int_rn(a * (1.f - b) * 16384.f);
    w10 = __float2int_rn((1.f - a) * b * 16384.f);
    w11 = 16384 - w00 - w01 - w10;
}

// Stages the RW x RH window of img whose top-left pixel is (x0, y0) into dst (row pitch DP bytes).
// Inside the image: aligned 32-bit loads, the first needed column sits at byte offset (x0 & 3), returned.
// Touching the border: REFLECT_101 byte gathers, offset 0.
template <int RW, int RH, int DP>
__device__ __forceinline__ int lk_stage(uint8_t* dst, const Level& L, int x0, int y0, int tid)
{
    if (x0 >= 0 && y0 >= 0 && x0 + RW <= L.w && y0 + RH <= L.h) {
        const int xa = x0 & ~3, xoff = x0 - xa;
        constexpr int WPR = DP / 4;                      // words per staged row
        const int need = (xoff + RW + 3) >> 2;           // words actually needed per row
        uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
        for (int i = tid; i < RH * WPR; i += LK_THREADS) {
            int r = i / WPR, c = i - r * WPR;
            if (c < need) d32[i] = __ldg(reinterpret_cast<const uint32_t*>(L.ptr + (size_t)(y0 + r) * L.pitch + xa) + c);
        }
        return xoff;
    }
    for (int i = tid; i < RW * RH; i += LK_THREADS) {
        int r = i / RW, c = i - r * RW;
        int yy = reflect101(y0 + r, L.h), xx = reflect101(x0 + c, L.w);
        dst[r * DP + c] = __ldg(L.ptr + (size_t)yy * L.pitch + xx);
    }
    return 0;
}

// Same staging executed by a subset of the CTA (thread index t of nt), and the byte offset lk_stage would return.
template <int RW, int RH, int DP>
__device__ __forceinline__ int lk_stage_part(uint8_t* dst, const Level& L, int x0, int y0, int t, int nt)
{
    if (x0 >= 0 && y0 >= 0 && x0 + RW <= L.w && y0 + RH <= L.h) {
        const int xa = x0 & ~3, xoff = x0 - xa;
        constexpr int WPR = DP / 4;
        const int need = (xoff + RW + 3) >> 2;
        uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
        for (int i = t; i < RH * WPR; i += nt) {
            int r = i / WPR, c = i - r * WPR;
            if (c < need) d32[i] = __ldg(reinterpret_cast<const uint32_t*>(L.ptr + (size_t)(y0 + r) * L.pitch + xa) + c);
        }
        return xoff;
    }
    for (int i = t; i < RW * RH; i += nt) {
        int r = i / RW, c = i - r * RW;
        int yy = reflect101(y0 + r, L.h), xx = reflect101(x0 + c, L.w);
        dst[r * DP + c] = __ldg(L.ptr + (size_t)yy * L.pitch + xx);
    }
    return 0;
}
template <int RW, int RH>
__device__ __forceinline__ int lk_stage_offset(const Level& L, int x0, int y0, bool tma = false)
{
    return (x0 >= 0 && y0 >= 0 && x0 + RW <= L.w && y0 + RH <= L.h) ? (tma ? (x0 & 15) : (x0 & 3)) : 0;
}

// One sequential float chain per lane: lane (q*5 + c) of the first nq*5 lanes adds the 105 slots of chain c of
// quantity q in order.  Chains shorter than 105 are padded with +0.0f, so the loop is a bare LDS + FADD.
__device__ __forceinline__ float lk_chain(const float* T, int lane, int nq)
{
    float acc = 0.f;
    if (lane < nq * 5) {
        const int q = lane / 5, c = lane - q * 5;
        const float* p = T + q * LK_Q + c;
#pragma unroll
        for (int s = 0; s < LK_TAIL; s++) acc += p[5 * s];
    }
    return acc;
}

// b1 and b2 from the chain results held in lanes comp*5 + c (the layout of lk_chain), OpenCV's final combination
__device__ __forceinline__ void lk_bcombine(float acc, float& b1, float& b2)
{
    float s[2];
#pragma unroll
    for (int comp = 0; comp < 2; comp++) {
        float c0 = __shfl_sync(0xffffffffu, acc, comp * 5 + 0), c1 = __shfl_sync(0xffffffffu, acc, comp * 5 + 1);
        float c2 = __shfl_sync(0xffffffffu, acc, comp * 5 + 2), c3 = __shfl_sync(0xffffffffu, acc, comp * 5 + 3);
        float t = __shfl_sync(0xffffffffu, acc, comp * 5 + 4);
        float x02 = c0 + c2, x13 = c1 + c3;
        s[comp] = t + ((x02 + 0.f) + (x13 + 0.f));
    }
    b1 = s[0];
    b2 = s[1];
}

__device__ __forceinline__ void lk_split(int v, unsigned& pos, unsigned& neg)
{
    pos += v > 0 ? (unsigned)v : 0u;
    neg += v < 0 ? (unsigned)-v : 0u;
}

// Per-warp integer partials of the b chains from a consumer thread's shares (x+, x-, y+, y-) of its pair chain (v, chain
// lane & 3) and of the tail chain (tv).  No sum can wrap: a term is below 2^26 in magnitude (|d| <= 8160, |g| <= 4080,
// two products per pair), and a whole chain (42 pair terms or 105 tail products) stays below 2^32.
__device__ __forceinline__ void lk_bpart_write(unsigned (*P)[4], int tid, const unsigned (&v)[4], const unsigned (&tv)[4])
{
    const int w = tid >> 5, lane = tid & 31;
    // Reduce-scatter over the 8 lanes of each pair chain (equal lane & 3), four shuffles, three deep: across lane bit 4
    // a lane keeps values {0,1} or {2,3}, across bit 3 one of them, across bit 2 it completes value (lane >> 3) & 3.
    const bool h4 = lane & 16, h3 = lane & 8;
    unsigned a0 = h4 ? v[2] : v[0], a1 = h4 ? v[3] : v[1];
    const unsigned s0 = h4 ? v[0] : v[2], s1 = h4 ? v[1] : v[3];
    a0 += __shfl_xor_sync(0xffffffffu, s0, 16);
    a1 += __shfl_xor_sync(0xffffffffu, s1, 16);
    unsigned c = (h3 ? a1 : a0) + __shfl_xor_sync(0xffffffffu, h3 ? a0 : a1, 8);
    c += __shfl_xor_sync(0xffffffffu, c, 4);
    if (!(lane & 4)) P[w * 4 + (lane & 3)][(lane >> 3) & 3] = c;
    unsigned s[4];
#pragma unroll
    for (int k = 0; k < 4; k++) s[k] = __reduce_add_sync(0xffffffffu, tv[k]);
    if (lane == 0) *reinterpret_cast<uint4*>(P[4 * LK_CWARPS + w]) = make_uint4(s[0], s[1], s[2], s[3]);
}

// b1 and b2 from the per-warp integer partials, computed by every consumer warp, when all ten chains are within the exactness
// bound; returns whether they are (the same answer in every warp).  Lane comp*8 + c (c < 5) sums chain c of component comp.
// OpenCV's combination t + ((c0 + c2) + (c1 + c3)) then pairs c0/c2 and c1/c3 across lane bit 1 and the two pair sums
// across lane bit 0; float addition is commutative, so the bits do not depend on which lane of a pair adds.
__device__ __forceinline__ bool lk_bsum_int(const unsigned (*P)[4], int lane, float& b1, float& b2)
{
    const int comp = lane >> 3, c = lane & 7;
    bool ok = true;
    float acc = 0.f;
    if (comp < 2 && c < 5) {
        unsigned pos = 0, neg = 0;
#pragma unroll
        for (int w = 0; w < LK_CWARPS; w++) {
            const uint2 v = reinterpret_cast<const uint2*>(P[c < 4 ? w * 4 + c : 4 * LK_CWARPS + w])[comp];
            pos += v.x;
            neg += v.y;
        }
        ok = pos < (1u << 24) && neg < (1u << 24);
        acc = (float)(int)(pos - neg);
    }
    if (!__all_sync(0xffffffffu, ok)) return false;
    const float t = __shfl_xor_sync(0xffffffffu, acc, 4);                 // lane comp*8: the tail chain
    const float x = acc + __shfl_xor_sync(0xffffffffu, acc, 2);           // lanes comp*8 + 0, 1: c0 + c2, c1 + c3
    const float s = t + ((x + 0.f) + (__shfl_xor_sync(0xffffffffu, x, 1) + 0.f));
    b1 = __shfl_sync(0xffffffffu, s, 0);
    b2 = __shfl_sync(0xffffffffu, s, 8);
    return true;
}

// One pyramid level for one point.  All LK_THREADS threads of the CTA call this with identical scalar arguments
// and keep identical copies of the scalar state; warp 0 owns the sequential chains.
#ifdef GF_PROFILE
#define LKP(i) do { long long t_ = gf_clock(); pc[i] += t_ - tl; tl = t_; } while (0)
#else
#define LKP(i) do { } while (0)
#endif

// Window origin of a point on one level (OpenCV: prevPt = prevPts[i] * (1/(1<<level)) - halfWin, then floor)
__device__ __forceinline__ void lk_origin(float2 p, int l, float& ppx, float& ppy, int& ipx, int& ipy)
{
    const float sc = (float)(1. / (double)(1 << l));
    ppx = p.x * sc - 10.f;
    ppy = p.y * sc - 10.f;
    ipx = __float2int_rd(ppx);
    ipy = __float2int_rd(ppy);
}

// Search window a level starts with when the pass's initial guess g needs no correction from the coarser levels: origin
// floor(g / 2^l - 10) - 9, as lk_iterate places it; false when that guess is out of range (the level's first iteration
// then ends the level).  The producers stage these windows (lk_build).  A window only caches the image, so a
// level whose iterate leaves it restages, and a better or worse guess changes no result.
__device__ __forceinline__ bool lk_jwin0(float2 g, int l, const Level& J, int& jx0, int& jy0)
{
    const float sc = (float)(1. / (double)(1 << l));
    const int iqx = __float2int_rd(g.x * sc - 10.f), iqy = __float2int_rd(g.y * sc - 10.f);
    jx0 = iqx - 9;
    jy0 = iqy - 9;
    return !(iqx < -LK_WIN || iqx >= J.w || iqy < -LK_WIN || iqy >= J.h);
}

// Producer role: builds one pyramid level of point p into level buffer buf -- the template patch S.tpl[buf] and the
// gradient matrix S.lv[buf] -- from the staged window S.ireg[level], and fetches the level's first search window
// (from the pass's initial guess g) into S.jreg[level & 1].  Run by the LK_PTHREADS producer threads (pt is the
// index among them) with identical arguments; warp 0 of the role runs the A chains.  The role's barriers are all
// skipped together when the level lies outside the image.
__device__ __forceinline__ void lk_build(LKSmem& S, int pt, const Level& I, const Level& J, float2 p, float2 g, int level,
                                         int buf, const LKTma& T)
{
    const bool tma_on = T.on;
    // ---- the level's first search window (lk_jwin0) into S.jreg[level & 1], whose last readers (the consumers of level
    //      level+2) passed the hand-over before this build.  A box completes on S.mbar_p[level & 1], which the consumers
    //      wait on; gathered bytes are published by the next hand-over ----
    {
        int jx0, jy0;
        if (lk_jwin0(g, level, J, jx0, jy0)) {
            if (tma_on && lk_inside<LK_JR, LK_JR>(J, jx0, jy0)) {
                if (pt == 0) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    mbar_expect_tx(&S.mbar_p[level & 1], LK_JR * LK_JPITCH);
                    lk_tma_box(S.jreg[level & 1], T.mj + level, jx0 & ~15, jy0, &S.mbar_p[level & 1]);
                }
            } else {
                lk_stage_part<LK_JR, LK_JR, LK_JPITCH>(S.jreg[level & 1], J, jx0, jy0, pt, LK_PTHREADS);
            }
        }
    }
    float ppx, ppy;
    int ipx, ipy;
    lk_origin(p, level, ppx, ppy, ipx, ipy);
    LKLevelA& R = S.lv[buf];
    if (ipx < -LK_WIN || ipx >= I.w || ipy < -LK_WIN || ipy >= I.h) {
        if (pt == 0) R.ok = 0;
        return;
    }
    const float a = ppx - (float)ipx, b = ppy - (float)ipy;
    int iw00, iw01, iw10, iw11;
    lk_weights(a, b, iw00, iw01, iw10, iw11);
    const uint8_t* ireg = S.ireg[level];
    const int ioff = lk_stage_offset<LK_IREG, LK_IREG>(I, ipx - 1, ipy - 1, tma_on);
    // ---- Scharr derivative at the 22x22 integer positions (0 outside the image).  The previous build's readers of
    //      S.sch passed its second role barrier before this build began ----
    for (int i = pt; i < LK_SCH * LK_SCH; i += LK_PTHREADS) {
        int r = i / LK_SCH, c = i - r * LK_SCH;
        int X = ipx + c, Y = ipy + r;
        int ix = 0, iy = 0;
        if (X >= 0 && X < I.w && Y >= 0 && Y < I.h) {
            const uint8_t* u = ireg + r * LK_IPITCH + ioff + c;  // row above, column left of the centre
            const uint8_t* m = u + LK_IPITCH;
            const uint8_t* d = m + LK_IPITCH;
            int t0l = (u[0] + d[0]) * 3 + m[0] * 10, t0r = (u[2] + d[2]) * 3 + m[2] * 10;
            int t1l = d[0] - u[0], t1c = d[1] - u[1], t1r = d[2] - u[2];
            ix = t0r - t0l;
            iy = (t1r + t1l) * 3 + t1c * 10;
        }
        reinterpret_cast<int*>(S.sch)[i] = (ix & 0xffff) | (iy << 16);
    }
    lk_bar(LK_BAR_PROD, LK_PTHREADS);
    // ---- bilinear 21x21 patches I*32, (Ix, Iy), and the gradient-matrix terms in chain order.  The previous build's
    //      A chains finished before warp 0 of the role reached the barrier above ----
    short4* tpl = S.tpl[buf];
    for (int i = pt; i < LK_NPIX; i += LK_PTHREADS) {
        int y = i / LK_WIN, x = i - y * LK_WIN;
        const uint8_t* q = ireg + (y + 1) * LK_IPITCH + ioff + (x + 1);
        int iv = q[0] * iw00 + q[1] * iw01 + q[LK_IPITCH] * iw10 + q[LK_IPITCH + 1] * iw11;
        const int pv = lk_descale(iv, 9);
        const int16_t* s = S.sch + 2 * (y * LK_SCH + x);
        int dxv = s[0] * iw00 + s[2] * iw01 + s[2 * LK_SCH] * iw10 + s[2 * LK_SCH + 2] * iw11;
        int dyv = s[1] * iw00 + s[3] * iw01 + s[2 * LK_SCH + 1] * iw10 + s[2 * LK_SCH + 3] * iw11;
        int gx = (int16_t)lk_descale(dxv, 14), gy = (int16_t)lk_descale(dyv, 14);
        tpl[i] = make_short4((short)pv, (short)gx, (short)gy, 0);
        // products are exact integers below 2^24, so (float)(int product) == fx*fy of OpenCV's float path
        int slot = (x < 16) ? (y * 4 + (x >> 2)) * 5 + (x & 3) : (y * 5 + (x - 16)) * 5 + 4;     // [step][chain]
        S.aterms[slot] = (float)(gx * gx);
        S.aterms[LK_Q + slot] = (float)(gx * gy);
        S.aterms[2 * LK_Q + slot] = (float)(gy * gy);
    }
    lk_bar(LK_BAR_PROD, LK_PTHREADS);
    // ---- gradient matrix, OpenCV lane order, minEig and the determinant ----
    if (pt < 32) {
        const float acc = lk_chain(S.aterms, pt, 3);
        float sum[3];
#pragma unroll
        for (int q = 0; q < 3; q++) {
            float l0 = __shfl_sync(0xffffffffu, acc, q * 5 + 0), l1 = __shfl_sync(0xffffffffu, acc, q * 5 + 1);
            float l2 = __shfl_sync(0xffffffffu, acc, q * 5 + 2), l3 = __shfl_sync(0xffffffffu, acc, q * 5 + 3);
            float t = __shfl_sync(0xffffffffu, acc, q * 5 + 4);
            sum[q] = t + ((l0 + l2) + (l1 + l3));
        }
        if (pt == 0) {
            const float FLT_SCALE = 1.f / (1 << 20);
            const float A11 = sum[0] * FLT_SCALE, A12 = sum[1] * FLT_SCALE, A22 = sum[2] * FLT_SCALE;
            const float D = A11 * A22 - A12 * A12;
            const float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / 882.f;
            R.A11 = A11;
            R.A12 = A12;
            R.A22 = A22;
            R.ok = !(minEig < 1e-4f || D < 1.1920928955078125e-07f);
            R.D = 1.f / D;
        }
    }
}

// Consumer role: the LK iterations of one pyramid level for one point, on the level built into buffer buf.  Run by the
// LK_CTHREADS consumer threads (tid < LK_CTHREADS) with identical scalar arguments; each keeps identical copies of the
// scalar state.  Warp 0 runs the sequential b chains of the fallback.
__device__ __forceinline__ void lk_iterate(LKSmem& S, int tid, const Level& J, float2 g, float& nx, float& ny, int level,
                                           int buf, int& status, int& iters, int& fallbacks, long long* pc, LKTma& T)
{
    [[maybe_unused]] long long tl = gf_clock();
    const float FLT_SCALE = 1.f / (1 << 20);
    uint8_t* jreg = S.jreg[level & 1];
    int jx0, jy0;
    bool jvalid = lk_jwin0(g, level, J, jx0, jy0);     // the window the producers staged for this level
    int joff = jvalid ? lk_stage_offset<LK_JR, LK_JR>(J, jx0, jy0, T.on) : 0;
    if (jvalid && T.on && lk_inside<LK_JR, LK_JR>(J, jx0, jy0)) {     // on every path: the barrier's next use needs it
        while (!mbar_try_wait(&S.mbar_p[level & 1], (T.phase_p >> (level & 1)) & 1u)) { }
        T.phase_p ^= 1u << (level & 1);
    }
    const LKLevelA R = S.lv[buf];
    if (!R.ok) {                 // outside the image, or minEig / determinant below the thresholds
        if (level == 0) status = 0;
        return;
    }
    const short4* tpl = S.tpl[buf];
    // this thread's pixels (the unit map above LK_BSLOTS): pair unit tid at template index p0 and p0 + 4, then either the
    // second pair unit (p0 + 336, p0 + 340) or tail unit tid - 40 at e0, and for 17 threads tail unit tid + 48 at e1
    const bool pair2 = tid < LK_PAIR2, tail2 = !pair2 && tid < LK_PAIR2 + LK_TAIL2;
    const int p0 = (tid >> 3) * LK_WIN + 8 * ((tid & 7) >> 2) + (tid & 3);
    const int po = (tid >> 3) * LK_JPITCH + 8 * ((tid & 7) >> 2) + (tid & 3);
    const int pslot = ((tid >> 3) * 2 + ((tid & 7) >> 2)) * 5 + (tid & 3);
    const int v0 = tid - LK_PAIR2, v1 = tid + (LK_TAIL - LK_TAIL2 - LK_PAIR2);     // tail unit indices (used when valid)
    const int e0 = (v0 / 5) * LK_WIN + 16 + v0 % 5, e1 = (v1 / 5) * LK_WIN + 16 + v1 % 5;
    const int eo0 = (v0 / 5) * LK_JPITCH + 16 + v0 % 5, eo1 = (v1 / 5) * LK_JPITCH + 16 + v1 % 5;
    constexpr int P2I = 16 * LK_WIN, P2O = 16 * LK_JPITCH, P2S = 16 * 2 * 5;        // unit + 128: 16 template rows down

    float A11 = R.A11, A12 = R.A12, A22 = R.A22, D = R.D;
    float qx = nx - 10.f, qy = ny - 10.f;
    float pdx_ = 0.f, pdy_ = 0.f;
    LKP(3);
    for (int j = 0; j < 30; j++) {
        int iqx = __float2int_rd(qx), iqy = __float2int_rd(qy);
        if (iqx < -LK_WIN || iqx >= J.w || iqy < -LK_WIN || iqy >= J.h) {
            if (level == 0) status = 0;
            break;
        }
        if (!(jvalid && iqx >= jx0 && iqy >= jy0 && iqx + 22 <= jx0 + LK_JR && iqy + 22 <= jy0 + LK_JR)) {
            jx0 = iqx - 9;
            jy0 = iqy - 9;
            lk_bar(LK_BAR_CONS, LK_CTHREADS);     // the readers of the previous window are done
            if (T.on && lk_inside<LK_JR, LK_JR>(J, jx0, jy0)) {
                if (tid == 0) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    mbar_expect_tx(&S.mbar_j, LK_JR * LK_JPITCH);
                    lk_tma_box(jreg, T.mj + level, jx0 & ~15, jy0, &S.mbar_j);
                }
                lk_tma_wait(&S.mbar_j, T.phase_j);     // every consumer waits: the box is visible to all without a barrier
                joff = jx0 & 15;
            } else {
                joff = lk_stage_part<LK_JR, LK_JR, LK_JPITCH>(jreg, J, jx0, jy0, tid, LK_CTHREADS);
                lk_bar(LK_BAR_CONS, LK_CTHREADS);
            }
            jvalid = true;
            LKP(4);
        }
        int iw00, iw01, iw10, iw11;
        lk_weights(qx - (float)iqx, qy - (float)iqy, iw00, iw01, iw10, iw11);
        const uint8_t* jb = jreg + (iqy - jy0) * LK_JPITCH + joff + (iqx - jx0);
        // No barrier here: the window staged by the producers or in this level was published by its barrier or mbarrier, the level's template
        // and matrix by the handoff; the previous iteration's fallback terms and sums were consumed before its last
        // barrier (the fast path reads neither), and its integer partials sit in the other half of S.bpart.
        // ---- mismatch terms: (d * Ix, d * Iy) of one template pixel ----
        auto pix = [&](int i, int off, int& px, int& py) {
            const uint8_t* q = jb + off;
            const int jv = q[0] * iw00 + q[1] * iw01 + q[LK_JPITCH] * iw10 + q[LK_JPITCH + 1] * iw11;
            const short4 t = tpl[i];
            const int d = lk_descale(jv, 9) - t.x;
            px = d * t.y;
            py = d * t.z;
        };
        // units: pair unit (ux, uy) -- pmaddwd, an exact int32 pair sum converted once; second unit (vx, vy), a pair or a
        // tail pixel; second tail pixel (wx, wy) or 0
        auto unit_terms = [&](int& ux, int& uy, int& vx, int& vy, int& wx, int& wy) {
            int x1, y1;
            pix(p0, po, ux, uy);
            pix(p0 + 4, po + 4, x1, y1);
            ux += x1;
            uy += y1;
            wx = wy = 0;
            if (pair2) {
                pix(p0 + P2I, po + P2O, vx, vy);
                pix(p0 + P2I + 4, po + P2O + 4, x1, y1);
                vx += x1;
                vy += y1;
            } else {
                pix(e0, eo0, vx, vy);
                if (tail2) pix(e1, eo1, wx, wy);
            }
        };
        int ux, uy, vx, vy, wx, wy;
        unit_terms(ux, uy, vx, vy, wx, wy);
        unsigned part[4] = {0u, 0u, 0u, 0u}, tpart[4] = {0u, 0u, 0u, 0u};     // x+, x-, y+, y- of the pair / tail chain
        lk_split(ux, part[0], part[1]);
        lk_split(uy, part[2], part[3]);
        unsigned vpart[4] = {0u, 0u, 0u, 0u};
        lk_split(vx, vpart[0], vpart[1]);
        lk_split(vy, vpart[2], vpart[3]);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            part[k] += pair2 ? vpart[k] : 0u;
            tpart[k] += pair2 ? 0u : vpart[k];
        }
        lk_split(wx, tpart[0], tpart[1]);
        lk_split(wy, tpart[2], tpart[3]);
        lk_bpart_write(S.bpart[j & 1], tid, part, tpart);
        lk_bar(LK_BAR_CONS, LK_CTHREADS);
        LKP(5);
        float s1, s2;
        if (!lk_bsum_int(S.bpart[j & 1], tid & 31, s1, s2)) {
            // Some chain may round: OpenCV's order.  The terms are computed again rather than kept in registers across
            // the barrier, stored in chain order, summed by warp 0 and broadcast.
            unit_terms(ux, uy, vx, vy, wx, wy);
            S.bterms[pslot] = (float)ux;
            S.bterms[LK_Q + pslot] = (float)uy;
            const int vslot = pair2 ? pslot + P2S : v0 * 5 + 4;
            S.bterms[vslot] = (float)vx;
            S.bterms[LK_Q + vslot] = (float)vy;
            if (tail2) {
                S.bterms[v1 * 5 + 4] = (float)wx;
                S.bterms[LK_Q + v1 * 5 + 4] = (float)wy;
            }
            lk_bar(LK_BAR_CONS, LK_CTHREADS);
            if (tid < 32) {
                lk_bcombine(lk_chain(S.bterms, tid, 2), s1, s2);
                if (tid == 0) { S.bsums[0] = s1; S.bsums[1] = s2; }
            }
            lk_bar(LK_BAR_CONS, LK_CTHREADS);
            s1 = S.bsums[0];
            s2 = S.bsums[1];
            fallbacks++;
        }
        LKP(6);
        iters++;
        float b1 = s1 * FLT_SCALE, b2 = s2 * FLT_SCALE;
        float dx = (A12 * b2 - A22 * b1) * D, dy = (A12 * b1 - A11 * b2) * D;
        qx += dx;
        qy += dy;
        nx = qx + 10.f;
        ny = qy + 10.f;
        if ((double)dx * (double)dx + (double)dy * (double)dy <= 0.01 * 0.01) break;
        if (j > 0 && fabs((double)(dx + pdx_)) < 0.01 && fabs((double)(dy + pdy_)) < 0.01) {
            nx -= dx * 0.5f;
            ny -= dy * 0.5f;
            break;
        }
        pdx_ = dx;
        pdy_ = dy;
        LKP(7);
    }
    // epilogue of OpenCV's err computation (level 0): final window origin must still be in range
    if (level == 0 && status) {
        int fx = __float2int_rd(nx - 10.f), fy = __float2int_rd(ny - 10.f);
        if (fx < -LK_WIN || fx >= J.w || fy < -LK_WIN || fy >= J.h) status = 0;
    }
}

// Whole pyramid for one point.  init is only read when use_init.  Every thread of the CTA calls this with identical
// arguments and receives the same out / status; iters, fallbacks and pc are counted by the consumer threads (thread 0
// reports them).  Level l is iterated by the consumers while the producers build level l-1; the roles meet at one
// handoff barrier per level (and one before the first), which both pass on every path: a level that is out of the image
// or rejected by minEig is built as "not ok" and skipped by the consumers, and the producers of level 0 build nothing.
__device__ __forceinline__ void lk_track_point(LKSmem& S, int tid, const Pyramid& I, const Pyramid& J,
                                               float2 p, float2 init, bool use_init, int max_level,
                                               float2& out, int& status, int& iters, int& fallbacks, long long* pc, LKTma& T)
{
    status = 1;
    [[maybe_unused]] long long tl = gf_clock();
    __syncthreads();     // the previous pass's readers of every buffer are done
    // the template windows of all levels depend only on p: fetch them together (one memory latency instead of one per level)
    const float2 g = use_init ? init : p;
    int n_box = 0;
    for (int l = 0; l <= max_level; l++) {
        float ppx, ppy;
        int ipx, ipy;
        lk_origin(p, l, ppx, ppy, ipx, ipy);
        if (ipx < -LK_WIN || ipx >= I.lv[l].w || ipy < -LK_WIN || ipy >= I.lv[l].h) continue;
        if (T.on && lk_inside<LK_IREG, LK_IREG>(I.lv[l], ipx - 1, ipy - 1)) n_box++;
        else lk_stage<LK_IREG, LK_IREG, LK_IPITCH>(S.ireg[l], I.lv[l], ipx - 1, ipy - 1, tid);
    }
    if (n_box) {            // the same test again by the issuing thread: one transaction count for all boxes of this point
        if (tid == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&S.mbar_i, n_box * LK_IREG * LK_IPITCH);
            for (int l = 0; l <= max_level; l++) {
                float ppx, ppy;
                int ipx, ipy;
                lk_origin(p, l, ppx, ppy, ipx, ipy);
                if (ipx < -LK_WIN || ipx >= I.lv[l].w || ipy < -LK_WIN || ipy >= I.lv[l].h) continue;
                if (lk_inside<LK_IREG, LK_IREG>(I.lv[l], ipx - 1, ipy - 1)) lk_tma_box(S.ireg[l], T.mi + l, (ipx - 1) & ~15, ipy - 1, &S.mbar_i);
            }
        }
        lk_tma_wait(&S.mbar_i, T.phase_i);
    }
    __syncthreads();
    LKP(0);
    if (tid >= LK_CTHREADS) {
        const int pt = tid - LK_CTHREADS;
        lk_build(S, pt, I.lv[max_level], J.lv[max_level], p, g, max_level, max_level & 1, T);
        lk_bar(LK_BAR_HANDOFF, LK_THREADS);
        for (int l = max_level; l >= 0; l--) {
            if (l > 0) lk_build(S, pt, I.lv[l - 1], J.lv[l - 1], p, g, l - 1, (l - 1) & 1, T);    // the buffer of level l+1, free
            lk_bar(LK_BAR_HANDOFF, LK_THREADS);
        }
    } else {
        float nx = 0.f, ny = 0.f;
        lk_bar(LK_BAR_HANDOFF, LK_THREADS);
        LKP(1);
        for (int l = max_level; l >= 0; l--) {
            float sc = (float)(1. / (double)(1 << l));
            if (l == max_level) {
                if (use_init) { nx = init.x * sc; ny = init.y * sc; }
                else { nx = p.x * sc; ny = p.y * sc; }
            } else { nx = nx * 2.f; ny = ny * 2.f; }
            lk_iterate(S, tid, J.lv[l], g, nx, ny, l, l & 1, status, iters, fallbacks, pc, T);
            if (l == 0 && tid == 0) { S.res = make_float2(nx, ny); S.res_status = status; }
            tl = gf_clock();
            lk_bar(LK_BAR_HANDOFF, LK_THREADS);
            LKP(2);
        }
    }
    out = S.res;
    status = S.res_status;
}

}  // namespace gf
