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

struct __align__(128) LKSmem {
    uint8_t ireg[LK_MAXLEV][LK_IREG * LK_IPITCH];   // per level: raw bytes, row r at r*32, first needed column at byte xoff
    uint8_t jreg[LK_JR * LK_JPITCH];                // 128-byte aligned like ireg[l]: both are TMA box destinations
    int16_t sch[LK_SCH * LK_SCH * 2];
    int16_t pI[LK_NPIX + 1];
    int16_t pdx[LK_NPIX + 1];
    int16_t pdy[LK_NPIX + 1];
    float terms[3 * LK_Q];                 // [quantity][step][chain]; slots beyond a chain's length hold +0.0f (x + 0 is exact)
    float sums[4];                         // chain results broadcast from warp 0
    unsigned long long mbar;               // completion barrier of the window loads
};
static_assert((LK_IREG * LK_IPITCH) % 128 == 0 && (LK_MAXLEV * LK_IREG * LK_IPITCH) % 128 == 0, "TMA destinations must be 128-byte aligned");

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
struct LKTma { const CUtensorMap* mi; const CUtensorMap* mj; unsigned phase; bool on; };

__device__ __forceinline__ void lk_tma_box(void* dst, const CUtensorMap* map, int x, int y, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(x), "r"(y), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void lk_tma_wait(LKSmem& S, LKTma& T)
{
    while (!mbar_try_wait(&S.mbar, T.phase)) { }
    T.phase ^= 1u;
}
// once per kernel, before the first lk_track_point
__device__ __forceinline__ void lk_tma_init(LKSmem& S, int tid)
{
    if (tid == 0) {
        mbar_init(&S.mbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}
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

// A thread's fixed share of the mismatch terms: one unit of the chain layout (a pmaddwd pair or a tail pixel) plus,
// for 17 threads, a second tail pixel -- at most two pixels per thread, the same for every level and iteration.
struct LKUnit { int i0, i1, slot, off0, off1; };
__device__ __forceinline__ LKUnit lk_unit(int u)
{
    LKUnit U;
    if (u < 4 * LK_BCHAIN) {
        int y = u >> 3, r = u & 7, k = r & 3, hh = r >> 2;
        U.i0 = y * LK_WIN + 8 * hh + k;
        U.i1 = U.i0 + 4;
        U.slot = (y * 2 + hh) * 5 + k;
    } else {
        int t = u - 4 * LK_BCHAIN, y = t / 5, x = 16 + (t - y * 5);
        U.i0 = U.i1 = y * LK_WIN + x;
        U.slot = t * 5 + 4;
    }
    U.off0 = (U.i0 / LK_WIN) * LK_JPITCH + (U.i0 % LK_WIN);
    U.off1 = (U.i1 / LK_WIN) * LK_JPITCH + (U.i1 % LK_WIN);
    return U;
}

// One pyramid level for one point.  All LK_THREADS threads of the CTA call this with identical scalar arguments
// and keep identical copies of the scalar state; warp 0 owns the sequential chains.  The level's 24x24 window of I
// is already staged in S.ireg[level] (lk_track_point).
__device__ __forceinline__ void lk_level(LKSmem& S, int tid, const Level& I, const Level& J, float2 p,
                                         float& nx, float& ny, int level, int& status, int& iters, long long* pc, LKTma& T)
{
    [[maybe_unused]] long long tl = gf_clock();
    const float FLT_SCALE = 1.f / (1 << 20);
    float ppx, ppy;
    int ipx, ipy;
    lk_origin(p, level, ppx, ppy, ipx, ipy);
    if (ipx < -LK_WIN || ipx >= I.w || ipy < -LK_WIN || ipy >= I.h) {
        if (level == 0) status = 0;
        return;
    }
    float a = ppx - (float)ipx, b = ppy - (float)ipy;
    int iw00, iw01, iw10, iw11;
    lk_weights(a, b, iw00, iw01, iw10, iw11);
    const uint8_t* ireg = S.ireg[level];
    const int ioff = lk_stage_offset<LK_IREG, LK_IREG>(I, ipx - 1, ipy - 1, T.on);
    __syncthreads();     // previous level's readers of sch / pI / terms are done
    // ---- Scharr derivative at the 22x22 integer positions (0 outside the image) ----
    for (int i = tid; i < LK_SCH * LK_SCH; i += LK_THREADS) {
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
    __syncthreads();
    LKP(1);
    // ---- bilinear 21x21 patches I*32, (Ix, Iy), and the gradient-matrix terms in chain order ----
    for (int i = tid; i < LK_NPIX; i += LK_THREADS) {
        int y = i / LK_WIN, x = i - y * LK_WIN;
        const uint8_t* q = ireg + (y + 1) * LK_IPITCH + ioff + (x + 1);
        int iv = q[0] * iw00 + q[1] * iw01 + q[LK_IPITCH] * iw10 + q[LK_IPITCH + 1] * iw11;
        S.pI[i] = (int16_t)lk_descale(iv, 9);
        const int16_t* s = S.sch + 2 * (y * LK_SCH + x);
        int dxv = s[0] * iw00 + s[2] * iw01 + s[2 * LK_SCH] * iw10 + s[2 * LK_SCH + 2] * iw11;
        int dyv = s[1] * iw00 + s[3] * iw01 + s[2 * LK_SCH + 1] * iw10 + s[2 * LK_SCH + 3] * iw11;
        int gx = (int16_t)lk_descale(dxv, 14), gy = (int16_t)lk_descale(dyv, 14);
        S.pdx[i] = (int16_t)gx;
        S.pdy[i] = (int16_t)gy;
        // products are exact integers below 2^24, so (float)(int product) == fx*fy of OpenCV's float path
        int slot = (x < 16) ? (y * 4 + (x >> 2)) * 5 + (x & 3) : (y * 5 + (x - 16)) * 5 + 4;     // [step][chain]
        S.terms[slot] = (float)(gx * gx);
        S.terms[LK_Q + slot] = (float)(gx * gy);
        S.terms[2 * LK_Q + slot] = (float)(gy * gy);
    }
    __syncthreads();
    LKP(2);
    // ---- gradient matrix, OpenCV lane order: warp 0 runs the 15 chains while the other warps already stage the
    //      search window of the first iteration (its position does not depend on A) ----
    float qx = nx - 10.f, qy = ny - 10.f;
    int jx0 = 0, jy0 = 0, joff = 0;
    bool jvalid = false;
    {
        int iqx = __float2int_rd(qx), iqy = __float2int_rd(qy);
        const bool inwin = !(iqx < -LK_WIN || iqx >= J.w || iqy < -LK_WIN || iqy >= J.h);
        if (inwin) { jx0 = iqx - 9; jy0 = iqy - 9; jvalid = true; }
        if (tid < 32) {
            const float acc = lk_chain(S.terms, tid, 3);
#pragma unroll
            for (int q = 0; q < 3; q++) {
                float l0 = __shfl_sync(0xffffffffu, acc, q * 5 + 0), l1 = __shfl_sync(0xffffffffu, acc, q * 5 + 1);
                float l2 = __shfl_sync(0xffffffffu, acc, q * 5 + 2), l3 = __shfl_sync(0xffffffffu, acc, q * 5 + 3);
                float t = __shfl_sync(0xffffffffu, acc, q * 5 + 4);
                if (tid == 0) S.sums[q] = t + ((l0 + l2) + (l1 + l3));
            }
        } else if (inwin) {
            if (T.on && lk_inside<LK_JR, LK_JR>(J, jx0, jy0)) {
                if (tid == 32) {     // previous readers / writers of jreg finished before the barrier at the top of this level
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    mbar_expect_tx(&S.mbar, LK_JR * LK_JPITCH);
                    lk_tma_box(S.jreg, T.mj + level, jx0 & ~15, jy0, &S.mbar);
                }
            } else {
                joff = lk_stage_part<LK_JR, LK_JR, LK_JPITCH>(S.jreg, J, jx0, jy0, tid - 32, LK_THREADS - 32);
            }
        }
        if (inwin) {
            joff = lk_stage_offset<LK_JR, LK_JR>(J, jx0, jy0, T.on);
            if (T.on && lk_inside<LK_JR, LK_JR>(J, jx0, jy0)) lk_tma_wait(S, T);
        }
    }
    // this thread's share of the mismatch terms and the template values it needs (constant over the iterations)
    const LKUnit U1 = lk_unit(tid < LK_BT ? tid : 0);
    const bool has2 = (tid >= 4 * LK_BCHAIN) && (LK_THREADS + tid - 4 * LK_BCHAIN < LK_BT);
    const LKUnit U2 = lk_unit(has2 ? LK_THREADS + tid - 4 * LK_BCHAIN : 4 * LK_BCHAIN);
    const int t1I0 = S.pI[U1.i0], t1x0 = S.pdx[U1.i0], t1y0 = S.pdy[U1.i0];
    const int t1I1 = S.pI[U1.i1], t1x1 = S.pdx[U1.i1], t1y1 = S.pdy[U1.i1];
    const int t2I = S.pI[U2.i0], t2x = S.pdx[U2.i0], t2y = S.pdy[U2.i0];
    __syncthreads();
    LKP(3);
    float A11 = S.sums[0] * FLT_SCALE, A12 = S.sums[1] * FLT_SCALE, A22 = S.sums[2] * FLT_SCALE;
    // the mismatch chains are 42 pair terms long: clear steps 42..83 of the SIMD chains of the two quantities they reuse
    for (int i = tid; i < 2 * 4 * (LK_CHAIN - LK_BCHAIN); i += LK_THREADS) {
        int q = i / (4 * (LK_CHAIN - LK_BCHAIN)), r = i - q * 4 * (LK_CHAIN - LK_BCHAIN);
        S.terms[q * LK_Q + (LK_BCHAIN + (r >> 2)) * 5 + (r & 3)] = 0.f;
    }
    float D = A11 * A22 - A12 * A12;
    float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / 882.f;
    if (minEig < 1e-4f || D < 1.1920928955078125e-07f) {
        if (level == 0) status = 0;
        return;
    }
    D = 1.f / D;

    float pdx_ = 0.f, pdy_ = 0.f;
    LKP(4);
    for (int j = 0; j < 30; j++) {
        int iqx = __float2int_rd(qx), iqy = __float2int_rd(qy);
        if (iqx < -LK_WIN || iqx >= J.w || iqy < -LK_WIN || iqy >= J.h) {
            if (level == 0) status = 0;
            break;
        }
        if (!(jvalid && iqx >= jx0 && iqy >= jy0 && iqx + 22 <= jx0 + LK_JR && iqy + 22 <= jy0 + LK_JR)) {
            jx0 = iqx - 9;
            jy0 = iqy - 9;
            __syncthreads();
            if (T.on && lk_inside<LK_JR, LK_JR>(J, jx0, jy0)) {
                if (tid == 0) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    mbar_expect_tx(&S.mbar, LK_JR * LK_JPITCH);
                    lk_tma_box(S.jreg, T.mj + level, jx0 & ~15, jy0, &S.mbar);
                }
                lk_tma_wait(S, T);
                joff = jx0 & 15;
            } else {
                joff = lk_stage<LK_JR, LK_JR, LK_JPITCH>(S.jreg, J, jx0, jy0, tid);
            }
            jvalid = true;
        }
        a = qx - (float)iqx;
        b = qy - (float)iqy;
        lk_weights(a, b, iw00, iw01, iw10, iw11);
        const uint8_t* jb = S.jreg + (iqy - jy0) * LK_JPITCH + joff + (iqx - jx0);
        __syncthreads();    // staged window and cleared/previous terms are visible; previous sums have been read
        // ---- mismatch terms in chain order: 168 pmaddwd pair units (row y, k in 0..3, half h) + 105 tail pixels ----
        if (tid < LK_BT) {
            const uint8_t* q = jb + U1.off0;
            int jv = q[0] * iw00 + q[1] * iw01 + q[LK_JPITCH] * iw10 + q[LK_JPITCH + 1] * iw11;
            int d0 = lk_descale(jv, 9) - t1I0;
            int sx = d0 * t1x0, sy = d0 * t1y0;
            if (tid < 4 * LK_BCHAIN) {
                q = jb + U1.off1;
                jv = q[0] * iw00 + q[1] * iw01 + q[LK_JPITCH] * iw10 + q[LK_JPITCH + 1] * iw11;
                int d1 = lk_descale(jv, 9) - t1I1;
                sx += d1 * t1x1;   // pmaddwd: exact int32 pair sum, converted once
                sy += d1 * t1y1;
            }
            S.terms[U1.slot] = (float)sx;
            S.terms[LK_Q + U1.slot] = (float)sy;
        }
        if (has2) {
            const uint8_t* q = jb + U2.off0;
            int jv = q[0] * iw00 + q[1] * iw01 + q[LK_JPITCH] * iw10 + q[LK_JPITCH + 1] * iw11;
            int d0 = lk_descale(jv, 9) - t2I;
            S.terms[U2.slot] = (float)(d0 * t2x);
            S.terms[LK_Q + U2.slot] = (float)(d0 * t2y);
        }
        __syncthreads();
        LKP(5);
        if (tid < 32) {
            const float bacc = lk_chain(S.terms, tid, 2);
#pragma unroll
            for (int comp = 0; comp < 2; comp++) {
                float c0 = __shfl_sync(0xffffffffu, bacc, comp * 5 + 0), c1 = __shfl_sync(0xffffffffu, bacc, comp * 5 + 1);
                float c2 = __shfl_sync(0xffffffffu, bacc, comp * 5 + 2), c3 = __shfl_sync(0xffffffffu, bacc, comp * 5 + 3);
                float t = __shfl_sync(0xffffffffu, bacc, comp * 5 + 4);
                float x02 = c0 + c2, x13 = c1 + c3;
                if (tid == 0) S.sums[comp] = t + ((x02 + 0.f) + (x13 + 0.f));
            }
        }
        __syncthreads();
        LKP(6);
        iters++;
        float b1 = S.sums[0] * FLT_SCALE, b2 = S.sums[1] * FLT_SCALE;
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

// Whole pyramid for one point.  init is only read when use_init.
__device__ __forceinline__ void lk_track_point(LKSmem& S, int tid, const Pyramid& I, const Pyramid& J,
                                               float2 p, float2 init, bool use_init, int max_level,
                                               float2& out, int& status, int& iters, long long* pc, LKTma& T)
{
    status = 1;
    float nx = 0.f, ny = 0.f;
    [[maybe_unused]] long long tl = gf_clock();
    __syncthreads();
    for (int i = tid; i < 3 * LK_Q; i += LK_THREADS) S.terms[i] = 0.f;    // chain padding must read +0.0f
    // the template windows of all levels depend only on p: fetch them together (one memory latency instead of one per level)
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
            mbar_expect_tx(&S.mbar, n_box * LK_IREG * LK_IPITCH);
            for (int l = 0; l <= max_level; l++) {
                float ppx, ppy;
                int ipx, ipy;
                lk_origin(p, l, ppx, ppy, ipx, ipy);
                if (ipx < -LK_WIN || ipx >= I.lv[l].w || ipy < -LK_WIN || ipy >= I.lv[l].h) continue;
                if (lk_inside<LK_IREG, LK_IREG>(I.lv[l], ipx - 1, ipy - 1)) lk_tma_box(S.ireg[l], T.mi + l, (ipx - 1) & ~15, ipy - 1, &S.mbar);
            }
        }
        lk_tma_wait(S, T);
    }
    __syncthreads();
    LKP(0);
    for (int l = max_level; l >= 0; l--) {
        float sc = (float)(1. / (double)(1 << l));
        if (l == max_level) {
            if (use_init) { nx = init.x * sc; ny = init.y * sc; }
            else { nx = p.x * sc; ny = p.y * sc; }
        } else { nx = nx * 2.f; ny = ny * 2.f; }
        lk_level(S, tid, I.lv[l], J.lv[l], p, nx, ny, l, status, iters, pc, T);
    }
    out = make_float2(nx, ny);
}

}  // namespace gf
