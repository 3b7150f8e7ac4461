// fe_lk_single.cuh -- the single-role form of fe_lk.cuh's pyramidal Lucas-Kanade: all 8 warps of the CTA set up a level, then
// all 8 iterate it.  Bit-exact with the two-role form (lk_track_point in fe_lk.cuh) and with OpenCV 4.13.
//
// The two-role form shortens each feature's dependent chain, which is what one tracker alone on the GPU waits for.  When
// several trackers share the GPU, the work of all their features counts instead, and there this form measured faster
// (DESIGN.md §1.3), so fe_tracker.cu launches it whenever more than one tracker is live on the device.  It shares
// fe_lk.cuh's window staging, chain and weight helpers; what differs is kept here, in namespace gf::lk1: the shared
// memory layout, the mbarrier bookkeeping, the mismatch-term units of 256 threads, the level and the pyramid.
#pragma once
#include "fe_lk.cuh"

namespace gf {
namespace lk1 {
// Units of the b terms per thread (lk_unit): thread u < 4 * LK_BCHAIN holds pair unit u, of chain u & 3; the others hold
// tail units (chain 4).  So warps 0..LK_PAIR_WARPS-1 carry pair units and warps LK_TAIL_WARP0.. carry tail units.
constexpr int LK_PAIR_WARPS = (4 * LK_BCHAIN + 31) / 32;            // 6
constexpr int LK_TAIL_WARP0 = 4 * LK_BCHAIN / 32;                   // 5
constexpr int LK_TAIL_WARPS = LK_THREADS / 32 - LK_TAIL_WARP0;       // 3
constexpr int LK_BSLOTS = 5 * LK_PAIR_WARPS;         // per-warp partials; the tail chain's slots beyond LK_TAIL_WARPS stay 0
static_assert(LK_PAIR_WARPS >= LK_TAIL_WARPS, "lk_bsum_int sums LK_PAIR_WARPS partials per chain");

struct __align__(128) LKSmem {
    uint8_t ireg[LK_MAXLEV][LK_IREG * LK_IPITCH];   // per level: raw bytes, row r at r*32, first needed column at byte xoff
    uint8_t jreg[LK_JR * LK_JPITCH];                // 128-byte aligned like ireg[l]: both are TMA box destinations
    int16_t sch[LK_SCH * LK_SCH * 2];
    short4 tpl[LK_NPIX + 1];               // template patch per pixel: (I*32, Ix, Iy, 0), one 8-byte load per pixel
    float terms[3 * LK_Q];                 // [quantity][step][chain]; slots beyond a chain's length hold +0.0f (x + 0 is exact)
    float sums[4];                         // chain results broadcast from warp 0
    // [iteration parity][slot][x+, x-, y+, y-]: per-warp sums of the positive b terms and of the magnitudes of the negative
    // ones of one chain; slot w*4 + k: pair chain k of warp w, slot 4*LK_PAIR_WARPS + w - LK_TAIL_WARP0: tail chain of warp w
    // (the tail chain's remaining slots are zeroed once per point, so every chain sums LK_PAIR_WARPS slots)
    alignas(16) unsigned bpart[2][LK_BSLOTS][4];
    unsigned long long mbar;               // completion barrier of the window loads
};
static_assert((LK_IREG * LK_IPITCH) % 128 == 0 && (LK_MAXLEV * LK_IREG * LK_IPITCH) % 128 == 0, "TMA destinations must be 128-byte aligned");
struct LKTma { const CUtensorMap* mi; const CUtensorMap* mj; unsigned phase; bool on; };

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
// Per-warp integer partials of the b chains from this thread's share v = (x+, x-, y+, y-) of its chain's terms.
// No sum can wrap: a term is below 2^26 in magnitude (|d| <= 8160, |g| <= 4080, two products per pair), and a whole
// chain (42 pair terms or 105 tail products) stays below 2^32.
__device__ __forceinline__ void lk_bpart_write(unsigned (*P)[4], int tid, const unsigned (&v)[4])
{
    const int w = tid >> 5, lane = tid & 31;
    const bool pair = tid < 4 * LK_BCHAIN;
    if (w < LK_PAIR_WARPS) {
        // Reduce-scatter over the 8 lanes of each pair chain (equal lane & 3), four shuffles, three deep: across lane bit 4
        // a lane keeps values {0,1} or {2,3}, across bit 3 one of them, across bit 2 it completes value (lane >> 3) & 3.
        const bool h4 = lane & 16, h3 = lane & 8;
        unsigned a0 = pair ? (h4 ? v[2] : v[0]) : 0u, a1 = pair ? (h4 ? v[3] : v[1]) : 0u;
        const unsigned s0 = pair ? (h4 ? v[0] : v[2]) : 0u, s1 = pair ? (h4 ? v[1] : v[3]) : 0u;
        a0 += __shfl_xor_sync(0xffffffffu, s0, 16);
        a1 += __shfl_xor_sync(0xffffffffu, s1, 16);
        unsigned c = (h3 ? a1 : a0) + __shfl_xor_sync(0xffffffffu, h3 ? a0 : a1, 8);
        c += __shfl_xor_sync(0xffffffffu, c, 4);
        if (!(lane & 4)) P[w * 4 + (lane & 3)][(lane >> 3) & 3] = c;
    }
    if (w >= LK_TAIL_WARP0) {           // every tail unit belongs to chain 4
        unsigned s[4];
#pragma unroll
        for (int k = 0; k < 4; k++) s[k] = __reduce_add_sync(0xffffffffu, pair ? 0u : v[k]);
        if (lane == 0) *reinterpret_cast<uint4*>(P[4 * LK_PAIR_WARPS + w - LK_TAIL_WARP0]) = make_uint4(s[0], s[1], s[2], s[3]);
    }
}

// b1 and b2 from the per-warp integer partials, computed by every warp, when all ten chains are within the exactness
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
        for (int w = 0; w < LK_PAIR_WARPS; w++) {
            const uint2 v = reinterpret_cast<const uint2*>(P[c < 4 ? w * 4 + c : 4 * LK_PAIR_WARPS + w])[comp];
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
                                         float& nx, float& ny, int level, int& status, int& iters, int& fallbacks,
                                         long long* pc, LKTma& T)
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
    __syncthreads();     // previous level's readers of sch / tpl / terms are done
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
        const int pv = lk_descale(iv, 9);
        const int16_t* s = S.sch + 2 * (y * LK_SCH + x);
        int dxv = s[0] * iw00 + s[2] * iw01 + s[2 * LK_SCH] * iw10 + s[2 * LK_SCH + 2] * iw11;
        int dyv = s[1] * iw00 + s[3] * iw01 + s[2 * LK_SCH + 1] * iw10 + s[2 * LK_SCH + 3] * iw11;
        int gx = (int16_t)lk_descale(dxv, 14), gy = (int16_t)lk_descale(dyv, 14);
        S.tpl[i] = make_short4((short)pv, (short)gx, (short)gy, 0);
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
    // this thread's share of the mismatch terms (constant over the iterations).  Its template values are read from
    // S.tpl in every iteration rather than held in registers: the loads overlap the weight arithmetic,
    // and the nine registers they would pin make the 80-register k_track serialise its iteration.
    const LKUnit U1 = lk_unit(tid < LK_BT ? tid : 0);
    const bool has2 = (tid >= 4 * LK_BCHAIN) && (LK_THREADS + tid - 4 * LK_BCHAIN < LK_BT);
    const LKUnit U2 = lk_unit(has2 ? LK_THREADS + tid - 4 * LK_BCHAIN : 4 * LK_BCHAIN);
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
                lk_tma_wait(S, T);     // every thread waits: the box is visible to all without a barrier
                joff = jx0 & 15;
            } else {
                joff = lk_stage<LK_JR, LK_JR, LK_JPITCH>(S.jreg, J, jx0, jy0, tid);
                __syncthreads();
            }
            jvalid = true;
        }
        a = qx - (float)iqx;
        b = qy - (float)iqy;
        lk_weights(a, b, iw00, iw01, iw10, iw11);
        const uint8_t* jb = S.jreg + (iqy - jy0) * LK_JPITCH + joff + (iqx - jx0);
        // No barrier here: the window staged before the loop, the cleared terms and the A sums were published by the
        // barrier before the loop; the previous iteration's terms and sums were consumed before its last barrier (the
        // fast path reads neither), and its integer partials sit in the other half of S.bpart.
        // ---- mismatch terms: 168 pmaddwd pair units (row y, k in 0..3, half h) + 105 tail pixels; this thread's unit
        //      U1 gives (sx, sy), the second tail unit U2 of 17 threads (ex, ey) ----
        auto unit_terms = [&](int& sx, int& sy, int& ex, int& ey) {
            sx = sy = ex = ey = 0;
            if (tid < LK_BT) {
                const uint8_t* q = jb + U1.off0;
                int jv = q[0] * iw00 + q[1] * iw01 + q[LK_JPITCH] * iw10 + q[LK_JPITCH + 1] * iw11;
                const short4 t0 = S.tpl[U1.i0];
                int d0 = lk_descale(jv, 9) - t0.x;
                sx = d0 * t0.y;
                sy = d0 * t0.z;
                if (tid < 4 * LK_BCHAIN) {
                    q = jb + U1.off1;
                    jv = q[0] * iw00 + q[1] * iw01 + q[LK_JPITCH] * iw10 + q[LK_JPITCH + 1] * iw11;
                    const short4 t1 = S.tpl[U1.i1];
                    int d1 = lk_descale(jv, 9) - t1.x;
                    sx += d1 * t1.y;   // pmaddwd: exact int32 pair sum, converted once
                    sy += d1 * t1.z;
                }
            }
            if (has2) {
                const uint8_t* q = jb + U2.off0;
                int jv = q[0] * iw00 + q[1] * iw01 + q[LK_JPITCH] * iw10 + q[LK_JPITCH + 1] * iw11;
                const short4 t2 = S.tpl[U2.i0];
                int d0 = lk_descale(jv, 9) - t2.x;
                ex = d0 * t2.y;
                ey = d0 * t2.z;
            }
        };
        int sx, sy, ex, ey;
        unit_terms(sx, sy, ex, ey);
        unsigned part[4] = {0u, 0u, 0u, 0u};     // this thread's x+, x-, y+, y- (all its units are of one chain)
        lk_split(sx, part[0], part[1]);
        lk_split(sy, part[2], part[3]);
        lk_split(ex, part[0], part[1]);
        lk_split(ey, part[2], part[3]);
        lk_bpart_write(S.bpart[j & 1], tid, part);
        __syncthreads();
        LKP(5);
        float s1, s2;
        if (!lk_bsum_int(S.bpart[j & 1], tid & 31, s1, s2)) {
            // Some chain may round: OpenCV's order.  The terms are computed again rather than kept in registers across
            // the barrier, stored in chain order, summed by warp 0 and broadcast.
            unit_terms(sx, sy, ex, ey);
            if (tid < LK_BT) {
                S.terms[U1.slot] = (float)sx;
                S.terms[LK_Q + U1.slot] = (float)sy;
            }
            if (has2) {
                S.terms[U2.slot] = (float)ex;
                S.terms[LK_Q + U2.slot] = (float)ey;
            }
            __syncthreads();
            if (tid < 32) {
                lk_bcombine(lk_chain(S.terms, tid, 2), s1, s2);
                if (tid == 0) { S.sums[0] = s1; S.sums[1] = s2; }
            }
            __syncthreads();
            s1 = S.sums[0];
            s2 = S.sums[1];
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

// Whole pyramid for one point.  init is only read when use_init.
__device__ __forceinline__ void lk_track_point(LKSmem& S, int tid, const Pyramid& I, const Pyramid& J,
                                               float2 p, float2 init, bool use_init, int max_level,
                                               float2& out, int& status, int& iters, int& fallbacks, long long* pc, LKTma& T)
{
    status = 1;
    float nx = 0.f, ny = 0.f;
    [[maybe_unused]] long long tl = gf_clock();
    __syncthreads();
    for (int i = tid; i < 3 * LK_Q; i += LK_THREADS) S.terms[i] = 0.f;    // chain padding must read +0.0f
    constexpr int NPAD = (LK_BSLOTS - 4 * LK_PAIR_WARPS - LK_TAIL_WARPS) * 4;      // and the unused tail partials 0
    for (int i = tid; i < 2 * NPAD; i += LK_THREADS) (&S.bpart[i / NPAD][4 * LK_PAIR_WARPS + LK_TAIL_WARPS][0])[i % NPAD] = 0u;
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
        lk_level(S, tid, I.lv[l], J.lv[l], p, nx, ny, l, status, iters, fallbacks, pc, T);
    }
    out = make_float2(nx, ny);
}

}  // namespace lk1
}  // namespace gf
