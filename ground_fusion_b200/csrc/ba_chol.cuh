// ba_chol.cuh -- dense FP64 linear algebra of the sliding-window solve on 8x8 tiles with FP64 tensor-core MMAs
// (mma.sync m8n8k4 f64 = SASS DMMA.8x8x4; latency and rate per SM: tools/dmma_probe.cu).
//
// Replaces Ceres' DENSE_SCHUR linear solver (SchurEliminator + dense Cholesky; reference call site estimator.cpp:3303-3318):
//   schur_tile      one 8x8 tile of the reduced camera system  S = H' + mu D^2 - W'^T C W'  (rank-L update on DMMA)
//   chol_factor     left-looking tiled Cholesky of the (nc+1)-row augmented system (row nc = right-hand side) by one CTA:
//                   tile (I,J) = A_IJ - sum_p L_Ip L_Jp^T accumulated in registers by DMMAs, 8x8 diagonal factorisation
//                   + inverse by one warp in registers, TRSM as two DMMAs against the published inverse
//   chol_backsubst  L^T y = z by one warp
// Tile storage ("fragment order"): tile element [r][c] at  (c/4)*32 + r*4 + c%4 , so that the k-half h of a tile is the
// contiguous run [h*32, h*32+32): lane l of an m8n8k4 operand fragment reads element h*32 + l.
#pragma once
#include <cfloat>
#include "gf_common.cuh"

#ifndef GF_CHOL_STAMP
#define GF_CHOL_STAMP(k) do { } while (0)     // tools/chol_bench.cu records per-warp, per-panel clock64() stamps through this hook
#define GF_CHOL_STAMP_AFTER(k, dep) do { } while (0)
#endif

namespace gfba {

#ifndef GF_ST_THREADS
#define GF_ST_THREADS 256
#endif
constexpr int ST_THREADS = GF_ST_THREADS;       // k_ba_step block size: 8 warps x 255 registers (the 8x8 diagonal factorisation lives in registers)
constexpr int ST_WARPS = ST_THREADS / 32;
constexpr int TILE_CAP = 376;                   // factor tiles resident in shared memory (512 B each); the rest spills to L2
constexpr int MAX_N8 = 48;                      // block rows of the augmented system
constexpr int MAX_NC = 8 * MAX_N8 - 1;          // reduced dimension supported by the solver (383)
constexpr int MAXR = 2 * ((MAX_N8 + 2 * (ST_WARPS - 1) - 1) / (2 * (ST_WARPS - 1)));   // block rows per bulk warp, even; kernels are instantiated for MAXR / 2 and MAXR

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b)
{
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__host__ __device__ __forceinline__ int tix(int I, int J) { return I * (I + 1) / 2 + J; }

// Factor tiles live in shared memory up to `cap` tiles, beyond that in a global (L2-resident) spill buffer.  SPILL = false is
// the common case (everything fits: <= 26 block rows = 351 tiles, nc <= 207): the accessors are plain LDS / STS with no second path.
// The tile slots start at offset 0 of the dynamic shared memory of the calling kernel.  Their 32-bit shared address is taken
// ONCE (ch_tiles_u32, made opaque to the compiler) and every access in the hot loops is an explicit ld.shared / st.shared with
// an immediate offset: left to itself nvcc rematerialises the address of the extern array (S2R SR_CgaCtaId + shifts, a
// long-latency special-register read) next to every load.
__device__ __forceinline__ unsigned ch_tiles_u32()
{
    extern __shared__ __align__(128) double gf_dyn_smem[];
    unsigned a = (unsigned)__cvta_generic_to_shared(gf_dyn_smem);
    asm volatile("" : "+r"(a));
    return a;
}
__device__ __forceinline__ double lds_f64(unsigned a) { double v; asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ double2 lds_v2f64(unsigned a) { double2 v; asm volatile("ld.shared.v2.f64 {%0,%1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void sts_v2f64(unsigned a, double x, double y) { asm volatile("st.shared.v2.f64 [%0], {%1,%2};" ::"r"(a), "d"(x), "d"(y) : "memory"); }

template <bool SPILL>
struct TileStoreT {
    unsigned sb;              // shared address of tile 0 (ch_tiles_u32)
    double* Lg;
    int cap;                  // tiles [0, cap) in shared memory (<= TILE_CAP; smaller only in tests of the spill path)
    __device__ __forceinline__ double frag(int t, int h, int lane) const
    {
        if (!SPILL || t < cap) return lds_f64(sb + 8u * (unsigned)(t * 64 + h * 32 + lane));
        return __ldcg(Lg + (size_t)(t - cap) * 64 + h * 32 + lane);
    }
    __device__ __forceinline__ double at(int t, int r, int c) const
    {
        const int o = (c >> 2) * 32 + r * 4 + (c & 3);
        if (!SPILL || t < cap) return lds_f64(sb + 8u * (unsigned)(t * 64 + o));
        return __ldcg(Lg + (size_t)(t - cap) * 64 + o);
    }
    // C-fragment (row l/4, columns 2(l%4), 2(l%4)+1) of an MMA result into fragment order
    __device__ __forceinline__ void store_c(int t, int lane, double x0, double x1) const
    {
        const int q = lane & 3, o = (q >> 1) * 32 + (lane >> 2) * 4 + 2 * (q & 1);
        if (!SPILL || t < cap) sts_v2f64(sb + 8u * (unsigned)(t * 64 + o), x0, x1);
        else *reinterpret_cast<double2*>(Lg + (size_t)(t - cap) * 64 + o) = make_double2(x0, x1);
    }
};

// ------------------------------------------------------------------------------------------------
// Cholesky of one 8x8 diagonal tile and the inverse of its factor, computed redundantly by every lane of a warp in
// registers (no shuffles: the chain per column is rsqrt -> mul -> fma).  S8: the updated tile, row-major, lower triangle.
// Columns >= ncol are padding and behave as identity columns (the right-hand-side row of the augmented system keeps its
// entries in the genuine columns).  Outputs: inverse of the factor in fragment order (the B operand of the TRSM MMAs and
// the diagonal solve of the back substitution); the factor itself row-major when Lout is given (last tile: it holds z).
// sqrt and 1/sqrt of a positive, normal double without the special-case branch of the CUDA math library (a branch would
// cut the factorisation below into basic blocks the scheduler cannot overlap).  The argument is brought into [1, 4) by its
// even exponent, the seed is the single-precision MUFU.RSQ (2^-22), two coupled Newton / Goldschmidt steps (g -> sqrt(x),
// h -> 1 / (2 sqrt(x))) square the error twice and a last correction fixes the square root itself.  Zero, negative,
// subnormal and non-finite x are the caller's failure case (the result is then garbage and never used: the exponent trick
// gives 1e-310 a root of 1.06e-154 and +inf a finite one, so chol8_inv accepts a pivot only in [DBL_MIN, DBL_MAX]).
__device__ __forceinline__ void sqrt_rsqrt(double x, double& sq, double& rs)
{
    const int hi = __double2hiint(x), lo = __double2loint(x);
    const int e = (((hi >> 20) & 0x7ff) - 1023) & ~1;
    const double xs = __hiloint2double(hi - (e << 20), lo);          // x * 2^-e
    const double y = (double)rsqrtf((float)xs);
    double g = xs * y, h = 0.5 * y;
    double r = fma(-g, h, 0.5);
    g = fma(g, r, g); h = fma(h, r, h);
    r = fma(-g, h, 0.5);
    g = fma(g, r, g); h = fma(h, r, h);
    r = fma(-g, g, xs);
    g = fma(r, h, g);
    h = h + h;
    const int he = (e >> 1) << 20;
    sq = __hiloint2double(__double2hiint(g) + he, __double2loint(g));
    rs = __hiloint2double(__double2hiint(h) - he, __double2loint(h));
}

__device__ __forceinline__ bool chol8_inv(const double* __restrict__ S8, int ncol, double* __restrict__ Linv, double* __restrict__ Lout)
{
    double a[8][8];
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int c2 = 0; c2 <= r / 2; c2++) {
            const double2 v = *reinterpret_cast<const double2*>(S8 + r * 8 + 2 * c2);
            a[r][2 * c2] = v.x; a[r][2 * c2 + 1] = v.y;
        }
    bool ok = true;
    double inv[8];
    // one straight-line block: padding columns (k >= ncol) are turned into identity columns by selects, not by branches
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const bool live = k < ncol;
        const double dk = live ? a[k][k] : 1.0;
        ok = ok & (dk >= DBL_MIN) & (dk <= DBL_MAX);      // positive and normal (NaN fails both); a select, not a branch
        double sq, r;
        sqrt_rsqrt(dk, sq, r);
        inv[k] = r;
        a[k][k] = sq;
#pragma unroll
        for (int i = k + 1; i < 8; i++) a[i][k] = live ? a[i][k] * r : 0.0;
#pragma unroll
        for (int i = k + 1; i < 8; i++)
#pragma unroll
            for (int j = k + 1; j <= i; j++) a[i][j] = fma(-a[i][k], a[j][k], a[i][j]);
    }
    if (Lout) {
#pragma unroll
        for (int r = 0; r < 8; r++)
#pragma unroll
            for (int c2 = 0; c2 < 4; c2++)
                *reinterpret_cast<double2*>(Lout + r * 8 + 2 * c2) = make_double2(2 * c2 <= r ? a[r][2 * c2] : 0.0, 2 * c2 + 1 <= r ? a[r][2 * c2 + 1] : 0.0);
    }
    // inverse of the lower-triangular factor, row by row: li[r][c] = -(sum_{c<=m<r} l[r][m] li[m][c]) / l[r][r]
    double li[8][8];
#pragma unroll
    for (int r = 0; r < 8; r++) {
#pragma unroll
        for (int c = 0; c < r; c++) {
            double s0 = 0.0, s1 = 0.0;
#pragma unroll
            for (int m = c; m < r; m += 2) {
                s0 = fma(a[r][m], li[m][c], s0);
                if (m + 1 < r) s1 = fma(a[r][m + 1], li[m + 1][c], s1);
            }
            li[r][c] = -(s0 + s1) * inv[r];
        }
        li[r][r] = inv[r];
    }
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
        for (int r = 0; r < 8; r++)
#pragma unroll
            for (int c2 = 0; c2 < 2; c2++) {
                const int c = 4 * h + 2 * c2;
                *reinterpret_cast<double2*>(Linv + h * 32 + r * 4 + 2 * c2) = make_double2(c <= r ? li[r][c] : 0.0, c + 1 <= r ? li[r][c + 1] : 0.0);   // (the zeros above the diagonal are part of the MMA operand)
            }
    return ok;
}

// ------------------------------------------------------------------------------------------------
// named barriers, mbarrier and the 1-D TMA bulk copy (the reduced system is pulled into shared memory by the copy engine)
__device__ __forceinline__ void nb_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void nb_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ unsigned ch_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ch_mbar_init(unsigned long long* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ch_smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void ch_mbar_expect_tx(unsigned long long* bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ch_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ch_tma_load_1d(void* dst, const void* src, unsigned bytes, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(ch_smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(ch_smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void ch_mbar_wait(unsigned long long* bar, unsigned parity)
{
    unsigned ok = 0, spins = 0;
    while (!ok) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(ch_smem_u32(bar)), "r"(parity) : "memory");
        if (!ok && ++spins > (1u << 24)) __trap();        // a lost copy must not hang the GPU
    }
}
// One elected thread: pull the first `ntl` tiles of the reduced system (row-major 8x8 tiles, 512 B each) into the factor's
// own tile slots.  The left-looking factorisation reads A_IJ exactly once, just before it writes L_IJ into the same slot.
__device__ __forceinline__ void chol_issue_load(const double* Ag, double* Ls, int ntl, unsigned long long* bar)
{
    const unsigned total = (unsigned)ntl * 512u;
    if (total == 0) return;
    ch_mbar_expect_tx(bar, total);
    for (unsigned off = 0; off < total; off += 32768u) {
        const unsigned nb = total - off < 32768u ? total - off : 32768u;
        ch_tma_load_1d(reinterpret_cast<char*>(Ls) + off, reinterpret_cast<const char*>(Ag) + off, nb, bar);
    }
}

// C-fragment (row l/4, columns 2(l%4), 2(l%4)+1) -> the two A/B operand fragments (row l/4, column 4h + l%4) of the same tile:
// lane (r, k) needs column 4h+k, held by lane 4r + 2h + k/2 as element k%2.
__device__ __forceinline__ void c_to_frags(double c0, double c1, int lane, double& f0, double& f1)
{
    const int src0 = (lane & ~3) + ((lane & 3) >> 1), src1 = src0 + 2;
    const double v00 = __shfl_sync(0xffffffffu, c0, src0), v01 = __shfl_sync(0xffffffffu, c1, src0);
    const double v10 = __shfl_sync(0xffffffffu, c0, src1), v11 = __shfl_sync(0xffffffffu, c1, src1);
    f0 = (lane & 1) ? v01 : v00;
    f1 = (lane & 1) ? v11 : v10;
}

// ------------------------------------------------------------------------------------------------
// Left-looking tiled Cholesky of the (nc+1)-row augmented system (row nc = right-hand side), one CTA with warp roles:
//   warp 0  "diagonal warp" owns the critical chain and never waits for bulk work: per panel J it turns the parked tile
//           c_{J,J-1} into L_{J,J-1} itself (two MMAs against the inverse it has just computed), subtracts L_{J,J-1} L_{J,J-1}^T
//           from the parked partial diagonal tile, factors the 8x8 result and inverts the factor (chol8_inv, in registers).
//   warps 1.. "bulk warps": block row I belongs to bulk warp I % CH_BULK.  Per panel J (after inv(L_J-1,J-1) is published):
//           TRSM of its tiles of panel J-1 (row J is the diagonal warp's) -> the owner of row J+1 prepares the next diagonal
//           ahead of time (partial tile A - sum_{p<J} L_{J+1,p} L_{J+1,p}^T, parked in S8) -> barrier (all tiles of panel J-1
//           incl. L_{J,J-1} visible) -> finishes its tiles of panel J (c = A - sums, parked in the tile's own slot in fragment
//           order; row J+1 first, then the diagonal warp is signalled) -> sums of panel J+1 over the panels < J.
// The inner loops are address walks over block rows (LDS with immediate offsets + MMAs): the factorisation is bound by the
// issue latency of a few warps on ONE SM, so every instruction next to an MMA counts.
// A: tiles [0, cap) already sit in their slots, row-major (chol_issue_load); others are read from Ag.  L: fragment order, same
// slots.  Linv: n8 tiles (fragment order), kept for the back substitution.  S8: 2 scratch tiles.  Ld: the factor of the last
// diagonal tile, row-major (it holds the tail of z).  Returns false if a pivot was not a positive normal number.
constexpr int CH_BULK = ST_WARPS - 1;
template <int R, bool SPILL>
__device__ __forceinline__ bool chol_factor(const double* __restrict__ Ag, const TileStoreT<SPILL>& T, double* Linv, double* S8, double* Ld,
                                            int nc, int n8, int* s_fail)
{
    const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
    const int coff = (lane >> 2) * 8 + 2 * (lane & 3);
    constexpr int NB_ALL = 32 * (CH_BULK + 1);
    auto a_pair = [&](int t) {
        if (!SPILL || t < T.cap) return lds_v2f64(T.sb + 8u * (unsigned)(t * 64 + coff));
        return __ldcg(reinterpret_cast<const double2*>(Ag + (size_t)t * 64 + coff));
    };
    if (w == 0) {
        // ---------------- diagonal warp ----------------
        for (int J = 0; J < n8; J++) {
            double* Sd = S8 + 64 * (J & 1);
            GF_CHOL_STAMP(0);
            if (J > 0) {
                nb_sync(1, 64);                                 // c_{J,J-1} parked in its slot, partial c_JJ in Sd
                const int t = tix(J, J - 1);
                const double a0 = T.frag(t, 0, lane), a1 = T.frag(t, 1, lane);
                GF_CHOL_STAMP(1);
                const double b0 = Linv[64 * (J - 1) + lane], b1 = Linv[64 * (J - 1) + 32 + lane];
                double x0 = 0.0, x1 = 0.0;
                dmma884(x0, x1, a0, b0);
                dmma884(x0, x1, a1, b1);
                T.store_c(t, lane, x0, x1);                     // L_{J,J-1}
                __syncwarp();
                const double f0 = T.frag(t, 0, lane), f1 = T.frag(t, 1, lane);
                __threadfence_block();
                nb_arrive(2, NB_ALL);                           // panel J-1 is complete once the bulk warps have arrived too
                double d0[2] = {0.0, 0.0}, d1[2] = {0.0, 0.0};
                dmma884(d0[0], d0[1], f0, f0);
                dmma884(d1[0], d1[1], f1, f1);
                const double2 cp = *reinterpret_cast<const double2*>(Sd + coff);
                *reinterpret_cast<double2*>(Sd + coff) = make_double2(cp.x - (d0[0] + d1[0]), cp.y - (d0[1] + d1[1]));
            } else {
                const double2 av = a_pair(0);
                *reinterpret_cast<double2*>(Sd + coff) = av;
                GF_CHOL_STAMP(1);
            }
            __syncwarp();
            GF_CHOL_STAMP(2);
            const bool okd = chol8_inv(Sd, min(8, nc - 8 * J), Linv + 64 * J, J == n8 - 1 ? Ld : nullptr);
            if (!okd && lane == 0) *s_fail = 1;
            // inv(L_JJ) published.  The diagonal warp may run one panel ahead of the slowest bulk warp: two barriers, by parity
            if (J + 1 < n8) { __threadfence_block(); nb_arrive(3 + (J & 1), NB_ALL); }
            GF_CHOL_STAMP(3);
        }
    } else {
        // ---------------- bulk warps ----------------
        // Every phase first issues ALL of its shared-memory loads and only then its MMAs: a warp issues in order, and an MMA
        // that waits for its own operand load (LDS ~30 cycles) while nothing else is in flight costs 3-4x its issue slot.
        const int bi = w - 1;
        double acc[R][4][2];      // sums of the panel being prepared: [row slot][k-half + 2 * panel parity][2]
        double dsum[R][2][2];     // running sums of the diagonal tile of every owned row: sum_p L_{row,p} L_{row,p}^T over the finished panels
#pragma unroll
        for (int s = 0; s < R; s++) {
#pragma unroll
            for (int k = 0; k < 4; k++) acc[s][k][0] = acc[s][k][1] = 0.0;
            dsum[s][0][0] = dsum[s][0][1] = dsum[s][1][0] = dsum[s][1][1] = 0.0;
        }
        for (int J = 0; J < n8; J++) {
            GF_CHOL_STAMP(0);
            const bool own_next = (J + 1 < n8) && ((J + 1) % CH_BULK == bi);       // this warp owns block row J+1
            if (J > 0) {
                nb_sync(3 + ((J - 1) & 1), NB_ALL);             // inv(L_J-1,J-1) published
                const double b0 = Linv[64 * (J - 1) + lane], b1 = Linv[64 * (J - 1) + 32 + lane];
                GF_CHOL_STAMP(1);
                // TRSM of panel J-1, rows > J (row J belongs to the diagonal warp): loads, MMAs, stores
                double ta0[R], ta1[R];
#pragma unroll
                for (int s = 0; s < R; s++) {
                    const int row = bi + CH_BULK * s;
                    ta0[s] = ta1[s] = 0.0;
                    if (row > J && row < n8) { const int t = tix(row, J - 1); ta0[s] = T.frag(t, 0, lane); ta1[s] = T.frag(t, 1, lane); }
                }
#pragma unroll
                for (int s = 0; s < R; s++) {
                    const int row = bi + CH_BULK * s;
                    if (row > J && row < n8) {
                        double x0 = 0.0, x1 = 0.0;
                        dmma884(x0, x1, ta0[s], b0);
                        dmma884(x0, x1, ta1[s], b1);
                        T.store_c(tix(row, J - 1), lane, x0, x1);
                    }
                }
                __syncwarp();
                // the new tiles join the running diagonal sums of their rows
#pragma unroll
                for (int s = 0; s < R; s++) {
                    const int row = bi + CH_BULK * s;
                    if (row > J && row < n8) { const int t = tix(row, J - 1); ta0[s] = T.frag(t, 0, lane); ta1[s] = T.frag(t, 1, lane); }
                }
#pragma unroll
                for (int s = 0; s < R; s++) {
                    const int row = bi + CH_BULK * s;
                    if (row > J && row < n8) {
                        dmma884(dsum[s][0][0], dsum[s][0][1], ta0[s], ta0[s]);
                        dmma884(dsum[s][1][0], dsum[s][1][1], ta1[s], ta1[s]);
                    }
                }
            }
            if (own_next) {
                // partial next diagonal tile: A_{J+1,J+1} - sum_{p<J} L_{J+1,p} L_{J+1,p}^T, parked in S8 for the diagonal warp
                const double2 av = a_pair(tix(J + 1, J + 1));
                double c0 = av.x, c1 = av.y;
#pragma unroll
                for (int s = 0; s < R; s++)
                    if (bi + CH_BULK * s == J + 1) { c0 -= dsum[s][0][0] + dsum[s][1][0]; c1 -= dsum[s][0][1] + dsum[s][1][1]; }
                *reinterpret_cast<double2*>(S8 + 64 * ((J + 1) & 1) + coff) = make_double2(c0, c1);
            }
            GF_CHOL_STAMP(2);
            if (J > 0) nb_sync(2, NB_ALL);                      // panel J-1 complete (bulk tiles + the diagonal warp's L_{J,J-1})
            GF_CHOL_STAMP(3);
            // ---- finish the tiles (row, J), row > J: c = A - sums, parked in the tile's slot in fragment order ----
            {
                double fa0[R], fa1[R], fb0 = 0.0, fb1 = 0.0;
                double2 fav[R];
                if (J > 0) { const int tb = tix(J, J - 1); fb0 = T.frag(tb, 0, lane); fb1 = T.frag(tb, 1, lane); }
#pragma unroll
                for (int s = 0; s < R; s++) {
                    const int row = bi + CH_BULK * s;
                    fa0[s] = fa1[s] = 0.0; fav[s] = make_double2(0.0, 0.0);
                    if (row > J && row < n8) {
                        const int t = tix(row, J);
                        if (J > 0) { fa0[s] = T.frag(t - 1, 0, lane); fa1[s] = T.frag(t - 1, 1, lane); }
                        fav[s] = a_pair(t);
                    }
                }
#pragma unroll
                for (int pass = 0; pass < 2; pass++) {          // row J+1 first: the diagonal warp waits for it
#pragma unroll
                    for (int s = 0; s < R; s++) {
                        const int row = bi + CH_BULK * s;
                        if (row > J && row < n8 && ((row == J + 1) == (pass == 0))) {
                            if (J > 0) {
                                dmma884(acc[s][0][0], acc[s][0][1], fa0[s], fb0);
                                dmma884(acc[s][1][0], acc[s][1][1], fa1[s], fb1);
                            }
                            const double c0 = fav[s].x - ((acc[s][0][0] + acc[s][1][0]) + (acc[s][2][0] + acc[s][3][0]));
                            const double c1 = fav[s].y - ((acc[s][0][1] + acc[s][1][1]) + (acc[s][2][1] + acc[s][3][1]));
                            T.store_c(tix(row, J), lane, c0, c1);
                        }
                    }
                    if (pass == 0 && own_next) { __threadfence_block(); nb_arrive(1, 64); }        // the diagonal warp may start panel J+1
                }
            }
            GF_CHOL_STAMP(4);
            // ---- sums of panel J+1 over the panels < J (final), rows > J+1: address walk, four panels (16 loads, 8 MMAs per row) per step ----
            if (J + 2 < n8) {
                const int tb0 = tix(J + 1, 0);
                bool act[R];
                unsigned ua[R];
#pragma unroll
                for (int s = 0; s < R; s++) {
                    const int row = bi + CH_BULK * s;
                    act[s] = row > J + 1 && row < n8;
                    ua[s] = T.sb + 8u * (unsigned)(tix(row, 0) * 64 + lane);
#pragma unroll
                    for (int k = 0; k < 4; k++) acc[s][k][0] = acc[s][k][1] = 0.0;
                }
                if (!SPILL) {
                    const unsigned ub = T.sb + 8u * (unsigned)(tb0 * 64 + lane);
                    unsigned off = 0;
                    int p = 0;
                    for (; p + 3 < J; p += 4, off += 2048u) {
                        double bq[8];
#pragma unroll
                        for (int k = 0; k < 8; k++) bq[k] = lds_f64(ub + off + 256u * k);
#pragma unroll
                        for (int s = 0; s < R; s++)
                            if (act[s]) {
                                double aq[8];
#pragma unroll
                                for (int k = 0; k < 8; k++) aq[k] = lds_f64(ua[s] + off + 256u * k);
#pragma unroll
                                for (int k = 0; k < 8; k++) dmma884(acc[s][k & 3][0], acc[s][k & 3][1], aq[k], bq[k]);
                            }
                    }
                    if (p + 1 < J) {
                        double bq[4];
#pragma unroll
                        for (int k = 0; k < 4; k++) bq[k] = lds_f64(ub + off + 256u * k);
#pragma unroll
                        for (int s = 0; s < R; s++)
                            if (act[s]) {
                                double aq[4];
#pragma unroll
                                for (int k = 0; k < 4; k++) aq[k] = lds_f64(ua[s] + off + 256u * k);
#pragma unroll
                                for (int k = 0; k < 4; k++) dmma884(acc[s][k][0], acc[s][k][1], aq[k], bq[k]);
                            }
                        p += 2; off += 1024u;
                    }
                    if (p < J) {
                        const double b00 = lds_f64(ub + off), b01 = lds_f64(ub + off + 256u);
#pragma unroll
                        for (int s = 0; s < R; s++)
                            if (act[s]) {
                                const double a00 = lds_f64(ua[s] + off), a01 = lds_f64(ua[s] + off + 256u);
                                dmma884(acc[s][2][0], acc[s][2][1], a00, b00);
                                dmma884(acc[s][3][0], acc[s][3][1], a01, b01);
                            }
                    }
                } else {
                    for (int p = 0; p < J; p++) {
                        const double b0 = T.frag(tb0 + p, 0, lane), b1 = T.frag(tb0 + p, 1, lane);
#pragma unroll
                        for (int s = 0; s < R; s++)
                            if (act[s]) {
                                const int ta = tix(bi + CH_BULK * s, p);
                                const double a0 = T.frag(ta, 0, lane), a1 = T.frag(ta, 1, lane);
                                if (p & 1) { dmma884(acc[s][2][0], acc[s][2][1], a0, b0); dmma884(acc[s][3][0], acc[s][3][1], a1, b1); }
                                else { dmma884(acc[s][0][0], acc[s][0][1], a0, b0); dmma884(acc[s][1][0], acc[s][1][1], a1, b1); }
                            }
                    }
                }
            }
            GF_CHOL_STAMP(5);
        }
    }
    __syncthreads();
    return *reinterpret_cast<volatile int*>(s_fail) == 0;
}

// ------------------------------------------------------------------------------------------------
// Back substitution  L^T y = z  over the leading nc x nc part of the factor (z = row nc of the factor), the whole CTA, as a
// two-stage pipeline so that the dependent chain is ~220 cycles per 8x8 block and meets no CTA-wide barrier:
//   warp 0 ("chain")  per block J from the bottom: rhs_J = zz_J - L_{J+1,J}^T y_{J+1} (its own, freshest term, in registers),
//                     y_J = L_JJ^-T rhs_J through the stored inverse, publish y_J.
//   warps 1.. ("helpers")  when y_I is published: zz_K -= L_{I,K}^T y_I for all columns of the blocks K < I-1, one column per
//                     thread, all loads issued before the 2 x 4-deep FMA chains.  Their result for y_I is needed by the chain
//                     two blocks later, so it never waits for them in steady state.
// zz: nr doubles of shared memory (running right-hand side), y: nc doubles (output).  Named barriers 5,6 (y_I published, by
// parity) and 7,8 (helpers done with y_I, by parity); the analysis of why two of each suffice is in DESIGN.md.
template <bool SPILL>
__device__ __forceinline__ void chol_backsubst(const TileStoreT<SPILL>& T, const double* __restrict__ Linv, const double* __restrict__ Ld,
                                               double* __restrict__ y, double* __restrict__ zz, int nc)
{
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int ir = nc >> 3, rr = nc & 7;              // tile row / local row of the right-hand-side row
    for (int c = tid; c < nc; c += ST_THREADS) zz[c] = (c >> 3) == ir ? Ld[rr * 8 + (c & 7)] : T.at(tix(ir, c >> 3), rr, c & 7);
    __syncthreads();
    const int jtop = (nc - 1) >> 3;
    constexpr int NB_ALL = ST_THREADS;
    if (w == 0) {
        const int k = lane & 7;
        double yprev = 0.0;                                   // y_{J+1}[k] (lane k, replicated in the four lane groups)
        for (int J = jtop; J >= 0; J--) {
            const int c0 = 8 * J;
            // operands that do not depend on the helpers: the inverse column and the tile column of the chain's own term
            const double* Li = Linv + 64 * J + (k >> 2) * 32 + (k & 3);
            double li[8], lt[8];
#pragma unroll
            for (int r = 0; r < 8; r++) li[r] = Li[r * 4];
            if (J < jtop) {
                const int t = tix(J + 1, J);
#pragma unroll
                for (int q = 0; q < 8; q++) lt[q] = T.at(t, q, k);
            }
            if (J + 2 <= jtop) nb_sync(7 + ((J + 2) & 1), NB_ALL);          // helpers are done with y_{J+2}: zz_J is final up to the chain's own term
            double rhs = (c0 + k < nc) ? zz[c0 + k] : 0.0;
            if (J < jtop) {
                double u0 = 0.0, u1 = 0.0;
#pragma unroll
                for (int q = 0; q < 8; q += 2) {
                    u0 = fma(lt[q], __shfl_sync(0xffffffffu, yprev, q), u0);
                    u1 = fma(lt[q + 1], __shfl_sync(0xffffffffu, yprev, q + 1), u1);
                }
                rhs -= u0 + u1;
            }
            double s0 = 0.0, s1 = 0.0;
#pragma unroll
            for (int r = 0; r < 8; r += 2) {
                s0 = fma((r >= k) ? li[r] : 0.0, __shfl_sync(0xffffffffu, rhs, r), s0);
                s1 = fma((r + 1 >= k) ? li[r + 1] : 0.0, __shfl_sync(0xffffffffu, rhs, r + 1), s1);
            }
            const double yk = (c0 + k < nc) ? s0 + s1 : 0.0;
            if (lane < 8 && c0 + lane < nc) y[c0 + lane] = yk;
            yprev = yk;
            if (J >= 2) { __threadfence_block(); nb_arrive(5 + (J & 1), NB_ALL); }      // y_J published (helpers have columns to update only for J >= 2)
        }
    } else {
        const int ht = tid - 32;                              // helper thread index, ST_THREADS - 32 of them
        for (int I = jtop; I >= 2; I--) {
            nb_sync(5 + (I & 1), NB_ALL);
            const int c0 = 8 * I, cend = 8 * (I - 1);        // columns [0, cend)
            double yv[8];
#pragma unroll
            for (int r = 0; r < 8; r++) yv[r] = (c0 + r < nc) ? y[c0 + r] : 0.0;
            for (int c = ht; c < cend; c += ST_THREADS - 32) {
                const int t = tix(I, c >> 3);
                double lv[8];
#pragma unroll
                for (int r = 0; r < 8; r++) lv[r] = T.at(t, r, c & 7);
                double u0 = zz[c], u1 = 0.0;
#pragma unroll
                for (int r = 0; r < 8; r += 2) { u0 = fma(-lv[r], yv[r], u0); u1 = fma(-lv[r + 1], yv[r + 1], u1); }
                zz[c] = u0 + u1;
            }
            __threadfence_block();
            nb_arrive(7 + (I & 1), NB_ALL);
        }
    }
    __syncthreads();
}

}  // namespace gfba
