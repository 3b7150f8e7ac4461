// fe_eig.cuh -- cv::pyrDown (u8) and cv::cornerMinEigenVal(blockSize 3, Sobel 3), bit-exact with cv2 4.13.
//
// Replaces the dense part of cv::goodFeaturesToTrack (reference feature_tracker.cpp:198) and the
// pyramid construction inside cv::calcOpticalFlowPyrLK (:118-153).  Arithmetic: oracle/fe_cv_restate.c.
//
// Min-eig, one fused kernel (u8 image in, float map out; no Sobel/cov image in HBM):
//   dx = fma(d0+d2, s, 2s*d1)                 d  = P[x+1]-P[x-1] per row           (float32)
//   dy = r2 - r0,  r = fma(s,P[x+1], fma(2s,P[x], s*P[x-1]))   (columns >= (w/32)*32: (s*P[x-1]+2s*P[x])+s*P[x+1])
//   cov = (dx*dx, dx*dy, dy*dy)  float32
//   box: row sums (S0+S1)+S2 in double; column sums are ONE RUNNING double sum per column and channel
//        down the whole image in OpenCV (s0 = SUM + D[y+1]; out = (float)s0; SUM = s0 - D[y-1]).
//        That chain is inherently sequential per column, but it is only two dependent DADDs per row; everything
//        else is not.  So the work is split in three kernels:
//          k_cov_rows    (parallel)  D[y][x] = the three row sums, as doubles, in a column-block-tiled layout with
//                                    the two reflected border rows materialised, so that the rows one chain warp needs
//                                    are one contiguous stream
//          k_box_chain   (serial)    one lane per (column, channel); the D stream is fetched ahead of the chain by
//                                    1-D TMA bulk copies into a shared-memory ring (cp.async.bulk + mbarrier), so the
//                                    chain runs at DADD latency: ~16 cycles per image row
//          k_eig_from_box (parallel) min-eig from the float box sums
//   eig = (a+c) - sqrt((a-c)^2 + b*b), a = c0/2, b = c1, c = c2/2                 (float32)
// Compile with -fmad=false.
#pragma once
#include "gf_common.cuh"

namespace gf {

// ------------------------------------------------------------------------------------------------
// pyrDown: out(y,x) = (sum_ij k_i k_j P[2y+i-2][2x+j-2] + 128) >> 8, k=[1 4 6 4 1], REFLECT_101
// ------------------------------------------------------------------------------------------------
constexpr int PD_TX = 32, PD_TY = 8;
// one PD_TX x PD_TY tile of the destination (blockIdx.x, blockIdx.y); k_pyr_down and the group form k_pyr_down_g
template <int V>
__device__ __forceinline__ void pyr_down_tile(const Level& src, uint8_t* dst, int dw, int dh, int dpitch)
{
    __shared__ uint8_t tile[2 * PD_TY + 3][2 * PD_TX + 4];
    __shared__ int rowf[2 * PD_TY + 3][PD_TX];
    const int ox = blockIdx.x * PD_TX, oy = blockIdx.y * PD_TY;
    const int tid = threadIdx.y * PD_TX + threadIdx.x;
    for (int i = tid; i < (2 * PD_TY + 3) * (2 * PD_TX + 3); i += PD_TX * PD_TY) {
        int r = i / (2 * PD_TX + 3), c = i - r * (2 * PD_TX + 3);
        int yy = reflect101(2 * oy - 2 + r, src.h), xx = reflect101(2 * ox - 2 + c, src.w);
        // tiles at the right/bottom edge may index beyond the last needed pixel: clamp keeps it legal
        yy = min(max(yy, 0), src.h - 1);
        xx = min(max(xx, 0), src.w - 1);
        tile[r][c] = __ldg(src.ptr + (size_t)yy * src.pitch + xx);
    }
    __syncthreads();
    for (int i = tid; i < (2 * PD_TY + 3) * PD_TX; i += PD_TX * PD_TY) {
        int r = i / PD_TX, c = i - r * PD_TX;
        const uint8_t* p = &tile[r][2 * c];
        rowf[r][c] = p[0] + 4 * p[1] + 6 * p[2] + 4 * p[3] + p[4];
    }
    __syncthreads();
    int x = ox + threadIdx.x, y = oy + threadIdx.y;
    if (x < dw && y < dh) {
        int r = 2 * threadIdx.y, c = threadIdx.x;
        int v = rowf[r][c] + 4 * rowf[r + 1][c] + 6 * rowf[r + 2][c] + 4 * rowf[r + 3][c] + rowf[r + 4][c];
        dst[(size_t)y * dpitch + x] = (uint8_t)((v + 128) >> 8);
    }
}
__global__ void __launch_bounds__(PD_TX* PD_TY) k_pyr_down(Level src, uint8_t* dst, int dw, int dh, int dpitch)
{
    pyr_down_tile<0>(src, dst, dw, dh, dpitch);
}

// ------------------------------------------------------------------------------------------------
// min-eig
// ------------------------------------------------------------------------------------------------
constexpr int EIG_TX = 128;   // columns per CTA (= threads per CTA) of k_cov_rows
constexpr int EIG_BAND = 16;  // rows per CTA of k_cov_rows
constexpr int BC_R = 16;      // padded rows per TMA chunk of k_box_chain (16 * 768 B = 12 KB)
constexpr int BC_NST = 6;     // ring stages: the chain runs 5 chunks (80 rows, > 1200 cycles) behind the copies
constexpr int BC_ROW = 96;    // doubles per padded row of one 32-column block: [channel 3][column 32]
constexpr size_t BC_SMEM = (size_t)BC_NST * BC_R * BC_ROW * sizeof(double);

// size in doubles of the tiled D buffer for a w x h image
__host__ __device__ inline size_t cov_rows_elems(int w, int h) { return (size_t)((w + 31) / 32) * (h + 2) * BC_ROW; }
// size in floats of the box-sum buffer
__host__ __device__ inline size_t box_elems(int w, int h) { return (size_t)3 * ((w + 31) / 32 * 32) * h; }

// tail: column >= (w/32)*32, where cv2's row filter runs its scalar (non-FMA) remainder loop
__device__ __forceinline__ void sobel_dxdy(int p00, int p01, int p02, int p10, int p11, int p12, int p20,
                                           int p21, int p22, bool tail, float& dx, float& dy)
{
    const float s = (float)(1.0 / (4.0 * 3.0 * 255.0));
    const float s2 = 2.f * s;
    (void)p11;
    int d0 = p02 - p00, d1 = p12 - p10, d2 = p22 - p20;
    dx = __fmaf_rn((float)(d0 + d2), s, s2 * (float)d1);
    float r0, r2;
    if (!tail) {
        r0 = __fmaf_rn(s, (float)p02, __fmaf_rn(s2, (float)p01, s * (float)p00));
        r2 = __fmaf_rn(s, (float)p22, __fmaf_rn(s2, (float)p21, s * (float)p20));
    } else {
        r0 = __fadd_rn(__fadd_rn(__fmul_rn(s, (float)p00), __fmul_rn(s2, (float)p01)), __fmul_rn(s, (float)p02));
        r2 = __fadd_rn(__fadd_rn(__fmul_rn(s, (float)p20), __fmul_rn(s2, (float)p21)), __fmul_rn(s, (float)p22));
    }
    dy = r2 - r0;
}

__device__ __forceinline__ float eig_from_box(double c0, double c1, double c2)
{
    float a = (float)c0 * 0.5f, b = (float)c1, c = (float)c2 * 0.5f;
    float t = a - c;
    return (a + c) - sqrtf(t * t + b * b);
}

// D in the layout k_box_chain streams: [column block x/32][padded row y+1][channel][x%32]; padded row 0 = D[1],
// padded row h+1 = D[h-2] (cv::boxFilter's BORDER_REFLECT_101 applied to the cov rows).
template <int V>
__device__ __forceinline__ void cov_rows_tile(const Level& img, double* __restrict__ Dt)
{
    constexpr int IH = EIG_BAND + 2, IWW = EIG_TX / 4 + 2, IP = 4 * IWW;   // image tile rows y0-1.., cols x0-4.. as 34 aligned words
    constexpr int CH = EIG_BAND, CW = EIG_TX + 2;         // dx/dy tile rows y0.., cols x0-1..
    __shared__ __align__(4) uint8_t timg[IH][IP];
    __shared__ float tdx[CH][CW + 2];
    __shared__ float tdy[CH][CW + 2];
    const int w = img.w, h = img.h;
    const int x0 = blockIdx.x * EIG_TX, y0 = blockIdx.y * EIG_BAND;
    const int tid = threadIdx.x;
    // aligned 32-bit loads (x0 is a multiple of 128, the pitch of 16): all of a thread's loads are in flight together.
    // Words left of the image or beyond the row pitch are skipped; the two border columns Sobel reads outside the image
    // (REFLECT_101: -1 -> 1, w -> w-2) are patched afterwards.
#pragma unroll
    for (int it = 0; it < (IH * IWW + EIG_TX - 1) / EIG_TX; it++) {
        const int i = tid + it * EIG_TX;
        if (i < IH * IWW) {
            const int r = i / IWW, j = i - r * IWW;
            const int yy = reflect101(min(max(y0 - 1 + r, -1), h), h);
            const int xa = x0 - 4 + 4 * j;
            if (xa >= 0 && xa < img.pitch)
                reinterpret_cast<uint32_t*>(&timg[r][0])[j] = __ldg(reinterpret_cast<const uint32_t*>(img.ptr + (size_t)yy * img.pitch + xa));
        }
    }
    __syncthreads();
    for (int r = tid; r < IH; r += EIG_TX) {
        if (x0 == 0) timg[r][3] = timg[r][5];                               // column -1 := column 1
        const int cw = w - (x0 - 4);                                          // tile slot of column w
        if (cw >= 2 && cw < IP) timg[r][cw] = timg[r][cw - 2];              // column w := column w-2
    }
    __syncthreads();
    // Sobel at slots whose (row, col) is inside the image; the column ring is filled by reflection below
    for (int i = tid; i < CH * CW; i += EIG_TX) {
        int r = i / CW, c = i - r * CW;
        int yy = y0 + r, xx = x0 - 1 + c;
        if (yy < h && xx >= 0 && xx < w) {
            const uint8_t* p = &timg[r][c + 2];  // timg row r <-> image row yy-1, byte c+2 <-> column xx-1
            float dx, dy;
            sobel_dxdy(p[0], p[1], p[2], p[IP], p[IP + 1], p[IP + 2], p[2 * IP], p[2 * IP + 1],
                       p[2 * IP + 2], xx >= (w / 32) * 32, dx, dy);
            tdx[r][c] = dx;
            tdy[r][c] = dy;
        }
    }
    __syncthreads();
    // cov is extended by REFLECT_101 at the *cov* level: column slot (-1) := slot (+1), slot (w) := slot (w-2)
    for (int i = tid; i < CH * 2; i += EIG_TX) {
        int r = i >> 1, c = (i & 1) ? CW - 1 : 0;
        int xx = x0 - 1 + c;
        if (xx == -1 || xx == w) {
            int rx = reflect101(xx, w) - (x0 - 1);
            if (rx >= 0 && rx < CW) { tdx[r][c] = tdx[r][rx]; tdy[r][c] = tdy[r][rx]; }
        }
    }
    if (x0 + EIG_TX > w) {   // last column block: the slot right of the image is not the tile's last slot
        for (int r = tid; r < CH; r += EIG_TX) {
            int c = w - (x0 - 1);           // slot of column w
            if (c >= 0 && c < CW && c - 2 >= 0) { tdx[r][c] = tdx[r][c - 2]; tdy[r][c] = tdy[r][c - 2]; }
        }
    }
    __syncthreads();
    const int x = x0 + tid;
    if (x >= w) return;
    const int nrows = min(EIG_BAND, h - y0);
    const size_t rows = (size_t)h + 2;
    double* dst = Dt + (size_t)(x >> 5) * rows * BC_ROW + (x & 31);
    for (int r = 0; r < nrows; r++) {
        const float* ax = &tdx[r][tid];  // cols x-1, x, x+1 <-> tid, tid+1, tid+2
        const float* ay = &tdy[r][tid];
        float xl = ax[0], xc = ax[1], xr = ax[2], yl = ay[0], yc = ay[1], yr = ay[2];
        double d0 = ((double)(xl * xl) + (double)(xc * xc)) + (double)(xr * xr);
        double d1 = ((double)(xl * yl) + (double)(xc * yc)) + (double)(xr * yr);
        double d2 = ((double)(yl * yl) + (double)(yc * yc)) + (double)(yr * yr);
        const int y = y0 + r;
        double* o = dst + (size_t)(y + 1) * BC_ROW;
        o[0] = d0; o[32] = d1; o[64] = d2;
        if (y == 1) { o = dst; o[0] = d0; o[32] = d1; o[64] = d2; }
        if (y == h - 2) { o = dst + (size_t)(h + 1) * BC_ROW; o[0] = d0; o[32] = d1; o[64] = d2; }
    }
}
__global__ void __launch_bounds__(EIG_TX) k_cov_rows(Level img, double* __restrict__ Dt)
{
    cov_rows_tile<0>(img, Dt);
}

// ---- mbarrier / 1-D TMA bulk copy (sm_90+) ----
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, unsigned bytes, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity)
{
    unsigned ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}

// The running column sums: one CTA of 3 warps per 32-column block, warp q <-> channel q, lane <-> column.
//   SUM = (0 + D[-1]) + D[0];  per row: s = SUM + D[y+1]; box[y] = (float)s; SUM = s - D[y-1]
// box: [channel][y][x] floats, row pitch bp = w rounded up to 32 (every lane stores).
template <int V>
__device__ __forceinline__ void box_chain_block(const double* __restrict__ Dt, float* __restrict__ box, int bp, int w, int h)
{
    extern __shared__ __align__(128) unsigned char bc_smem[];
    __shared__ __align__(8) unsigned long long mbar[BC_NST];
    double* buf = reinterpret_cast<double*>(bc_smem);              // [stage][row][channel][32]
    const int tid = threadIdx.x, lane = tid & 31, q = tid >> 5;
    const int x = blockIdx.x * 32 + lane;
    const int rows = h + 2, nchunk = (rows + BC_R - 1) / BC_R;
    const double* src = Dt + (size_t)blockIdx.x * rows * BC_ROW;
    if (tid == 0) {
        for (int i = 0; i < BC_NST; i++) mbar_init(&mbar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](int k) {
        const int r0 = k * BC_R, nr = min(BC_R, rows - r0);
        const unsigned bytes = (unsigned)(nr * BC_ROW * sizeof(double));
        mbar_expect_tx(&mbar[k % BC_NST], bytes);
        tma_load_1d(buf + (size_t)(k % BC_NST) * BC_R * BC_ROW, src + (size_t)r0 * BC_ROW, bytes, &mbar[k % BC_NST]);
    };
    if (tid == 0)
        for (int k = 0; k < BC_NST - 1 && k < nchunk; k++) issue(k);
    float* o = box + (size_t)q * bp * h + x;               // next output row of this lane (pitch bp >= 32-aligned w: no bounds test)
    double a = 0.0, b = 0.0, S = 0.0;
    for (int k = 0; k < nchunk; k++) {
        __syncthreads();                                   // everyone is done with the stage that is refilled next
        if (tid == 0 && k + BC_NST - 1 < nchunk) issue(k + BC_NST - 1);
        {
            unsigned spins = 0;
            while (!mbar_try_wait(&mbar[k % BC_NST], (unsigned)((k / BC_NST) & 1)))
                if (++spins > (1u << 24)) __trap();        // a lost copy must not hang the GPU
        }
        const double* B = buf + (size_t)(k % BC_NST) * BC_R * BC_ROW + q * 32 + lane;
        const int nr = min(BC_R, rows - k * BC_R);
        int r = 0;
        if (k == 0) {                                      // padded rows 0 and 1: D[-1] and D[0]
            a = B[0];
            b = B[BC_ROW];
            S = (0.0 + a) + b;
            r = 2;
        }
        if (r == 0 && nr == BC_R) {
#pragma unroll
            for (int rr = 0; rr < BC_R; rr++) {
                const double c = B[rr * BC_ROW];
                const double s = S + c;
                *o = (float)s;
                o += bp;
                S = s - a;
                a = b;
                b = c;
            }
        } else {
            for (; r < nr; r++) {
                const double c = B[r * BC_ROW];
                const double s = S + c;
                *o = (float)s;
                o += bp;
                S = s - a;
                a = b;
                b = c;
            }
        }
    }
}
__global__ void __launch_bounds__(96) k_box_chain(const double* __restrict__ Dt, float* __restrict__ box, int bp, int w, int h)
{
    box_chain_block<0>(Dt, box, bp, w, h);
}

template <int V>
__device__ __forceinline__ void eig_from_box_tile(const float* __restrict__ box, int bp, float* __restrict__ eig, int epitch, int w, int h)
{
    const int x = blockIdx.x * 64 + (threadIdx.x & 63);
    const int yb = blockIdx.y * 16 + (threadIdx.x >> 6);
    if (x >= w) return;
    const size_t plane = (size_t)bp * h;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int y = yb + 4 * j;
        if (y < h) {
            const size_t o = (size_t)y * bp + x;
            float a = box[o] * 0.5f, b = box[plane + o], c = box[2 * plane + o] * 0.5f;
            float t = a - c;
            eig[(size_t)y * epitch + x] = (a + c) - sqrtf(t * t + b * b);
        }
    }
}
__global__ void __launch_bounds__(256) k_eig_from_box(const float* __restrict__ box, int bp, float* __restrict__ eig, int epitch, int w, int h)
{
    eig_from_box_tile<0>(box, bp, eig, epitch, w, h);
}

}  // namespace gf
