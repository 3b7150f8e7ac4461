// fe_clahe.cuh -- cv::CLAHE::apply for 8-bit images (cv::createCLAHE(clip, Size(tiles_x, tiles_y))), the equalisation the
// reference applies to every camera image when the config key `equalize` is set (rosNodeTest.cpp:256-261).  Bit-exact with
// OpenCV 4.13; the op order follows the plain-C restatement tests/clahe_restate.c, which tests/test_clahe_oracle.py pins to cv2.
//
//   k_clahe_lut   one CTA per tile: histogram of the tile (the source read through the REFLECT_101 index map of the padded
//                 histogram source), clip, redistribution, 256-wide scan, u8 LUT
//   k_clahe_apply all tile LUTs staged in shared memory, bilinear blend of the four neighbouring tiles' LUTs, 16 px per thread
#pragma once
#include "gf_common.cuh"

namespace gf {

constexpr int CLAHE_MAX_TILES = 16;            // per dimension
constexpr int CLAHE_LUT_THREADS = 512;
constexpr int CLAHE_LUT_UNROLL = 4;
constexpr int CLAHE_APPLY_THREADS = 256;
constexpr int CLAHE_APPLY_ROWS = 8;            // image rows per CTA of k_clahe_apply

// Tile geometry as CLAHE_Impl::apply derives it (host side; see clahe_geometry)
struct ClaheGeom {
    int w, h, tiles_x, tiles_y, tw, th;
    int limit;                                 // integer clip limit, 0: no clipping
    float lut_scale, inv_tw, inv_th;           // 255.f / (tw * th), 1.f / tw, 1.f / th
};

inline int clahe_geometry(ClaheGeom& g, int w, int h, double clip_limit, int tiles_x, int tiles_y)
{
    if (tiles_x < 1 || tiles_y < 1 || tiles_x > CLAHE_MAX_TILES || tiles_y > CLAHE_MAX_TILES)
        return set_err(GF_ERR_INVALID_ARG, "CLAHE tile grid must be 1..16 x 1..16");
    if (!(clip_limit == clip_limit) || clip_limit > 1e6) return set_err(GF_ERR_INVALID_ARG, "CLAHE clip limit must be a number <= 1e6");
    // the histogram source is extended by REFLECT_101 on the bottom / right when EITHER dimension does not divide -- by a whole
    // tile row / column on a dimension that does
    const bool padded = (w % tiles_x) != 0 || (h % tiles_y) != 0;
    const int ew = padded ? w + tiles_x - w % tiles_x : w, eh = padded ? h + tiles_y - h % tiles_y : h;
    g.w = w; g.h = h; g.tiles_x = tiles_x; g.tiles_y = tiles_y;
    g.tw = ew / tiles_x; g.th = eh / tiles_y;
    const int area = g.tw * g.th;
    g.lut_scale = 255.f / (float)area;
    g.limit = 0;
    if (clip_limit > 0.0) {
        g.limit = (int)(clip_limit * area / 256);
        if (g.limit < 1) g.limit = 1;
    }
    g.inv_tw = 1.f / (float)g.tw; g.inv_th = 1.f / (float)g.th;
    return GF_OK;
}

// grid = tiles_x * tiles_y CTAs; lut: [tiles_y][tiles_x][256]
template <int V>
__device__ __forceinline__ void clahe_lut_tile(const uint8_t* src, long long pitch, const ClaheGeom& g, uint8_t* __restrict__ lut)
{
    constexpr int NW = CLAHE_LUT_THREADS / 32;
    __shared__ int wh[NW][256];                // per-warp histograms
    __shared__ int red[8], scan[8];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int tx = blockIdx.x % g.tiles_x, ty = blockIdx.x / g.tiles_x;
    for (int i = tid; i < NW * 256; i += CLAHE_LUT_THREADS) (&wh[0][0])[i] = 0;
    __syncthreads();
    const int area = g.tw * g.th, x0 = tx * g.tw, y0 = ty * g.th;
    // every lane of a warp runs the same trip count, so __match_any_sync sees the whole warp: lanes holding the same value
    // (a flat tile puts most of its pixels in one bin) add once, with the count of their group
    // (CLAHE_LUT_UNROLL independent loads in flight per thread before the first of them is binned)
    for (int i0 = 0; i0 < area; i0 += CLAHE_LUT_THREADS * CLAHE_LUT_UNROLL) {
        int v[CLAHE_LUT_UNROLL];
        #pragma unroll
        for (int u = 0; u < CLAHE_LUT_UNROLL; u++) {
            const int i = i0 + u * CLAHE_LUT_THREADS + tid;
            v[u] = 256;                        // no pixel
            if (i < area) {
                const int r = i / g.tw, c = i - r * g.tw;
                v[u] = __ldg(src + (long long)reflect101(y0 + r, g.h) * pitch + reflect101(x0 + c, g.w));
            }
        }
        #pragma unroll
        for (int u = 0; u < CLAHE_LUT_UNROLL; u++) {
            const unsigned peers = __match_any_sync(0xffffffffu, v[u]);
            if (v[u] < 256 && lane == __ffs(peers) - 1) atomicAdd(&wh[wid][v[u]], __popc(peers));
        }
    }
    __syncthreads();
    const bool bin = tid < 256;                // warps 0..7 own one bin per thread from here on
    int hv = 0, incl = 0;
    if (bin) {
        #pragma unroll
        for (int k = 0; k < NW; k++) hv += wh[k][tid];
        // clip: excess = sum of max(h - limit, 0)
        if (g.limit > 0) {
            int ex = hv > g.limit ? hv - g.limit : 0;
            hv = min(hv, g.limit);
            for (int o = 16; o > 0; o >>= 1) ex += __shfl_xor_sync(0xffffffffu, ex, o);
            if (lane == 0) red[wid] = ex;
        }
    }
    __syncthreads();
    if (bin) {
        // redistribution: every bin gets excess / 256, and the residual single increments go to bins 0, step, 2 step, ...
        // (step = max(256 / residual, 1)) until `residual` of them have been given
        if (g.limit > 0) {
            int excess = 0;
            #pragma unroll
            for (int k = 0; k < 8; k++) excess += red[k];
            const int batch = excess / 256, residual = excess - 256 * batch;
            hv += batch;
            if (residual) {
                const int step = max(256 / residual, 1);
                if (tid % step == 0 && tid / step < residual) hv += 1;
            }
        }
        // inclusive scan of the 256 bins
        incl = hv;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) scan[wid] = incl;
    }
    __syncthreads();
    if (bin) {
        int sum = incl;
        for (int k = 0; k < wid; k++) sum += scan[k];
        // lut = saturate_cast<uchar>(sum * lutScale): int -> float, one rounded product, round half to even
        const int q = __float2int_rn(__fmul_rn(__int2float_rn(sum), g.lut_scale));
        lut[(size_t)blockIdx.x * 256 + tid] = (uint8_t)min(max(q, 0), 255);
    }
}
__global__ void __launch_bounds__(CLAHE_LUT_THREADS) k_clahe_lut(const uint8_t* src, long long pitch, ClaheGeom g, uint8_t* __restrict__ lut)
{
    clahe_lut_tile<0>(src, pitch, g, lut);
}

// grid = ceil(h / CLAHE_APPLY_ROWS) CTAs, dynamic shared memory tiles_x * tiles_y * 256 bytes.
template <int V>
__device__ __forceinline__ void clahe_apply_rows(const uint8_t* src, long long pitch, const ClaheGeom& g, const uint8_t* __restrict__ lut,
                                                 uint8_t* __restrict__ dst, int dst_pitch)
{
    extern __shared__ __align__(16) uint8_t s_lut[];
    const int n16 = g.tiles_x * g.tiles_y * 16;
    for (int i = threadIdx.x; i < n16; i += CLAHE_APPLY_THREADS) ((uint4*)s_lut)[i] = __ldg((const uint4*)lut + i);
    __syncthreads();
    const int chunks = (g.w + 15) >> 4, y_begin = blockIdx.x * CLAHE_APPLY_ROWS, y_end = min(y_begin + CLAHE_APPLY_ROWS, g.h);
    for (int item = threadIdx.x; item < (y_end - y_begin) * chunks; item += CLAHE_APPLY_THREADS) {
        const int y = y_begin + item / chunks, x0 = (item % chunks) << 4;
        const float tyf = __fsub_rn(__fmul_rn((float)y, g.inv_th), 0.5f);
        int ty1 = __float2int_rd(tyf), ty2 = ty1 + 1;
        const float ya = __fsub_rn(tyf, (float)ty1), ya1 = __fsub_rn(1.f, ya);
        ty1 = max(ty1, 0); ty2 = min(ty2, g.tiles_y - 1);
        const uint8_t* L1 = s_lut + ty1 * g.tiles_x * 256;
        const uint8_t* L2 = s_lut + ty2 * g.tiles_x * 256;
        const uint8_t* sp = src + (long long)y * pitch + x0;
        uint8_t* dp = dst + (size_t)y * dst_pitch + x0;
        const int n = min(16, g.w - x0);
        const bool vec = n == 16 && ((((uintptr_t)sp) | ((uintptr_t)dp)) & 15) == 0;
        uint4 vin = make_uint4(0, 0, 0, 0), vout;
        uint8_t* in = (uint8_t*)&vin;
        uint8_t* out = (uint8_t*)&vout;
        if (vec) vin = __ldg((const uint4*)sp);
        else {
            #pragma unroll
            for (int k = 0; k < 16; k++) if (k < n) in[k] = __ldg(sp + k);
        }
        #pragma unroll
        for (int k = 0; k < 16; k++) {
            const int x = x0 + k;
            const float txf = __fsub_rn(__fmul_rn((float)x, g.inv_tw), 0.5f);
            int tx1 = __float2int_rd(txf), tx2 = tx1 + 1;
            const float xa = __fsub_rn(txf, (float)tx1), xa1 = __fsub_rn(1.f, xa);
            tx1 = max(tx1, 0); tx2 = min(tx2, g.tiles_x - 1);
            const int v = in[k];
            const float l11 = L1[tx1 * 256 + v], l12 = L1[tx2 * 256 + v], l21 = L2[tx1 * 256 + v], l22 = L2[tx2 * 256 + v];
            const float res = __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(l11, xa1), __fmul_rn(l12, xa)), ya1),
                                        __fmul_rn(__fadd_rn(__fmul_rn(l21, xa1), __fmul_rn(l22, xa)), ya));
            out[k] = (uint8_t)min(max(__float2int_rn(res), 0), 255);
        }
        if (vec) *(uint4*)dp = vout;
        else {
            #pragma unroll
            for (int k = 0; k < 16; k++) if (k < n) dp[k] = out[k];
        }
    }
}
__global__ void __launch_bounds__(CLAHE_APPLY_THREADS) k_clahe_apply(const uint8_t* src, long long pitch, ClaheGeom g,
                                                                     const uint8_t* __restrict__ lut, uint8_t* __restrict__ dst, int dst_pitch)
{
    clahe_apply_rows<0>(src, pitch, g, lut, dst, dst_pitch);
}

inline size_t clahe_lut_bytes(const ClaheGeom& g) { return (size_t)g.tiles_x * g.tiles_y * 256; }

// Once per device before the first enqueue_clahe (up to 64 KB of LUTs in k_clahe_apply's shared memory)
inline int clahe_prepare()
{
    static bool attr_done[64] = {};     // per device
    int dev = 0;
    GF_CUDA(cudaGetDevice(&dev));
    if (!attr_done[dev & 63]) {
        GF_CUDA(cudaFuncSetAttribute(k_clahe_apply, cudaFuncAttributeMaxDynamicSharedMemorySize, CLAHE_MAX_TILES * CLAHE_MAX_TILES * 256));
        attr_done[dev & 63] = true;
    }
    return GF_OK;
}

// Both kernels on s; lut: clahe_lut_bytes(g) bytes of device memory (16-byte aligned)
inline int enqueue_clahe(cudaStream_t s, const uint8_t* src, long long pitch, const ClaheGeom& g, uint8_t* lut, uint8_t* dst, int dst_pitch)
{
    k_clahe_lut<<<g.tiles_x * g.tiles_y, CLAHE_LUT_THREADS, 0, s>>>(src, pitch, g, lut); GF_LAUNCHED();
    k_clahe_apply<<<(g.h + CLAHE_APPLY_ROWS - 1) / CLAHE_APPLY_ROWS, CLAHE_APPLY_THREADS, clahe_lut_bytes(g), s>>>(src, pitch, g, lut, dst, dst_pitch); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

}  // namespace gf
