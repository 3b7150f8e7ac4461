// yolo_kernels.cuh -- the device half of gf_detector: darknet's inference forward pass (network_predict on the CPU build),
// bit for bit.  Built with -fmad=false, and every float operation whose rounding matters is written with an _rn intrinsic, so
// nothing is contracted or reordered:
//   letterbox   BGR8 -> planar float / 255 (the node's mat_to_image; its rgbgr_image and fetchInThread's undo each other) ->
//               resize_image's two bilinear passes -> embedded at the centre of a 0.5 fill, one thread per output value
//   conv        implicit GEMM, out[m][p] = 0 + w[m][0] x[0][p] + w[m][1] x[1][p] + ... in gemm_nn's k = c size^2 + ky size + kx
//               order, as one sequential FMUL / FADD chain per output in registers; the padding's zero products are skipped
//               (adding +-0 to a sum that starts at +0 never changes it).  Epilogue: normalize_cpu's double division by
//               sqrt(var) + 1e-6f (the denominator precomputed on the host in double), scale_bias, add_bias, activation.
//   the rest    maxpool, reorg (darknet's forward = 0 mapping), upsample, shortcut, and the [region] / [yolo] heads'
//               logistic / softmax with their exp in double by gm_exp (correctly rounded)
// Every kernel runs a batch of images: image i's values sit at i * (the layer's per-image size) in each buffer.  A conv CTA's
// pixel tile lies within one image, so each output keeps its sequential k order whatever the batch.  Maxpool, upsample and the
// heads see the batch as more channels (anchors), which their per-channel mapping already handles; reorg and shortcut take the
// image from blockIdx.y.
#pragma once
#include <cfloat>
#include <cstdint>

#include "gm_math.h"

namespace gfy {

// leaky_activate: (x > 0) ? x : .1 * x, the product in double
__device__ __forceinline__ float act_leaky(float x) { return x > 0.f ? x : __double2float_rn(__dmul_rn(0.1, (double)x)); }
__device__ __forceinline__ float act(float x, int a) { return a ? act_leaky(x) : x; }
// logistic_activate: 1. / (1. + exp(-x)) in double
__device__ __forceinline__ float logistic(float x) { return __double2float_rn(__ddiv_rn(1.0, __dadd_rn(1.0, gm_exp(-(double)x)))); }

constexpr int LB_MAX = 64;                 // frames per letterbox launch (GF_DETECTOR_BATCH_MAX)

// per-frame geometry of one letterbox launch: the frame, its size and its letterboxed size at the net size
struct LbFrames {
    const uint8_t* bgr[LB_MAX];
    int pitch[LB_MAX], w[LB_MAX], h[LB_MAX], new_w[LB_MAX], new_h[LB_MAX];
};

// one output value of letterbox_image(mat_to_image(frame), nw, nh) per thread; blockIdx.z = 3 frame + channel; out is
// [frame][3][nh][nw]
__global__ void k_yolo_letterbox(const __grid_constant__ LbFrames f, int nw, int nh, float* __restrict__ out)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, k = blockIdx.z % 3, im = blockIdx.z / 3;
    if (x >= nw) return;
    const uint8_t* __restrict__ bgr = f.bgr[im];
    const int pitch = f.pitch[im], w = f.w[im], h = f.h[im], new_w = f.new_w[im], new_h = f.new_h[im];
    const int dx = (nw - new_w) / 2, dy = (nh - new_h) / 2;
    const int c = x - dx, r = y - dy;
    float v = 0.5f;
    if (c >= 0 && c < new_w && r >= 0 && r < new_h) {
        const float w_scale = __fdiv_rn((float)(w - 1), (float)(new_w - 1));
        const float h_scale = __fdiv_rn((float)(h - 1), (float)(new_h - 1));
        auto px = [&](int ix, int iy) { return __double2float_rn(__ddiv_rn((double)bgr[(size_t)iy * pitch + 3 * ix + k], 255.0)); };
        auto part = [&](int row) {            // resize_image's first (horizontal) pass at column c
            if (c == new_w - 1 || w == 1) return px(w - 1, row);
            const float sx = __fmul_rn((float)c, w_scale);
            const int ix = (int)sx;
            const float fx = __fsub_rn(sx, (float)ix);
            return __fadd_rn(__fmul_rn(__fsub_rn(1.f, fx), px(ix, row)), __fmul_rn(fx, px(ix + 1, row)));
        };
        const float sy = __fmul_rn((float)r, h_scale);
        const int iy = (int)sy;
        const float fy = __fsub_rn(sy, (float)iy);
        v = __fmul_rn(__fsub_rn(1.f, fy), part(iy));
        if (!(r == new_h - 1 || h == 1)) v = __fadd_rn(v, __fmul_rn(fy, part(iy + 1)));
    }
    out[(((size_t)im * 3 + k) * nh + y) * nw + x] = v;
}

struct ConvArgs {
    const float* in;       // [image][C][H][W]
    const float* w;        // [M][K], K = C size^2
    float* out;            // [image][M][OH][OW]
    const float* bias;
    const float* scale;    // batch norm only
    const float* mean;
    const double* den;     // sqrt((double)var) + (double)1e-6f
    int C, H, W, M, K, OW, N, size, stride, pad, bn, act;
};

constexpr int CONV_THREADS = 256, CONV_BK = 8;

// CTA tile BM filters x BN pixels of one image, 256 threads each holding (BM / 16) x (BN / 16) sums; K staged through shared
// memory in chunks of CONV_BK, double-buffered, the next chunk's loads issued before the current chunk's arithmetic.
// BATCH: blockIdx.x = image * ceil(N / BN) + pixel tile.  Without it (one image) the image terms fold away and the loop keeps
// one image's addressing: the image offset costs the gather loop instructions, so a lone frame does not pay for it.
template <int BM, int BN, bool BATCH>
__device__ __forceinline__ void conv_body(const ConvArgs& a)
{
    constexpr int TM = BM / 16, TN = BN / 16;
    constexpr int WL = BM * CONV_BK / CONV_THREADS, XL = BN * CONV_BK / CONV_THREADS;
    __shared__ float Ws[2][CONV_BK][BM];
    __shared__ float Xs[2][CONV_BK][BN];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    // the image's channels continue the batch's: channel ch of image im is channel im C + ch of the buffer (a.in stays the
    // kernel parameter, so the loop's addressing is that of one image)
    const int tiles = (a.N + BN - 1) / BN, im = BATCH ? blockIdx.x / tiles : 0, imc = im * a.C;
    const int m0 = blockIdx.y * BM, n0 = (blockIdx.x - im * tiles) * BN;
    const int ss = a.size * a.size;
    // the pixel this thread gathers for the X tile, fixed over all chunks
    const int xp = tid % BN, xk0 = tid / BN;
    const int gp = n0 + xp;
    const bool pix_ok = gp < a.N;
    const int oy = pix_ok ? gp / a.OW : 0, ox = pix_ok ? gp - (gp / a.OW) * a.OW : 0;
    const int iy0 = oy * a.stride - a.pad, ix0 = ox * a.stride - a.pad;
    const size_t HW = (size_t)a.H * a.W;

    float wr[WL], xr[XL];
    auto load = [&](int k0) {
#pragma unroll
        for (int r = 0; r < WL; r++) {
            const int e = tid + CONV_THREADS * r, m = e / CONV_BK, kk = e % CONV_BK;
            const int gm = m0 + m, gk = k0 + kk;
            wr[r] = (gm < a.M && gk < a.K) ? __ldg(a.w + (size_t)gm * a.K + gk) : 0.f;
        }
#pragma unroll
        for (int r = 0; r < XL; r++) {
            const int gk = k0 + xk0 + r * (CONV_THREADS / BN);
            float v = 0.f;
            if (pix_ok && gk < a.K) {
                const int ch = gk / ss, rem = gk - ch * ss, ky = rem / a.size, kx = rem - ky * a.size;
                const int iy = iy0 + ky, ix = ix0 + kx;
                if (iy >= 0 && iy < a.H && ix >= 0 && ix < a.W) v = __ldg(a.in + (imc + ch) * HW + (size_t)iy * a.W + ix);
            }
            xr[r] = v;
        }
    };
    auto store = [&](int b) {
#pragma unroll
        for (int r = 0; r < WL; r++) {
            const int e = tid + CONV_THREADS * r;
            Ws[b][e % CONV_BK][e / CONV_BK] = wr[r];
        }
#pragma unroll
        for (int r = 0; r < XL; r++) Xs[b][xk0 + r * (CONV_THREADS / BN)][xp] = xr[r];
    };

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = 0.f;

    const int nk = (a.K + CONV_BK - 1) / CONV_BK;
    load(0);
    store(0);
    __syncthreads();
    for (int kc = 0; kc < nk; kc++) {
        const int b = kc & 1;
        if (kc + 1 < nk) load((kc + 1) * CONV_BK);
#pragma unroll
        for (int kk = 0; kk < CONV_BK; kk++) {
            float wv[TM], xv[TN];
#pragma unroll
            for (int i = 0; i < TM; i++) wv[i] = Ws[b][kk][ty + 16 * i];
#pragma unroll
            for (int j = 0; j < TN; j++) xv[j] = Xs[b][kk][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < TM; i++)
#pragma unroll
                for (int j = 0; j < TN; j++) acc[i][j] = __fadd_rn(acc[i][j], __fmul_rn(wv[i], xv[j]));
        }
        if (kc + 1 < nk) store(b ^ 1);
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < TM; i++) {
        const int m = m0 + ty + 16 * i;
        if (m >= a.M) continue;
        const float bias = a.bias[m];
        float sc = 0.f, mu = 0.f;
        double den = 1.0;
        if (a.bn) { sc = a.scale[m]; mu = a.mean[m]; den = a.den[m]; }
#pragma unroll
        for (int j = 0; j < TN; j++) {
            const int p = n0 + tx + 16 * j;
            if (p >= a.N) continue;
            float v = acc[i][j];
            if (a.bn) {
                v = __double2float_rn(__ddiv_rn((double)__fsub_rn(v, mu), den));
                v = __fmul_rn(v, sc);
            }
            v = __fadd_rn(v, bias);
            a.out[((size_t)im * a.M + m) * a.N + p] = act(v, a.act);
        }
    }
}

// one image / a batch of images: the same body (so the same sums), compiled for each
template <int BM, int BN>
__global__ void __launch_bounds__(CONV_THREADS) k_yolo_conv(ConvArgs a) { conv_body<BM, BN, false>(a); }
template <int BM, int BN>
__global__ void __launch_bounds__(CONV_THREADS) k_yolo_conv_batch(ConvArgs a) { conv_body<BM, BN, true>(a); }

// forward_maxpool_layer: the first strictly larger value wins, outside the input counts as -FLT_MAX
__global__ void k_yolo_maxpool(const float* __restrict__ in, float* __restrict__ out, int W, int H, int C, int OW, int OH,
                               int size, int stride, int pad)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)OW * OH * C) return;
    const int j = (int)(idx % OW), i = (int)(idx / OW % OH), k = (int)(idx / ((long)OW * OH));
    const int off = -pad / 2;
    float mx = -FLT_MAX;
    for (int n = 0; n < size; n++)
        for (int m = 0; m < size; m++) {
            const int y = off + i * stride + n, x = off + j * stride + m;
            const float v = (y >= 0 && y < H && x >= 0 && x < W) ? in[((size_t)k * H + y) * W + x] : -FLT_MAX;
            mx = v > mx ? v : mx;
        }
    out[idx] = mx;
}

// forward_reorg_layer without reverse: reorg_cpu(in, w, h, c, batch, stride, forward = 0), out[in_index] = in[out_index];
// blockIdx.y = image (reorg_cpu's batch term is one image's w h c values)
__global__ void k_yolo_reorg(const float* __restrict__ in, float* __restrict__ out, int w, int h, int c, int stride)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)w * h * c) return;
    in += (size_t)blockIdx.y * w * h * c;
    out += (size_t)blockIdx.y * w * h * c;
    const int i = (int)(idx % w), j = (int)(idx / w % h), k = (int)(idx / ((long)w * h));
    const int out_c = c / (stride * stride);
    const int c2 = k % out_c, offset = k / out_c;
    const int w2 = i * stride + offset % stride, h2 = j * stride + offset / stride;
    out[idx] = in[w2 + (long)w * stride * (h2 + (long)h * stride * c2)];
}

// forward_upsample_layer: out = scale * in at (x / stride, y / stride)
__global__ void k_yolo_upsample(const float* __restrict__ in, float* __restrict__ out, int w, int h, int c, int stride, float scale)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const int OW = w * stride, OH = h * stride;
    if (idx >= (long)OW * OH * c) return;
    const int x = (int)(idx % OW), y = (int)(idx / OW % OH), k = (int)(idx / ((long)OW * OH));
    out[idx] = __fmul_rn(scale, in[((size_t)k * h + y / stride) * w + x / stride]);
}

// forward_shortcut_layer: out = prev; out[mapped] = alpha out + beta add over shortcut_cpu's overlap; then the activation;
// blockIdx.y = image
__global__ void k_yolo_shortcut(const float* __restrict__ prev, const float* __restrict__ add, float* __restrict__ out,
                                int w1, int h1, int c1, int w2, int h2, int c2, float alpha, float beta, int act_)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)w2 * h2 * c2) return;
    prev += (size_t)blockIdx.y * w2 * h2 * c2;
    out += (size_t)blockIdx.y * w2 * h2 * c2;
    add += (size_t)blockIdx.y * w1 * h1 * c1;
    int stride = w1 / w2, sample = w2 / w1;
    if (stride < 1) stride = 1;
    if (sample < 1) sample = 1;
    const int minw = w1 < w2 ? w1 : w2, minh = h1 < h2 ? h1 : h2, minc = c1 < c2 ? c1 : c2;
    const int x = (int)(idx % w2), y = (int)(idx / w2 % h2), k = (int)(idx / ((long)w2 * h2));
    float v = prev[idx];
    if (k < minc && x % sample == 0 && y % sample == 0 && x / sample < minw && y / sample < minh) {
        const int i = x / sample, j = y / sample;
        v = __fadd_rn(__fmul_rn(alpha, v), __fmul_rn(beta, add[i * stride + (size_t)w1 * (j * stride + (size_t)h1 * k)]));
    }
    out[idx] = act(v, act_);
}

// forward_region_layer / forward_yolo_layer on the CPU build: one thread per (anchor, cell) over its (classes + coords + 1)
// entries.  Region: logistic on x, y and objectness, then softmax over the classes (of the raw input) or logistic on them.
// Yolo: logistic on everything but w and h.
__global__ void k_yolo_head(const float* __restrict__ in, float* __restrict__ out, int wh, int num, int classes, int yolo, int softmax)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= wh * num) return;
    const int n = t / wh, loc = t - n * wh;
    const int E = classes + 5;
    const size_t base = (size_t)n * wh * E + loc;
    for (int e = 0; e < 5; e++) {
        const float x = in[base + (size_t)e * wh];
        out[base + (size_t)e * wh] = (e == 2 || e == 3) ? x : logistic(x);
    }
    if (yolo || !softmax) {
        for (int j = 0; j < classes; j++) out[base + (size_t)(5 + j) * wh] = logistic(in[base + (size_t)(5 + j) * wh]);
        return;
    }
    // softmax(input, classes, temp = 1, stride = wh): e = exp(x / 1 - largest / 1), sum += e, then e / sum
    float largest = -FLT_MAX;
    for (int j = 0; j < classes; j++) {
        const float x = in[base + (size_t)(5 + j) * wh];
        if (x > largest) largest = x;
    }
    float sum = 0.f;
    for (int j = 0; j < classes; j++) {
        const float e = __double2float_rn(gm_exp((double)__fsub_rn(in[base + (size_t)(5 + j) * wh], largest)));
        sum = __fadd_rn(sum, e);
        out[base + (size_t)(5 + j) * wh] = e;
    }
    for (int j = 0; j < classes; j++) out[base + (size_t)(5 + j) * wh] = __fdiv_rn(out[base + (size_t)(5 + j) * wh], sum);
}

}  // namespace gfy
