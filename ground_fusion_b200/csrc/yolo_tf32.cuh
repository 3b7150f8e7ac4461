// yolo_tf32.cuh -- the detector's TF32 convolution (gf_detector_set_precision(GF_DETECTOR_TF32)): the same implicit GEMM as
// k_yolo_conv, out[M filters][N pixels] over K = C size^2, on Hopper's tensor cores.  Not bit-exact with darknet; DESIGN.md
// "YOLO detector: the TF32 mode" has the contract and its error bound.
//   operands    both rounded to TF32 by cvt.rna.tf32.f32 (round to nearest, ties away from zero; low 13 bits zero): the weights
//               once, into a [M][Kp] copy zero-padded to Kp = K rounded up to 4 (k_yolo_round_weights_tf32); the im2col values
//               as they are gathered.  wgmma never sees an unrounded FP32 value, so its own truncation of the low bits never acts.
//   tile        64 x 64 outputs per CTA, one warpgroup, one m64n64k8 wgmma per k-step into FP32 accumulators in registers.  For
//               .tf32 both operands must be K-major in shared memory (the transpose bits exist only for 16-bit types), in the
//               no-swizzle canonical layout: 8 rows x 16 bytes per core matrix, core matrices of one k-chunk of 4 adjacent in
//               M (N), the next k-chunk BM * 16 (BN * 16) bytes on.
//   pipeline    K in stages of TC_BK = 32, two shared-memory buffers: every thread loads stage s + 1 from global memory (the
//               weights as float4, the im2col gather one value at a time with its padding zeros) while the tensor cores
//               run stage s, then rounds the gathered values and stores them into the other buffer, and the CTA barrier
//               hands it over.  The rounding waits for the store so that no gathered load waits on another.
//   im2col      a per-layer table of k -> (c H W + ky W + kx, ky, kx): two bounds tests and one load per value, no division.
//   split-K     layers with too few tiles to fill the GPU (the 13^2 and 26^2 layers) split K over blockIdx.z; the splits'
//               FP32 partial sums are added in split order by k_yolo_splitk_reduce.  No atomics: the order is fixed by the
//               layer's per-image shape, so the same input always gives the same bits, whatever the batch around it.
//   batch       blockIdx.x = image * ceil(N / BN) + pixel tile; each image has its own [splits][M][N] partial sums.
//   epilogue    k_yolo_conv's, op for op (conv_epilogue_tf32 below restates it), so the modes differ only in the sums.
#pragma once
#include <cstdint>

#include "yolo_kernels.cuh"

namespace gfy {

constexpr int TC_BK = 32;

// cvt.rna.tf32.f32: nearest value with an 11-bit significand, ties away from zero, as an FP32 bit pattern
__device__ __forceinline__ float tf32_rna(float x)
{
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// the TF32 weight copy: out[m][k] = rna(w[m][k]) for k < K, 0 for K <= k < Kp
__global__ void k_yolo_round_weights_tf32(const float* __restrict__ w, int M, int K, int Kp, float* __restrict__ out)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)M * Kp) return;
    const int m = (int)(idx / Kp), k = (int)(idx - (long)m * Kp);
    out[idx] = k < K ? tf32_rna(w[(size_t)m * K + k]) : 0.f;
}

// shared-memory matrix descriptor, no swizzle: start address, leading (K) and stride (M / N) byte offsets, all in 16-byte units
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo, uint32_t sbo)
{
    return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)((lbo & 0x3FFFF) >> 4) << 16) | ((uint64_t)((sbo & 0x3FFFF) >> 4) << 32);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }
// generic-proxy st.shared made visible to the async proxy (wgmma's operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// D[64][64] += A[64][8] B[64][8]^T: both operands K-major in shared memory (descriptors), FP32 accumulators
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t da, uint64_t db)
{
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
                 "}, %32, %33, p, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(1));
}

template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t da, uint64_t db)
{
    static_assert(BN == 64, "only the m64n64k8 form is wrapped");
    wgmma_tf32_n64(d, da, db);
}

// k_yolo_conv's epilogue for output (m, p) of the image whose outputs start at out: normalize_cpu (double division), scale_bias,
// add_bias, the activation
__device__ __forceinline__ void conv_epilogue_tf32(const ConvArgs& a, float* out, int m, int p, float v)
{
    const float bias = a.bias[m];
    float sc = 0.f, mu = 0.f;
    double den = 1.0;
    if (a.bn) {
        sc = a.scale[m]; mu = a.mean[m]; den = a.den[m];
        v = __double2float_rn(__ddiv_rn((double)__fsub_rn(v, mu), den));
        v = __fmul_rn(v, sc);
    }
    v = __fadd_rn(v, bias);
    out[(size_t)m * a.N + p] = act(v, a.act);
}

// One gather-table entry per k of the layer (host-built, tf32_ktab in yolo_detector.cu): x = c H W + ky W + kx, y = ky << 16 | kx;
// entries past K carry ky = 0x7FFF, so their bounds test fails and they gather zeros.  The im2col address of a pixel whose
// window starts at (iy0, ix0) is then in + x + iy0 W + ix0 after two bounds tests, with no division in the loop.
constexpr int TC_KTAB_PAD = 0x7FFF;

// Split-K: the CTA at blockIdx.z runs stages [z nsp, (z + 1) nsp) of the layer's K / TC_BK stages.  With part == nullptr there
// is one split and the CTA applies the epilogue; otherwise it writes its raw sums to part[z][M][N] and
// k_yolo_splitk_reduce adds the splits in z order (a fixed order, so the result does not depend on scheduling).
//
// a.w is the TF32 copy [M][Kp].  64 filters x 64 pixels per CTA, one warpgroup (128 threads), several CTAs per SM so that one
// CTA's loads overlap another's tensor-core work.  Every thread stages 4 k-chunks of 4 values of A and of B per stage, and
// gathers B for one fixed pixel.
//
// BATCH: blockIdx.x = image * ceil(N / BN) + pixel tile; without it (one image) the image terms fold away.
template <int BM, int BN, bool BATCH>
__device__ __forceinline__ void conv_tf32_body(const ConvArgs& a, int Kp, const int4* __restrict__ ktab, int nsp,
                                               float* __restrict__ part)
{
    constexpr int T = BM * 2;
    constexpr int A_BYTES = BM * TC_BK * 4, B_BYTES = BN * TC_BK * 4, STAGE = A_BYTES + B_BYTES;
    constexpr int AR = BM * (TC_BK / 4) / T, BR = BN * (TC_BK / 4) / T;
    static_assert(AR == 4 && BR >= 1 && T % BN == 0, "tile shape");
    static_assert(BM * (BN + 1) * 4 <= 2 * STAGE, "epilogue staging fits the pipeline buffers");
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
    const int tid = threadIdx.x, wg = tid / 128, lane = tid % 32, warp = (tid % 128) / 32;
    const int tiles = (a.N + BN - 1) / BN, im = BATCH ? blockIdx.x / tiles : 0;
    const int m0 = blockIdx.y * BM, n0 = (blockIdx.x - im * tiles) * BN;

    // B: this thread's pixel and its k-chunks bj0, bj0 + T / BN, ...; a pixel past N gets a window no bounds test accepts
    const int bp = tid % BN, bj0 = tid / BN;
    const int gp = n0 + bp;
    const bool pix_ok = gp < a.N;
    const int oy = pix_ok ? gp / a.OW : 0, ox = pix_ok ? gp - (gp / a.OW) * a.OW : 0;
    const int iy0 = pix_ok ? oy * a.stride - a.pad : -0x40000000, ix0 = ox * a.stride - a.pad;
    const float* in0 = a.in + (size_t)im * a.C * a.H * a.W + (pix_ok ? (long)iy0 * a.W + ix0 : 0l);

    float4 ar[AR], br[BR];
    // A chunk c = tid + T r: a group of 64 chunks is 8 rows x 8 k-chunks, rows fastest, so each quarter warp stores one
    // 128-byte core matrix row block without bank conflicts
    auto a_row = [&](int r) { const int c = tid + T * r; return (c / 64) * 8 + c % 8; };
    auto a_chk = [&](int r) { return ((tid + T * r) % 64) / 8; };
    auto gather = [&](int x, int y) {
        const int iy = iy0 + (y >> 16), ix = ix0 + (y & 0xFFFF);
        return ((unsigned)iy < (unsigned)a.H && (unsigned)ix < (unsigned)a.W) ? __ldg(in0 + x) : 0.f;
    };
    auto load = [&](int k0) {
#pragma unroll
        for (int r = 0; r < AR; r++) {
            const int gm = m0 + a_row(r), gk = k0 + 4 * a_chk(r);
            ar[r] = (gm < a.M && gk < Kp) ? __ldg(reinterpret_cast<const float4*>(a.w + (size_t)gm * Kp + gk)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int r = 0; r < BR; r++) {
            const int kb = k0 + 4 * (bj0 + r * (T / BN));
            const int4 t0 = __ldg(ktab + kb / 2), t1 = __ldg(ktab + kb / 2 + 1);
            br[r] = make_float4(gather(t0.x, t0.y), gather(t0.z, t0.w), gather(t1.x, t1.y), gather(t1.z, t1.w));
        }
    };
    auto store = [&](int b) {
        uint8_t* sa = smem + b * STAGE;
        uint8_t* sb = sa + A_BYTES;
#pragma unroll
        for (int r = 0; r < AR; r++) {
            const int m = a_row(r), j = a_chk(r);
            *reinterpret_cast<float4*>(sa + (j * (BM / 8) + m / 8) * 128 + (m % 8) * 16) = ar[r];
        }
#pragma unroll
        for (int r = 0; r < BR; r++) {
            const int j = bj0 + r * (T / BN);
            const float4 v = make_float4(tf32_rna(br[r].x), tf32_rna(br[r].y), tf32_rna(br[r].z), tf32_rna(br[r].w));
            *reinterpret_cast<float4*>(sb + (j * (BN / 8) + bp / 8) * 128 + (bp % 8) * 16) = v;
        }
    };

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;

    const int ns = (a.K + TC_BK - 1) / TC_BK;
    const int s0 = blockIdx.z * nsp, s1 = min(ns, s0 + nsp);
    load(s0 * TC_BK);
    store(0);
    fence_proxy_async();
    __syncthreads();
    for (int s = s0; s < s1; s++) {
        const int b = (s - s0) & 1;
        if (s + 1 < s1) load((s + 1) * TC_BK);
        const uint32_t sa = sbase + b * STAGE + wg * 8 * 128, sb = sbase + b * STAGE + A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < TC_BK / 8; ks++)
            wgmma_tf32<BN>(acc, smem_desc(sa + ks * 2 * BM * 16, BM * 16, 128), smem_desc(sb + ks * 2 * BN * 16, BN * 16, 128));
        wgmma_commit();
        if (s + 1 < s1) store(b ^ 1);      // the other buffer: its wgmmas (stage s - 1) completed before the last barrier
        wgmma_wait_all();
        fence_proxy_async();
        __syncthreads();
    }

    // the accumulators through shared memory (the pipeline buffers are free after the last barrier), so that each warp writes
    // whole rows of 64 outputs.  Accumulator i of a thread: row 16 warp + lane / 4 + 8 ((i / 2) % 2), column
    // 8 (i / 4) + 2 (lane % 4) + i % 2
    float* tile = reinterpret_cast<float*>(smem);
#pragma unroll
    for (int i = 0; i < BN / 2; i++)
        tile[(wg * 64 + warp * 16 + lane / 4 + 8 * ((i / 2) % 2)) * (BN + 1) + 8 * (i / 4) + 2 * (lane % 4) + i % 2] = acc[i];
    __syncthreads();
    for (int e = tid; e < BM * BN; e += T) {
        const int m = m0 + e / BN, p = n0 + e % BN;
        if (m >= a.M || p >= a.N) continue;
        const float v = tile[(e / BN) * (BN + 1) + e % BN];
        if (part) part[(((size_t)im * gridDim.z + blockIdx.z) * a.M + m) * a.N + p] = v;
        else conv_epilogue_tf32(a, a.out + (size_t)im * a.M * a.N, m, p, v);
    }
}

// one image / a batch of images: the same body (so the same sums), compiled for each
template <int BM, int BN>
__global__ void __launch_bounds__(BM * 2, 4) k_yolo_conv_tf32(ConvArgs a, int Kp, const int4* __restrict__ ktab, int nsp,
                                                             float* __restrict__ part)
{
    conv_tf32_body<BM, BN, false>(a, Kp, ktab, nsp, part);
}
template <int BM, int BN>
__global__ void __launch_bounds__(BM * 2, 4) k_yolo_conv_tf32_batch(ConvArgs a, int Kp, const int4* __restrict__ ktab, int nsp,
                                                                   float* __restrict__ part)
{
    conv_tf32_body<BM, BN, true>(a, Kp, ktab, nsp, part);
}

// the splits of a split-K layer added in split order, then k_yolo_conv's epilogue; one thread per output, blockIdx.y = image
__global__ void k_yolo_splitk_reduce(ConvArgs a, const float* __restrict__ part, int splits)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long MN = (long)a.M * a.N;
    if (idx >= MN) return;
    part += blockIdx.y * splits * MN;
    float v = part[idx];
    for (int z = 1; z < splits; z++) v = __fadd_rn(v, part[z * MN + idx]);
    conv_epilogue_tf32(a, a.out + blockIdx.y * MN, (int)(idx / a.N), (int)(idx % a.N), v);
}

}  // namespace gfy
