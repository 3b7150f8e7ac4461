// yolo_detector.cu -- gf_detector_* (C ABI): the use_yolo front end's detector, the darknet_ros node
// (vins_estimator/src/YoloObjectDetector.cpp) with the vendored darknet's CPU forward pass, on the GPU and bit-exact with it.
//   create   the cfg and .weights read on the host (yolo_cfg.cuh), every parameter in HBM once, the forward pass of one image
//            captured as one CUDA graph: the layers' kernels (yolo_kernels.cuh) and the copies of the [region] / [yolo] outputs
//            to pinned memory
//   detect   n frames (detect is the batch of one): the frames to the device, k_yolo_letterbox, the graph of n images
//            (captured on the first call with that n and kept), then per frame on the host darknet's decoding
//            (get_network_boxes(w, h, thresh, 0.5, 0, 1)), do_nms_obj(0.4) with libc qsort, and darknet_ros's extraction.
//            The per-image buffers hold gf_detector_set_max_batch images; image i's values sit at i * the per-image size.
// DESIGN.md "YOLO detector" has the arithmetic and why the default mode uses no tensor cores; gf_detector_set_precision
// selects the TF32 tensor-core convolutions (yolo_tf32.cuh) instead, every other kernel unchanged.
// Built as its own library, libgf_yolo.so, with its own error text (gf_detector_last_error); libgf_b200.so exports the same
// entry points as forwarders (yolo_forward.cpp) and carries none of this device code, so a tracker / estimator process that
// never detects loads exactly what it loaded before.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "gf_common.cuh"
#include "yolo_cfg.cuh"
#include "yolo_kernels.cuh"
#include "yolo_tf32.cuh"

using namespace gf;
using namespace gfy;

namespace gf {
thread_local char g_err[512] = "";           // this library's error text (set_err, GF_CUDA)
std::atomic<uint64_t> g_launches{0};
}  // namespace gf

namespace gfy {

struct DevLayer {
    float* out = nullptr;
    float *w = nullptr, *bias = nullptr, *scale = nullptr, *mean = nullptr;
    double* den = nullptr;
    float* w_tf32 = nullptr;             // the weights rounded to TF32, [n][kp], allocated by the first switch to TF32
    int kp = 0;                          // K rounded up to 4
    int* ktab = nullptr;                 // the TF32 kernel's im2col table (tf32_ktab), allocated with w_tf32
    float* host_out = nullptr;           // pinned copy of a [region] / [yolo] output
};

// darknet's detection struct, field for field, so that qsort sees elements of the same size and order as the oracle's
struct Det {
    float x, y, w, h;
    int classes;
    float* prob;
    float* mask;
    float objectness;
    int sort_class;
};
static_assert(sizeof(Det) == 48, "Det must have darknet's detection layout");

}  // namespace gfy

struct gf_detector {
    int device = 0;
    float thresh = 0.3f;
    Net net;
    std::vector<DevLayer> dl;
    int max_batch = 1;                   // images the per-image buffers hold
    float* d_input = nullptr;            // [max_batch][3][h][w]
    uint8_t* d_frame = nullptr;          // the host frames of a call, staged one after another
    size_t frame_cap = 0;
    cudaStream_t st = nullptr;
    cudaGraphExec_t exec[GF_DETECTOR_BATCH_MAX + 1] = {};     // exec[n]: the forward pass of n images, once used
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    int precision = GF_DETECTOR_EXACT;
    bool tf32_ready = false;             // the TF32 weights, tables and workspace exist
    float* d_part = nullptr;             // the TF32 split-K partial sums, [max_batch] x the layer that needs most
    std::vector<float> prob_store;
    bool ran = false;
    int last_n = 0;                      // frames of the last detect
};
static_assert(LB_MAX == GF_DETECTOR_BATCH_MAX, "one letterbox launch takes a whole batch");

namespace {

int select_device(int device)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return set_err(GF_ERR_NO_DEVICE, "no CUDA device visible; libgf_b200 has no CPU fallback");
    if (device < 0 || device >= n) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    return GF_OK;
}

void drop_graphs(gf_detector* d)
{
    for (cudaGraphExec_t& x : d->exec)
        if (x) { cudaGraphExecDestroy(x); x = nullptr; }
}

void free_detector(gf_detector* d)
{
    if (!d) return;
    drop_graphs(d);
    for (DevLayer& l : d->dl) {
        cudaFree(l.out); cudaFree(l.w); cudaFree(l.bias); cudaFree(l.scale); cudaFree(l.mean); cudaFree(l.den); cudaFree(l.w_tf32); cudaFree(l.ktab);
        if (l.host_out) cudaFreeHost(l.host_out);
    }
    cudaFree(d->d_input);
    cudaFree(d->d_part);
    cudaFree(d->d_frame);
    if (d->ev0) cudaEventDestroy(d->ev0);
    if (d->ev1) cudaEventDestroy(d->ev1);
    if (d->st) cudaStreamDestroy(d->st);
    delete d;
}

template <typename T>
int upload(T** dst, const std::vector<T>& v)
{
    GF_CUDA(cudaMalloc(dst, sizeof(T) * v.size()));
    GF_CUDA(cudaMemcpy(*dst, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
    return GF_OK;
}

inline unsigned blocks(long n, int t) { return (unsigned)((n + t - 1) / t); }

// darknet's letterbox geometry: the frame scaled to fit the net size, aspect kept
void letterbox_size(int w, int h, int nw, int nh, int& new_w, int& new_h)
{
    if ((float)nw / w < (float)nh / h) { new_w = nw; new_h = (h * nw) / w; }
    else { new_h = nh; new_w = (w * nh) / h; }
}

template <int BM, int BN>
void launch_conv(const ConvArgs& a, int n, cudaStream_t s)
{
    dim3 g(blocks(a.N, BN) * n, blocks(a.M, BM));
    if (n == 1) k_yolo_conv<BM, BN><<<g, CONV_THREADS, 0, s>>>(a);
    else k_yolo_conv_batch<BM, BN><<<g, CONV_THREADS, 0, s>>>(a);
    GF_LAUNCHED();
}

// a TF32 convolution's device operands: the rounded weights [M][kp], the im2col table, the split-K workspace (if it splits)
struct Tf32Operands {
    const float* w = nullptr;
    int kp = 0;
    const int* ktab = nullptr;
    float* part = nullptr;
};

// split-K of a TF32 layer from its shape alone: enough 64 x 64 CTAs for four per SM of the H100's 132 (the kernel's occupancy),
// each split at least 4 stages of TC_BK; splits = 1 for layers whose tiles already fill the GPU.  Per image, not per batch:
// the split order sets the bits of every output, so a frame's result must not depend on the frames batched with it.
struct Tf32Plan { int splits, nsp; };
Tf32Plan tf32_plan(int M, int N, int K)
{
    const int ns = (K + TC_BK - 1) / TC_BK;
    const long tiles = (long)blocks(N, 64) * blocks(M, 64);
    int want = (int)std::min<long>(std::max<long>(528 / tiles, 1), std::max(ns / 4, 1));
    const int nsp = (ns + want - 1) / want;
    return Tf32Plan{(ns + nsp - 1) / nsp, nsp};
}

// the im2col table of a layer (yolo_tf32.cuh): per k, c H W + ky W + kx and ky << 16 | kx; padded to whole stages with
// entries no bounds test accepts
std::vector<int> tf32_ktab(int C, int H, int W, int size)
{
    const int K = C * size * size, ns = (K + TC_BK - 1) / TC_BK;
    std::vector<int> t(2 * (size_t)ns * TC_BK);
    for (int k = 0; k < ns * TC_BK; k++) {
        if (k >= K) { t[2 * k] = 0; t[2 * k + 1] = TC_KTAB_PAD << 16; continue; }
        const int c = k / (size * size), ky = k / size % size, kx = k % size;
        t[2 * k] = c * H * W + ky * W + kx;
        t[2 * k + 1] = ky << 16 | kx;
    }
    return t;
}

size_t tf32_part_floats(int M, int N, int K)
{
    const Tf32Plan pl = tf32_plan(M, N, K);
    return pl.splits > 1 ? (size_t)pl.splits * M * N : 0;
}

// the split-K workspace one image needs: the largest of the network's layers
size_t tf32_part_max(const Net& net)
{
    size_t part = 0;
    for (const Layer& l : net.layers)
        if (l.type == L_CONV) part = std::max(part, tf32_part_floats(l.n, l.ow * l.oh, l.c * l.size * l.size));
    return part;
}

// the TF32 kernel's dynamic shared memory (32 KB); before any launch or capture
int tf32_setup()
{
    GF_CUDA(cudaFuncSetAttribute(k_yolo_conv_tf32<64, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (64 + 64) * TC_BK * 8));
    GF_CUDA(cudaFuncSetAttribute(k_yolo_conv_tf32_batch<64, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (64 + 64) * TC_BK * 8));
    return GF_OK;
}

// one convolution of n images at `precision` (the detector and gf_stage_yolo_conv both come here).  The TF32 split comes from
// the layer's per-image shape alone; the exact tile may look at the whole batch, since it does not change an output's sum.
void launch_conv_layer(ConvArgs a, int precision, const Tf32Operands& t, int n, cudaStream_t s)
{
    if (precision == GF_DETECTOR_TF32) {
        a.w = t.w;
        const Tf32Plan pl = tf32_plan(a.M, a.N, a.K);
        float* part = pl.splits > 1 ? t.part : nullptr;
        const dim3 g(blocks(a.N, 64) * n, blocks(a.M, 64), pl.splits);
        const int4* ktab = reinterpret_cast<const int4*>(t.ktab);
        if (n == 1) k_yolo_conv_tf32<64, 64><<<g, 128, (64 + 64) * TC_BK * 8, s>>>(a, t.kp, ktab, pl.nsp, part);
        else k_yolo_conv_tf32_batch<64, 64><<<g, 128, (64 + 64) * TC_BK * 8, s>>>(a, t.kp, ktab, pl.nsp, part);
        GF_LAUNCHED();
        if (part) {
            k_yolo_splitk_reduce<<<dim3(blocks((long)a.M * a.N, 256), n), 256, 0, s>>>(a, part, pl.splits);
            GF_LAUNCHED();
        }
        return;
    }
    // 64 x 64 tiles where they fill the GPU twice over, 32 x 32 where the layer is small
    if ((long)blocks(a.N, 64) * blocks(a.M, 64) * n >= 264) launch_conv<64, 64>(a, n, s);
    else launch_conv<32, 32>(a, n, s);
}

// a layer's TF32 weight copy, rounded on the device by k_yolo_round_weights_tf32
int round_weights_tf32(const float* w, int M, int K, int kp, float** out, cudaStream_t s)
{
    GF_CUDA(cudaMalloc(out, 4 * (size_t)M * kp));
    k_yolo_round_weights_tf32<<<blocks((long)M * kp, 256), 256, 0, s>>>(w, M, K, kp, *out);
    GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

// layer i's kernels for n images on stream s (captured into the graph)
int enqueue_layer(gf_detector* d, int i, int n, cudaStream_t s)
{
    const Layer& l = d->net.layers[i];
    DevLayer& o = d->dl[i];
    const float* in = i == 0 ? d->d_input : d->dl[i - 1].out;
    constexpr int T = 256;
    switch (l.type) {
    case L_CONV: {
        ConvArgs a{in, o.w, o.out, o.bias, o.scale, o.mean, o.den, l.c, l.h, l.w, l.n, l.c * l.size * l.size, l.ow, l.ow * l.oh,
                   l.size, l.stride, l.pad, l.bn, l.act};
        Tf32Operands t;
        t.w = o.w_tf32; t.kp = o.kp; t.ktab = o.ktab; t.part = d->d_part;
        launch_conv_layer(a, d->precision, t, n, s);
        break;
    }
    case L_MAXPOOL:
        k_yolo_maxpool<<<blocks(l.outputs * n, T), T, 0, s>>>(in, o.out, l.w, l.h, l.c * n, l.ow, l.oh, l.size, l.stride, l.pad);
        GF_LAUNCHED();
        break;
    case L_ROUTE: {           // each input's n images into their rows of the concatenation
        size_t off = 0;
        for (int k : l.in) {
            const size_t m = (size_t)d->net.layers[k].outputs;
            if (n == 1) GF_CUDA(cudaMemcpyAsync(o.out + off, d->dl[k].out, 4 * m, cudaMemcpyDeviceToDevice, s));
            else GF_CUDA(cudaMemcpy2DAsync(o.out + off, 4 * (size_t)l.outputs, d->dl[k].out, 4 * m, 4 * m, n, cudaMemcpyDeviceToDevice, s));
            off += m;
        }
        break;
    }
    case L_REORG:
        k_yolo_reorg<<<dim3(blocks(l.outputs, T), n), T, 0, s>>>(in, o.out, l.w, l.h, l.c, l.stride); GF_LAUNCHED();
        break;
    case L_UPSAMPLE:
        k_yolo_upsample<<<blocks(l.outputs * n, T), T, 0, s>>>(in, o.out, l.w, l.h, l.c * n, l.stride, l.scale); GF_LAUNCHED();
        break;
    case L_SHORTCUT:
        k_yolo_shortcut<<<dim3(blocks(l.outputs, T), n), T, 0, s>>>(in, d->dl[l.in[0]].out, o.out, l.w, l.h, l.c, l.ow, l.oh, l.oc,
                                                                    l.alpha, l.beta, l.act);
        GF_LAUNCHED();
        break;
    case L_REGION:
    case L_YOLO:
        k_yolo_head<<<blocks((long)l.ow * l.oh * l.num * n, 128), 128, 0, s>>>(in, o.out, l.ow * l.oh, l.num * n, l.classes,
                                                                               l.type == L_YOLO, l.softmax);
        GF_LAUNCHED();
        GF_CUDA(cudaMemcpyAsync(o.host_out, o.out, 4 * (size_t)n * l.outputs, cudaMemcpyDeviceToHost, s));
        break;
    }
    GF_CUDA(cudaGetLastError());
    return GF_OK;
}

// the per-image buffers of nb images: every layer's output, the heads' pinned copies, the letterboxed input and, with part > 0,
// the TF32 split-K workspace of part floats per image
struct BatchBufs {
    std::vector<float*> out, host_out;
    float* input = nullptr;
    float* part = nullptr;
};

void free_bufs(BatchBufs& b)
{
    for (float* p : b.out) cudaFree(p);
    for (float* p : b.host_out) if (p) cudaFreeHost(p);
    cudaFree(b.input);
    cudaFree(b.part);
    b = BatchBufs();
}

// all or nothing: on failure every buffer allocated here is freed again
int alloc_bufs(const gf_detector* d, int nb, size_t part, BatchBufs& b)
{
    const size_t nl = d->net.layers.size();
    b.out.assign(nl, nullptr);
    b.host_out.assign(nl, nullptr);
    cudaError_t e = cudaMalloc(&b.input, 4 * (size_t)nb * 3 * d->net.w * d->net.h);
    for (size_t i = 0; i < nl && e == cudaSuccess; i++) {
        const Layer& l = d->net.layers[i];
        e = cudaMalloc(&b.out[i], 4 * (size_t)nb * l.outputs);
        if (e == cudaSuccess && (l.type == L_REGION || l.type == L_YOLO)) e = cudaMallocHost(&b.host_out[i], 4 * (size_t)nb * l.outputs);
    }
    if (e == cudaSuccess && part) e = cudaMalloc(&b.part, 4 * (size_t)nb * part);
    if (e != cudaSuccess) {
        free_bufs(b);
        cudaGetLastError();
        return set_err(GF_ERR_CUDA, "allocating the buffers of %s images failed: %s", std::to_string(nb).c_str(), cudaGetErrorString(e));
    }
    return GF_OK;
}

// b's buffers into the handle, the handle's previous ones into b
void swap_bufs(gf_detector* d, BatchBufs& b)
{
    for (size_t i = 0; i < d->dl.size(); i++) {
        std::swap(d->dl[i].out, b.out[i]);
        std::swap(d->dl[i].host_out, b.host_out[i]);
    }
    std::swap(d->d_input, b.input);
    std::swap(d->d_part, b.part);
}

int capture(gf_detector* d, int n, cudaGraphExec_t* out);

int detector_init(gf_detector* d)
{
    GF_CUDA(cudaStreamCreateWithFlags(&d->st, cudaStreamNonBlocking));
    GF_CUDA(cudaEventCreate(&d->ev0));
    GF_CUDA(cudaEventCreate(&d->ev1));
    d->dl.resize(d->net.layers.size());
    BatchBufs b;
    int rc = alloc_bufs(d, 1, 0, b);
    if (rc) return rc;
    swap_bufs(d, b);
    for (size_t i = 0; i < d->net.layers.size(); i++) {
        const Layer& l = d->net.layers[i];
        DevLayer& o = d->dl[i];
        if (l.type == L_CONV) {
            int rc = upload(&o.w, l.weights);
            if (!rc) rc = upload(&o.bias, l.biases);
            if (!rc && l.bn) {
                std::vector<double> den(l.n);
                for (int m = 0; m < l.n; m++) den[m] = sqrt((double)l.var[m]) + (double).000001f;   // normalize_cpu's denominator
                rc = upload(&o.scale, l.scales);
                if (!rc) rc = upload(&o.mean, l.mean);
                if (!rc) rc = upload(&o.den, den);
            }
            if (rc) return rc;
        }
    }
    return capture(d, 1, &d->exec[1]);
}

// the forward pass of n images at d->precision captured as one graph and instantiated into *out (untouched on failure)
int capture(gf_detector* d, int n, cudaGraphExec_t* out)
{
    GF_CUDA(cudaStreamBeginCapture(d->st, cudaStreamCaptureModeThreadLocal));
    int rc = GF_OK;
    for (size_t i = 0; i < d->net.layers.size() && !rc; i++) rc = enqueue_layer(d, (int)i, n, d->st);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(d->st, &g);
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    GF_CUDA(e);
    cudaGraphExec_t x = nullptr;
    const cudaError_t ei = cudaGraphInstantiate(&x, g, 0);
    cudaGraphDestroy(g);
    if (ei != cudaSuccess) return set_err(GF_ERR_CUDA, "cudaGraphInstantiate failed");
    *out = x;
    return GF_OK;
}

// ---- host: darknet's decoding, NMS and darknet_ros's extraction ----------------------------------------------------------

// correct_region_boxes / correct_yolo_boxes with relative = 1
void correct_boxes(Det* dets, int n, int w, int h, int netw, int neth)
{
    int new_w = 0, new_h = 0;
    if (((float)netw / w) < ((float)neth / h)) { new_w = netw; new_h = (h * netw) / w; }
    else { new_h = neth; new_w = (w * neth) / h; }
    for (int i = 0; i < n; i++) {
        Det& b = dets[i];
        b.x = (float)((b.x - (netw - new_w) / 2. / netw) / ((float)new_w / netw));
        b.y = (float)((b.y - (neth - new_h) / 2. / neth) / ((float)new_h / neth));
        b.w *= (float)netw / new_w;
        b.h *= (float)neth / new_h;
    }
}

// get_network_boxes(net, w, h, thresh, hier, 0, 1, &n) of image im of the last batch: every layer's detections in layer order
void network_boxes(gf_detector* d, int im, int w, int h, std::vector<Det>& dets)
{
    const Net& net = d->net;
    const float thresh = d->thresh;
    const int classes = net.layers.back().classes;
    size_t total = 0;
    for (size_t li = 0; li < net.layers.size(); li++) {
        const Layer& l = net.layers[li];
        const int wh = l.ow * l.oh, E = l.classes + 5;
        const float* p = d->dl[li].host_out + (size_t)im * l.outputs;
        if (l.type == L_REGION) total += (size_t)wh * l.num;
        if (l.type == L_YOLO)
            for (int i = 0; i < wh; i++)
                for (int n = 0; n < l.num; n++) total += p[(size_t)n * wh * E + 4 * wh + i] > thresh;
    }
    dets.assign(total, Det{});
    d->prob_store.assign(total * classes, 0.f);
    for (size_t i = 0; i < total; i++) { dets[i].prob = d->prob_store.data() + i * classes; dets[i].mask = nullptr; }
    size_t at = 0;
    for (size_t li = 0; li < net.layers.size(); li++) {
        const Layer& l = net.layers[li];
        if (l.type != L_REGION && l.type != L_YOLO) continue;
        const int wh = l.ow * l.oh, E = l.classes + 5;
        const float* p = d->dl[li].host_out + (size_t)im * l.outputs;
        const size_t first = at;
        for (int i = 0; i < wh; i++) {
            const int row = i / l.ow, col = i % l.ow;
            for (int n = 0; n < l.num; n++) {
                const size_t base = (size_t)n * wh * E + i;
                const float obj = p[base + 4 * (size_t)wh];
                if (l.type == L_YOLO && obj <= thresh) continue;
                // a [yolo] layer appends its detections above thresh; a [region] layer fills all of its own at n * wh + i
                Det& b = l.type == L_YOLO ? dets[at++] : dets[first + (size_t)n * wh + i];
                const int a = l.type == L_YOLO ? l.mask[n] : n;
                const int bw = l.type == L_YOLO ? net.w : l.ow, bh = l.type == L_YOLO ? net.h : l.oh;
                b.x = (col + p[base]) / l.ow;                                  // get_region_box / get_yolo_box
                b.y = (row + p[base + wh]) / l.oh;
                b.w = (float)(exp((double)p[base + 2 * (size_t)wh]) * l.anchors[2 * a] / bw);    // exp in double, as in C
                b.h = (float)(exp((double)p[base + 3 * (size_t)wh]) * l.anchors[2 * a + 1] / bh);
                if (l.type == L_YOLO) {
                    b.objectness = obj;
                    b.classes = l.classes;
                } else {
                    b.objectness = obj > thresh ? obj : 0;
                    if (!b.objectness) continue;
                }
                for (int j = 0; j < l.classes; j++) {
                    const float prob = b.objectness * p[base + (size_t)(5 + j) * wh];
                    b.prob[j] = (prob > thresh) ? prob : 0;
                }
            }
        }
        if (l.type == L_REGION) at = first + (size_t)wh * l.num;
        correct_boxes(dets.data() + first, (int)(at - first), w, h, net.w, net.h);
    }
}

// darknet's nms_comparator: descending by objectness (sort_class is -1 throughout do_nms_obj)
int nms_cmp(const void* pa, const void* pb)
{
    const Det* a = (const Det*)pa;
    const Det* b = (const Det*)pb;
    float diff = 0;
    if (b->sort_class >= 0) diff = a->prob[b->sort_class] - b->prob[b->sort_class];
    else diff = a->objectness - b->objectness;
    if (diff < 0) return 1;
    if (diff > 0) return -1;
    return 0;
}

float overlap1(float x1, float w1, float x2, float w2)
{
    const float l1 = x1 - w1 / 2, l2 = x2 - w2 / 2;
    const float left = l1 > l2 ? l1 : l2;
    const float r1 = x1 + w1 / 2, r2 = x2 + w2 / 2;
    const float right = r1 < r2 ? r1 : r2;
    return right - left;
}

float iou(const Det& a, const Det& b)
{
    const float w = overlap1(a.x, a.w, b.x, b.w), h = overlap1(a.y, a.h, b.y, b.h);
    const float inter = (w < 0 || h < 0) ? 0 : w * h;
    const float uni = a.w * a.h + b.w * b.h - inter;
    return inter / uni;
}

// do_nms_obj(dets, total, classes, 0.4): zero-objectness detections swapped to the end, qsort, greedy suppression
void nms_obj(std::vector<Det>& dets, int classes, float thresh)
{
    int k = (int)dets.size() - 1;
    for (int i = 0; i <= k; i++) {
        if (dets[i].objectness == 0) {
            std::swap(dets[i], dets[k]);
            --k;
            --i;
        }
    }
    const int total = k + 1;
    for (int i = 0; i < total; i++) dets[i].sort_class = -1;
    qsort(dets.data(), total, sizeof(Det), nms_cmp);
    for (int i = 0; i < total; i++) {
        if (dets[i].objectness == 0) continue;
        for (int j = i + 1; j < total; j++) {
            if (dets[j].objectness == 0) continue;
            if (iou(dets[i], dets[j]) > thresh) {
                dets[j].objectness = 0;
                for (int c = 0; c < classes; c++) dets[j].prob[c] = 0;
            }
        }
    }
}

struct RoiBox { float x, y, w, h, prob; int cls; };

// detectInThread's extraction (clamped to [0, 1], > 1 % of the frame, one entry per class with a non-zero probability) and the
// publishing loop (count 1..100, grouped by class in class order, corners by int truncation of (centre -+ size / 2) * frame size)
int extract(const std::vector<Det>& dets, int classes, int fw, int fh, gf_box* boxes, int* cls, float* probs, int cap)
{
    std::vector<RoiBox> roi;
    for (const Det& d : dets) {
        float xmin = (float)(d.x - d.w / 2.), xmax = (float)(d.x + d.w / 2.);
        float ymin = (float)(d.y - d.h / 2.), ymax = (float)(d.y + d.h / 2.);
        if (xmin < 0) xmin = 0;
        if (ymin < 0) ymin = 0;
        if (xmax > 1) xmax = 1;
        if (ymax > 1) ymax = 1;
        for (int j = 0; j < classes; j++) {
            if (d.prob[j]) {
                const float xc = (xmin + xmax) / 2, yc = (ymin + ymax) / 2;
                const float bw = xmax - xmin, bh = ymax - ymin;
                if (bw > 0.01 && bh > 0.01) roi.push_back(RoiBox{xc, yc, bw, bh, d.prob[j], j});
            }
        }
    }
    const int num = (int)roi.size();
    if (num <= 0 || num > GF_MAX_BOXES) return 0;
    int n = 0;
    for (int c = 0; c < classes; c++)
        for (const RoiBox& r : roi) {
            if (r.cls != c) continue;
            if (n < cap) {
                boxes[n].xmin = (int)((r.x - r.w / 2) * fw);
                boxes[n].ymin = (int)((r.y - r.h / 2) * fh);
                boxes[n].xmax = (int)((r.x + r.w / 2) * fw);
                boxes[n].ymax = (int)((r.y + r.h / 2) * fh);
                if (cls) cls[n] = c;
                if (probs) probs[n] = r.prob;
            }
            n++;
        }
    return n;
}

int check_frame(const void* bgr, size_t pitch, int w, int h)
{
    if (!bgr || w < 1 || h < 1 || w > 16384 || h > 16384 || pitch < (size_t)3 * w || pitch > (1u << 30))
        return set_err(GF_ERR_INVALID_ARG, "bad frame (BGR8, 1..16384 pixels a side, pitch >= 3 * width)");
    return GF_OK;
}

void set_frame(LbFrames& f, int i, const uint8_t* src, int pitch, int w, int h, int nw, int nh)
{
    f.bgr[i] = src; f.pitch[i] = pitch; f.w[i] = w; f.h[i] = h;
    letterbox_size(w, h, nw, nh, f.new_w[i], f.new_h[i]);
}

void launch_letterbox(const LbFrames& f, int n, int nw, int nh, float* out, cudaStream_t s)
{
    k_yolo_letterbox<<<dim3(blocks(nw, 128), nh, 3 * n), 128, 0, s>>>(f, nw, nh, out);
    GF_LAUNCHED();
}

// the n frames for the letterbox: device frames in place, host frames copied one after another into the staging buffer
int stage_frames(gf_detector* d, int n, const void* const* bgr, const size_t* pitch, const int* w, const int* h, int on_device,
                 LbFrames& f)
{
    size_t need = 0;
    for (int i = 0; i < n && !on_device; i++) need += (size_t)3 * w[i] * h[i];
    if (need > d->frame_cap) {
        cudaFree(d->d_frame);
        d->d_frame = nullptr; d->frame_cap = 0;
        GF_CUDA(cudaMalloc(&d->d_frame, need));
        d->frame_cap = need;
    }
    size_t off = 0;
    for (int i = 0; i < n; i++) {
        const uint8_t* src = (const uint8_t*)bgr[i];
        int sp = (int)pitch[i];
        if (!on_device) {
            GF_CUDA(cudaMemcpy2DAsync(d->d_frame + off, 3 * (size_t)w[i], bgr[i], pitch[i], 3 * (size_t)w[i], h[i], cudaMemcpyHostToDevice, d->st));
            src = d->d_frame + off; sp = 3 * w[i];
            off += (size_t)3 * w[i] * h[i];
        }
        set_frame(f, i, src, sp, w[i], h[i], d->net.w, d->net.h);
    }
    return GF_OK;
}

// the forward pass of n checked frames and the host decoding of each; frame i's boxes at box_start[i] .. box_start[i + 1],
// nothing written at or past cap
int detect_frames(gf_detector* d, int n, const void* const* bgr, const size_t* pitch, const int* w, const int* h, int on_device,
                  gf_box* boxes, int* class_ids, float* probs, int cap, int* box_start)
{
    GF_CUDA(cudaSetDevice(d->device));
    if (!d->exec[n]) {
        const int rc = capture(d, n, &d->exec[n]);
        if (rc) return rc;
    }
    LbFrames f;
    const int rc = stage_frames(d, n, bgr, pitch, w, h, on_device, f);
    if (rc) return rc;
    GF_CUDA(cudaEventRecord(d->ev0, d->st));
    launch_letterbox(f, n, d->net.w, d->net.h, d->d_input, d->st);
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaGraphLaunch(d->exec[n], d->st));
    GF_CUDA(cudaEventRecord(d->ev1, d->st));
    GF_CUDA(cudaStreamSynchronize(d->st));
    d->ran = true;
    d->last_n = n;
    const int classes = d->net.layers.back().classes;
    std::vector<Det> dets;
    box_start[0] = 0;
    for (int i = 0; i < n; i++) {
        network_boxes(d, i, w[i], h[i], dets);
        nms_obj(dets, classes, .4f);
        const int at = box_start[i], room = std::max(cap - at, 0);
        box_start[i + 1] = at + extract(dets, classes, w[i], h[i], room ? boxes + at : nullptr,
                                        room && class_ids ? class_ids + at : nullptr, room && probs ? probs + at : nullptr, room);
    }
    if (box_start[n] > cap) return set_err(GF_ERR_CAPACITY, "more boxes than cap");
    return GF_OK;
}

}  // namespace

extern "C" {

const char* gf_detector_last_error(void) { return g_err; }

int gf_detector_create(gf_detector** out, int device, const char* cfg_path, const char* weights_path, float thresh)
{
    if (!out || !cfg_path || !weights_path) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    if (!(thresh >= 0.f && thresh < 1.f)) return set_err(GF_ERR_INVALID_ARG, "thresh must lie in [0, 1)");
    gf_detector* d = new (std::nothrow) gf_detector();
    if (!d) return set_err(GF_ERR_CUDA, "out of host memory");
    d->device = device;
    d->thresh = thresh;
    // the files first: an unsupported network is refused by name before any device is touched
    std::string err;
    int rc = GF_OK;
    if (!parse_net(cfg_path, d->net, err)) rc = set_err(GF_ERR_UNSUPPORTED, "%s", err.c_str());
    else if (!load_weights(weights_path, d->net, err)) rc = set_err(GF_ERR_INVALID_ARG, "%s", err.c_str());
    if (rc) { delete d; return rc; }
    rc = select_device(device);
    if (!rc) rc = detector_init(d);
    if (rc) {
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        free_detector(d);
        cudaGetLastError();
        memcpy(g_err, keep, sizeof(keep));
        return rc;
    }
    *out = d;
    return GF_OK;
}

void gf_detector_destroy(gf_detector* d)
{
    if (!d) return;
    cudaSetDevice(d->device);
    if (d->st) cudaStreamSynchronize(d->st);
    free_detector(d);
}

int gf_detector_info(gf_detector* d, int* net_wh, int* n_layers, int* classes)
{
    if (!d) return set_err(GF_ERR_INVALID_ARG, "null detector");
    if (net_wh) { net_wh[0] = d->net.w; net_wh[1] = d->net.h; }
    if (n_layers) *n_layers = (int)d->net.layers.size();
    if (classes) *classes = d->net.layers.back().classes;
    return GF_OK;
}

int gf_detector_layer_shape(gf_detector* d, int layer, int* whc)
{
    if (!d || !whc || layer < -1 || layer >= (int)d->net.layers.size()) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (layer < 0) { whc[0] = d->net.w; whc[1] = d->net.h; whc[2] = 3; return GF_OK; }
    const Layer& l = d->net.layers[layer];
    whc[0] = l.ow; whc[1] = l.oh; whc[2] = l.oc;
    return GF_OK;
}

int gf_detector_detect(gf_detector* d, const void* bgr, size_t pitch, int w, int h, int on_device, gf_box* boxes, int* class_ids,
                       float* probs, int cap, int* n_out)
{
    if (!d || !n_out || cap < 0 || (cap > 0 && !boxes)) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    const int rc0 = check_frame(bgr, pitch, w, h);
    if (rc0) return rc0;
    int box_start[2];
    const int rc = detect_frames(d, 1, &bgr, &pitch, &w, &h, on_device, boxes, class_ids, probs, cap, box_start);
    if (rc == GF_OK || rc == GF_ERR_CAPACITY) *n_out = box_start[1];
    return rc;
}

int gf_detector_detect_batch(gf_detector* d, int n, const void* const* bgr, const size_t* pitch, const int* w, const int* h,
                             int on_device, gf_box* boxes, int* class_ids, float* probs, int cap, int* box_start)
{
    if (!d || !bgr || !pitch || !w || !h || !box_start || cap < 0 || (cap > 0 && !boxes) || n < 1)
        return set_err(GF_ERR_INVALID_ARG, "bad argument");
    for (int i = 0; i < n; i++)          // the frames before the handle: every argument error is found without touching it
        if (check_frame(bgr[i], pitch[i], w[i], h[i]))
            return set_err(GF_ERR_INVALID_ARG, "frame %s: bad frame (BGR8, 1..16384 pixels a side, pitch >= 3 * width)", std::to_string(i).c_str());
    if (n > d->max_batch) return set_err(GF_ERR_CAPACITY, "%s frames exceed the handle's max_batch of %s", std::to_string(n).c_str(), std::to_string(d->max_batch).c_str());
    return detect_frames(d, n, bgr, pitch, w, h, on_device, boxes, class_ids, probs, cap, box_start);
}

int gf_detector_set_max_batch(gf_detector* d, int max_batch)
{
    if (!d) return set_err(GF_ERR_INVALID_ARG, "null detector");
    if (max_batch < 1 || max_batch > GF_DETECTOR_BATCH_MAX) return set_err(GF_ERR_INVALID_ARG, "max_batch must lie in [1, GF_DETECTOR_BATCH_MAX]");
    if (max_batch == d->max_batch) return GF_OK;
    GF_CUDA(cudaSetDevice(d->device));
    GF_CUDA(cudaStreamSynchronize(d->st));
    BatchBufs b;
    const int rc = alloc_bufs(d, max_batch, d->tf32_ready ? tf32_part_max(d->net) : 0, b);
    if (rc) return rc;
    drop_graphs(d);                      // they name the old buffers
    swap_bufs(d, b);
    free_bufs(b);
    d->max_batch = max_batch;
    d->ran = false;
    d->last_n = 0;
    return GF_OK;
}

int gf_detector_last_device_ms(gf_detector* d, float* ms)
{
    if (!d || !ms || !d->ran) return set_err(GF_ERR_INVALID_ARG, "no detection has run");
    GF_CUDA(cudaEventElapsedTime(ms, d->ev0, d->ev1));
    return GF_OK;
}

int gf_detector_member_layer_output(gf_detector* d, int member, int layer, float* out, size_t n)
{
    if (!d || !out || layer < -1 || layer >= (int)d->net.layers.size()) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (!d->ran) return set_err(GF_ERR_INVALID_ARG, "no detection has run");
    if (member < 0 || member >= d->last_n) return set_err(GF_ERR_INVALID_ARG, "member %s outside the last call's %s frames", std::to_string(member).c_str(), std::to_string(d->last_n).c_str());
    const size_t need = layer < 0 ? (size_t)3 * d->net.w * d->net.h : (size_t)d->net.layers[layer].outputs;
    if (n < need) return set_err(GF_ERR_CAPACITY, "output buffer too small");
    GF_CUDA(cudaSetDevice(d->device));
    GF_CUDA(cudaMemcpy(out, (layer < 0 ? d->d_input : d->dl[layer].out) + member * need, 4 * need, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_detector_layer_output(gf_detector* d, int layer, float* out, size_t n)
{
    return gf_detector_member_layer_output(d, 0, layer, out, n);
}

int gf_detector_layer_times(gf_detector* d, int reps, float* ms)
{
    if (!d || !ms || reps < 1) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (!d->ran) return set_err(GF_ERR_INVALID_ARG, "no detection has run");
    GF_CUDA(cudaSetDevice(d->device));
    cudaEvent_t a, b;
    GF_CUDA(cudaEventCreate(&a));
    GF_CUDA(cudaEventCreate(&b));
    int rc = GF_OK;
    for (size_t i = 0; i < d->net.layers.size() && !rc; i++) {
        cudaEventRecord(a, d->st);
        for (int r = 0; r < reps && !rc; r++) rc = enqueue_layer(d, (int)i, d->last_n, d->st);
        cudaEventRecord(b, d->st);
        if (cudaEventSynchronize(b) != cudaSuccess || cudaEventElapsedTime(ms + i, a, b) != cudaSuccess) rc = set_err(GF_ERR_CUDA, "timing failed");
        else ms[i] /= reps;
    }
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    return rc;
}

int gf_stage_letterbox(int device, const void* bgr, size_t pitch, int w, int h, int on_device, int net_w, int net_h, float* out)
{
    if (!out || net_w < 1 || net_h < 1 || net_w > 8192 || net_h > 8192) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    int rc = check_frame(bgr, pitch, w, h);
    if (rc) return rc;
    rc = select_device(device);
    if (rc) return rc;
    const uint8_t* src = (const uint8_t*)bgr;
    uint8_t* tmp = nullptr;
    float* d_out = nullptr;
    const size_t n = (size_t)3 * net_w * net_h;
    if (!on_device) {
        GF_CUDA(cudaMalloc(&tmp, (size_t)3 * w * h));
        if (cudaMemcpy2D(tmp, 3 * (size_t)w, bgr, pitch, 3 * (size_t)w, h, cudaMemcpyHostToDevice) != cudaSuccess) {
            cudaFree(tmp);
            return set_err(GF_ERR_CUDA, "frame upload failed");
        }
        src = tmp; pitch = 3 * (size_t)w;
    }
    if (cudaMalloc(&d_out, 4 * n) != cudaSuccess) { cudaFree(tmp); return set_err(GF_ERR_CUDA, "cudaMalloc failed"); }
    LbFrames f;
    set_frame(f, 0, src, (int)pitch, w, h, net_w, net_h);
    launch_letterbox(f, 1, net_w, net_h, d_out, 0);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, 4 * n, cudaMemcpyDeviceToHost);
    cudaFree(d_out);
    cudaFree(tmp);
    if (e != cudaSuccess) return set_err(GF_ERR_CUDA, "letterbox failed: %s", cudaGetErrorString(e));
    return GF_OK;
}

int gf_detector_set_precision(gf_detector* d, int precision)
{
    if (!d) return set_err(GF_ERR_INVALID_ARG, "null detector");
    if (precision != GF_DETECTOR_EXACT && precision != GF_DETECTOR_TF32)
        return set_err(GF_ERR_INVALID_ARG, "precision must be GF_DETECTOR_EXACT (0) or GF_DETECTOR_TF32 (1)");
    if (precision == d->precision) return GF_OK;
    GF_CUDA(cudaSetDevice(d->device));
    GF_CUDA(cudaStreamSynchronize(d->st));
    if (precision == GF_DETECTOR_TF32 && !d->tf32_ready) {
        int rc = tf32_setup();
        for (size_t i = 0; i < d->net.layers.size() && !rc; i++) {
            const Layer& l = d->net.layers[i];
            DevLayer& o = d->dl[i];
            if (l.type != L_CONV || o.w_tf32) continue;
            const int K = l.c * l.size * l.size;
            o.kp = (K + 3) / 4 * 4;
            rc = round_weights_tf32(o.w, l.n, K, o.kp, &o.w_tf32, d->st);
            if (!rc) rc = upload(&o.ktab, tf32_ktab(l.c, l.h, l.w, l.size));
        }
        const size_t part = tf32_part_max(d->net) * d->max_batch;
        if (!rc && part && !d->d_part && cudaMalloc(&d->d_part, 4 * part) != cudaSuccess) rc = set_err(GF_ERR_CUDA, "cudaMalloc failed");
        if (!rc && cudaStreamSynchronize(d->st) != cudaSuccess) rc = set_err(GF_ERR_CUDA, "rounding the weights to TF32 failed");
        if (rc) return rc;
        d->tf32_ready = true;
    }
    // every batch size in use re-captured; the old graphs stay in place unless all succeed
    const int keep = d->precision;
    d->precision = precision;
    cudaGraphExec_t fresh[GF_DETECTOR_BATCH_MAX + 1] = {};
    int rc = GF_OK;
    for (int n = 1; n <= GF_DETECTOR_BATCH_MAX && !rc; n++)
        if (d->exec[n]) rc = capture(d, n, &fresh[n]);
    if (rc) {
        d->precision = keep;
        for (cudaGraphExec_t x : fresh) if (x) cudaGraphExecDestroy(x);
        return rc;
    }
    drop_graphs(d);
    std::copy(fresh, fresh + GF_DETECTOR_BATCH_MAX + 1, d->exec);
    return GF_OK;
}

int gf_detector_get_precision(gf_detector* d, int* precision)
{
    if (!d || !precision) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    *precision = d->precision;
    return GF_OK;
}

int gf_stage_yolo_conv(int device, int precision, const int* shape, const float* in, const float* w, const float* bias,
                       const float* scale, const float* mean, const float* var, float* out)
{
    if (!shape || !in || !w || !bias || !out) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (precision != GF_DETECTOR_EXACT && precision != GF_DETECTOR_TF32) return set_err(GF_ERR_INVALID_ARG, "bad precision");
    const int C = shape[0], H = shape[1], W = shape[2], M = shape[3], size = shape[4], stride = shape[5], pad = shape[6];
    const int bn = shape[7], act_ = shape[8];
    if (C < 1 || H < 1 || W < 1 || M < 1 || size < 1 || stride < 1 || pad < 0 || (bn != 0 && bn != 1) || (act_ != 0 && act_ != 1) ||
        (long)C * H * W > (1l << 28) || (long)C * size * size > (1l << 20) || (bn && (!scale || !mean || !var)))
        return set_err(GF_ERR_INVALID_ARG, "bad shape (C H W M size stride pad bn act)");
    const int OW = (W + 2 * pad - size) / stride + 1, OH = (H + 2 * pad - size) / stride + 1;
    if (OW < 1 || OH < 1) return set_err(GF_ERR_INVALID_ARG, "empty output");
    const int K = C * size * size, N = OW * OH, kp = (K + 3) / 4 * 4;
    if ((long)M * N > (1l << 28) || (long)M * K > (1l << 28)) return set_err(GF_ERR_INVALID_ARG, "layer too large");
    int rc = select_device(device);
    if (!rc && precision == GF_DETECTOR_TF32) rc = tf32_setup();
    if (rc) return rc;
    std::vector<double> den(bn ? M : 0);
    for (int m = 0; m < (bn ? M : 0); m++) den[m] = sqrt((double)var[m]) + (double).000001f;     // as detector_init
    float *d_in = nullptr, *d_w = nullptr, *d_b = nullptr, *d_sc = nullptr, *d_mu = nullptr, *d_out = nullptr, *d_wt = nullptr;
    float* d_part = nullptr;
    int* d_ktab = nullptr;
    double* d_den = nullptr;
    cudaError_t e = cudaSuccess;
    auto put = [&](auto** dst, const auto* src, size_t n) {
        if (e == cudaSuccess) e = cudaMalloc(dst, sizeof(*src) * n);
        if (e == cudaSuccess) e = cudaMemcpy(*dst, src, sizeof(*src) * n, cudaMemcpyHostToDevice);
    };
    put(&d_in, in, (size_t)C * H * W);
    put(&d_w, w, (size_t)M * K);
    put(&d_b, bias, (size_t)M);
    if (bn) { put(&d_sc, scale, (size_t)M); put(&d_mu, mean, (size_t)M); put(&d_den, den.data(), (size_t)M); }
    if (e == cudaSuccess) e = cudaMalloc(&d_out, 4 * (size_t)M * N);
    if (e == cudaSuccess && precision == GF_DETECTOR_TF32) {
        rc = round_weights_tf32(d_w, M, K, kp, &d_wt, 0);
        const std::vector<int> tab = tf32_ktab(C, H, W, size);
        if (!rc) put(&d_ktab, tab.data(), tab.size());
        const size_t np = tf32_part_floats(M, N, K);
        if (!rc && np && e == cudaSuccess) e = cudaMalloc(&d_part, 4 * np);
        if (rc) e = cudaErrorUnknown;
    }
    if (e == cudaSuccess) {
        const ConvArgs a{d_in, d_w, d_out, d_b, d_sc, d_mu, d_den, C, H, W, M, K, OW, N, size, stride, pad, bn, act_};
        Tf32Operands t;
        t.w = d_wt; t.kp = kp; t.ktab = d_ktab; t.part = d_part;
        launch_conv_layer(a, precision, t, 1, 0);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, 4 * (size_t)M * N, cudaMemcpyDeviceToHost);
    cudaFree(d_in); cudaFree(d_w); cudaFree(d_b); cudaFree(d_sc); cudaFree(d_mu); cudaFree(d_den); cudaFree(d_out); cudaFree(d_wt);
    cudaFree(d_part); cudaFree(d_ktab);
    if (rc) return rc;
    if (e != cudaSuccess) return set_err(GF_ERR_CUDA, "convolution stage failed: %s", cudaGetErrorString(e));
    return GF_OK;
}

}  // extern "C"
