// gm_grid.cu -- gf_grid_map_* (C ABI): the 2-D occupancy grid of the reference's grid_mapping tool on the GPU
// (support_files/grid_mapping: main.cpp:114-120, grid_mapper.cpp, grid_map.cpp), built online from the dense map's keyframe
// points and rebuilt after a pose correction.
//   rays     one thread per point: world point, z band [0.1, 0.5], then the tool's ray from the body position in steps of one
//            cell (a sequential double sum r += cs), counted, scanned, and emitted as one 32-bit record per step,
//            cell << 2 | kind, in the tool's (keyframe, point, step) order; a skipped step is SENTINEL
//   sort     a stable LSD radix sort on the cell bits keeps each cell's updates in the tool's order
//   apply    the first thread of each cell's run applies the run's log-odds updates one after another
// The semantics these restate are in one place each below (gm_cell, gm_emit_ray, gm_update, gm_apply_run's shortcuts) and are
// described in DESIGN.md "Occupancy grid".  Built with -fmad=false: bel is bit-identical to oracle/gm_oracle.c in its shared mode.
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "gf_pose.cuh"
#include "gm_math.h"

using namespace gf;

namespace gfgm {

constexpr double Z_LO = 0.1, Z_HI = 0.5;           // main.cpp:117: kept iff !(z > 0.5 || z < 0.1)
constexpr uint32_t SENTINEL = 0xffffffffu;         // cell bits 2^30 - 1: no cell of a grid of < 2^30 cells; sorts last
constexpr long long MAX_STEPS = 1ll << 24;         // steps of one ray (GF_ERR_CAPACITY beyond)
enum { FREE = 0, OCC = 1, PRIOR = 2 };

struct Grid {
    int sx, sy, ix, iy;
    double cs;
    double c[3];                                   // log(p / (1 - p)) by kind, by gm_log
};

// GridMap::getIdx (grid_map.cpp:19-32): cvFloor(x / cs) + init.  The tool's x86 cvFloor turns NaN and values outside int into
// INT_MIN (or a wrapped value), which the range test rejects; CUDA's conversion of NaN gives 0, so the test is made on the floored
// double itself, in exact arithmetic.  Returns the column-major cell x + sx * y, or -1.
__device__ __forceinline__ int gm_cell(const Grid& g, double x, double y)
{
    const double fx = floor(x / g.cs), fy = floor(y / g.cs);
    if (!(fx >= -(double)g.ix && fx < (double)g.sx - (double)g.ix && fy >= -(double)g.iy && fy < (double)g.sy - (double)g.iy)) return -1;
    return ((int)fx + g.ix) + g.sx * ((int)fy + g.iy);
}

// The ray of GridMapper::updateMap (grid_mapper.cpp:12-36) from the body (T0, T1) to (px, py); the unused atan is dropped.  A
// point straight above or below the body gives z = 0, cosz = NaN and one step at a NaN position, which gm_cell rejects.
struct Ray {
    double T0, T1, z, cosz, sinz;
};
__device__ __forceinline__ bool gm_ray(const Ext& e, const Pose& T, const float* l, Ray& q)
{
    double w[3];
    to_world(e, T, l, w);
    if (w[2] > Z_HI || w[2] < Z_LO) return false;
    q.T0 = T.P[0]; q.T1 = T.P[1];
    const double dx = w[0] - q.T0, dy = w[1] - q.T1;
    q.z = sqrt(dy * dy + dx * dx);
    q.cosz = dx / q.z; q.sinz = dy / q.z;
    return true;
}

// one update of GridMapper::updateGrid (:38-46) with GridMap's log / exp round trip (grid_map.cpp:52-67)
__device__ __forceinline__ double gm_update(double bel, double c)
{
    double l = gm_log(bel / (1.0 - bel));
    l = l + c;
    return 1.0 - 1.0 / (1 + gm_exp(l));
}

// point i (of [p0, p0 + n)) of keyframe kf[i] into the packed float3 store, from rows of `stride` floats; bad = a non-finite value
__global__ void k_gm_pack(int n, const float* __restrict__ in, int stride, float* __restrict__ out, int* bad)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int k = 0; k < 3; k++) {
        const float v = in[(size_t)stride * i + k];
        if (!isfinite(v)) atomicExch(bad, 1);
        out[3 * (size_t)i + k] = v;
    }
}

// the number of steps of the ray of camera-frame point l under T (0 outside the band); *bad set beyond MAX_STEPS
__device__ __forceinline__ long long gm_steps(const Ext& e, const Pose& T, const Grid& g, const float* l, int* bad)
{
    Ray q;
    long long c = 0;
    if (gm_ray(e, T, l, q)) {
        for (double r = 0; r < q.z + g.cs; r += g.cs)
            if (++c > MAX_STEPS) { atomicExch(bad, 1); break; }
    }
    return c;
}
// the number of steps of each point's ray; cnt[n] = 0 for the exclusive scan's total
__global__ void k_gm_count(int n, int p0, const float* __restrict__ pts, const int* __restrict__ kf, const Pose* __restrict__ poses, Ext e, Grid g,
                           long long* __restrict__ cnt, int* bad)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > n) return;
    if (j == n) { cnt[n] = 0; return; }
    const int i = p0 + j;
    cnt[j] = gm_steps(e, poses[kf[i]], g, pts + 3 * (size_t)i, bad);
}

// records [a, b) of the ray steps of camera-frame point l, whose steps are records [o, ...): hi | (cell << 2 | kind)
template <typename T>
__device__ __forceinline__ void gm_emit_ray(const Ext& e, const Pose& P, const Grid& g, const float* l, long long o, long long a, long long b, T hi,
                                            T* __restrict__ rec)
{
    Ray q;
    gm_ray(e, P, l, q);
    const double cs = g.cs;
    double lx = -1.0, ly = -1.0;                   // Eigen::Vector2d(Eigen::Infinity, Eigen::Infinity): Infinity is the integer -1
    long long s = o;
    for (double r = 0; r < q.z + cs && s < b; r += cs, s++) {
        const double px = r * q.cosz + q.T0, py = r * q.sinz + q.T1;
        uint32_t v = SENTINEL;
        if (!(px == lx && py == ly)) {             // the tool skips a step that repeats the last position
            const int kind = r < (q.z - 0.5 * cs) ? FREE : (r > (q.z + 0.5 * cs) ? PRIOR : OCC);   // laserInvModel, :48-57
            const int cell = gm_cell(g, px, py);
            if (cell >= 0) v = (uint32_t)cell << 2 | (uint32_t)kind;
            lx = px; ly = py;
        }
        if (s >= a) rec[s - a] = hi | (T)v;
    }
}
// records [a, b) of the ray steps, in (point, step) order: step s of point j is record off[j] + s
__global__ void k_gm_emit(int n, int p0, const float* __restrict__ pts, const int* __restrict__ kf, const Pose* __restrict__ poses, Ext e, Grid g,
                          const long long* __restrict__ off, long long a, long long b, uint32_t* __restrict__ rec)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const long long o = off[j], o1 = off[j + 1];
    if (o1 == o || o1 <= a || o >= b) return;
    const int i = p0 + j;
    gm_emit_ray<uint32_t>(e, poses[kf[i]], g, pts + 3 * (size_t)i, o, a, b, 0u, rec);
}

// Over the records sorted stably by (record >> 2): the first thread of each cell's run applies the run in order.  Two shortcuts
// are exact: an update that leaves bel unchanged leaves it unchanged again, so the records of the same kind that follow it are
// skipped; and 0 and 1 absorb every kind (log(0) = -inf, log(inf) = inf).  stats: updates applied, updates skipped, longest run.
template <typename T>
__device__ __forceinline__ void gm_apply_run(int i, int n, const T* __restrict__ srec, const Grid& g, double* __restrict__ bel, unsigned long long* stats)
{
    const T v = srec[i];
    if ((uint32_t)v == SENTINEL) return;
    const uint32_t cell = (uint32_t)v >> 2;
    const T run = v >> 2;
    if (i > 0 && (srec[i - 1] >> 2) == run) return;
    int end = i + 1;
    while (end < n && (srec[end] >> 2) == run) end++;
    double b = bel[cell];
    int j = i;
    unsigned long long applied = 0;
    while (j < end && b != 0.0 && b != 1.0) {
        const uint32_t kind = (uint32_t)srec[j] & 3u;
        const double nb = gm_update(b, kind == FREE ? g.c[FREE] : (kind == OCC ? g.c[OCC] : g.c[PRIOR]));
        applied++;
        j++;
        if (nb == b)
            while (j < end && ((uint32_t)srec[j] & 3u) == kind) j++;
        b = nb;
    }
    bel[cell] = b;
    atomicAdd(&stats[0], applied);
    atomicAdd(&stats[1], (unsigned long long)(end - i) - applied);
    atomicMax(&stats[2], (unsigned long long)(end - i));
}
__global__ void k_gm_apply(int n, const uint32_t* __restrict__ srec, Grid g, double* __restrict__ bel, unsigned long long* stats)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    gm_apply_run<uint32_t>(i, n, srec, g, bel, stats);
}

// GridMap::saveMap's pixels (grid_map.cpp:74-87, 113-118): 1 - bel, rows = x, flipped, * 255, converted to 8 bits with round
// half to even and saturation; and the node's OccupancyGrid from those pixels (pose_graph_node.cpp:865-899): convertTo(CV_32F,
// 1 / 255.0), value = 1 - v, -1 unless |value - 0.5| > 0.005, else (signed char)(value * 100) at x + sx * y
__global__ void k_gm_outputs(int sx, int ncell, const double* __restrict__ bel, uint8_t* __restrict__ img, int8_t* __restrict__ occ)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ncell) return;
    const int x = i % sx, y = i / sx, sy = ncell / sx;
    const double m = rint((1.0 - bel[i]) * 255.0);
    const int px = m <= 0 ? 0 : (m >= 255 ? 255 : (int)m);
    img[(size_t)(sx - 1 - x) * sy + y] = (uint8_t)px;
    const float f = (float)px * (float)(1 / 255.0);
    const double value = 1.0 - 1.0 * (double)f;
    occ[i] = fabs(value - 0.5) > 0.005 ? (int8_t)(value * 100) : (int8_t)-1;
}

}  // namespace gfgm

using namespace gfgm;

struct gf_grid_map {
    int device = 0;
    cudaStream_t st = nullptr;
    gf_grid_map_cfg cfg;
    Grid grid;
    Ext ext;
    int ncell = 0;
    // host state
    int n_points = 0;
    std::vector<Pose> poses;                       // the pose each keyframe was last applied with
    std::vector<int> kf_off{0};                    // keyframe k's points are [kf_off[k], kf_off[k+1])
    long long stats[4] = {0, 0, 0, 0};             // last call: records, applied, skipped, longest run
    // device
    double* bel = nullptr;
    float* pts = nullptr;                          // [max_points][3] camera-frame points
    int* kf = nullptr;                             // keyframe of each point
    Pose *dposes = nullptr, *dposes2 = nullptr;    // current poses; a rebuild's new poses until it commits
    long long* cnt = nullptr; long long* off = nullptr;
    uint32_t *rec = nullptr, *srec = nullptr;
    uint8_t* img = nullptr; int8_t* occ = nullptr;
    int* bad = nullptr;
    unsigned long long* dstats = nullptr;
    void* tmp = nullptr; size_t tmp_bytes = 0;
    long long* h_pin = nullptr;                    // pinned: total records, bad flag, stats
};

static int gm_device(int device)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return set_err(GF_ERR_NO_DEVICE, "no CUDA device visible; libgf_b200 has no CPU fallback");
    if (device < 0 || device >= n) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    return GF_OK;
}

static void gm_free(gf_grid_map* m)
{
    for (void* p : {(void*)m->bel, (void*)m->pts, (void*)m->kf, (void*)m->dposes, (void*)m->dposes2, (void*)m->cnt, (void*)m->off, (void*)m->rec,
                    (void*)m->srec, (void*)m->img, (void*)m->occ, (void*)m->bad, (void*)m->dstats, m->tmp})
        if (p) cudaFree(p);
    if (m->h_pin) cudaFreeHost(m->h_pin);
    if (m->st) cudaStreamDestroy(m->st);
    delete m;
}

static bool finite_all(const double* v, size_t n)
{
    for (size_t i = 0; i < n; i++) if (!std::isfinite(v[i])) return false;
    return true;
}

// Rays of the points [p0, p0 + n) under `poses`: count their steps; on return h_pin[0] = total records, h_pin[1] = a ray longer
// than MAX_STEPS.  Nothing of the grid's state is written.
static int gm_count(gf_grid_map* m, int p0, int n, const Pose* poses)
{
    GF_CUDA(cudaMemsetAsync(m->bad, 0, 4, m->st));
    k_gm_count<<<(n + 1 + 127) / 128, 128, 0, m->st>>>(n, p0, m->pts, m->kf, poses, m->ext, m->grid, m->cnt, m->bad);
    GF_LAUNCHED();
    size_t b = m->tmp_bytes;
    GF_CUDA(cub::DeviceScan::ExclusiveSum(m->tmp, b, m->cnt, m->off, n + 1, m->st));
    m->h_pin[1] = 0;
    GF_CUDA(cudaMemcpyAsync(m->h_pin, m->off + n, 8, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaMemcpyAsync(m->h_pin + 1, m->bad, 4, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaStreamSynchronize(m->st));
    return GF_OK;
}

// Emit, sort and apply the counted records in chunks of at most max_records: each cell's updates stay in order across chunks
static int gm_apply(gf_grid_map* m, int p0, int n, const Pose* poses, long long total)
{
    GF_CUDA(cudaMemsetAsync(m->dstats, 0, 3 * sizeof(unsigned long long), m->st));
    const long long M = m->cfg.max_records;
    for (long long a = 0; a < total; a += M) {
        const long long b = std::min(total, a + M);
        const int nr = (int)(b - a);
        k_gm_emit<<<(n + 127) / 128, 128, 0, m->st>>>(n, p0, m->pts, m->kf, poses, m->ext, m->grid, m->off, a, b, m->rec);
        GF_LAUNCHED();
        size_t tb = m->tmp_bytes;
        GF_CUDA(cub::DeviceRadixSort::SortKeys(m->tmp, tb, m->rec, m->srec, nr, 2, 32, m->st));
        k_gm_apply<<<(nr + 127) / 128, 128, 0, m->st>>>(nr, m->srec, m->grid, m->bel, m->dstats);
        GF_LAUNCHED();
    }
    GF_CUDA(cudaMemcpyAsync(m->h_pin + 2, m->dstats, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaStreamSynchronize(m->st));
    m->stats[0] = total; m->stats[1] = m->h_pin[2]; m->stats[2] = m->h_pin[3]; m->stats[3] = m->h_pin[4];
    return GF_OK;
}

extern "C" {

int gf_grid_map_create(gf_grid_map** out, int device, const gf_grid_map_cfg* cfg)
{
    if (!out || !cfg) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    *out = nullptr;
    const gf_grid_map_cfg& c = *cfg;
    const double ps[3] = {c.p_occ, c.p_free, c.p_prior};
    if (c.size_x < 1 || c.size_y < 1 || (long long)c.size_x * c.size_y >= (1ll << 30))
        return set_err(GF_ERR_INVALID_ARG, "bad grid size (size_x, size_y >= 1, size_x * size_y < 2^30)");
    if (!(c.cell_size > 0) || !std::isfinite(c.cell_size)) return set_err(GF_ERR_INVALID_ARG, "cell_size must be positive and finite");
    for (double p : ps) if (!(p > 0 && p < 1)) return set_err(GF_ERR_INVALID_ARG, "probabilities must lie in (0, 1)");
    if (!finite_all(c.ric, 9) || !finite_all(c.tic, 3)) return set_err(GF_ERR_INVALID_ARG, "ric / tic not finite");
    if (c.max_points < 1 || c.max_keyframes < 1 || c.max_records < 1) return set_err(GF_ERR_INVALID_ARG, "capacities must be >= 1");
    if (c.max_points > (1 << 29) || c.max_records > (1 << 30)) return set_err(GF_ERR_CAPACITY, "max_points above 2^29 or max_records above 2^30");
    int rc = gm_device(device);
    if (rc) return rc;
    gf_grid_map* m = new gf_grid_map();
    m->device = device;
    m->cfg = c;
    m->grid.sx = c.size_x; m->grid.sy = c.size_y; m->grid.ix = c.init_x; m->grid.iy = c.init_y; m->grid.cs = c.cell_size;
    m->grid.c[FREE] = gm_log(c.p_free / (1.0 - c.p_free));
    m->grid.c[OCC] = gm_log(c.p_occ / (1.0 - c.p_occ));
    m->grid.c[PRIOR] = gm_log(c.p_prior / (1.0 - c.p_prior));
    memcpy(m->ext.ric, c.ric, sizeof(m->ext.ric)); memcpy(m->ext.tic, c.tic, sizeof(m->ext.tic));
    m->ncell = c.size_x * c.size_y;
    m->poses.reserve(c.max_keyframes);
    const size_t N = (size_t)c.max_points, R = (size_t)c.max_records, C = (size_t)m->ncell;
#define GM_ALLOC(p, bytes) do { if (cudaMalloc(&(p), (bytes)) != cudaSuccess) { cudaGetLastError(); gm_free(m); return set_err(GF_ERR_CUDA, "cudaMalloc failed (grid map)"); } } while (0)
    if (cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking) != cudaSuccess) { gm_free(m); return set_err(GF_ERR_CUDA, "stream creation failed"); }
    GM_ALLOC(m->bel, 8 * C); GM_ALLOC(m->img, C); GM_ALLOC(m->occ, C);
    GM_ALLOC(m->pts, 12 * N); GM_ALLOC(m->kf, 4 * N); GM_ALLOC(m->cnt, 8 * (N + 1)); GM_ALLOC(m->off, 8 * (N + 1));
    GM_ALLOC(m->dposes, sizeof(Pose) * (size_t)c.max_keyframes); GM_ALLOC(m->dposes2, sizeof(Pose) * (size_t)c.max_keyframes);
    GM_ALLOC(m->rec, 4 * R); GM_ALLOC(m->srec, 4 * R);
    GM_ALLOC(m->bad, 4); GM_ALLOC(m->dstats, 3 * sizeof(unsigned long long));
#undef GM_ALLOC
    size_t b1 = 0, b2 = 0;
    if (cub::DeviceRadixSort::SortKeys(nullptr, b1, m->rec, m->srec, c.max_records, 2, 32) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, b2, m->cnt, m->off, c.max_points + 1) != cudaSuccess) { gm_free(m); return set_err(GF_ERR_CUDA, "cub sizing failed"); }
    m->tmp_bytes = std::max(b1, b2);
    if (cudaMalloc(&m->tmp, m->tmp_bytes) != cudaSuccess || cudaMallocHost(&m->h_pin, 8 * sizeof(long long)) != cudaSuccess) {
        cudaGetLastError(); gm_free(m); return set_err(GF_ERR_CUDA, "allocation failed (grid map)");
    }
    std::vector<double> half(C, 0.5);
    if (cudaMemcpy(m->bel, half.data(), 8 * C, cudaMemcpyHostToDevice) != cudaSuccess) { gm_free(m); return set_err(GF_ERR_CUDA, "initialisation failed (grid map)"); }
    *out = m;
    return GF_OK;
}

void gf_grid_map_destroy(gf_grid_map* m)
{
    if (!m) return;
    cudaSetDevice(m->device);
    cudaStreamSynchronize(m->st);
    gm_free(m);
}

int gf_grid_map_add_keyframe(gf_grid_map* m, const double* R, const double* P, const float* pts, int n, int stride_floats, int on_device)
{
    if (!m || !R || !P || n < 0 || (n > 0 && !pts) || stride_floats < 3) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (!finite_all(R, 9) || !finite_all(P, 3)) return set_err(GF_ERR_INVALID_ARG, "pose not finite");
    const int k = (int)m->poses.size();
    if (k >= m->cfg.max_keyframes) return set_err(GF_ERR_CAPACITY, "max_keyframes reached");
    if ((long long)m->n_points + n > m->cfg.max_points) return set_err(GF_ERR_CAPACITY, "max_points reached");
    if (!on_device)
        for (size_t i = 0; i < (size_t)n; i++)
            for (int a = 0; a < 3; a++) if (!std::isfinite(pts[(size_t)stride_floats * i + a])) return set_err(GF_ERR_INVALID_ARG, "point not finite");
    GF_CUDA(cudaSetDevice(m->device));
    Pose T;
    memcpy(T.R, R, sizeof(T.R)); memcpy(T.P, P, sizeof(T.P));
    const int p0 = m->n_points;
    // the new points, keyframe ids and pose go past the committed ends: the state is unchanged until they are counted in
    if (n > 0) {
        float* dst = m->pts + 3 * (size_t)p0;
        GF_CUDA(cudaMemsetAsync(m->bad, 0, 4, m->st));
        if (on_device) {
            k_gm_pack<<<(n + 255) / 256, 256, 0, m->st>>>(n, pts, stride_floats, dst, m->bad);
            GF_LAUNCHED();
        } else {
            GF_CUDA(cudaMemcpy2DAsync(dst, 12, pts, 4 * (size_t)stride_floats, 12, n, cudaMemcpyHostToDevice, m->st));
        }
        std::vector<int> ids(n, k);
        GF_CUDA(cudaMemcpyAsync(m->kf + p0, ids.data(), 4 * (size_t)n, cudaMemcpyHostToDevice, m->st));
        GF_CUDA(cudaMemcpyAsync(m->dposes + k, &T, sizeof(Pose), cudaMemcpyHostToDevice, m->st));
        m->h_pin[1] = 0;
        GF_CUDA(cudaMemcpyAsync(m->h_pin + 1, m->bad, 4, cudaMemcpyDeviceToHost, m->st));
        GF_CUDA(cudaStreamSynchronize(m->st));
        if ((int)m->h_pin[1]) return set_err(GF_ERR_INVALID_ARG, "point not finite");
        int rc = gm_count(m, p0, n, m->dposes);
        if (rc) return rc;
        if ((int)m->h_pin[1]) return set_err(GF_ERR_CAPACITY, "a ray longer than 2^24 steps");
        // commit
        if ((rc = gm_apply(m, p0, n, m->dposes, m->h_pin[0]))) return rc;
    } else {
        GF_CUDA(cudaMemcpy(m->dposes + k, &T, sizeof(Pose), cudaMemcpyHostToDevice));
        m->stats[0] = m->stats[1] = m->stats[2] = m->stats[3] = 0;
    }
    m->n_points += n;
    m->kf_off.push_back(m->n_points);
    m->poses.push_back(T);
    return GF_OK;
}

int gf_grid_map_update_poses(gf_grid_map* m, int n_keyframes, const double* R, const double* P)
{
    if (!m || (n_keyframes > 0 && (!R || !P))) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n_keyframes != (int)m->poses.size()) return set_err(GF_ERR_INVALID_ARG, "n_keyframes differs from the number of keyframes added");
    if (!finite_all(R, 9 * (size_t)n_keyframes) || !finite_all(P, 3 * (size_t)n_keyframes)) return set_err(GF_ERR_INVALID_ARG, "pose not finite");
    GF_CUDA(cudaSetDevice(m->device));
    std::vector<Pose> np(n_keyframes);
    for (int k = 0; k < n_keyframes; k++) { memcpy(np[k].R, R + 9 * (size_t)k, sizeof(np[k].R)); memcpy(np[k].P, P + 3 * (size_t)k, sizeof(np[k].P)); }
    const int n = m->n_points;
    long long total = 0;
    if (n_keyframes > 0) GF_CUDA(cudaMemcpyAsync(m->dposes2, np.data(), sizeof(Pose) * (size_t)n_keyframes, cudaMemcpyHostToDevice, m->st));
    if (n > 0) {
        int rc = gm_count(m, 0, n, m->dposes2);
        if (rc) return rc;
        if ((int)m->h_pin[1]) return set_err(GF_ERR_CAPACITY, "a ray longer than 2^24 steps");
        total = m->h_pin[0];
    }
    // commit: the grid back to 0.5, then every keyframe again in order
    std::vector<double> half((size_t)m->ncell, 0.5);
    GF_CUDA(cudaMemcpyAsync(m->bel, half.data(), 8 * (size_t)m->ncell, cudaMemcpyHostToDevice, m->st));
    std::swap(m->dposes, m->dposes2);
    m->poses = np;
    if (n > 0) return gm_apply(m, 0, n, m->dposes, total);
    GF_CUDA(cudaStreamSynchronize(m->st));
    m->stats[0] = m->stats[1] = m->stats[2] = m->stats[3] = 0;
    return GF_OK;
}

int gf_grid_map_read(gf_grid_map* m, int which, void* out)
{
    if (!m || !out || which < GF_GRID_MAP_BEL || which > GF_GRID_MAP_OCCUPANCY) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    GF_CUDA(cudaSetDevice(m->device));
    const size_t C = (size_t)m->ncell;
    if (which == GF_GRID_MAP_BEL) {
        GF_CUDA(cudaMemcpyAsync(out, m->bel, 8 * C, cudaMemcpyDeviceToHost, m->st));
    } else {
        k_gm_outputs<<<(m->ncell + 255) / 256, 256, 0, m->st>>>(m->cfg.size_x, m->ncell, m->bel, m->img, m->occ);
        GF_LAUNCHED();
        GF_CUDA(cudaMemcpyAsync(out, which == GF_GRID_MAP_IMAGE ? (void*)m->img : (void*)m->occ, C, cudaMemcpyDeviceToHost, m->st));
    }
    GF_CUDA(cudaStreamSynchronize(m->st));
    return GF_OK;
}

int gf_grid_map_size(gf_grid_map* m, int* size_x, int* size_y, int* n_keyframes, int* n_points)
{
    if (!m) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (size_x) *size_x = m->cfg.size_x;
    if (size_y) *size_y = m->cfg.size_y;
    if (n_keyframes) *n_keyframes = (int)m->poses.size();
    if (n_points) *n_points = m->n_points;
    return GF_OK;
}

int gf_grid_map_stats(gf_grid_map* m, int64_t* out4)
{
    if (!m || !out4) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    for (int i = 0; i < 4; i++) out4[i] = m->stats[i];
    return GF_OK;
}

}  // extern "C"

// ---- gf_grid_map_group: one keyframe for each of several grids with one launch chain ----
// The members' points are concatenated (member a's are [base[a], base[a + 1])) and so are their records, in (member, point,
// step) order.  A record is member << 32 | cell << 2 | kind: sorting it stably on bits [2, 38) keeps every member's cells
// apart and each cell's updates in the member's order.  Chunks of max_records cut that sequence in order, so each member's
// updates stay in order across chunks as in the single grid.
namespace gfgm {

constexpr int GROUP_MAX = 64;

struct GmMember {                                     // one member of a group call
    Grid grid; Ext ext; Pose T;
    const float* src; int stride, on_device;          // the caller's points (device ones are packed here)
    float* pts; int* kf; Pose* dposes; double* bel;
    int p0, k;
};

__device__ __forceinline__ int gm_seg(const int* __restrict__ base, int F, int i)
{
    int lo = 0, hi = F;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (base[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// every member's pose; then per point: device points packed into the member's store, the keyframe id
__global__ void k_gmg_poses(int A, const GmMember* __restrict__ mb)
{
    const int a = threadIdx.x;
    if (a < A) mb[a].dposes[mb[a].k] = mb[a].T;
}
__global__ void k_gmg_prep(int N, const GmMember* __restrict__ mb, const int* __restrict__ base, int A, int* bad)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N) return;
    const int a = gm_seg(base, A, t), l = t - base[a];
    const GmMember& M = mb[a];
    if (M.on_device)
        for (int k = 0; k < 3; k++) {
            const float v = M.src[(size_t)M.stride * l + k];
            if (!isfinite(v)) atomicExch(&bad[a], 1);
            M.pts[3 * ((size_t)M.p0 + l) + k] = v;
        }
    M.kf[M.p0 + l] = M.k;
}
// cnt[t] = the steps of point t (0 for a member with a non-finite point); cnt[N] = 0
__global__ void k_gmg_count(int N, const GmMember* __restrict__ mb, const int* __restrict__ base, int A, const int* __restrict__ bad,
                            int* __restrict__ longray, long long* __restrict__ cnt)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t > N) return;
    if (t == N) { cnt[N] = 0; return; }
    const int a = gm_seg(base, A, t);
    const GmMember& M = mb[a];
    cnt[t] = bad[a] ? 0 : gm_steps(M.ext, M.T, M.grid, M.pts + 3 * ((size_t)M.p0 + t - base[a]), &longray[a]);
}
// res[3 a] = member a's records, res[3 a + 1] its non-finite flag, res[3 a + 2] its long-ray flag
__global__ void k_gmg_totals(int A, const int* __restrict__ base, const long long* __restrict__ off, const int* __restrict__ bad,
                             const int* __restrict__ longray, long long* __restrict__ res)
{
    const int a = threadIdx.x;
    if (a >= A) return;
    res[3 * a] = off[base[a + 1]] - off[base[a]];
    res[3 * a + 1] = bad[a];
    res[3 * a + 2] = longray[a];
}
// the points of the members not in ok cast no ray
__global__ void k_gmg_drop(int N, const int* __restrict__ base, int A, uint64_t ok, long long* __restrict__ cnt)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N) return;
    if (!((ok >> gm_seg(base, A, t)) & 1)) cnt[t] = 0;
}
__global__ void k_gmg_emit(int N, const GmMember* __restrict__ mb, const int* __restrict__ base, int A, const long long* __restrict__ off,
                           long long a, long long b, uint64_t* __restrict__ rec)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N) return;
    const long long o = off[t], o1 = off[t + 1];
    if (o1 == o || o1 <= a || o >= b) return;
    const int s = gm_seg(base, A, t);
    const GmMember& M = mb[s];
    gm_emit_ray<uint64_t>(M.ext, M.T, M.grid, M.pts + 3 * ((size_t)M.p0 + t - base[s]), o, a, b, (uint64_t)s << 32, rec);
}
__global__ void k_gmg_apply(int n, const uint64_t* __restrict__ srec, const GmMember* __restrict__ mb, unsigned long long* stats)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = (int)(srec[i] >> 32);
    gm_apply_run<uint64_t>(i, n, srec, mb[s].grid, mb[s].bel, stats + 3 * s);
}

}  // namespace gfgm

struct GmCall {
    GmMember mb[GROUP_MAX];
    int base[GROUP_MAX + 1];
};

struct gf_grid_map_group {
    int device = 0, n = 0;
    long long pcap = 0, max_records = 0;
    std::vector<gf_grid_map*> m;
    cudaStream_t st = nullptr;
    cudaEvent_t ev = nullptr;
    GmCall* h = nullptr;                              // pageable host copy of the descriptors
    GmCall* d = nullptr;
    long long *cnt = nullptr, *off = nullptr, *res = nullptr;
    uint64_t *rec = nullptr, *srec = nullptr;
    int *bad = nullptr, *longray = nullptr;
    unsigned long long* dstats = nullptr;
    void* tmp = nullptr; size_t tmp_bytes = 0;
    long long* h_res = nullptr;                       // pinned: per member 3 totals / flags, then 3 stats
};

static int gm_member_err(int rc, int k)
{
    char keep[sizeof(g_err)];
    memcpy(keep, g_err, sizeof(keep));
    snprintf(g_err, sizeof(g_err), "member %d: %s", k, keep);
    return rc;
}

static void gmg_free(gf_grid_map_group* g)
{
    for (void* p : {(void*)g->d, (void*)g->cnt, (void*)g->off, (void*)g->res, (void*)g->rec, (void*)g->srec, (void*)g->bad, (void*)g->longray,
                    (void*)g->dstats, g->tmp})
        if (p) cudaFree(p);
    if (g->h_res) cudaFreeHost(g->h_res);
    if (g->ev) cudaEventDestroy(g->ev);
    if (g->st) cudaStreamDestroy(g->st);
    delete g->h;
    delete g;
}

gf_dense_map* gf_dense_map_group_member(gf_dense_map_group* g, int k);
int gf_dense_map_last_keyframe_device(gf_dense_map* m, const float** xyz, int* n, cudaStream_t* st, int* device);

// The group call over m members with per-member point sources; dense_st (nullable): the streams that wrote them.
static int gmg_add(gf_grid_map_group* g, const int32_t* members, int m, const double* R, const double* P, const float* const* pts, const int* n_pts,
                   const int* stride, int on_device, const cudaStream_t* dense_st, int32_t* status)
{
    std::vector<int> st(m, GF_OK), act;
    int first = GF_OK;
    char first_err[sizeof(g_err)] = "";
    auto fail = [&](int j, int rc) { st[j] = gm_member_err(rc, j); if (first == GF_OK) { first = rc; memcpy(first_err, g_err, sizeof(first_err)); } };
    for (int j = 0; j < m; j++) {                     // the single call's checks, in its order
        gf_grid_map* gm = g->m[members[j]];
        const int n = n_pts[j];
        if (!finite_all(R + 9 * (size_t)j, 9) || !finite_all(P + 3 * (size_t)j, 3)) { fail(j, set_err(GF_ERR_INVALID_ARG, "pose not finite")); continue; }
        if ((int)gm->poses.size() >= gm->cfg.max_keyframes) { fail(j, set_err(GF_ERR_CAPACITY, "max_keyframes reached")); continue; }
        if ((long long)gm->n_points + n > gm->cfg.max_points) { fail(j, set_err(GF_ERR_CAPACITY, "max_points reached")); continue; }
        bool finite = true;
        if (!on_device)
            for (size_t i = 0; i < (size_t)n && finite; i++)
                for (int a = 0; a < 3; a++) if (!std::isfinite(pts[j][(size_t)stride[j] * i + a])) finite = false;
        if (!finite) { fail(j, set_err(GF_ERR_INVALID_ARG, "point not finite")); continue; }
        act.push_back(j);
    }
    const int A = (int)act.size();
    if (A > 0) {
        GF_CUDA(cudaSetDevice(g->device));
        GmCall& c = *g->h;
        c.base[0] = 0;
        for (int a = 0; a < A; a++) {
            const int j = act[a];
            gf_grid_map* gm = g->m[members[j]];
            GF_CUDA(cudaEventRecord(g->ev, gm->st));
            GF_CUDA(cudaStreamWaitEvent(g->st, g->ev, 0));
            if (dense_st) {
                GF_CUDA(cudaEventRecord(g->ev, dense_st[j]));
                GF_CUDA(cudaStreamWaitEvent(g->st, g->ev, 0));
            }
            GmMember& M = c.mb[a];
            M.grid = gm->grid; M.ext = gm->ext;
            memcpy(M.T.R, R + 9 * (size_t)j, sizeof(M.T.R)); memcpy(M.T.P, P + 3 * (size_t)j, sizeof(M.T.P));
            M.src = pts[j]; M.stride = stride[j]; M.on_device = on_device;
            M.pts = gm->pts; M.kf = gm->kf; M.dposes = gm->dposes; M.bel = gm->bel;
            M.p0 = gm->n_points; M.k = (int)gm->poses.size();
            c.base[a + 1] = c.base[a] + n_pts[j];
            if (!on_device && n_pts[j] > 0)
                GF_CUDA(cudaMemcpy2DAsync(gm->pts + 3 * (size_t)M.p0, 12, pts[j], 4 * (size_t)stride[j], 12, n_pts[j], cudaMemcpyHostToDevice, g->st));
        }
        const int N = c.base[A];
        GF_CUDA(cudaMemcpyAsync(g->d->mb, c.mb, sizeof(GmMember) * A, cudaMemcpyHostToDevice, g->st));
        GF_CUDA(cudaMemcpyAsync(g->d->base, c.base, 4 * (size_t)(A + 1), cudaMemcpyHostToDevice, g->st));
        GF_CUDA(cudaMemsetAsync(g->bad, 0, 4 * A, g->st));
        GF_CUDA(cudaMemsetAsync(g->longray, 0, 4 * A, g->st));
        GF_CUDA(cudaMemsetAsync(g->dstats, 0, 3 * sizeof(unsigned long long) * A, g->st));
        k_gmg_poses<<<1, GROUP_MAX, 0, g->st>>>(A, g->d->mb);
        GF_LAUNCHED();
        if (N > 0) {
            k_gmg_prep<<<(N + 255) / 256, 256, 0, g->st>>>(N, g->d->mb, g->d->base, A, g->bad);
            GF_LAUNCHED();
        }
        k_gmg_count<<<(N + 1 + 127) / 128, 128, 0, g->st>>>(N, g->d->mb, g->d->base, A, g->bad, g->longray, g->cnt);
        GF_LAUNCHED();
        size_t b = g->tmp_bytes;
        GF_CUDA(cub::DeviceScan::ExclusiveSum(g->tmp, b, g->cnt, g->off, N + 1, g->st));
        k_gmg_totals<<<1, GROUP_MAX, 0, g->st>>>(A, g->d->base, g->off, g->bad, g->longray, g->res);
        GF_LAUNCHED();
        GF_CUDA(cudaMemcpyAsync(g->h_res, g->res, 3 * sizeof(long long) * A, cudaMemcpyDeviceToHost, g->st));
        GF_CUDA(cudaStreamSynchronize(g->st));
        uint64_t ok = 0;
        long long total = 0;
        std::vector<long long> recs(A);
        for (int a = 0; a < A; a++) {
            const int j = act[a];
            recs[a] = g->h_res[3 * a];
            if (g->h_res[3 * a + 1]) fail(j, set_err(GF_ERR_INVALID_ARG, "point not finite"));
            else if (g->h_res[3 * a + 2]) fail(j, set_err(GF_ERR_CAPACITY, "a ray longer than 2^24 steps"));
            else { ok |= 1ull << a; total += recs[a]; }
        }
        if (ok != (A == 64 ? ~0ull : (1ull << A) - 1) && N > 0) {   // the failed members' rays leave the sequence
            k_gmg_drop<<<(N + 255) / 256, 256, 0, g->st>>>(N, g->d->base, A, ok, g->cnt);
            GF_LAUNCHED();
            b = g->tmp_bytes;
            GF_CUDA(cub::DeviceScan::ExclusiveSum(g->tmp, b, g->cnt, g->off, N + 1, g->st));
        }
        const long long M = g->max_records;
        for (long long a0 = 0; a0 < total; a0 += M) {
            const long long b1 = std::min(total, a0 + M);
            const int nr = (int)(b1 - a0);
            k_gmg_emit<<<(N + 127) / 128, 128, 0, g->st>>>(N, g->d->mb, g->d->base, A, g->off, a0, b1, g->rec);
            GF_LAUNCHED();
            size_t tb = g->tmp_bytes;
            GF_CUDA(cub::DeviceRadixSort::SortKeys(g->tmp, tb, g->rec, g->srec, nr, 2, 38, g->st));
            k_gmg_apply<<<(nr + 127) / 128, 128, 0, g->st>>>(nr, g->srec, g->d->mb, g->dstats);
            GF_LAUNCHED();
        }
        GF_CUDA(cudaMemcpyAsync(g->h_res + 3 * GROUP_MAX, g->dstats, 3 * sizeof(unsigned long long) * A, cudaMemcpyDeviceToHost, g->st));
        GF_CUDA(cudaStreamSynchronize(g->st));
        GF_CUDA(cudaEventRecord(g->ev, g->st));
        for (int a = 0; a < A; a++) {
            gf_grid_map* gm = g->m[members[act[a]]];
            GF_CUDA(cudaStreamWaitEvent(gm->st, g->ev, 0));
            if (!((ok >> a) & 1)) continue;
            gm->n_points += c.base[a + 1] - c.base[a];
            gm->kf_off.push_back(gm->n_points);
            gm->poses.push_back(c.mb[a].T);
            const long long* s3 = g->h_res + 3 * GROUP_MAX + 3 * a;
            gm->stats[0] = recs[a]; gm->stats[1] = s3[0]; gm->stats[2] = s3[1]; gm->stats[3] = s3[2];
        }
    }
    if (status) for (int j = 0; j < m; j++) status[j] = st[j];
    if (first != GF_OK) memcpy(g_err, first_err, sizeof(first_err));
    return first;
}

static int gmg_check_members(gf_grid_map_group* g, const int32_t* members, int m)
{
    if (m < 1 || m > g->n) return set_err(GF_ERR_INVALID_ARG, "m must lie in [1, group size]");
    uint64_t seen = 0;
    for (int j = 0; j < m; j++) {
        const int k = members[j];
        if (k < 0 || k >= g->n) return gm_member_err(set_err(GF_ERR_INVALID_ARG, "member index out of range"), j);
        if ((seen >> k) & 1) return gm_member_err(set_err(GF_ERR_INVALID_ARG, "the member is listed twice"), j);
        seen |= 1ull << k;
    }
    return GF_OK;
}

extern "C" {

int gf_grid_map_group_create(gf_grid_map_group** out, gf_grid_map* const* grids, int n)
{
    if (!out || !grids) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    if (n < 1) return set_err(GF_ERR_INVALID_ARG, "a group has at least one grid");
    if (n > GROUP_MAX) return set_err(GF_ERR_INVALID_ARG, "a group has at most GF_GRID_MAP_GROUP_MAX (64) grids");
    long long pcap = 0, mr = grids[0] ? grids[0]->cfg.max_records : 0;
    for (int k = 0; k < n; k++) {
        if (!grids[k]) return gm_member_err(set_err(GF_ERR_INVALID_ARG, "null grid"), k);
        for (int j = 0; j < k; j++) if (grids[j] == grids[k]) return gm_member_err(set_err(GF_ERR_INVALID_ARG, "the grid is listed twice"), k);
        if (grids[k]->device != grids[0]->device) return gm_member_err(set_err(GF_ERR_INVALID_ARG, "bound to another device than member 0"), k);
        pcap += grids[k]->cfg.max_points;
        mr = std::min(mr, (long long)grids[k]->cfg.max_records);
    }
    if (pcap >= (1ll << 31) - 1) return set_err(GF_ERR_CAPACITY, "the members' max_points add up to 2^31 or more");
    GF_CUDA(cudaSetDevice(grids[0]->device));
    gf_grid_map_group* g = new gf_grid_map_group();
    g->device = grids[0]->device; g->n = n; g->pcap = pcap; g->max_records = mr;
    g->m.assign(grids, grids + n);
    g->h = new GmCall();
    const size_t N = (size_t)pcap, Rn = (size_t)mr;
#define GMG_ALLOC(p, bytes) do { if (cudaMalloc(&(p), (bytes)) != cudaSuccess) { cudaGetLastError(); gmg_free(g); return set_err(GF_ERR_CUDA, "cudaMalloc failed (grid map group)"); } } while (0)
    if (cudaStreamCreateWithFlags(&g->st, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&g->ev, cudaEventDisableTiming) != cudaSuccess) {
        cudaGetLastError(); gmg_free(g); return set_err(GF_ERR_CUDA, "stream creation failed");
    }
    GMG_ALLOC(g->d, sizeof(GmCall));
    GMG_ALLOC(g->cnt, 8 * (N + 1)); GMG_ALLOC(g->off, 8 * (N + 1)); GMG_ALLOC(g->res, 3 * 8 * GROUP_MAX);
    GMG_ALLOC(g->rec, 8 * Rn); GMG_ALLOC(g->srec, 8 * Rn);
    GMG_ALLOC(g->bad, 4 * GROUP_MAX); GMG_ALLOC(g->longray, 4 * GROUP_MAX); GMG_ALLOC(g->dstats, 3 * sizeof(unsigned long long) * GROUP_MAX);
#undef GMG_ALLOC
    size_t b1 = 0, b2 = 0;
    if (cub::DeviceRadixSort::SortKeys(nullptr, b1, g->rec, g->srec, (int)mr, 2, 38) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, b2, g->cnt, g->off, (int)(N + 1)) != cudaSuccess) { gmg_free(g); return set_err(GF_ERR_CUDA, "cub sizing failed"); }
    g->tmp_bytes = std::max(b1, b2);
    if (cudaMalloc(&g->tmp, g->tmp_bytes) != cudaSuccess || cudaMallocHost(&g->h_res, 6 * sizeof(long long) * GROUP_MAX) != cudaSuccess) {
        cudaGetLastError(); gmg_free(g); return set_err(GF_ERR_CUDA, "allocation failed (grid map group)");
    }
    *out = g;
    return GF_OK;
}

void gf_grid_map_group_destroy(gf_grid_map_group* g)
{
    if (!g) return;
    cudaSetDevice(g->device);
    cudaStreamSynchronize(g->st);
    gmg_free(g);
}

int gf_grid_map_group_size(gf_grid_map_group* g, int* n)
{
    if (!g || !n) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *n = g->n;
    return GF_OK;
}

int gf_grid_map_group_add_keyframes(gf_grid_map_group* g, const int32_t* members, int m, const double* R, const double* P, const float* const* pts,
                                    const int32_t* n_pts, const int32_t* stride_floats, int on_device, int32_t* status)
{
    if (!g || !members || !R || !P || !pts || !n_pts || !stride_floats) return set_err(GF_ERR_INVALID_ARG, "null argument");
    int rc = gmg_check_members(g, members, m);
    if (rc) return rc;
    for (int j = 0; j < m; j++)
        if (n_pts[j] < 0 || (n_pts[j] > 0 && !pts[j]) || stride_floats[j] < 3) return gm_member_err(set_err(GF_ERR_INVALID_ARG, "bad argument"), j);
    return gmg_add(g, members, m, R, P, pts, n_pts, stride_floats, on_device, nullptr, status);
}

int gf_grid_map_group_add_dense_keyframes(gf_grid_map_group* g, gf_dense_map_group* dg, const int32_t* members, int m, const double* R, const double* P,
                                          int32_t* status)
{
    if (!g || !dg || !members || !R || !P) return set_err(GF_ERR_INVALID_ARG, "null argument");
    int rc = gmg_check_members(g, members, m);
    if (rc) return rc;
    std::vector<const float*> pts(m);
    std::vector<int> n(m), stride(m, 3);
    std::vector<cudaStream_t> dense_st(m);
    for (int j = 0; j < m; j++) {
        gf_dense_map* dm = gf_dense_map_group_member(dg, members[j]);
        if (!dm) return gm_member_err(set_err(GF_ERR_INVALID_ARG, "member index beyond the dense-map group"), j);
        int dev;
        if ((rc = gf_dense_map_last_keyframe_device(dm, &pts[j], &n[j], &dense_st[j], &dev))) return gm_member_err(rc, j);
        if (dev != g->device) return gm_member_err(set_err(GF_ERR_INVALID_ARG, "the dense map is bound to another device"), j);
    }
    return gmg_add(g, members, m, R, P, pts.data(), n.data(), stride.data(), 1, dense_st.data(), status);
}

}  // extern "C"
