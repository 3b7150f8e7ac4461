// gm_grid.cu -- gf_grid_map_* (C ABI): the 2-D occupancy grid of the reference's grid_mapping tool on the GPU
// (support_files/grid_mapping: main.cpp:114-120, grid_mapper.cpp, grid_map.cpp), built online from the dense map's keyframe
// points and rebuilt after a pose correction.
//   rays     one thread per point: world point, z band [0.1, 0.5], then the tool's ray from the body position in steps of one
//            cell (a sequential double sum r += cs), counted, scanned, and emitted as one 32-bit record per step,
//            cell << 2 | kind, in the tool's (keyframe, point, step) order; a skipped step is SENTINEL
//   sort     a stable LSD radix sort on the cell bits keeps each cell's updates in the tool's order
//   apply    the first thread of each cell's run applies the run's log-odds updates one after another
// The semantics these restate are in one place each below (gm_cell, k_gm_emit's ray, gm_update, k_gm_apply's shortcuts) and are
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

// the number of steps of each point's ray (0 outside the band); cnt[n] = 0 for the exclusive scan's total
__global__ void k_gm_count(int n, int p0, const float* __restrict__ pts, const int* __restrict__ kf, const Pose* __restrict__ poses, Ext e, Grid g,
                           long long* __restrict__ cnt, int* bad)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > n) return;
    if (j == n) { cnt[n] = 0; return; }
    const int i = p0 + j;
    Ray q;
    long long c = 0;
    if (gm_ray(e, poses[kf[i]], pts + 3 * (size_t)i, q)) {
        for (double r = 0; r < q.z + g.cs; r += g.cs)
            if (++c > MAX_STEPS) { atomicExch(bad, 1); break; }
    }
    cnt[j] = c;
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
    Ray q;
    gm_ray(e, poses[kf[i]], pts + 3 * (size_t)i, q);
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
        if (s >= a) rec[s - a] = v;
    }
}

// Over the records sorted stably by cell: the first thread of each cell's run applies the run in order.  Two shortcuts are
// exact: an update that leaves bel unchanged leaves it unchanged again, so the records of the same kind that follow it are
// skipped; and 0 and 1 absorb every kind (log(0) = -inf, log(inf) = inf).  stats: updates applied, updates skipped, longest run.
__global__ void k_gm_apply(int n, const uint32_t* __restrict__ srec, Grid g, double* __restrict__ bel, unsigned long long* stats)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t v = srec[i];
    if (v == SENTINEL) return;
    const uint32_t cell = v >> 2;
    if (i > 0 && (srec[i - 1] >> 2) == cell) return;
    int end = i + 1;
    while (end < n && (srec[end] >> 2) == cell) end++;
    double b = bel[cell];
    int j = i;
    unsigned long long applied = 0;
    while (j < end && b != 0.0 && b != 1.0) {
        const uint32_t kind = srec[j] & 3u;
        const double nb = gm_update(b, kind == FREE ? g.c[FREE] : (kind == OCC ? g.c[OCC] : g.c[PRIOR]));
        applied++;
        j++;
        if (nb == b)
            while (j < end && (srec[j] & 3u) == kind) j++;
        b = nb;
    }
    bel[cell] = b;
    atomicAdd(&stats[0], applied);
    atomicAdd(&stats[1], (unsigned long long)(end - i) - applied);
    atomicMax(&stats[2], (unsigned long long)(end - i));
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
