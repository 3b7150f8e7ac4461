// dm_map.cu -- gf_dense_map_* (C ABI): dense_map's colour point map on the GPU (reference dense_map/src).
//   keyframe points   pose_graph_node.cpp:598-623: every depth_dist-th pixel lifted (PinholeCamera::liftProjective), depth in
//                     metres, white (> 240 in all channels) and out-of-range (d < 0.1 or >= 7) samples dropped
//   insertion         PoseGraph::addKeyFrame, pose_graph.cpp:191-221: world point, z band [-0.5, 2], then inserted iff the
//                     0.01 m voxel of an OctreePointCloudDensity holds < 3 points; the keyframe keeps the inserted points
//   filter            pose_graph.cpp:228-239: RadiusOutlierRemoval, radius 0.8, 10 neighbours
//   rebuild           PoseGraph::updatePath, pose_graph.cpp:997-1058: fresh octree over a wider box, every keyframe's kept points
//                     re-inserted with its corrected pose under the gate < 5, no z band, then the filter again
// The PCL semantics these restate are in one place each below (dm_octree_anchor, dm_voxel_key, k_dm_count) and are described in
// DESIGN.md "Dense colour map".  Built with -fmad=false: every float/double result is bit-identical to oracle/dm_oracle.c.
#include <cub/cub.cuh>
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <limits>
#include <vector>

#include "gf_camera.cuh"
#include "gf_pose.cuh"

using namespace gf;

namespace gfdm {

constexpr double VOXEL = 0.01;                    // OctreePointCloudDensity<PointXYZRGB>(0.01), pose_graph.cpp:29
constexpr int GATE_ADD = 3, GATE_REBUILD = 5;     // getVoxelDensityAtPoint(p) < 3 (:210), < 5 (:1041)
constexpr double Z_HI = 2.0, Z_LO = -0.5;         // pose_graph.cpp:200
constexpr double RADIUS = 0.8;                    // setRadiusSearch(0.8), :235
constexpr int MIN_PTS = 10;                       // setMinNeighborsInRadius(10), :237
constexpr uint64_t EMPTY = ~0ull;                 // free hash slot
constexpr uint64_t INVALID = 1ull << 63;          // sorts after every packed 3 x 21-bit key
constexpr int CELL_OFF = 1 << 20;                 // cell coordinates are stored biased into 21 bits

// PCL 1.10 OctreePointCloud::defineBoundingBox -> getKeyBitSize (unverified restatement: PCL is not vendored).  With no leaf
// yet, the box is widened symmetrically on every axis to 2^depth voxels, depth = ceil(log2(max key)); the voxel key of a point
// is then (unsigned)((double(p) - min) / resolution).  Returns the widened min and max.
static void dm_octree_anchor(const double lo[3], const double hi[3], double mn[3], double mx[3])
{
    const float min_value = std::numeric_limits<float>::epsilon();
    unsigned mk[3];
    for (int a = 0; a < 3; a++) mk[a] = (unsigned)std::ceil((hi[a] - lo[a] - min_value) / VOXEL);
    const unsigned max_voxels = std::max(std::max(std::max(mk[0], mk[1]), mk[2]), 2u);
    const unsigned depth = std::min(32u, (unsigned)std::ceil(std::log2((double)max_voxels) - min_value));
    const double side = (double)(1ull << depth) * VOXEL;
    for (int a = 0; a < 3; a++) {
        const double over = (side - (hi[a] - lo[a])) / 2.0;
        mn[a] = lo[a] - over;
        mx[a] = hi[a] + over;
    }
}
// PoseGraph::PoseGraph (:34) and updatePath (:1002): note y-min -1000 in the constructor's box
static const double BOX_INIT_LO[3] = {-10000, -1000, -10000}, BOX_REBUILD_LO[3] = {-10000, -10000, -10000}, BOX_HI[3] = {10000, 10000, 10000};

struct Anchor { double mn[3], mx[3]; };

// the voxel key of a float point inside the anchored box, packed 3 x 21 bits; INVALID (and *bad set) outside the box
__device__ __forceinline__ uint64_t dm_voxel_key(const Anchor& A, const float* f, int* bad)
{
    uint64_t key = 0;
    for (int a = 0; a < 3; a++) {
        const double x = (double)f[a];
        if (!(x >= A.mn[a] && x < A.mx[a])) { atomicExch(bad, 1); return INVALID; }
        key = (key << 21) | (uint64_t)(unsigned)((x - A.mn[a]) / VOXEL);
    }
    return key;
}

__device__ __forceinline__ uint32_t hslot(uint64_t k, uint32_t mask)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (uint32_t)k & mask;
}
__device__ __forceinline__ int hfind(const uint64_t* keys, uint32_t mask, uint64_t k)
{
    for (uint32_t s = hslot(k, mask);; s = (s + 1) & mask) {
        const uint64_t x = keys[s];
        if (x == k) return (int)s;
        if (x == EMPTY) return -1;
    }
}
__device__ __forceinline__ uint32_t hinsert(uint64_t* keys, uint32_t mask, uint64_t k)
{
    for (uint32_t s = hslot(k, mask);; s = (s + 1) & mask) {
        const uint64_t x = atomicCAS((unsigned long long*)&keys[s], (unsigned long long)EMPTY, (unsigned long long)k);
        if (x == EMPTY || x == k) return s;
    }
}

// one thread per sample: lift, depth / colour tests, local point, world point, z band, voxel key
__global__ void k_dm_sample(CamParams cam, int su, int n, int B, int D, const uint8_t* __restrict__ rgb, size_t rgb_pitch,
                            const uint16_t* __restrict__ depth, size_t depth_pitch, Ext e, Pose T, Anchor A, uint64_t* __restrict__ key,
                            uint32_t* __restrict__ idx, float* __restrict__ loc, uchar4* __restrict__ col, float* __restrict__ wxyz, int* bad)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    idx[s] = s;
    key[s] = INVALID;
    const int u = B + (s % su) * D, v = B + (s / su) * D;
    const uint8_t* c = rgb + (size_t)v * rgb_pitch + 3 * (size_t)u;
    const uint8_t r = c[0], g = c[1], b = c[2];
    float d = (float)(int)*(const uint16_t*)((const uint8_t*)depth + (size_t)v * depth_pitch + 2 * (size_t)u);
    d = d / 1000;
    if (r > 240 && g > 240 && b > 240) return;
    if ((double)d < 0.1 || (double)d >= 7.0) return;
    double ax, ay;
    cam_lift(cam, (double)u, (double)v, ax, ay);
    const float l[3] = {(float)(ax * d), (float)(ay * d), d};
    double w[3];
    to_world(e, T, l, w);
    if (w[2] > Z_HI || w[2] < Z_LO) return;
    const float f[3] = {(float)w[0], (float)w[1], (float)w[2]};
    for (int k = 0; k < 3; k++) { loc[3 * s + k] = l[k]; wxyz[3 * s + k] = f[k]; }
    col[s] = make_uchar4(r, g, b, 0);
    key[s] = dm_voxel_key(A, f, bad);
}

// one thread per kept keyframe point: its world point under the keyframe's current pose (updatePath: no z band)
__global__ void k_dm_rebuild_xform(int n, const float* __restrict__ kf_xyz, const int* __restrict__ kf_id, const Pose* __restrict__ poses, Ext e,
                                   Anchor A, uint64_t* __restrict__ key, uint32_t* __restrict__ idx, float* __restrict__ wxyz, int* bad)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double w[3];
    to_world(e, poses[kf_id[i]], kf_xyz + 3 * (size_t)i, w);
    const float f[3] = {(float)w[0], (float)w[1], (float)w[2]};
    for (int k = 0; k < 3; k++) wxyz[3 * (size_t)i + k] = f[k];
    idx[i] = i;
    key[i] = dm_voxel_key(A, f, bad);
}

// Over the (key, index) pairs sorted stably by key: the first thread of each voxel's run reads the voxel's count c and accepts
// the run's j-th point iff c + j < cap -- the sequential rule, since the run lists the voxel's points in input order.
// add[i] = the number accepted (at the run's first position, 0 elsewhere).
__global__ void k_dm_gate(int n, const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sidx, const uint64_t* __restrict__ vkeys,
                          const int* __restrict__ vcnt, uint32_t vmask, int cap, int* __restrict__ flag, int* __restrict__ add)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = skey[i];
    add[i] = 0;
    if (k == INVALID) { flag[sidx[i]] = 0; return; }
    if (i > 0 && skey[i - 1] == k) return;
    const int s = hfind(vkeys, vmask, k);
    const int c = s < 0 ? 0 : vcnt[s];
    int a = 0;
    for (int j = i; j < n && skey[j] == k; j++) {
        const int ok = c + (j - i) < cap;
        flag[sidx[j]] = ok;
        a += ok;
    }
    add[i] = a;
}
__global__ void k_dm_hash_add(int n, const uint64_t* __restrict__ skey, const int* __restrict__ add, uint64_t* vkeys, int* vcnt, uint32_t vmask)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || add[i] == 0) return;
    atomicAdd(&vcnt[hinsert(vkeys, vmask, skey[i])], add[i]);
}
// stable compaction of the accepted points: cloud at c0 (+ the keyframe's kept local points at k0 when loc != nullptr)
__global__ void k_dm_scatter(int n, const int* __restrict__ flag, const int* __restrict__ pos, const float* __restrict__ wxyz, const uchar4* __restrict__ col,
                             float* __restrict__ cxyz, uchar4* __restrict__ ccol, int c0, const float* __restrict__ loc, float* __restrict__ kxyz,
                             uchar4* __restrict__ kcol, int* __restrict__ kid, int k0, int kf)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flag[i]) return;
    const size_t c = (size_t)c0 + pos[i];
    for (int k = 0; k < 3; k++) cxyz[3 * c + k] = wxyz[3 * (size_t)i + k];
    ccol[c] = col[i];
    if (loc) {
        const size_t q = (size_t)k0 + pos[i];
        for (int k = 0; k < 3; k++) kxyz[3 * q + k] = loc[3 * (size_t)i + k];
        kcol[q] = col[i];
        kid[q] = kf;
    }
}

// ---- radius filter over a cell index: cells of side >= radius (slightly larger, so that rounding of the cell coordinate
// never moves a neighbour two cells away); a point's neighbours are in its 27-cell stencil ----
__device__ __forceinline__ int cell_of(float x, double inv_cell) { return (int)floor((double)x * inv_cell); }
__device__ __forceinline__ uint64_t cell_key(int cx, int cy, int cz)
{
    return ((uint64_t)(unsigned)(cx + CELL_OFF) << 42) | ((uint64_t)(unsigned)(cy + CELL_OFF) << 21) | (uint64_t)(unsigned)(cz + CELL_OFF);
}
__global__ void k_dm_cell_keys(int n, const float* __restrict__ xyz, double inv_cell, uint64_t* __restrict__ key, uint32_t* __restrict__ idx)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    key[i] = cell_key(cell_of(xyz[3 * (size_t)i], inv_cell), cell_of(xyz[3 * (size_t)i + 1], inv_cell), cell_of(xyz[3 * (size_t)i + 2], inv_cell));
    idx[i] = i;
}
// the runs of the sorted cell keys become (start, end) entries of the cell hash; the points are gathered in cell order
__global__ void k_dm_cell_build(int n, const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sidx, const float* __restrict__ xyz,
                                uint64_t* hkeys, int2* hrange, uint32_t hmask, float4* __restrict__ sxyz)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t p = sidx[i];
    sxyz[i] = make_float4(xyz[3 * p], xyz[3 * p + 1], xyz[3 * p + 2], 0.f);
    const uint64_t k = skey[i];
    if (i == 0 || skey[i - 1] != k) hrange[hinsert(hkeys, hmask, k)].x = i;
    if (i == n - 1 || skey[i + 1] != k) hrange[hinsert(hkeys, hmask, k)].y = i + 1;
}
// the cells holding a point with index >= from are dirty: only points in their stencil can gain neighbours
__global__ void k_dm_mark_dirty(int n, int from, const float* __restrict__ xyz, double inv_cell, const uint64_t* __restrict__ hkeys, uint32_t hmask,
                                uint8_t* __restrict__ dirty)
{
    const int i = from + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = cell_key(cell_of(xyz[3 * (size_t)i], inv_cell), cell_of(xyz[3 * (size_t)i + 1], inv_cell), cell_of(xyz[3 * (size_t)i + 2], inv_cell));
    dirty[hfind(hkeys, hmask, k)] = 1;
}
// RadiusOutlierRemoval (PCL 1.10, unverified restatement): a point is kept iff a radius search capped at min_pts + 1 results
// returns more than min_pts points, itself and duplicates included; FLANN's L2_Simple distance ((dx*dx) + dy*dy) + dz*dz in
// float, compared strictly with float(radius^2).  A kept point stays kept (its count can only grow until the next rebuild), so
// only points not yet kept whose stencil touches a dirty cell are counted.
__global__ void k_dm_count(int n, const float* __restrict__ xyz, double inv_cell, const uint64_t* __restrict__ hkeys, const int2* __restrict__ hrange,
                           const uint8_t* __restrict__ dirty, uint32_t hmask, const float4* __restrict__ sxyz, float r2, int min_pts, uint8_t* __restrict__ kept)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || kept[i]) return;
    const float qx = xyz[3 * (size_t)i], qy = xyz[3 * (size_t)i + 1], qz = xyz[3 * (size_t)i + 2];
    const int cx = cell_of(qx, inv_cell), cy = cell_of(qy, inv_cell), cz = cell_of(qz, inv_cell);
    int slots[27];
    bool any = false;
    for (int t = 0; t < 27; t++) {
        slots[t] = hfind(hkeys, hmask, cell_key(cx + t % 3 - 1, cy + (t / 3) % 3 - 1, cz + t / 9 - 1));
        if (slots[t] >= 0 && dirty[slots[t]]) any = true;
    }
    if (!any) return;
    int cnt = 0;
    for (int t = 0; t < 27 && cnt <= min_pts; t++) {
        if (slots[t] < 0) continue;
        const int2 r = hrange[slots[t]];
        for (int j = r.x; j < r.y; j++) {
            const float4 p = sxyz[j];
            const float dx = qx - p.x, dy = qy - p.y, dz = qz - p.z;
            const float dist = dx * dx + dy * dy + dz * dz;
            if (dist < r2 && ++cnt > min_pts) break;
        }
    }
    kept[i] = cnt > min_pts;
}

// scratch of the radius filter over up to cap points
struct Filter {
    int cap = 0;
    uint32_t hmask = 0;
    uint64_t *key = nullptr, *skey = nullptr, *hkeys = nullptr;
    uint32_t *idx = nullptr, *sidx = nullptr;
    int2* hrange = nullptr;
    uint8_t* dirty = nullptr;
    float4* sxyz = nullptr;
    void* tmp = nullptr;
    size_t tmp_bytes = 0;

    int alloc(int n)
    {
        cap = std::max(n, 1);
        uint32_t hc = 64;
        while (hc < 2u * (uint32_t)cap) hc <<= 1;
        hmask = hc - 1;
        GF_CUDA(cudaMalloc(&key, 8 * (size_t)cap)); GF_CUDA(cudaMalloc(&skey, 8 * (size_t)cap));
        GF_CUDA(cudaMalloc(&idx, 4 * (size_t)cap)); GF_CUDA(cudaMalloc(&sidx, 4 * (size_t)cap));
        GF_CUDA(cudaMalloc(&sxyz, 16 * (size_t)cap));
        GF_CUDA(cudaMalloc(&hkeys, 8 * (size_t)hc)); GF_CUDA(cudaMalloc(&hrange, 8 * (size_t)hc)); GF_CUDA(cudaMalloc(&dirty, hc));
        size_t b1 = 0, b2 = 0;
        GF_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b1, key, skey, idx, sidx, cap, 0, 63));
        GF_CUDA(cub::DeviceSelect::Flagged(nullptr, b2, cub::CountingInputIterator<int>(0), dirty, (int*)idx, (int*)idx, cap));
        tmp_bytes = std::max(b1, b2);
        GF_CUDA(cudaMalloc(&tmp, tmp_bytes));
        return GF_OK;
    }
    void release()
    {
        for (void* p : {(void*)key, (void*)skey, (void*)hkeys, (void*)idx, (void*)sidx, (void*)hrange, (void*)dirty, (void*)sxyz, tmp}) if (p) cudaFree(p);
        *this = Filter();
    }
    // kept[0, from) holds the result over the points [0, from) (nothing kept when from == 0); afterwards kept[0, n) is the
    // result over [0, n).  Then (when sel != nullptr) the indices of the kept points in order and their number.
    int run(int n, int from, const float* xyz, uint8_t* kept, double radius, int min_pts, int* sel, int* d_nsel, cudaStream_t st)
    {
        const double inv_cell = 1.0 / (radius * (65.0 / 64.0));
        const float r2 = (float)(radius * radius);
        GF_CUDA(cudaMemsetAsync(kept + from, 0, (size_t)(n - from), st));
        if (n == 0) return sel ? (cudaMemsetAsync(d_nsel, 0, 4, st) == cudaSuccess ? GF_OK : GF_ERR_CUDA) : GF_OK;
        if (n > from) {                                   // no new point: nothing can change
            // the cell hash is sized by the points of this call (at least 2 n slots), not by the capacity
            uint32_t hm = 63;
            while (hm < hmask && (size_t)hm + 1 < 2 * (size_t)n) hm = (hm << 1) | 1;
            const int nb = (n + 255) / 256;
            k_dm_cell_keys<<<nb, 256, 0, st>>>(n, xyz, inv_cell, key, idx);
            GF_LAUNCHED();
            size_t b = tmp_bytes;
            GF_CUDA(cub::DeviceRadixSort::SortPairs(tmp, b, key, skey, idx, sidx, n, 0, 63, st));
            GF_CUDA(cudaMemsetAsync(hkeys, 0xff, 8 * ((size_t)hm + 1), st));
            GF_CUDA(cudaMemsetAsync(dirty, 0, (size_t)hm + 1, st));
            k_dm_cell_build<<<nb, 256, 0, st>>>(n, skey, sidx, xyz, hkeys, hrange, hm, sxyz);
            GF_LAUNCHED();
            k_dm_mark_dirty<<<(n - from + 255) / 256, 256, 0, st>>>(n, from, xyz, inv_cell, hkeys, hm, dirty);
            GF_LAUNCHED();
            k_dm_count<<<(n + 127) / 128, 128, 0, st>>>(n, xyz, inv_cell, hkeys, hrange, dirty, hm, sxyz, r2, min_pts, kept);
            GF_LAUNCHED();
        }
        if (sel) {
            size_t b = tmp_bytes;
            GF_CUDA(cub::DeviceSelect::Flagged(tmp, b, cub::CountingInputIterator<int>(0), kept, sel, d_nsel, n, st));
        }
        GF_CUDA(cudaGetLastError());
        return GF_OK;
    }
};

}  // namespace gfdm

using namespace gfdm;

struct gf_dense_map {
    int device = 0;
    cudaStream_t st = nullptr;
    gf_dense_map_cfg cfg;
    CamParams cam;
    Ext ext;
    Anchor anchor;
    int su = 0, sv = 0, ns = 0;                      // sample grid
    int max_points = 0, work = 0;                    // work = max(max_points, samples per keyframe)
    uint32_t vmask = 0;
    // host state
    int n_cloud = 0, n_filtered = 0, n_kf_points = 0;
    std::vector<Pose> poses;                         // pose each keyframe was last inserted with
    std::vector<int> kf_off{0};                      // keyframe k's kept points are [kf_off[k], kf_off[k+1])
    // device
    uint8_t* rgb = nullptr; uint16_t* depth = nullptr;           // staging frame (host intake)
    uint64_t *key = nullptr, *skey = nullptr, *vkeys = nullptr;
    uint32_t *idx = nullptr, *sidx = nullptr;
    int *flag = nullptr, *pos = nullptr, *add = nullptr, *bad = nullptr, *nsel = nullptr, *fidx = nullptr;
    int* vcnt = nullptr;
    float *loc = nullptr, *wxyz = nullptr;
    uchar4* col = nullptr;
    float* cxyz = nullptr; uchar4* ccol = nullptr; uint8_t* kept = nullptr;
    float* kxyz = nullptr; uchar4* kcol = nullptr; int* kid = nullptr;
    Pose* dposes = nullptr;
    void* tmp = nullptr; size_t tmp_bytes = 0;
    int* h_pin = nullptr;                            // pinned: total accepted, bad flag
    Filter filt;
};

static int dm_device(int device)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return set_err(GF_ERR_NO_DEVICE, "no CUDA device visible; libgf_b200 has no CPU fallback");
    if (device < 0 || device >= n) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    return GF_OK;
}

static void dm_free(gf_dense_map* m)
{
    for (void* p : {(void*)m->rgb, (void*)m->depth, (void*)m->key, (void*)m->skey, (void*)m->vkeys, (void*)m->idx, (void*)m->sidx, (void*)m->flag,
                    (void*)m->pos, (void*)m->add, (void*)m->bad, (void*)m->nsel, (void*)m->fidx, (void*)m->vcnt, (void*)m->loc, (void*)m->wxyz,
                    (void*)m->col, (void*)m->cxyz, (void*)m->ccol, (void*)m->kept, (void*)m->kxyz, (void*)m->kcol, (void*)m->kid, (void*)m->dposes, m->tmp})
        if (p) cudaFree(p);
    if (m->h_pin) cudaFreeHost(m->h_pin);
    m->filt.release();
    if (m->st) cudaStreamDestroy(m->st);
    delete m;
}

// sort the (key, index) pairs of n points, gate them against the voxel counts with cap, and count the accepted ones; on return
// h_pin[0] = accepted, h_pin[1] = a point fell outside the octree's box.  Nothing of the map's state is written.
static int dm_gate(gf_dense_map* m, int n, int cap)
{
    size_t b = m->tmp_bytes;
    GF_CUDA(cub::DeviceRadixSort::SortPairs(m->tmp, b, m->key, m->skey, m->idx, m->sidx, n, 0, 64, m->st));
    k_dm_gate<<<(n + 255) / 256, 256, 0, m->st>>>(n, m->skey, m->sidx, m->vkeys, m->vcnt, m->vmask, cap, m->flag, m->add);
    GF_LAUNCHED();
    b = m->tmp_bytes;
    GF_CUDA(cub::DeviceScan::ExclusiveSum(m->tmp, b, m->flag, m->pos, n, m->st));
    GF_CUDA(cudaMemcpyAsync(m->h_pin, m->pos + (n - 1), 4, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaMemcpyAsync(m->h_pin + 2, m->flag + (n - 1), 4, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaMemcpyAsync(m->h_pin + 1, m->bad, 4, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaStreamSynchronize(m->st));
    m->h_pin[0] += m->h_pin[2];
    return GF_OK;
}

static int dm_filter(gf_dense_map* m, int from)
{
    int rc = m->filt.run(m->n_cloud, from, m->cxyz, m->kept, RADIUS, MIN_PTS, m->fidx, m->nsel, m->st);
    if (rc) return rc;
    GF_CUDA(cudaMemcpyAsync(&m->n_filtered, m->nsel, 4, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaStreamSynchronize(m->st));
    return GF_OK;
}

extern "C" {

int gf_dense_map_create(gf_dense_map** out, int device, const gf_dense_map_cfg* cfg)
{
    if (!out || !cfg) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    *out = nullptr;
    const gf_dense_map_cfg& c = *cfg;
    if (c.width < 1 || c.height < 1 || c.depth_dist < 1 || c.depth_boundary < 0 || 2 * c.depth_boundary >= c.width || 2 * c.depth_boundary >= c.height ||
        c.max_points < 1 || c.max_keyframes < 1 || c.pinhole[0] == 0.0 || c.pinhole[1] == 0.0)
        return set_err(GF_ERR_INVALID_ARG, "bad dense-map geometry (depth_dist >= 1, 2 * depth_boundary < width and height, capacities >= 1)");
    if (c.max_points > (1 << 29)) return set_err(GF_ERR_CAPACITY, "max_points above 2^29");
    int rc = dm_device(device);
    if (rc) return rc;
    gf_dense_map* m = new gf_dense_map();
    m->device = device;
    m->cfg = c;
    m->cam = make_cam(c.pinhole);
    memcpy(m->ext.ric, c.ric, sizeof(m->ext.ric)); memcpy(m->ext.tic, c.tic, sizeof(m->ext.tic));
    dm_octree_anchor(BOX_INIT_LO, BOX_HI, m->anchor.mn, m->anchor.mx);
    m->su = (c.width - 2 * c.depth_boundary + c.depth_dist - 1) / c.depth_dist;
    m->sv = (c.height - 2 * c.depth_boundary + c.depth_dist - 1) / c.depth_dist;
    m->ns = m->su * m->sv;
    m->max_points = c.max_points;
    m->work = std::max(c.max_points, m->ns);
    m->poses.reserve(c.max_keyframes);
    uint32_t hc = 64;
    while (hc < 2u * (uint32_t)c.max_points) hc <<= 1;
    m->vmask = hc - 1;
    const size_t W = (size_t)m->work, N = (size_t)c.max_points, S = (size_t)m->ns;
#define DM_ALLOC(p, bytes) do { if (cudaMalloc(&(p), (bytes)) != cudaSuccess) { cudaGetLastError(); dm_free(m); return set_err(GF_ERR_CUDA, "cudaMalloc failed (dense map)"); } } while (0)
    if (cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking) != cudaSuccess) { dm_free(m); return set_err(GF_ERR_CUDA, "stream creation failed"); }
    DM_ALLOC(m->rgb, (size_t)c.width * c.height * 3); DM_ALLOC(m->depth, (size_t)c.width * c.height * 2);
    DM_ALLOC(m->key, 8 * W); DM_ALLOC(m->skey, 8 * W); DM_ALLOC(m->idx, 4 * W); DM_ALLOC(m->sidx, 4 * W);
    DM_ALLOC(m->flag, 4 * W); DM_ALLOC(m->pos, 4 * W); DM_ALLOC(m->add, 4 * W); DM_ALLOC(m->wxyz, 12 * W);
    DM_ALLOC(m->loc, 12 * S); DM_ALLOC(m->col, 4 * S);
    DM_ALLOC(m->bad, 4); DM_ALLOC(m->nsel, 4); DM_ALLOC(m->fidx, 4 * N);
    DM_ALLOC(m->vkeys, 8 * (size_t)hc); DM_ALLOC(m->vcnt, 4 * (size_t)hc);
    DM_ALLOC(m->cxyz, 12 * N); DM_ALLOC(m->ccol, 4 * N); DM_ALLOC(m->kept, N);
    DM_ALLOC(m->kxyz, 12 * N); DM_ALLOC(m->kcol, 4 * N); DM_ALLOC(m->kid, 4 * N);
    DM_ALLOC(m->dposes, sizeof(Pose) * (size_t)c.max_keyframes);
#undef DM_ALLOC
    size_t b1 = 0, b2 = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, b1, m->key, m->skey, m->idx, m->sidx, m->work, 0, 64) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, b2, m->flag, m->pos, m->work) != cudaSuccess) { dm_free(m); return set_err(GF_ERR_CUDA, "cub sizing failed"); }
    m->tmp_bytes = std::max(b1, b2);
    if (cudaMalloc(&m->tmp, m->tmp_bytes) != cudaSuccess || cudaMallocHost(&m->h_pin, 16) != cudaSuccess || (rc = m->filt.alloc(c.max_points)) != GF_OK) {
        cudaGetLastError(); dm_free(m); return rc ? rc : set_err(GF_ERR_CUDA, "allocation failed (dense map)");
    }
    if (cudaMemsetAsync(m->vkeys, 0xff, 8 * (size_t)hc, m->st) != cudaSuccess || cudaMemsetAsync(m->vcnt, 0, 4 * (size_t)hc, m->st) != cudaSuccess ||
        cudaStreamSynchronize(m->st) != cudaSuccess) {
        dm_free(m); return set_err(GF_ERR_CUDA, "initialisation failed (dense map)");
    }
    *out = m;
    return GF_OK;
}

void gf_dense_map_destroy(gf_dense_map* m)
{
    if (!m) return;
    cudaSetDevice(m->device);
    cudaStreamSynchronize(m->st);
    dm_free(m);
}

int gf_dense_map_add_keyframe(gf_dense_map* m, const double* R, const double* P, const uint8_t* rgb, size_t rgb_pitch,
                              const uint16_t* depth, size_t depth_pitch, int on_device, int* n_inserted)
{
    if (!m || !R || !P || !rgb || !depth) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    const int w = m->cfg.width, h = m->cfg.height;
    if (rgb_pitch < 3 * (size_t)w || depth_pitch < 2 * (size_t)w) return set_err(GF_ERR_INVALID_ARG, "row pitch below the row width");
    if ((depth_pitch | (size_t)(uintptr_t)depth) & 1) return set_err(GF_ERR_INVALID_ARG, "depth rows must start at even addresses (uint16)");
    const int kf = (int)m->poses.size();
    if (kf >= m->cfg.max_keyframes) return set_err(GF_ERR_CAPACITY, "max_keyframes reached");
    GF_CUDA(cudaSetDevice(m->device));
    Pose T;
    memcpy(T.R, R, sizeof(T.R)); memcpy(T.P, P, sizeof(T.P));
    const uint8_t* d_rgb = rgb; const uint16_t* d_depth = depth;
    if (!on_device) {
        GF_CUDA(cudaMemcpy2DAsync(m->rgb, 3 * (size_t)w, rgb, rgb_pitch, 3 * (size_t)w, h, cudaMemcpyHostToDevice, m->st));
        GF_CUDA(cudaMemcpy2DAsync(m->depth, 2 * (size_t)w, depth, depth_pitch, 2 * (size_t)w, h, cudaMemcpyHostToDevice, m->st));
        d_rgb = m->rgb; d_depth = m->depth; rgb_pitch = 3 * (size_t)w; depth_pitch = 2 * (size_t)w;
    }
    const int n = m->ns;
    GF_CUDA(cudaMemsetAsync(m->bad, 0, 4, m->st));
    k_dm_sample<<<(n + 127) / 128, 128, 0, m->st>>>(m->cam, m->su, n, m->cfg.depth_boundary, m->cfg.depth_dist, d_rgb, rgb_pitch, d_depth, depth_pitch,
                                                    m->ext, T, m->anchor, m->key, m->idx, m->loc, m->col, m->wxyz, m->bad);
    GF_LAUNCHED();
    int rc = dm_gate(m, n, GATE_ADD);
    if (rc) return rc;
    const int acc = m->h_pin[0];
    if (m->h_pin[1]) return set_err(GF_ERR_INVALID_ARG, "a point of the keyframe falls outside the octree's bounding box");
    if (m->n_kf_points + acc > m->max_points) return set_err(GF_ERR_CAPACITY, "max_points reached");
    // commit
    k_dm_hash_add<<<(n + 255) / 256, 256, 0, m->st>>>(n, m->skey, m->add, m->vkeys, m->vcnt, m->vmask);
    GF_LAUNCHED();
    k_dm_scatter<<<(n + 255) / 256, 256, 0, m->st>>>(n, m->flag, m->pos, m->wxyz, m->col, m->cxyz, m->ccol, m->n_cloud, m->loc, m->kxyz, m->kcol,
                                                     m->kid, m->n_kf_points, kf);
    GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    const int from = m->n_cloud;
    m->n_cloud += acc;
    m->n_kf_points += acc;
    m->kf_off.push_back(m->n_kf_points);
    m->poses.push_back(T);
    if ((rc = dm_filter(m, from))) return rc;
    if (n_inserted) *n_inserted = acc;
    return GF_OK;
}

int gf_dense_map_update_poses(gf_dense_map* m, int n_keyframes, const double* R, const double* P)
{
    if (!m || (n_keyframes > 0 && (!R || !P))) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n_keyframes != (int)m->poses.size()) return set_err(GF_ERR_INVALID_ARG, "n_keyframes differs from the number of keyframes added");
    GF_CUDA(cudaSetDevice(m->device));
    std::vector<Pose> np(n_keyframes);
    for (int k = 0; k < n_keyframes; k++) { memcpy(np[k].R, R + 9 * (size_t)k, sizeof(np[k].R)); memcpy(np[k].P, P + 3 * (size_t)k, sizeof(np[k].P)); }
    Anchor A;
    dm_octree_anchor(BOX_REBUILD_LO, BOX_HI, A.mn, A.mx);
    const int n = m->n_kf_points;
    int acc = 0;
    if (n > 0) {
        GF_CUDA(cudaMemcpyAsync(m->dposes, np.data(), sizeof(Pose) * (size_t)n_keyframes, cudaMemcpyHostToDevice, m->st));
        GF_CUDA(cudaMemsetAsync(m->bad, 0, 4, m->st));
        k_dm_rebuild_xform<<<(n + 255) / 256, 256, 0, m->st>>>(n, m->kxyz, m->kid, m->dposes, m->ext, A, m->key, m->idx, m->wxyz, m->bad);
        GF_LAUNCHED();
        GF_CUDA(cudaMemcpyAsync(m->h_pin + 1, m->bad, 4, cudaMemcpyDeviceToHost, m->st));
        GF_CUDA(cudaStreamSynchronize(m->st));
        if (m->h_pin[1]) return set_err(GF_ERR_INVALID_ARG, "a point of the rebuilt map falls outside the octree's bounding box");
        // commit: deleteTree + defineBoundingBox, then re-insert in keyframe order
        GF_CUDA(cudaMemsetAsync(m->vkeys, 0xff, 8 * ((size_t)m->vmask + 1), m->st));
        GF_CUDA(cudaMemsetAsync(m->vcnt, 0, 4 * ((size_t)m->vmask + 1), m->st));
        int rc = dm_gate(m, n, GATE_REBUILD);
        if (rc) return rc;
        acc = m->h_pin[0];
        k_dm_hash_add<<<(n + 255) / 256, 256, 0, m->st>>>(n, m->skey, m->add, m->vkeys, m->vcnt, m->vmask);
        GF_LAUNCHED();
        k_dm_scatter<<<(n + 255) / 256, 256, 0, m->st>>>(n, m->flag, m->pos, m->wxyz, m->kcol, m->cxyz, m->ccol, 0, nullptr, nullptr, nullptr, nullptr, 0, 0);
        GF_LAUNCHED();
        GF_CUDA(cudaGetLastError());
    } else {
        GF_CUDA(cudaMemsetAsync(m->vkeys, 0xff, 8 * ((size_t)m->vmask + 1), m->st));
        GF_CUDA(cudaMemsetAsync(m->vcnt, 0, 4 * ((size_t)m->vmask + 1), m->st));
    }
    m->anchor = A;
    m->poses = np;
    m->n_cloud = acc;
    return dm_filter(m, 0);
}

int gf_dense_map_size(gf_dense_map* m, int* n_cloud, int* n_filtered, int* n_keyframes)
{
    if (!m) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n_cloud) *n_cloud = m->n_cloud;
    if (n_filtered) *n_filtered = m->n_filtered;
    if (n_keyframes) *n_keyframes = (int)m->poses.size();
    return GF_OK;
}

int gf_dense_map_read(gf_dense_map* m, int which, float* xyz, uint8_t* rgb, int32_t* idx)
{
    if (!m || (which != GF_DENSE_MAP_CLOUD && which != GF_DENSE_MAP_FILTERED)) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    GF_CUDA(cudaSetDevice(m->device));
    const int n = m->n_cloud;
    std::vector<float> cx(3 * (size_t)n);
    std::vector<uchar4> cc(n);
    if (n) {
        GF_CUDA(cudaMemcpyAsync(cx.data(), m->cxyz, 12 * (size_t)n, cudaMemcpyDeviceToHost, m->st));
        GF_CUDA(cudaMemcpyAsync(cc.data(), m->ccol, 4 * (size_t)n, cudaMemcpyDeviceToHost, m->st));
    }
    std::vector<int> sel;
    if (which == GF_DENSE_MAP_FILTERED) {
        sel.resize(m->n_filtered);
        if (m->n_filtered) GF_CUDA(cudaMemcpyAsync(sel.data(), m->fidx, 4 * (size_t)m->n_filtered, cudaMemcpyDeviceToHost, m->st));
    }
    GF_CUDA(cudaStreamSynchronize(m->st));
    const int nout = which == GF_DENSE_MAP_FILTERED ? m->n_filtered : n;
    for (int i = 0; i < nout; i++) {
        const int s = which == GF_DENSE_MAP_FILTERED ? sel[i] : i;
        if (xyz) for (int k = 0; k < 3; k++) xyz[3 * (size_t)i + k] = cx[3 * (size_t)s + k];
        if (rgb) { rgb[3 * (size_t)i] = cc[s].x; rgb[3 * (size_t)i + 1] = cc[s].y; rgb[3 * (size_t)i + 2] = cc[s].z; }
        if (idx) idx[i] = s;
    }
    return GF_OK;
}

int gf_dense_map_keyframe_points(gf_dense_map* m, int k, float* out6, int* n)
{
    if (!m || !n || k < 0 || k >= (int)m->poses.size()) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    const int o = m->kf_off[k], c = m->kf_off[k + 1] - o;
    *n = c;
    if (!out6 || c == 0) return GF_OK;
    GF_CUDA(cudaSetDevice(m->device));
    std::vector<float> x(3 * (size_t)c);
    std::vector<uchar4> cc(c);
    GF_CUDA(cudaMemcpyAsync(x.data(), m->kxyz + 3 * (size_t)o, 12 * (size_t)c, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaMemcpyAsync(cc.data(), m->kcol + o, 4 * (size_t)c, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaStreamSynchronize(m->st));
    for (int i = 0; i < c; i++) {
        float* r = out6 + 6 * (size_t)i;
        r[0] = x[3 * (size_t)i]; r[1] = x[3 * (size_t)i + 1]; r[2] = x[3 * (size_t)i + 2];
        r[3] = cc[i].x; r[4] = cc[i].y; r[5] = cc[i].z;
    }
    return GF_OK;
}

int gf_stage_radius_filter(int device, const float* xyz, int n, double radius, int min_pts, uint8_t* keep)
{
    if (n < 0 || (n > 0 && (!xyz || !keep)) || !(radius > 0) || min_pts < 0) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n == 0) return GF_OK;
    const double lim = (double)(CELL_OFF - 2) * radius * (65.0 / 64.0);
    for (size_t i = 0; i < 3 * (size_t)n; i++)
        if (!(std::fabs((double)xyz[i]) < lim)) return set_err(GF_ERR_INVALID_ARG, "coordinate not finite or beyond 2^20 filter cells");
    int rc = dm_device(device);
    if (rc) return rc;
    Filter f;
    float* d_xyz = nullptr;
    uint8_t* d_keep = nullptr;
    if ((rc = f.alloc(n)) == GF_OK) {
        if (cudaMalloc(&d_xyz, 12 * (size_t)n) != cudaSuccess || cudaMalloc(&d_keep, n) != cudaSuccess) rc = set_err(GF_ERR_CUDA, "cudaMalloc failed");
        else if (cudaMemcpy(d_xyz, xyz, 12 * (size_t)n, cudaMemcpyHostToDevice) != cudaSuccess) rc = set_err(GF_ERR_CUDA, "copy failed");
        else if ((rc = f.run(n, 0, d_xyz, d_keep, radius, min_pts, nullptr, nullptr, 0)) == GF_OK &&
                 cudaMemcpy(keep, d_keep, n, cudaMemcpyDeviceToHost) != cudaSuccess) rc = set_err(GF_ERR_CUDA, "copy failed");
    }
    f.release();
    if (d_xyz) cudaFree(d_xyz);
    if (d_keep) cudaFree(d_keep);
    return rc;
}

}  // extern "C"
