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

// sample s: lift, depth / colour tests, local point, world point, z band, voxel key
__device__ __forceinline__ void dm_sample(int s, const CamParams& cam, int su, int B, int D, const uint8_t* __restrict__ rgb, size_t rgb_pitch,
                                          const uint16_t* __restrict__ depth, size_t depth_pitch, const Ext& e, const Pose& T, const Anchor& A,
                                          uint64_t* __restrict__ key, uint32_t* __restrict__ idx, float* __restrict__ loc, uchar4* __restrict__ col,
                                          float* __restrict__ wxyz, int* bad)
{
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
// one thread per sample
__global__ void k_dm_sample(CamParams cam, int su, int n, int B, int D, const uint8_t* __restrict__ rgb, size_t rgb_pitch,
                            const uint16_t* __restrict__ depth, size_t depth_pitch, Ext e, Pose T, Anchor A, uint64_t* __restrict__ key,
                            uint32_t* __restrict__ idx, float* __restrict__ loc, uchar4* __restrict__ col, float* __restrict__ wxyz, int* bad)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    dm_sample(s, cam, su, B, D, rgb, rgb_pitch, depth, depth_pitch, e, T, A, key, idx, loc, col, wxyz, bad);
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
__device__ __forceinline__ void dm_gate_run(int i, int n, const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sidx,
                                            const uint64_t* __restrict__ vkeys, const int* __restrict__ vcnt, uint32_t vmask, int cap,
                                            int* __restrict__ flag, int* __restrict__ add)
{
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
__global__ void k_dm_gate(int n, const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sidx, const uint64_t* __restrict__ vkeys,
                          const int* __restrict__ vcnt, uint32_t vmask, int cap, int* __restrict__ flag, int* __restrict__ add)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    dm_gate_run(i, n, skey, sidx, vkeys, vcnt, vmask, cap, flag, add);
}
__global__ void k_dm_hash_add(int n, const uint64_t* __restrict__ skey, const int* __restrict__ add, uint64_t* vkeys, int* vcnt, uint32_t vmask)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || add[i] == 0) return;
    atomicAdd(&vcnt[hinsert(vkeys, vmask, skey[i])], add[i]);
}
// point i, accepted at position p of the compaction: cloud at c0 (+ the keyframe's kept local points at k0 when loc != nullptr)
__device__ __forceinline__ void dm_scatter_one(int i, int p, const float* __restrict__ wxyz, const uchar4* __restrict__ col, float* __restrict__ cxyz,
                                               uchar4* __restrict__ ccol, int c0, const float* __restrict__ loc, float* __restrict__ kxyz,
                                               uchar4* __restrict__ kcol, int* __restrict__ kid, int k0, int kf)
{
    const size_t c = (size_t)c0 + p;
    for (int k = 0; k < 3; k++) cxyz[3 * c + k] = wxyz[3 * (size_t)i + k];
    ccol[c] = col[i];
    if (loc) {
        const size_t q = (size_t)k0 + p;
        for (int k = 0; k < 3; k++) kxyz[3 * q + k] = loc[3 * (size_t)i + k];
        kcol[q] = col[i];
        kid[q] = kf;
    }
}
// stable compaction of the accepted points
__global__ void k_dm_scatter(int n, const int* __restrict__ flag, const int* __restrict__ pos, const float* __restrict__ wxyz, const uchar4* __restrict__ col,
                             float* __restrict__ cxyz, uchar4* __restrict__ ccol, int c0, const float* __restrict__ loc, float* __restrict__ kxyz,
                             uchar4* __restrict__ kcol, int* __restrict__ kid, int k0, int kf)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flag[i]) return;
    dm_scatter_one(i, pos[i], wxyz, col, cxyz, ccol, c0, loc, kxyz, kcol, kid, k0, kf);
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
// the count of a query point over its 27-cell stencil (slots: each cell's hash slot, -1 when empty): 1 / 0 = kept or not,
// -1 when no cell of the stencil is dirty (the point cannot have gained a neighbour)
__device__ __forceinline__ int dm_stencil_count(float qx, float qy, float qz, const int* slots, const int2* __restrict__ hrange,
                                                const uint8_t* __restrict__ dirty, const float4* __restrict__ sxyz, float r2, int min_pts)
{
    bool any = false;
    for (int t = 0; t < 27; t++) if (slots[t] >= 0 && dirty[slots[t]]) any = true;
    if (!any) return -1;
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
    return cnt > min_pts;
}
__global__ void k_dm_count(int n, const float* __restrict__ xyz, double inv_cell, const uint64_t* __restrict__ hkeys, const int2* __restrict__ hrange,
                           const uint8_t* __restrict__ dirty, uint32_t hmask, const float4* __restrict__ sxyz, float r2, int min_pts, uint8_t* __restrict__ kept)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || kept[i]) return;
    const float qx = xyz[3 * (size_t)i], qy = xyz[3 * (size_t)i + 1], qz = xyz[3 * (size_t)i + 2];
    const int cx = cell_of(qx, inv_cell), cy = cell_of(qy, inv_cell), cz = cell_of(qz, inv_cell);
    int slots[27];
    for (int t = 0; t < 27; t++) slots[t] = hfind(hkeys, hmask, cell_key(cx + t % 3 - 1, cy + (t / 3) % 3 - 1, cz + t / 9 - 1));
    const int r = dm_stencil_count(qx, qy, qz, slots, hrange, dirty, sxyz, r2, min_pts);
    if (r >= 0) kept[i] = r;
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
    bool nf_stale = false;                           // a group call filtered the cloud: n_filtered is in nsel on the device
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
    m->nf_stale = false;
    return GF_OK;
}

// n_filtered after a group call, read on the map's stream (which waits for the group's work)
static int dm_fetch_n_filtered(gf_dense_map* m)
{
    if (!m->nf_stale) return GF_OK;
    GF_CUDA(cudaSetDevice(m->device));
    GF_CUDA(cudaMemcpyAsync(&m->n_filtered, m->nsel, 4, cudaMemcpyDeviceToHost, m->st));
    GF_CUDA(cudaStreamSynchronize(m->st));
    m->nf_stale = false;
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
    int rc = dm_fetch_n_filtered(m);
    if (rc) return rc;
    if (n_cloud) *n_cloud = m->n_cloud;
    if (n_filtered) *n_filtered = m->n_filtered;
    if (n_keyframes) *n_keyframes = (int)m->poses.size();
    return GF_OK;
}

int gf_dense_map_read(gf_dense_map* m, int which, float* xyz, uint8_t* rgb, int32_t* idx)
{
    if (!m || (which != GF_DENSE_MAP_CLOUD && which != GF_DENSE_MAP_FILTERED)) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    int rc = dm_fetch_n_filtered(m);
    if (rc) return rc;
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

// ---- gf_dense_map_group: one keyframe for each of several maps with one launch chain ----
// Gate: every member has the same ns samples, so the samples of a call form equal segments; a segmented sort orders each
// member's (voxel key, sample) pairs as the single map's sort does (the 63-bit voxel key leaves no bits for a member index).
// Filter: the cloud points lie inside the octree's box (|coordinate| < 15000 m, < 2^18 filter cells), so a cell key of 3 x 19
// bits leaves the top bits for the member, and one device-wide sort keeps every member's cells apart.
namespace gfdm {

constexpr int GROUP_MAX = 64;
constexpr int GCELL_OFF = 1 << 18;

struct DmMember {                                     // one member of a group call
    CamParams cam; Ext ext; Pose T; Anchor A;
    const uint8_t* rgb; const uint16_t* depth; size_t rgb_pitch, depth_pitch;
    uint64_t* vkeys; int* vcnt; uint32_t vmask;
    float *cxyz, *kxyz; uchar4 *ccol, *kcol; int* kid;
    int c0, k0, kf;
};
struct DmFilt {                                       // one member of the group's radius filter: points [from, n) are new
    const float* xyz; uint8_t* kept; int* fidx; int* nsel;
    int n, from;
};

// the segment a of bases[0..F] (increasing, bases[0] = 0) holding i
__device__ __forceinline__ int dm_seg(const int* __restrict__ base, int F, int i)
{
    int lo = 0, hi = F;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (base[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ uint64_t gcell_key(int a, int cx, int cy, int cz)
{
    return ((uint64_t)a << 57) | ((uint64_t)(unsigned)(cx + GCELL_OFF) << 38) | ((uint64_t)(unsigned)(cy + GCELL_OFF) << 19) | (uint64_t)(unsigned)(cz + GCELL_OFF);
}

// grid (samples, members): member a's samples are [a n, (a + 1) n) of every scratch array
__global__ void k_dmg_sample(const DmMember* __restrict__ mb, int su, int n, int B, int D, uint64_t* __restrict__ key, uint32_t* __restrict__ idx,
                             float* __restrict__ loc, uchar4* __restrict__ col, float* __restrict__ wxyz, int* bad)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const DmMember& M = mb[blockIdx.y];
    const size_t o = (size_t)blockIdx.y * n;
    dm_sample(s, M.cam, su, B, D, M.rgb, M.rgb_pitch, M.depth, M.depth_pitch, M.ext, M.T, M.A, key + o, idx + o, loc + 3 * o, col + o, wxyz + 3 * o,
              bad + blockIdx.y);
}
__global__ void k_dmg_gate(const DmMember* __restrict__ mb, int n, const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sidx, int cap,
                           int* __restrict__ flag, int* __restrict__ add)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const DmMember& M = mb[blockIdx.y];
    const size_t o = (size_t)blockIdx.y * n;
    dm_gate_run(i, n, skey + o, sidx + o, M.vkeys, M.vcnt, M.vmask, cap, flag + o, add + o);
}
// res[2 a] = member a's accepted points, res[2 a + 1] = its out-of-box flag
__global__ void k_dmg_counts(int A, int n, const int* __restrict__ flag, const int* __restrict__ pos, const int* __restrict__ bad, int* __restrict__ res)
{
    const int a = threadIdx.x;
    if (a >= A) return;
    const size_t o = (size_t)a * n;
    res[2 * a] = pos[o + n - 1] - pos[o] + flag[o + n - 1];
    res[2 * a + 1] = bad[a];
}
// commit of the members whose bit is set in ok
__global__ void k_dmg_hash_add(const DmMember* __restrict__ mb, int n, uint64_t ok, const uint64_t* __restrict__ skey, const int* __restrict__ add)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !((ok >> blockIdx.y) & 1)) return;
    const size_t o = (size_t)blockIdx.y * n;
    if (add[o + i] == 0) return;
    const DmMember& M = mb[blockIdx.y];
    atomicAdd(&M.vcnt[hinsert(M.vkeys, M.vmask, skey[o + i])], add[o + i]);
}
__global__ void k_dmg_scatter(const DmMember* __restrict__ mb, int n, uint64_t ok, const int* __restrict__ flag, const int* __restrict__ pos,
                              const float* __restrict__ wxyz, const uchar4* __restrict__ col, const float* __restrict__ loc)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !((ok >> blockIdx.y) & 1)) return;
    const size_t o = (size_t)blockIdx.y * n;
    if (!flag[o + i]) return;
    const DmMember& M = mb[blockIdx.y];
    dm_scatter_one(i, pos[o + i] - pos[o], wxyz + 3 * o, col + o, M.cxyz, M.ccol, M.c0, loc + 3 * o, M.kxyz, M.kcol, M.kid, M.k0, M.kf);
}

// the radius filter over the clouds of F members, concatenated: member a's points are [fb[a], fb[a + 1]), its new ones
// [nb[a], nb[a + 1]) of the new points' concatenation
__global__ void k_dmg_cell_keys(int N, const DmFilt* __restrict__ f, const int* __restrict__ fb, int F, double inv_cell, uint64_t* __restrict__ key,
                                uint32_t* __restrict__ idx)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int a = dm_seg(fb, F, i);
    const float* x = f[a].xyz + 3 * (size_t)(i - fb[a]);
    key[i] = gcell_key(a, cell_of(x[0], inv_cell), cell_of(x[1], inv_cell), cell_of(x[2], inv_cell));
    idx[i] = i;
}
__global__ void k_dmg_cell_build(int N, const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sidx, const DmFilt* __restrict__ f,
                                 const int* __restrict__ fb, int F, uint64_t* hkeys, int2* hrange, uint32_t hmask, float4* __restrict__ sxyz)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int p = sidx[i], a = dm_seg(fb, F, p);
    const float* x = f[a].xyz + 3 * (size_t)(p - fb[a]);
    sxyz[i] = make_float4(x[0], x[1], x[2], 0.f);
    const uint64_t k = skey[i];
    if (i == 0 || skey[i - 1] != k) hrange[hinsert(hkeys, hmask, k)].x = i;
    if (i == N - 1 || skey[i + 1] != k) hrange[hinsert(hkeys, hmask, k)].y = i + 1;
}
// a new point: not kept yet, and its cell is dirty
__global__ void k_dmg_mark_dirty(int Nn, const DmFilt* __restrict__ f, const int* __restrict__ nb, int F, double inv_cell,
                                 const uint64_t* __restrict__ hkeys, uint32_t hmask, uint8_t* __restrict__ dirty)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= Nn) return;
    const int a = dm_seg(nb, F, t);
    const size_t l = (size_t)f[a].from + (t - nb[a]);
    f[a].kept[l] = 0;
    const float* x = f[a].xyz + 3 * l;
    dirty[hfind(hkeys, hmask, gcell_key(a, cell_of(x[0], inv_cell), cell_of(x[1], inv_cell), cell_of(x[2], inv_cell)))] = 1;
}
__global__ void k_dmg_count(int N, const DmFilt* __restrict__ f, const int* __restrict__ fb, int F, double inv_cell, const uint64_t* __restrict__ hkeys,
                            const int2* __restrict__ hrange, const uint8_t* __restrict__ dirty, uint32_t hmask, const float4* __restrict__ sxyz, float r2,
                            int min_pts)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int a = dm_seg(fb, F, i);
    const size_t l = (size_t)(i - fb[a]);
    uint8_t* kept = f[a].kept;
    if (kept[l]) return;
    const float* x = f[a].xyz + 3 * l;
    const float qx = x[0], qy = x[1], qz = x[2];
    const int cx = cell_of(qx, inv_cell), cy = cell_of(qy, inv_cell), cz = cell_of(qz, inv_cell);
    int slots[27];
    for (int t = 0; t < 27; t++) slots[t] = hfind(hkeys, hmask, gcell_key(a, cx + t % 3 - 1, cy + (t / 3) % 3 - 1, cz + t / 9 - 1));
    const int r = dm_stencil_count(qx, qy, qz, slots, hrange, dirty, sxyz, r2, min_pts);
    if (r >= 0) kept[l] = r;
}
__global__ void k_dmg_flags(int N, const DmFilt* __restrict__ f, const int* __restrict__ fb, int F, int* __restrict__ flg)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int a = dm_seg(fb, F, i);
    flg[i] = f[a].kept[i - fb[a]];
}
// each member's kept indices in order, and their number
__global__ void k_dmg_select(int N, const DmFilt* __restrict__ f, const int* __restrict__ fb, int F, const int* __restrict__ flg, const int* __restrict__ pos)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int a = dm_seg(fb, F, i), p0 = pos[fb[a]];
    if (flg[i]) f[a].fidx[pos[i] - p0] = i - fb[a];
    if (i == fb[a + 1] - 1) *f[a].nsel = pos[i] + flg[i] - p0;
}

}  // namespace gfdm

struct DmCall {                                       // a call's descriptors, uploaded to the device
    DmMember mb[GROUP_MAX];
    DmFilt fl[GROUP_MAX];
    int fb[GROUP_MAX + 1], nb[GROUP_MAX + 1];
};

struct gf_dense_map_group {
    int device = 0, n = 0, ns = 0, gcap = 0, fcap = 0;
    std::vector<gf_dense_map*> m;
    cudaStream_t st = nullptr;
    cudaEvent_t ev = nullptr;                         // orders the members' streams and the group's
    DmCall* h = nullptr;                              // host copy of the descriptors (pageable: reusable once its upload returns)
    DmCall* d = nullptr;
    // gate scratch, n * ns entries
    uint64_t *key = nullptr, *skey = nullptr;
    uint32_t *idx = nullptr, *sidx = nullptr;
    int *flag = nullptr, *pos = nullptr, *add = nullptr, *bad = nullptr, *res = nullptr, *seg = nullptr;
    float *loc = nullptr, *wxyz = nullptr;
    uchar4* col = nullptr;
    // filter scratch over the members' capacities together
    uint64_t *fkey = nullptr, *fskey = nullptr, *hkeys = nullptr;
    uint32_t *fidx = nullptr, *fsidx = nullptr, hmask = 0;
    int *flg = nullptr, *fpos = nullptr;
    int2* hrange = nullptr;
    uint8_t* dirty = nullptr;
    float4* sxyz = nullptr;
    void* tmp = nullptr; size_t tmp_bytes = 0;
    int* h_res = nullptr;                             // pinned: accepted, out-of-box flag per member
};

static int dm_member_err(int rc, int k)
{
    char keep[sizeof(g_err)];
    memcpy(keep, g_err, sizeof(keep));
    snprintf(g_err, sizeof(g_err), "member %d: %s", k, keep);
    return rc;
}

static void dmg_free(gf_dense_map_group* g)
{
    for (void* p : {(void*)g->d, (void*)g->key, (void*)g->skey, (void*)g->idx, (void*)g->sidx, (void*)g->flag, (void*)g->pos, (void*)g->add, (void*)g->bad,
                    (void*)g->res, (void*)g->seg, (void*)g->loc, (void*)g->wxyz, (void*)g->col, (void*)g->fkey, (void*)g->fskey, (void*)g->hkeys,
                    (void*)g->fidx, (void*)g->fsidx, (void*)g->flg, (void*)g->fpos, (void*)g->hrange, (void*)g->dirty, (void*)g->sxyz, g->tmp})
        if (p) cudaFree(p);
    if (g->h_res) cudaFreeHost(g->h_res);
    if (g->ev) cudaEventDestroy(g->ev);
    if (g->st) cudaStreamDestroy(g->st);
    delete g->h;
    delete g;
}

// the group's filter over the members listed in g->h->fl[0, F), fb / nb filled; N points, Nn of them new
static int dmg_filter(gf_dense_map_group* g, int F, int N, int Nn)
{
    const double inv_cell = 1.0 / (RADIUS * (65.0 / 64.0));
    const float r2 = (float)(RADIUS * RADIUS);
    const DmFilt* fl = g->d->fl;
    const int *fb = g->d->fb, *nb = g->d->nb;
    uint32_t hm = 63;
    while (hm < g->hmask && (size_t)hm + 1 < 2 * (size_t)N) hm = (hm << 1) | 1;
    const int blocks = (N + 255) / 256;
    k_dmg_cell_keys<<<blocks, 256, 0, g->st>>>(N, fl, fb, F, inv_cell, g->fkey, g->fidx);
    GF_LAUNCHED();
    size_t b = g->tmp_bytes;
    GF_CUDA(cub::DeviceRadixSort::SortPairs(g->tmp, b, g->fkey, g->fskey, g->fidx, g->fsidx, N, 0, 63, g->st));
    GF_CUDA(cudaMemsetAsync(g->hkeys, 0xff, 8 * ((size_t)hm + 1), g->st));
    GF_CUDA(cudaMemsetAsync(g->dirty, 0, (size_t)hm + 1, g->st));
    k_dmg_cell_build<<<blocks, 256, 0, g->st>>>(N, g->fskey, g->fsidx, fl, fb, F, g->hkeys, g->hrange, hm, g->sxyz);
    GF_LAUNCHED();
    k_dmg_mark_dirty<<<(Nn + 255) / 256, 256, 0, g->st>>>(Nn, fl, nb, F, inv_cell, g->hkeys, hm, g->dirty);
    GF_LAUNCHED();
    k_dmg_count<<<(N + 127) / 128, 128, 0, g->st>>>(N, fl, fb, F, inv_cell, g->hkeys, g->hrange, g->dirty, hm, g->sxyz, r2, MIN_PTS);
    GF_LAUNCHED();
    k_dmg_flags<<<blocks, 256, 0, g->st>>>(N, fl, fb, F, g->flg);
    GF_LAUNCHED();
    b = g->tmp_bytes;
    GF_CUDA(cub::DeviceScan::ExclusiveSum(g->tmp, b, g->flg, g->fpos, N, g->st));
    k_dmg_select<<<blocks, 256, 0, g->st>>>(N, fl, fb, F, g->flg, g->fpos);
    GF_LAUNCHED();
    return GF_OK;
}

extern "C" {

int gf_dense_map_group_create(gf_dense_map_group** out, gf_dense_map* const* maps, int n)
{
    if (!out || !maps) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    if (n < 1) return set_err(GF_ERR_INVALID_ARG, "a group has at least one map");
    if (n > GROUP_MAX) return set_err(GF_ERR_INVALID_ARG, "a group has at most GF_DENSE_MAP_GROUP_MAX (64) maps");
    long long fcap = 0;
    for (int k = 0; k < n; k++) {
        if (!maps[k]) return dm_member_err(set_err(GF_ERR_INVALID_ARG, "null map"), k);
        for (int j = 0; j < k; j++) if (maps[j] == maps[k]) return dm_member_err(set_err(GF_ERR_INVALID_ARG, "the map is listed twice"), k);
        const gf_dense_map_cfg &a = maps[0]->cfg, &c = maps[k]->cfg;
        if (maps[k]->device != maps[0]->device) return dm_member_err(set_err(GF_ERR_INVALID_ARG, "bound to another device than member 0"), k);
        if (c.width != a.width || c.height != a.height || c.depth_dist != a.depth_dist || c.depth_boundary != a.depth_boundary)
            return dm_member_err(set_err(GF_ERR_INVALID_ARG, "width, height, depth_dist or depth_boundary differ from member 0's"), k);
        fcap += c.max_points;
    }
    if (fcap > (1ll << 30)) return set_err(GF_ERR_CAPACITY, "the members' max_points add up to more than 2^30");
    GF_CUDA(cudaSetDevice(maps[0]->device));
    gf_dense_map_group* g = new gf_dense_map_group();
    g->device = maps[0]->device; g->n = n; g->ns = maps[0]->ns;
    g->m.assign(maps, maps + n);
    g->h = new DmCall();
    g->gcap = n * g->ns;
    g->fcap = (int)fcap;
    const size_t G = (size_t)g->gcap, C = (size_t)g->fcap;
    uint32_t hc = 64;
    while (hc < 2u * (uint32_t)C) hc <<= 1;
    g->hmask = hc - 1;
#define DMG_ALLOC(p, bytes) do { if (cudaMalloc(&(p), (bytes)) != cudaSuccess) { cudaGetLastError(); dmg_free(g); return set_err(GF_ERR_CUDA, "cudaMalloc failed (dense map group)"); } } while (0)
    if (cudaStreamCreateWithFlags(&g->st, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&g->ev, cudaEventDisableTiming) != cudaSuccess) {
        cudaGetLastError(); dmg_free(g); return set_err(GF_ERR_CUDA, "stream creation failed");
    }
    DMG_ALLOC(g->d, sizeof(DmCall));
    DMG_ALLOC(g->key, 8 * G); DMG_ALLOC(g->skey, 8 * G); DMG_ALLOC(g->idx, 4 * G); DMG_ALLOC(g->sidx, 4 * G);
    DMG_ALLOC(g->flag, 4 * G); DMG_ALLOC(g->pos, 4 * G); DMG_ALLOC(g->add, 4 * G);
    DMG_ALLOC(g->loc, 12 * G); DMG_ALLOC(g->wxyz, 12 * G); DMG_ALLOC(g->col, 4 * G);
    DMG_ALLOC(g->bad, 4 * GROUP_MAX); DMG_ALLOC(g->res, 8 * GROUP_MAX); DMG_ALLOC(g->seg, 4 * (GROUP_MAX + 1));
    DMG_ALLOC(g->fkey, 8 * C); DMG_ALLOC(g->fskey, 8 * C); DMG_ALLOC(g->fidx, 4 * C); DMG_ALLOC(g->fsidx, 4 * C);
    DMG_ALLOC(g->flg, 4 * C); DMG_ALLOC(g->fpos, 4 * C); DMG_ALLOC(g->sxyz, 16 * C);
    DMG_ALLOC(g->hkeys, 8 * (size_t)hc); DMG_ALLOC(g->hrange, 8 * (size_t)hc); DMG_ALLOC(g->dirty, hc);
#undef DMG_ALLOC
    size_t b[4] = {0, 0, 0, 0};
    if (cub::DeviceSegmentedRadixSort::SortPairs(nullptr, b[0], g->key, g->skey, g->idx, g->sidx, g->gcap, n, g->seg, g->seg + 1, 0, 64) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, b[1], g->flag, g->pos, g->gcap) != cudaSuccess ||
        cub::DeviceRadixSort::SortPairs(nullptr, b[2], g->fkey, g->fskey, g->fidx, g->fsidx, g->fcap, 0, 63) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, b[3], g->flg, g->fpos, g->fcap) != cudaSuccess) {
        dmg_free(g); return set_err(GF_ERR_CUDA, "cub sizing failed");
    }
    g->tmp_bytes = *std::max_element(b, b + 4);
    std::vector<int> seg(GROUP_MAX + 1);
    for (int a = 0; a <= GROUP_MAX; a++) seg[a] = a * g->ns;
    if (cudaMalloc(&g->tmp, g->tmp_bytes) != cudaSuccess || cudaMallocHost(&g->h_res, 8 * GROUP_MAX) != cudaSuccess ||
        cudaMemcpy(g->seg, seg.data(), 4 * seg.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaGetLastError(); dmg_free(g); return set_err(GF_ERR_CUDA, "allocation failed (dense map group)");
    }
    *out = g;
    return GF_OK;
}

void gf_dense_map_group_destroy(gf_dense_map_group* g)
{
    if (!g) return;
    cudaSetDevice(g->device);
    cudaStreamSynchronize(g->st);
    dmg_free(g);
}

int gf_dense_map_group_size(gf_dense_map_group* g, int* n)
{
    if (!g || !n) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *n = g->n;
    return GF_OK;
}

int gf_dense_map_group_add_keyframes(gf_dense_map_group* g, const int32_t* members, int m, const double* R, const double* P,
                                     const uint8_t* const* rgb, const size_t* rgb_pitch, const uint16_t* const* depth, const size_t* depth_pitch,
                                     int on_device, int32_t* n_inserted, int32_t* status)
{
    if (!g || !members || !R || !P || !rgb || !rgb_pitch || !depth || !depth_pitch) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (m < 1 || m > g->n) return set_err(GF_ERR_INVALID_ARG, "m must lie in [1, group size]");
    const int w = g->m[0]->cfg.width, h = g->m[0]->cfg.height, ns = g->ns;
    uint64_t seen = 0;
    for (int j = 0; j < m; j++) {
        const int k = members[j];
        if (k < 0 || k >= g->n) return dm_member_err(set_err(GF_ERR_INVALID_ARG, "member index out of range"), j);
        if ((seen >> k) & 1) return dm_member_err(set_err(GF_ERR_INVALID_ARG, "the member is listed twice"), j);
        seen |= 1ull << k;
        if (!rgb[j] || !depth[j]) return dm_member_err(set_err(GF_ERR_INVALID_ARG, "null frame"), j);
        if (rgb_pitch[j] < 3 * (size_t)w || depth_pitch[j] < 2 * (size_t)w) return dm_member_err(set_err(GF_ERR_INVALID_ARG, "row pitch below the row width"), j);
        if ((depth_pitch[j] | (size_t)(uintptr_t)depth[j]) & 1) return dm_member_err(set_err(GF_ERR_INVALID_ARG, "depth rows must start at even addresses (uint16)"), j);
    }
    GF_CUDA(cudaSetDevice(g->device));
    std::vector<int> st(m, GF_OK), act;                 // act: the call's j of each active member
    for (int j = 0; j < m; j++) {
        if (n_inserted) n_inserted[j] = 0;
        gf_dense_map* dm = g->m[members[j]];
        if ((int)dm->poses.size() >= dm->cfg.max_keyframes) st[j] = dm_member_err(set_err(GF_ERR_CAPACITY, "max_keyframes reached"), j);
        else act.push_back(j);
    }
    const int A = (int)act.size();
    int first = GF_OK;
    char first_err[sizeof(g_err)] = "";
    auto note = [&](int j) { if (first == GF_OK && st[j] != GF_OK) { first = st[j]; memcpy(first_err, g_err, sizeof(first_err)); } };
    for (int j = 0; j < m; j++) note(j);
    if (A > 0) {
        DmCall& c = *g->h;
        for (int a = 0; a < A; a++) {
            const int j = act[a];
            gf_dense_map* dm = g->m[members[j]];
            GF_CUDA(cudaEventRecord(g->ev, dm->st));
            GF_CUDA(cudaStreamWaitEvent(g->st, g->ev, 0));
            DmMember& M = c.mb[a];
            M.cam = dm->cam; M.ext = dm->ext; M.A = dm->anchor;
            memcpy(M.T.R, R + 9 * (size_t)j, sizeof(M.T.R)); memcpy(M.T.P, P + 3 * (size_t)j, sizeof(M.T.P));
            M.rgb = rgb[j]; M.depth = depth[j]; M.rgb_pitch = rgb_pitch[j]; M.depth_pitch = depth_pitch[j];
            if (!on_device) {
                GF_CUDA(cudaMemcpy2DAsync(dm->rgb, 3 * (size_t)w, rgb[j], rgb_pitch[j], 3 * (size_t)w, h, cudaMemcpyHostToDevice, g->st));
                GF_CUDA(cudaMemcpy2DAsync(dm->depth, 2 * (size_t)w, depth[j], depth_pitch[j], 2 * (size_t)w, h, cudaMemcpyHostToDevice, g->st));
                M.rgb = dm->rgb; M.depth = dm->depth; M.rgb_pitch = 3 * (size_t)w; M.depth_pitch = 2 * (size_t)w;
            }
            M.vkeys = dm->vkeys; M.vcnt = dm->vcnt; M.vmask = dm->vmask;
            M.cxyz = dm->cxyz; M.ccol = dm->ccol; M.kxyz = dm->kxyz; M.kcol = dm->kcol; M.kid = dm->kid;
            M.c0 = dm->n_cloud; M.k0 = dm->n_kf_points; M.kf = (int)dm->poses.size();
        }
        GF_CUDA(cudaMemcpyAsync(g->d->mb, c.mb, sizeof(DmMember) * A, cudaMemcpyHostToDevice, g->st));
        GF_CUDA(cudaMemsetAsync(g->bad, 0, 4 * A, g->st));
        const dim3 g128((ns + 127) / 128, A), g256((ns + 255) / 256, A);
        const gf_dense_map_cfg& cf = g->m[0]->cfg;
        k_dmg_sample<<<g128, 128, 0, g->st>>>(g->d->mb, g->m[0]->su, ns, cf.depth_boundary, cf.depth_dist, g->key, g->idx, g->loc, g->col, g->wxyz, g->bad);
        GF_LAUNCHED();
        size_t b = g->tmp_bytes;
        GF_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(g->tmp, b, g->key, g->skey, g->idx, g->sidx, A * ns, A, g->seg, g->seg + 1, 0, 64, g->st));
        k_dmg_gate<<<g256, 256, 0, g->st>>>(g->d->mb, ns, g->skey, g->sidx, GATE_ADD, g->flag, g->add);
        GF_LAUNCHED();
        b = g->tmp_bytes;
        GF_CUDA(cub::DeviceScan::ExclusiveSum(g->tmp, b, g->flag, g->pos, A * ns, g->st));
        k_dmg_counts<<<1, GROUP_MAX, 0, g->st>>>(A, ns, g->flag, g->pos, g->bad, g->res);
        GF_LAUNCHED();
        GF_CUDA(cudaMemcpyAsync(g->h_res, g->res, 8 * (size_t)A, cudaMemcpyDeviceToHost, g->st));
        GF_CUDA(cudaStreamSynchronize(g->st));           // the call's one wait: every member's accepted count and box flag
        uint64_t ok = 0;
        int F = 0, N = 0, Nn = 0;
        c.fb[0] = c.nb[0] = 0;
        for (int a = 0; a < A; a++) {
            const int j = act[a], acc = g->h_res[2 * a];
            gf_dense_map* dm = g->m[members[j]];
            if (g->h_res[2 * a + 1]) st[j] = dm_member_err(set_err(GF_ERR_INVALID_ARG, "a point of the keyframe falls outside the octree's bounding box"), j);
            else if (dm->n_kf_points + acc > dm->max_points) st[j] = dm_member_err(set_err(GF_ERR_CAPACITY, "max_points reached"), j);
            note(j);
            if (st[j] != GF_OK) continue;
            ok |= 1ull << a;
            if (n_inserted) n_inserted[j] = acc;
            const int from = dm->n_cloud;
            dm->n_cloud += acc;
            dm->n_kf_points += acc;
            dm->kf_off.push_back(dm->n_kf_points);
            dm->poses.push_back(c.mb[a].T);
            if (acc > 0) {                              // no new point: the filter's result stands
                c.fl[F] = DmFilt{dm->cxyz, dm->kept, dm->fidx, dm->nsel, dm->n_cloud, from};
                N += dm->n_cloud; Nn += acc;
                c.fb[F + 1] = N; c.nb[F + 1] = Nn;
                F++;
                dm->nf_stale = true;
            }
        }
        if (ok) {
            k_dmg_hash_add<<<g256, 256, 0, g->st>>>(g->d->mb, ns, ok, g->skey, g->add);
            GF_LAUNCHED();
            k_dmg_scatter<<<g256, 256, 0, g->st>>>(g->d->mb, ns, ok, g->flag, g->pos, g->wxyz, g->col, g->loc);
            GF_LAUNCHED();
        }
        if (F > 0) {
            GF_CUDA(cudaMemcpyAsync(g->d->fl, c.fl, sizeof(DmFilt) * F, cudaMemcpyHostToDevice, g->st));
            GF_CUDA(cudaMemcpyAsync(g->d->fb, c.fb, 4 * (size_t)(F + 1), cudaMemcpyHostToDevice, g->st));
            GF_CUDA(cudaMemcpyAsync(g->d->nb, c.nb, 4 * (size_t)(F + 1), cudaMemcpyHostToDevice, g->st));
            int rc = dmg_filter(g, F, N, Nn);
            if (rc) return rc;
        }
        GF_CUDA(cudaGetLastError());
        GF_CUDA(cudaEventRecord(g->ev, g->st));           // the members' later work follows the group's
        for (int a = 0; a < A; a++) GF_CUDA(cudaStreamWaitEvent(g->m[members[act[a]]]->st, g->ev, 0));
    }
    if (status) for (int j = 0; j < m; j++) status[j] = st[j];
    if (first != GF_OK) memcpy(g_err, first_err, sizeof(first_err));
    return first;
}

}  // extern "C"

// For gf_grid_map_group_add_dense_keyframes (gm_grid.cu; not exported): member k of a group, and the device points (packed
// float3) of the keyframe a map added last, with the stream their writes are ordered on.
gf_dense_map* gf_dense_map_group_member(gf_dense_map_group* g, int k) { return k >= 0 && k < g->n ? g->m[k] : nullptr; }
int gf_dense_map_last_keyframe_device(gf_dense_map* m, const float** xyz, int* n, cudaStream_t* st, int* device)
{
    const int k = (int)m->poses.size() - 1;
    if (k < 0) return set_err(GF_ERR_INVALID_ARG, "the dense map has no keyframe");
    *xyz = m->kxyz + 3 * (size_t)m->kf_off[k];
    *n = m->kf_off[k + 1] - m->kf_off[k];
    *st = m->st;
    *device = m->device;
    return GF_OK;
}
