// fm_kernels.cu -- gf_fm_* (C ABI): the per-landmark kernels of FeatureManager, the step either side of
// Estimator::optimization() (SURVEY 8(f) row 1; reference vins_estimator/src/estimator/feature_manager.cpp):
//   gf_fm_triangulate      triangulateWithDepth (:726-799) followed by triangulate (:668-723): depth of every landmark with
//                          >= 4 observations and no depth yet -- first from the RGB-D depths that re-project consistently into
//                          the other frames (mean of the verified depths, flag 1), else by DLT over all observations (flag 2)
//   gf_fm_parallax         compensatedParallax2 (:977-1011) summed over the landmarks tracked through frames count-2, count-1
//                          (addFeatureCheckParallax :96-104: the keyframe test)
//   gf_fm_back_shift_depth removeBackShiftDepth (:818-856): depth of a landmark transferred from the marginalised frame 0 to
//                          the new first frame
// and the per-landmark loops of the estimator that feed the front end back (estimator.cpp, after optimization()):
//   gf_fm_reprojection_errors  the sums behind Estimator::outliersRejection (:3909-3966) and movingConsistencyCheckW (:3968-4011):
//                          sum over the later observations of reprojectionError (:3888-3898) and reprojectionError3D (:3900-3907)
//   gf_fm_predict_next     Estimator::predictPtsInNextFrame (:3853-3886): landmarks carried into the constant-velocity prediction of
//                          the next frame's camera (the xyz that FeatureTracker::setPrediction takes)
// One thread per landmark: the work is O(obs^2) <= 121 small FP64 steps per landmark and there are <= a few hundred
// landmarks.  The arithmetic is in fm_device.cuh; these entry points take the lists flattened from the host, and
// gf_fm_window (fm_window.cu) runs the same functions over a table that stays on the device.
#include <vector>

#include "fm_device.cuh"

using namespace gf;

namespace gffm {

__global__ void k_fm_triangulate(int n, const int* __restrict__ start, const int* __restrict__ nobs, const int* __restrict__ off,
                                 const double* __restrict__ pts /* xyz per observation */, const double* __restrict__ dep,
                                 double* __restrict__ est, int* __restrict__ flag, FmPoses ps, double depth_threshold, double init_depth)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fm_triangulate_one(nobs[i], start[i], pts + 3 * (size_t)off[i], 3, dep + off[i], 1, est + i, flag + i, ps, depth_threshold, init_depth);
}

__global__ void k_fm_parallax(int n, const double* __restrict__ pi, const double* __restrict__ pj, double* __restrict__ out)
{
    __shared__ double sh[256];
    double s = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) s += fm_parallax_one(pi + 3 * i, pj + 3 * i);
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) atomicAdd(out, sh[0]);
}

__global__ void k_fm_back_shift(int n, const double* __restrict__ uv /* xyz */, double* __restrict__ est, const double* __restrict__ T /* marg_R 9, marg_P 3, new_R 9, new_P 3 */,
                                double init_depth)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    est[i] = fm_back_shift_one(uv + 3 * i, est[i], T, init_depth);
}

__global__ void k_fm_reproj(int nf, const int* __restrict__ start, const int* __restrict__ nobs, const int* __restrict__ off, const double* __restrict__ pts,
                            const double* __restrict__ depth, double* __restrict__ err2d, double* __restrict__ err3d, int* __restrict__ cnt, FmPoses ps)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    fm_reproj_one(start[i], nobs[i], pts + 3 * (size_t)off[i], 3, depth[i], ps, err2d + i, err3d + i, cnt + i);
}

__global__ void k_fm_predict(int n, const int* __restrict__ first, const double* __restrict__ uv, const double* __restrict__ depth, double* __restrict__ out,
                             FmPoses ps, const double* __restrict__ T)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fm_predict_one(first[i], uv + 3 * i, depth[i], ps, T, out + 3 * i);
}

}  // namespace gffm


using namespace gffm;

static int fm_device(int device)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return set_err(GF_ERR_NO_DEVICE, "no CUDA device visible; libgf_b200 has no CPU fallback");
    if (device < 0 || device >= n) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    return GF_OK;
}
struct FmBuf {
    void* p = nullptr;
    ~FmBuf() { if (p) cudaFree(p); }
    int put(const void* src, size_t bytes) { GF_CUDA(cudaMalloc(&p, bytes ? bytes : 8)); if (bytes) GF_CUDA(cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice)); return GF_OK; }
};

extern "C" {

int gf_fm_triangulate(int device, int n_features, const int32_t* start_frame, const int32_t* n_obs, const int32_t* obs_offset, int n_obs_total,
                      const double* points, const double* depths, double* estimated_depth, int32_t* estimate_flag,
                      int n_frames, const double* Ps, const double* Rs, const double* tic, const double* ric, double depth_threshold, double init_depth)
{
    if (n_features < 0 || n_frames < 1 || n_frames > GF_BA_MAX_FRAMES || (n_features > 0 && (!start_frame || !n_obs || !obs_offset || !points || !depths || !estimated_depth || !estimate_flag)) || !Ps || !Rs || !tic || !ric)
        return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n_features == 0) return GF_OK;
    for (int i = 0; i < n_features; i++)
        if (n_obs[i] < 0 || start_frame[i] < 0 || start_frame[i] + n_obs[i] > n_frames || obs_offset[i] < 0 || obs_offset[i] + n_obs[i] > n_obs_total)
            return set_err(GF_ERR_INVALID_ARG, "observation list out of range");
    int rc = fm_device(device);
    if (rc) return rc;
    FmPoses ps; memset(&ps, 0, sizeof(ps));
    memcpy(ps.P, Ps, sizeof(double) * 3 * n_frames); memcpy(ps.R, Rs, sizeof(double) * 9 * n_frames); memcpy(ps.tic, tic, 24); memcpy(ps.ric, ric, 72);
    FmBuf b_s, b_n, b_o, b_p, b_d, b_e, b_f;
    if ((rc = b_s.put(start_frame, 4 * (size_t)n_features)) || (rc = b_n.put(n_obs, 4 * (size_t)n_features)) || (rc = b_o.put(obs_offset, 4 * (size_t)n_features)) ||
        (rc = b_p.put(points, 24 * (size_t)n_obs_total)) || (rc = b_d.put(depths, 8 * (size_t)n_obs_total)) || (rc = b_e.put(estimated_depth, 8 * (size_t)n_features)) ||
        (rc = b_f.put(estimate_flag, 4 * (size_t)n_features))) return rc;
    k_fm_triangulate<<<(n_features + 63) / 64, 64>>>(n_features, (const int*)b_s.p, (const int*)b_n.p, (const int*)b_o.p, (const double*)b_p.p, (const double*)b_d.p,
                                                     (double*)b_e.p, (int*)b_f.p, ps, depth_threshold, init_depth);
    GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy(estimated_depth, b_e.p, 8 * (size_t)n_features, cudaMemcpyDeviceToHost));
    GF_CUDA(cudaMemcpy(estimate_flag, b_f.p, 4 * (size_t)n_features, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_fm_reprojection_errors(int device, int n_features, const int32_t* start_frame, const int32_t* n_obs, const int32_t* obs_offset, int n_obs_total,
                              const double* points, const double* estimated_depth, int n_frames, const double* Ps, const double* Rs, const double* tic,
                              const double* ric, double* err2d_sum, double* err3d_sum, int32_t* count)
{
    if (n_features < 0 || n_frames < 1 || n_frames > GF_BA_MAX_FRAMES || !Ps || !Rs || !tic || !ric ||
        (n_features > 0 && (!start_frame || !n_obs || !obs_offset || !points || !estimated_depth || !err2d_sum || !err3d_sum || !count)))
        return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n_features == 0) return GF_OK;
    for (int i = 0; i < n_features; i++)
        if (n_obs[i] < 1 || start_frame[i] < 0 || start_frame[i] + n_obs[i] > n_frames || obs_offset[i] < 0 || obs_offset[i] + n_obs[i] > n_obs_total)
            return set_err(GF_ERR_INVALID_ARG, "observation list out of range");
    int rc = fm_device(device);
    if (rc) return rc;
    FmPoses ps; memset(&ps, 0, sizeof(ps));
    memcpy(ps.P, Ps, sizeof(double) * 3 * n_frames); memcpy(ps.R, Rs, sizeof(double) * 9 * n_frames); memcpy(ps.tic, tic, 24); memcpy(ps.ric, ric, 72);
    FmBuf b_s, b_n, b_o, b_p, b_d, b_2, b_3, b_c;
    if ((rc = b_s.put(start_frame, 4 * (size_t)n_features)) || (rc = b_n.put(n_obs, 4 * (size_t)n_features)) || (rc = b_o.put(obs_offset, 4 * (size_t)n_features)) ||
        (rc = b_p.put(points, 24 * (size_t)n_obs_total)) || (rc = b_d.put(estimated_depth, 8 * (size_t)n_features))) return rc;
    GF_CUDA(cudaMalloc(&b_2.p, 8 * (size_t)n_features)); GF_CUDA(cudaMalloc(&b_3.p, 8 * (size_t)n_features)); GF_CUDA(cudaMalloc(&b_c.p, 4 * (size_t)n_features));
    k_fm_reproj<<<(n_features + 63) / 64, 64>>>(n_features, (const int*)b_s.p, (const int*)b_n.p, (const int*)b_o.p, (const double*)b_p.p, (const double*)b_d.p,
                                                (double*)b_2.p, (double*)b_3.p, (int*)b_c.p, ps);
    GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy(err2d_sum, b_2.p, 8 * (size_t)n_features, cudaMemcpyDeviceToHost));
    GF_CUDA(cudaMemcpy(err3d_sum, b_3.p, 8 * (size_t)n_features, cudaMemcpyDeviceToHost));
    GF_CUDA(cudaMemcpy(count, b_c.p, 4 * (size_t)n_features, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_fm_predict_next(int device, int n, const int32_t* first_frame, const double* uv_first, const double* estimated_depth, int n_frames, int frame_count,
                       const double* Ps, const double* Rs, const double* tic, const double* ric, double* pts_cam)
{
    if (n < 0 || n_frames < 2 || n_frames > GF_BA_MAX_FRAMES || frame_count < 1 || frame_count >= n_frames || !Ps || !Rs || !tic || !ric ||
        (n > 0 && (!first_frame || !uv_first || !estimated_depth || !pts_cam)))
        return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n == 0) return GF_OK;
    for (int i = 0; i < n; i++) if (first_frame[i] < 0 || first_frame[i] >= n_frames) return set_err(GF_ERR_INVALID_ARG, "frame index out of range");
    double T[12];
    fm_next_pose(Ps, Rs, frame_count, T);
    int rc = fm_device(device);
    if (rc) return rc;
    FmPoses ps; memset(&ps, 0, sizeof(ps));
    memcpy(ps.P, Ps, sizeof(double) * 3 * n_frames); memcpy(ps.R, Rs, sizeof(double) * 9 * n_frames); memcpy(ps.tic, tic, 24); memcpy(ps.ric, ric, 72);
    FmBuf b_f, b_u, b_d, b_t, b_o;
    if ((rc = b_f.put(first_frame, 4 * (size_t)n)) || (rc = b_u.put(uv_first, 24 * (size_t)n)) || (rc = b_d.put(estimated_depth, 8 * (size_t)n)) || (rc = b_t.put(T, sizeof(T))))
        return rc;
    GF_CUDA(cudaMalloc(&b_o.p, 24 * (size_t)n));
    k_fm_predict<<<(n + 63) / 64, 64>>>(n, (const int*)b_f.p, (const double*)b_u.p, (const double*)b_d.p, (double*)b_o.p, ps, (const double*)b_t.p);
    GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy(pts_cam, b_o.p, 24 * (size_t)n, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_fm_parallax(int device, int n, const double* pts_i, const double* pts_j, double* parallax_sum)
{
    if (n < 0 || !parallax_sum || (n > 0 && (!pts_i || !pts_j))) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    *parallax_sum = 0.0;
    if (n == 0) return GF_OK;
    int rc = fm_device(device);
    if (rc) return rc;
    FmBuf a, b, o;
    const double zero = 0.0;
    if ((rc = a.put(pts_i, 24 * (size_t)n)) || (rc = b.put(pts_j, 24 * (size_t)n)) || (rc = o.put(&zero, 8))) return rc;
    k_fm_parallax<<<1, 256>>>(n, (const double*)a.p, (const double*)b.p, (double*)o.p);      // one CTA: a fixed summation order
    GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy(parallax_sum, o.p, 8, cudaMemcpyDeviceToHost));
    return GF_OK;
}

int gf_fm_back_shift_depth(int device, int n, const double* uv_i, double* estimated_depth, const double* marg_R, const double* marg_P,
                           const double* new_R, const double* new_P, double init_depth)
{
    if (n < 0 || !marg_R || !marg_P || !new_R || !new_P || (n > 0 && (!uv_i || !estimated_depth))) return set_err(GF_ERR_INVALID_ARG, "bad argument");
    if (n == 0) return GF_OK;
    int rc = fm_device(device);
    if (rc) return rc;
    double T[24];
    memcpy(T, marg_R, 72); memcpy(T + 9, marg_P, 24); memcpy(T + 12, new_R, 72); memcpy(T + 21, new_P, 24);
    FmBuf a, e, t;
    if ((rc = a.put(uv_i, 24 * (size_t)n)) || (rc = e.put(estimated_depth, 8 * (size_t)n)) || (rc = t.put(T, sizeof(T)))) return rc;
    k_fm_back_shift<<<(n + 127) / 128, 128>>>(n, (const double*)a.p, (double*)e.p, (const double*)t.p, init_depth);
    GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    GF_CUDA(cudaMemcpy(estimated_depth, e.p, 8 * (size_t)n, cudaMemcpyDeviceToHost));
    return GF_OK;
}

}  // extern "C"
