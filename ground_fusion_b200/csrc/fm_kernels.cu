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
// landmarks; the list bookkeeping (std::list<FeaturePerId>) stays on the host (ground_fusion_b200/feature_manager.py).
#include <cfloat>
#include <vector>

#include "gf_common.cuh"

using namespace gf;

namespace gffm {

__device__ __forceinline__ void m3_mul(const double* a, const double* b, double* c)
{
    double t[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) t[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
    for (int i = 0; i < 9; i++) c[i] = t[i];
}
__device__ __forceinline__ void m3_T(const double* a, double* c)
{
    double t[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) t[i * 3 + j] = a[j * 3 + i];
    for (int i = 0; i < 9; i++) c[i] = t[i];
}
__device__ __forceinline__ void m3_v(const double* a, const double* b, double* c)
{
    const double t0 = a[0] * b[0] + a[1] * b[1] + a[2] * b[2], t1 = a[3] * b[0] + a[4] * b[1] + a[5] * b[2], t2 = a[6] * b[0] + a[7] * b[1] + a[8] * b[2];
    c[0] = t0; c[1] = t1; c[2] = t2;
}

struct FmPoses { double P[GF_BA_MAX_FRAMES][3]; double R[GF_BA_MAX_FRAMES][9]; double tic[3]; double ric[9]; };

// one row of the DLT matrix A folded into the upper-triangular R of A = QR by Givens rotations, so that A is never stored
__device__ __forceinline__ void qr_add_row4(double R[4][4], double r[4])
{
    for (int k = 0; k < 4; k++) {
        if (r[k] == 0.0) continue;
        const double h = hypot(R[k][k], r[k]), c = R[k][k] / h, s = r[k] / h;
        R[k][k] = h;
        for (int j = k + 1; j < 4; j++) { const double a = R[k][j], b = r[j]; R[k][j] = c * a + s * b; r[j] = c * b - s * a; }
    }
}
// right singular vector of the smallest singular value of R (hence of A) by one-sided (Hestenes) Jacobi on R's columns: the
// vector Eigen::JacobiSVD returns as matrixV().rightCols<1>(), up to sign (only the ratio v2 / v3 is used).  Working on R, not
// on A^T A, keeps the error of the null vector at eps kappa(A) instead of eps kappa(A)^2, which matters exactly where the DLT
// is used: far landmarks and windows that barely move.
__device__ inline void smallest_right_sv4(double R[4][4], double v[4])
{
    double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    for (int sweep = 0; sweep < 20; sweep++) {
        bool rotated = false;
        for (int p = 0; p < 3; p++)
            for (int q = p + 1; q < 4; q++) {
                double a = 0, b = 0, g = 0;
                for (int k = 0; k < 4; k++) { a += R[k][p] * R[k][p]; b += R[k][q] * R[k][q]; g += R[k][p] * R[k][q]; }
                if (fabs(g) <= DBL_EPSILON * sqrt(a) * sqrt(b)) continue;       // columns p, q already orthogonal (or one is zero)
                const double zeta = (b - a) / (2.0 * g);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + hypot(1.0, zeta));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 4; k++) { const double x = R[k][p], y = R[k][q]; R[k][p] = c * x - s * y; R[k][q] = s * x + c * y; }
                for (int k = 0; k < 4; k++) { const double x = V[k][p], y = V[k][q]; V[k][p] = c * x - s * y; V[k][q] = s * x + c * y; }
                rotated = true;
            }
        if (!rotated) break;
    }
    int m = 0;
    double nm = R[0][0] * R[0][0] + R[1][0] * R[1][0] + R[2][0] * R[2][0] + R[3][0] * R[3][0];
    for (int j = 1; j < 4; j++) {
        const double n2 = R[0][j] * R[0][j] + R[1][j] * R[1][j] + R[2][j] * R[2][j] + R[3][j] * R[3][j];
        if (n2 < nm) { nm = n2; m = j; }
    }
    for (int k = 0; k < 4; k++) v[k] = V[k][m];
}

__global__ void k_fm_triangulate(int n, const int* __restrict__ start, const int* __restrict__ nobs, const int* __restrict__ off,
                                 const double* __restrict__ pts /* xyz per observation */, const double* __restrict__ dep,
                                 double* __restrict__ est, int* __restrict__ flag, FmPoses ps, double depth_threshold, double init_depth)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int m = nobs[i], s0 = start[i];
    if (m < 4 || est[i] > 0) return;                                   // used_num < 4 / already has a depth (both loops skip it)
    const double* p = pts + 3 * (size_t)off[i];
    const double* dd = dep + off[i];
    auto cam = [&](int f, double* t, double* R) {                     // t = Ps + Rs tic, R = Rs ric
        double rt[3]; m3_v(ps.R[f], ps.tic, rt);
        for (int k = 0; k < 3; k++) t[k] = ps.P[f][k] + rt[k];
        m3_mul(ps.R[f], ps.ric, R);
    };
    // ---- triangulateWithDepth ----
    double tr[3], Rr[9], RrT[9];
    cam(s0, tr, Rr); m3_T(Rr, RrT);
    double sum = 0; int cnt = 0;
    for (int a = 0; a < m; a++) {
        if (dd[a] < 0.1 || dd[a] > depth_threshold) continue;
        double t0[3], R0[9], R0T[9];
        cam(s0 + a, t0, R0); m3_T(R0, R0T);
        const double point0[3] = {p[3 * a] * dd[a], p[3 * a + 1] * dd[a], p[3 * a + 2] * dd[a]};
        double d0[3] = {t0[0] - tr[0], t0[1] - tr[1], t0[2] - tr[2]}, t2r[3], R2r[9];
        m3_v(RrT, d0, t2r); m3_mul(RrT, R0, R2r);
        for (int b = 0; b < m; b++) {
            if (a == b) continue;
            double t1[3], R1[9];
            cam(s0 + b, t1, R1);
            double d1[3] = {t1[0] - t0[0], t1[1] - t0[1], t1[2] - t0[2]}, t20[3], R20[9], R20T[9];
            m3_v(R0T, d1, t20); m3_mul(R0T, R1, R20); m3_T(R20, R20T);
            double a1[3], a2[3];
            m3_v(R20T, point0, a1); m3_v(R20T, t20, a2);
            const double px = a1[0] - a2[0], py = a1[1] - a2[1], pz = a1[2] - a2[2];
            const double rx = p[3 * b] - px / pz, ry = p[3 * b + 1] - py / pz;
            if (sqrt(rx * rx + ry * ry) < 10.0 / 460) {
                double pr[3]; m3_v(R2r, point0, pr);
                sum += pr[2] + t2r[2]; cnt++;
            }
        }
    }
    if (cnt > 0) {
        double d = sum / cnt; int fl = 1;
        if (d < 0.1) { d = init_depth; fl = 0; }
        est[i] = d; flag[i] = fl;
        return;                                                       // triangulate() then skips it (estimated_depth > 0)
    }
    // ---- triangulate: DLT over all observations, reference frame = start frame ----
    double t0[3], R0[9], R0T[9];
    cam(s0, t0, R0); m3_T(R0, R0T);
    double QR[4][4] = {{0}};
    for (int a = 0; a < m; a++) {
        double t1[3], R1[9];
        cam(s0 + a, t1, R1);
        double d1[3] = {t1[0] - t0[0], t1[1] - t0[1], t1[2] - t0[2]}, t[3], R[9], RT[9], nt[3];
        m3_v(R0T, d1, t); m3_mul(R0T, R1, R); m3_T(R, RT); m3_v(RT, t, nt);
        double P[3][4];
        for (int r = 0; r < 3; r++) { for (int c = 0; c < 3; c++) P[r][c] = RT[r * 3 + c]; P[r][3] = -nt[r]; }
        const double nrm = sqrt(p[3 * a] * p[3 * a] + p[3 * a + 1] * p[3 * a + 1] + p[3 * a + 2] * p[3 * a + 2]);
        const double f[3] = {p[3 * a] / nrm, p[3 * a + 1] / nrm, p[3 * a + 2] / nrm};
        double r0[4], r1[4];
        for (int c = 0; c < 4; c++) { r0[c] = f[0] * P[2][c] - f[2] * P[0][c]; r1[c] = f[1] * P[2][c] - f[2] * P[1][c]; }
        qr_add_row4(QR, r0); qr_add_row4(QR, r1);
    }
    double v[4];
    smallest_right_sv4(QR, v);
    double d = v[2] / v[3]; int fl = 2;
    // NaN and +inf (v3 == 0: a window without translation leaves the depth undetermined) never reach estimated_depth, whose
    // inverse the solve takes
    if (!(d >= 0.1) || isinf(d)) { d = init_depth; fl = 0; }
    est[i] = d; flag[i] = fl;
}

// sum over i of sqrt(du^2 + dv^2) with (u, v) the normalised points of the two frames; the compensated variant of the reference
// is the identity (p_i_comp = p_i, :989), so min(.,.) is the plain distance
__global__ void k_fm_parallax(int n, const double* __restrict__ pi, const double* __restrict__ pj, double* __restrict__ out)
{
    __shared__ double sh[256];
    double s = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double ui = pi[3 * i] / pi[3 * i + 2], vi = pi[3 * i + 1] / pi[3 * i + 2];
        const double du = ui - pj[3 * i], dv = vi - pj[3 * i + 1];
        s += fmax(0.0, sqrt(fmin(du * du + dv * dv, du * du + dv * dv)));
    }
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
    const double d = est[i];
    const double pi_[3] = {uv[3 * i] * d, uv[3 * i + 1] * d, uv[3 * i + 2] * d};
    double w[3], nRT[9], pj[3];
    m3_v(T, pi_, w);
    for (int k = 0; k < 3; k++) w[k] += T[9 + k] - T[21 + k];
    m3_T(T + 12, nRT); m3_v(nRT, w, pj);
    est[i] = pj[2] > 0 ? pj[2] : init_depth;
}

// err2d[i] = sum_j |pi(T_cj^-1 T_ci (depth uv_i)) - uv_j|,  err3d[i] = sum_j |T_cj^-1 T_ci (depth uv_i) - uv_j| / depth over the
// observations j after the first; cnt[i] = their number
__global__ void k_fm_reproj(int nf, const int* __restrict__ start, const int* __restrict__ nobs, const int* __restrict__ off, const double* __restrict__ pts,
                            const double* __restrict__ depth, double* __restrict__ err2d, double* __restrict__ err3d, int* __restrict__ cnt, FmPoses ps)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    const int fi = start[i], n = nobs[i];
    const double d = depth[i];
    const double* uvi = pts + 3 * (size_t)off[i];
    double a[3] = {d * uvi[0], d * uvi[1], d * uvi[2]}, b[3], pw[3];
    m3_v(ps.ric, a, b);
    for (int k = 0; k < 3; k++) b[k] += ps.tic[k];
    m3_v(ps.R[fi], b, pw);
    for (int k = 0; k < 3; k++) pw[k] += ps.P[fi][k];
    double ricT[9];
    m3_T(ps.ric, ricT);
    double e2 = 0, e3 = 0;
    int c = 0;
    for (int j = 1; j < n; j++) {
        const int fj = fi + j;
        const double* uvj = pts + 3 * (size_t)(off[i] + j);
        double RjT[9], t[3], u[3], pc[3];
        m3_T(ps.R[fj], RjT);
        for (int k = 0; k < 3; k++) t[k] = pw[k] - ps.P[fj][k];
        m3_v(RjT, t, u);
        for (int k = 0; k < 3; k++) u[k] -= ps.tic[k];
        m3_v(ricT, u, pc);
        const double rx = pc[0] / pc[2] - uvj[0], ry = pc[1] / pc[2] - uvj[1];
        e2 += sqrt(rx * rx + ry * ry);
        const double dx = pc[0] - uvj[0], dy = pc[1] - uvj[1], dz = pc[2] - uvj[2];
        e3 += sqrt(dx * dx + dy * dy + dz * dz) / d;
        c++;
    }
    err2d[i] = e2; err3d[i] = e3; cnt[i] = c;
}

// out[i] = ric^T (nextR^T (Rs[f_i] (ric (depth uv_i) + tic) + Ps[f_i] - nextP) - tic),  nextT = curT (prevT^-1 curT) in T[0..11] (R 9, P 3)
__global__ void k_fm_predict(int n, const int* __restrict__ first, const double* __restrict__ uv, const double* __restrict__ depth, double* __restrict__ out,
                             FmPoses ps, const double* __restrict__ T)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int fi = first[i];
    const double d = depth[i];
    double a[3] = {d * uv[3 * i], d * uv[3 * i + 1], d * uv[3 * i + 2]}, b[3], pw[3], nRT[9], ricT[9], l[3], c[3];
    m3_v(ps.ric, a, b);
    for (int k = 0; k < 3; k++) b[k] += ps.tic[k];
    m3_v(ps.R[fi], b, pw);
    for (int k = 0; k < 3; k++) pw[k] += ps.P[fi][k] - T[9 + k];
    m3_T(T, nRT); m3_v(nRT, pw, l);
    for (int k = 0; k < 3; k++) l[k] -= ps.tic[k];
    m3_T(ps.ric, ricT); m3_v(ricT, l, c);
    out[3 * i] = c[0]; out[3 * i + 1] = c[1]; out[3 * i + 2] = c[2];
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
    // nextT = curT * (prevT^-1 * curT), constant-velocity motion (estimator.cpp:3859-3863); host side, 4x4 in FP64
    const double* Rc = Rs + 9 * frame_count; const double* Pc = Ps + 3 * frame_count;
    const double* Rp = Rs + 9 * (frame_count - 1); const double* Pp = Ps + 3 * (frame_count - 1);
    double dR[9], dP[3], t[3], T[12];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double v = 0; for (int k = 0; k < 3; k++) v += Rp[k * 3 + i] * Rc[k * 3 + j]; dR[i * 3 + j] = v; }   // Rp^T Rc
    for (int k = 0; k < 3; k++) t[k] = Pc[k] - Pp[k];
    for (int i = 0; i < 3; i++) dP[i] = Rp[0 * 3 + i] * t[0] + Rp[1 * 3 + i] * t[1] + Rp[2 * 3 + i] * t[2];                                                       // Rp^T (Pc - Pp)
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double v = 0; for (int k = 0; k < 3; k++) v += Rc[i * 3 + k] * dR[k * 3 + j]; T[i * 3 + j] = v; }
    for (int i = 0; i < 3; i++) T[9 + i] = Rc[i * 3] * dP[0] + Rc[i * 3 + 1] * dP[1] + Rc[i * 3 + 2] * dP[2] + Pc[i];
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
