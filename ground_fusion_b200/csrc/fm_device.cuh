// fm_device.cuh -- the per-landmark arithmetic of FeatureManager as __device__ functions, shared by the stateless gf_fm_*
// kernels (fm_kernels.cu: flattened lists from the host) and the resident landmark table (fm_window.cu: rows of the table).
// Both callers run the same instruction sequence on the same values, so their results are bit-equal.  Observations are
// addressed with a stride in doubles: 3 (points) / 1 (depths) in the flattened lists, the row length in the table.
#pragma once
#include <cfloat>

#include "gf_common.cuh"

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

// triangulateWithDepth (:726-799) followed by triangulate (:668-723) for one landmark of m observations from frame s0 on:
// observation a has its point (xyz) at p + a * pstr and its depth at dd + a * dstr.  *est / *flag are left alone when the
// landmark has fewer than four observations or a depth already.
__device__ __forceinline__ void fm_triangulate_one(int m, int s0, const double* __restrict__ p, int pstr, const double* __restrict__ dd, int dstr,
                                                   double* __restrict__ est, int* __restrict__ flag, const FmPoses& ps, double depth_threshold,
                                                   double init_depth)
{
    if (m < 4 || *est > 0) return;                                    // used_num < 4 / already has a depth (both loops skip it)
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
        const double da = dd[dstr * a];
        if (da < 0.1 || da > depth_threshold) continue;
        double t0[3], R0[9], R0T[9];
        cam(s0 + a, t0, R0); m3_T(R0, R0T);
        const double point0[3] = {p[pstr * a] * da, p[pstr * a + 1] * da, p[pstr * a + 2] * da};
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
            const double rx = p[pstr * b] - px / pz, ry = p[pstr * b + 1] - py / pz;
            if (sqrt(rx * rx + ry * ry) < 10.0 / 460) {
                double pr[3]; m3_v(R2r, point0, pr);
                sum += pr[2] + t2r[2]; cnt++;
            }
        }
    }
    if (cnt > 0) {
        double d = sum / cnt; int fl = 1;
        if (d < 0.1) { d = init_depth; fl = 0; }
        *est = d; *flag = fl;
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
        const double x = p[pstr * a], y = p[pstr * a + 1], z = p[pstr * a + 2];
        const double nrm = sqrt(x * x + y * y + z * z);
        const double f[3] = {x / nrm, y / nrm, z / nrm};
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
    *est = d; *flag = fl;
}

// one landmark's term of the keyframe parallax: sqrt(du^2 + dv^2) with (u, v) the normalised points of the two frames; the
// compensated variant of the reference is the identity (p_i_comp = p_i, :989), so min(.,.) is the plain distance
__device__ __forceinline__ double fm_parallax_one(const double* __restrict__ pi, const double* __restrict__ pj)
{
    const double ui = pi[0] / pi[2], vi = pi[1] / pi[2];
    const double du = ui - pj[0], dv = vi - pj[1];
    return fmax(0.0, sqrt(fmin(du * du + dv * dv, du * du + dv * dv)));
}

// removeBackShiftDepth's depth transfer: depth d of the point uv (xyz) seen from the marginalised frame, in the new first frame;
// T = marg_R 9, marg_P 3, new_R 9, new_P 3
__device__ __forceinline__ double fm_back_shift_one(const double* __restrict__ uv, double d, const double* __restrict__ T, double init_depth)
{
    const double pi_[3] = {uv[0] * d, uv[1] * d, uv[2] * d};
    double w[3], nRT[9], pj[3];
    m3_v(T, pi_, w);
    for (int k = 0; k < 3; k++) w[k] += T[9 + k] - T[21 + k];
    m3_T(T + 12, nRT); m3_v(nRT, w, pj);
    return pj[2] > 0 ? pj[2] : init_depth;
}

// *err2d = sum_j |pi(T_cj^-1 T_ci (depth uv_i)) - uv_j|,  *err3d = sum_j |T_cj^-1 T_ci (depth uv_i) - uv_j| / depth over the
// observations j after the first of a landmark with n observations from frame fi on (points at pts + j * pstr); *cnt = their number
__device__ __forceinline__ void fm_reproj_one(int fi, int n, const double* __restrict__ pts, int pstr, double d, const FmPoses& ps,
                                              double* __restrict__ err2d, double* __restrict__ err3d, int* __restrict__ cnt)
{
    const double* uvi = pts;
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
        const double* uvj = pts + (size_t)pstr * j;
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
    *err2d = e2; *err3d = e3; *cnt = c;
}

// out = ric^T (nextR^T (Rs[fi] (ric (depth uv) + tic) + Ps[fi] - nextP) - tic),  nextT = curT (prevT^-1 curT) in T[0..11] (R 9, P 3)
__device__ __forceinline__ void fm_predict_one(int fi, const double* __restrict__ uv, double d, const FmPoses& ps, const double* __restrict__ T,
                                               double* __restrict__ out)
{
    double a[3] = {d * uv[0], d * uv[1], d * uv[2]}, b[3], pw[3], nRT[9], ricT[9], l[3], c[3];
    m3_v(ps.ric, a, b);
    for (int k = 0; k < 3; k++) b[k] += ps.tic[k];
    m3_v(ps.R[fi], b, pw);
    for (int k = 0; k < 3; k++) pw[k] += ps.P[fi][k] - T[9 + k];
    m3_T(T, nRT); m3_v(nRT, pw, l);
    for (int k = 0; k < 3; k++) l[k] -= ps.tic[k];
    m3_T(ps.ric, ricT); m3_v(ricT, l, c);
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2];
}

// nextT = curT * (prevT^-1 * curT), the constant-velocity motion of predictPtsInNextFrame (estimator.cpp:3859-3863), on the
// host in FP64: T = R 9, P 3
inline void fm_next_pose(const double* Ps, const double* Rs, int frame_count, double T[12])
{
    const double* Rc = Rs + 9 * frame_count; const double* Pc = Ps + 3 * frame_count;
    const double* Rp = Rs + 9 * (frame_count - 1); const double* Pp = Ps + 3 * (frame_count - 1);
    double dR[9], dP[3], t[3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double v = 0; for (int k = 0; k < 3; k++) v += Rp[k * 3 + i] * Rc[k * 3 + j]; dR[i * 3 + j] = v; }   // Rp^T Rc
    for (int k = 0; k < 3; k++) t[k] = Pc[k] - Pp[k];
    for (int i = 0; i < 3; i++) dP[i] = Rp[0 * 3 + i] * t[0] + Rp[1 * 3 + i] * t[1] + Rp[2 * 3 + i] * t[2];                                                       // Rp^T (Pc - Pp)
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double v = 0; for (int k = 0; k < 3; k++) v += Rc[i * 3 + k] * dR[k * 3 + j]; T[i * 3 + j] = v; }
    for (int i = 0; i < 3; i++) T[9 + i] = Rc[i * 3] * dP[0] + Rc[i * 3 + 1] * dP[1] + Rc[i * 3 + 2] * dP[2] + Pc[i];
}

}  // namespace gffm
