/*
 * oracle/ba_oracle.c -- TEST INFRASTRUCTURE ONLY (CPU oracle for the back end; never shipped).
 *
 * FP64 restatement of Estimator::optimization() (reference vins_estimator/src/estimator/estimator.cpp:
 * 2890-3636): the analytic factors of vins_estimator/src/factor/ and the Ceres solve they are fed to.
 *
 * PARITY UNPINNED: the reference has no tests or golden vectors for this path and cannot be compiled
 * here (Ceres, Eigen, Sophus, ROS absent).  The trust-region loop lives in un-vendored Ceres Solver
 * 1.14 (README.md:84; internal/ceres/{trust_region_minimizer,dogleg_strategy,corrector,
 * residual_block}.cc) and is restated here from its published algorithm: Jacobi column scaling fixed at
 * iteration 0, traditional dogleg (radius 1e4, mu 1e-8..1, x10 on failure), step acceptance at relative
 * decrease > 1e-3, function/parameter/gradient tolerances 1e-6/1e-8/1e-10, DENSE_SCHUR = exact
 * elimination of the landmark blocks + dense Cholesky.  The factors are pinned by finite differences
 * (the method of ProjectionTwoFrameOneCamFactor::check, projectionTwoFrameOneCamFactor.cpp:153-275) and
 * the optimum by an independent SciPy solve (tests/test_ba_oracle.py).
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC (oracle/Makefile).
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/gf_b200.h"

#define GFO __attribute__((visibility("default")))

/* ------------------------------------------------------------------ small math ------------------ */
typedef double v3[3];
typedef double m3[9]; /* row-major */
typedef double q4[4]; /* x y z w */

static void m3_mul(const m3 a, const m3 b, m3 c)
{
    m3 t;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) t[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
    memcpy(c, t, sizeof(m3));
}
static void m3_T(const m3 a, m3 c)
{
    m3 t;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) t[i * 3 + j] = a[j * 3 + i];
    memcpy(c, t, sizeof(m3));
}
static void m3_v(const m3 a, const v3 b, v3 c)
{
    v3 t;
    for (int i = 0; i < 3; i++) t[i] = a[i * 3] * b[0] + a[i * 3 + 1] * b[1] + a[i * 3 + 2] * b[2];
    memcpy(c, t, sizeof(v3));
}
static void skew(const v3 q, m3 s)
{ /* Utility::skewSymmetric, utility/utility.h:38-46 */
    s[0] = 0; s[1] = -q[2]; s[2] = q[1];
    s[3] = q[2]; s[4] = 0; s[5] = -q[0];
    s[6] = -q[1]; s[7] = q[0]; s[8] = 0;
}
static void q_mul(const q4 a, const q4 b, q4 c)
{ /* Hamilton product, Eigen convention */
    q4 t;
    t[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    t[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    t[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    t[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
    memcpy(c, t, sizeof(q4));
}
static void q_inv(const q4 a, q4 c)
{ /* Eigen::Quaternion::inverse(): conjugate / squaredNorm */
    double n2 = a[0] * a[0] + a[1] * a[1] + a[2] * a[2] + a[3] * a[3];
    c[0] = -a[0] / n2; c[1] = -a[1] / n2; c[2] = -a[2] / n2; c[3] = a[3] / n2;
}
static void q_normalize(q4 a)
{
    double n = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2] + a[3] * a[3]);
    for (int i = 0; i < 4; i++) a[i] /= n;
}
static void q_to_R(const q4 q, m3 R)
{ /* Eigen::Quaternion::toRotationMatrix */
    double x = q[0], y = q[1], z = q[2], w = q[3];
    double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
static void q_rot(const q4 q, const v3 v, v3 out)
{
    m3 R;
    q_to_R(q, R);
    m3_v(R, v, out);
}
static void delta_q(const v3 theta, q4 dq)
{ /* Utility::deltaQ, utility/utility.h:23-36 */
    dq[0] = theta[0] / 2.0; dq[1] = theta[1] / 2.0; dq[2] = theta[2] / 2.0; dq[3] = 1.0;
    q_normalize(dq);
}
static void q_left_br(const q4 q, m3 out)
{ /* Utility::Qleft(q).bottomRightCorner<3,3>() = w I + skew(v) */
    m3 s; skew(q, s);
    for (int i = 0; i < 9; i++) out[i] = s[i];
    out[0] += q[3]; out[4] += q[3]; out[8] += q[3];
}
static void q_right_br(const q4 q, m3 out)
{ /* Utility::Qright(q).bottomRightCorner<3,3>() = w I - skew(v) */
    m3 s; skew(q, s);
    for (int i = 0; i < 9; i++) out[i] = -s[i];
    out[0] += q[3]; out[4] += q[3]; out[8] += q[3];
}

/* dense helpers (row-major) */
static int chol_lower(double* A, int n)
{ /* in place, lower triangle; returns 0 on success */
    for (int j = 0; j < n; j++) {
        double d = A[j * n + j];
        for (int k = 0; k < j; k++) d -= A[j * n + k] * A[j * n + k];
        if (!(d > 0.0)) return -1;
        d = sqrt(d);
        A[j * n + j] = d;
        for (int i = j + 1; i < n; i++) {
            double s = A[i * n + j];
            for (int k = 0; k < j; k++) s -= A[i * n + k] * A[j * n + k];
            A[i * n + j] = s / d;
        }
    }
    return 0;
}
static void chol_solve(const double* L, int n, double* b)
{
    for (int i = 0; i < n; i++) {
        double s = b[i];
        for (int k = 0; k < i; k++) s -= L[i * n + k] * b[k];
        b[i] = s / L[i * n + i];
    }
    for (int i = n - 1; i >= 0; i--) {
        double s = b[i];
        for (int k = i + 1; k < n; k++) s -= L[k * n + i] * b[k];
        b[i] = s / L[i * n + i];
    }
}
static int lu_inverse(const double* A, int n, double* inv)
{ /* Gauss-Jordan with partial pivoting (Eigen's inverse() for dynamic sizes is PartialPivLU-based) */
    double* M = (double*)malloc(sizeof(double) * n * 2 * n);
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) { M[i * 2 * n + j] = A[i * n + j]; M[i * 2 * n + n + j] = (i == j); }
    for (int c = 0; c < n; c++) {
        int piv = c;
        for (int r = c + 1; r < n; r++) if (fabs(M[r * 2 * n + c]) > fabs(M[piv * 2 * n + c])) piv = r;
        if (M[piv * 2 * n + c] == 0.0) { free(M); return -1; }
        if (piv != c) for (int j = 0; j < 2 * n; j++) { double t = M[c * 2 * n + j]; M[c * 2 * n + j] = M[piv * 2 * n + j]; M[piv * 2 * n + j] = t; }
        double d = M[c * 2 * n + c];
        for (int j = 0; j < 2 * n; j++) M[c * 2 * n + j] /= d;
        for (int r = 0; r < n; r++) if (r != c) {
            double f = M[r * 2 * n + c];
            if (f != 0.0) for (int j = 0; j < 2 * n; j++) M[r * 2 * n + j] -= f * M[c * 2 * n + j];
        }
    }
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) inv[i * n + j] = M[i * 2 * n + n + j];
    free(M);
    return 0;
}
/* sqrt_info = LLT(cov^-1).matrixL().transpose()  (imu_factor.h:73, wheel_factor.h:85): upper triangular U = L^T */
GFO int gfo_sqrt_info(const double* cov, int n, double* sqrt_info)
{
    double* inv = (double*)malloc(sizeof(double) * n * n);
    if (lu_inverse(cov, n, inv)) { free(inv); return -1; }
    if (chol_lower(inv, n)) { free(inv); return -2; }
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) sqrt_info[i * n + j] = (j >= i) ? inv[j * n + i] : 0.0;
    free(inv);
    return 0;
}

/* symmetric eigendecomposition, cyclic Jacobi: A = V diag(w) V^T (Eigen::SelfAdjointEigenSolver stand-in;
 * only V S V^T-type products are compared, which do not depend on the eigenvector basis) */
static void sym_eig(const double* Ain, int n, double* w, double* V)
{
    double* A = (double*)malloc(sizeof(double) * n * n);
    memcpy(A, Ain, sizeof(double) * n * n);
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) V[i * n + j] = (i == j);
    for (int sweep = 0; sweep < 60; sweep++) {
        double off = 0, diag = 0;
        for (int i = 0; i < n; i++) { diag += A[i * n + i] * A[i * n + i]; for (int j = i + 1; j < n; j++) off += A[i * n + j] * A[i * n + j]; }
        if (off <= 1e-30 * diag || off == 0) break;
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++) {
                double apq = A[p * n + q];
                if (apq == 0.0) continue;
                double theta = (A[q * n + q] - A[p * n + p]) / (2.0 * apq);
                double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < n; k++) {
                    double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s * akq; A[k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; k++) {
                    double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s * aqk; A[q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; k++) {
                    double vkp = V[k * n + p], vkq = V[k * n + q];
                    V[k * n + p] = c * vkp - s * vkq; V[k * n + q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < n; i++) w[i] = A[i * n + i];
    free(A);
}

/* Symmetric eigendecomposition the way Eigen's SelfAdjointEigenSolver does it -- Householder tridiagonalisation followed
 * by implicit-shift QL -- restated from the classic EISPACK tred2 / tql2 routines (public domain; Eigen's implementation
 * is the same algorithm family).  V: row-major n x n, columns = eigenvectors; w: eigenvalues (unsorted order of
 * deflation, as needed by the marginalisation, which is order-independent). */
static void sym_eig_ql(const double* Ain, int n, double* w, double* V)
{
    double* d = w;
    double* e = (double*)malloc(sizeof(double) * (n + 1));
    memcpy(V, Ain, sizeof(double) * n * n);          /* symmetric: row-major == column-major */
#define VV(i, j) V[(size_t)(j) * n + (i)]              /* column-major while working: the inner loops run down columns */
    for (int j = 0; j < n; j++) d[j] = VV(n - 1, j);
    for (int i = n - 1; i > 0; i--) {                       /* tred2 */
        double scale = 0.0, h = 0.0;
        for (int k = 0; k < i; k++) scale += fabs(d[k]);
        if (scale == 0.0) {
            e[i] = d[i - 1];
            for (int j = 0; j < i; j++) { d[j] = VV(i - 1, j); VV(i, j) = 0.0; VV(j, i) = 0.0; }
        } else {
            for (int k = 0; k < i; k++) { d[k] /= scale; h += d[k] * d[k]; }
            double f = d[i - 1], g = sqrt(h);
            if (f > 0) g = -g;
            e[i] = scale * g; h = h - f * g; d[i - 1] = f - g;
            for (int j = 0; j < i; j++) e[j] = 0.0;
            for (int j = 0; j < i; j++) {
                f = d[j]; VV(j, i) = f; g = e[j] + VV(j, j) * f;
                for (int k = j + 1; k <= i - 1; k++) { g += VV(k, j) * d[k]; e[k] += VV(k, j) * f; }
                e[j] = g;
            }
            f = 0.0;
            for (int j = 0; j < i; j++) { e[j] /= h; f += e[j] * d[j]; }
            double hh = f / (h + h);
            for (int j = 0; j < i; j++) e[j] -= hh * d[j];
            for (int j = 0; j < i; j++) {
                f = d[j]; g = e[j];
                for (int k = j; k <= i - 1; k++) VV(k, j) -= (f * e[k] + g * d[k]);
                d[j] = VV(i - 1, j); VV(i, j) = 0.0;
            }
        }
        d[i] = h;
    }
    for (int i = 0; i < n - 1; i++) {                       /* accumulate the transformations */
        VV(n - 1, i) = VV(i, i); VV(i, i) = 1.0;
        double h = d[i + 1];
        if (h != 0.0) {
            for (int k = 0; k <= i; k++) d[k] = VV(k, i + 1) / h;
            for (int j = 0; j <= i; j++) {
                double g = 0.0;
                for (int k = 0; k <= i; k++) g += VV(k, i + 1) * VV(k, j);
                for (int k = 0; k <= i; k++) VV(k, j) -= g * d[k];
            }
        }
        for (int k = 0; k <= i; k++) VV(k, i + 1) = 0.0;
    }
    for (int j = 0; j < n; j++) { d[j] = VV(n - 1, j); VV(n - 1, j) = 0.0; }
    VV(n - 1, n - 1) = 1.0; e[0] = 0.0;
    for (int i = 1; i < n; i++) e[i - 1] = e[i];            /* tql2 */
    e[n - 1] = 0.0;
    double f = 0.0, tst1 = 0.0;
    const double eps = 2.220446049250313e-16;
    for (int l = 0; l < n; l++) {
        double t = fabs(d[l]) + fabs(e[l]);
        if (t > tst1) tst1 = t;
        int m = l;
        while (m < n) { if (fabs(e[m]) <= eps * tst1) break; m++; }
        if (m > l) {
            int iter = 0;
            do {
                iter++;
                double g = d[l], p = (d[l + 1] - g) / (2.0 * e[l]), r = hypot(p, 1.0);
                if (p < 0) r = -r;
                d[l] = e[l] / (p + r); d[l + 1] = e[l] * (p + r);
                double dl1 = d[l + 1], h = g - d[l];
                for (int i = l + 2; i < n; i++) d[i] -= h;
                f += h;
                p = d[m];
                double c = 1.0, c2 = c, c3 = c, el1 = e[l + 1], s = 0.0, s2 = 0.0;
                for (int i = m - 1; i >= l; i--) {
                    c3 = c2; c2 = c; s2 = s;
                    g = c * e[i]; h = c * p; r = hypot(p, e[i]);
                    e[i + 1] = s * r; s = e[i] / r; c = p / r; p = c * d[i] - s * g; d[i + 1] = h + s * (c * g + s * d[i]);
                    for (int k = 0; k < n; k++) { h = VV(k, i + 1); VV(k, i + 1) = s * VV(k, i) + c * h; VV(k, i) = c * VV(k, i) - s * h; }
                }
                p = -s * s2 * c3 * el1 * e[l] / dl1; e[l] = s * p; d[l] = c * p;
            } while (fabs(e[l]) > eps * tst1 && iter < 200);
        }
        d[l] = d[l] + f; e[l] = 0.0;
    }
#undef VV
    for (int i = 0; i < n; i++) for (int j = i + 1; j < n; j++) { double t = V[(size_t)i * n + j]; V[(size_t)i * n + j] = V[(size_t)j * n + i]; V[(size_t)j * n + i] = t; }
    free(e);
}
GFO void gfo_sym_eig(const double* A, int n, double* w, double* V, int method) { if (method == 0) sym_eig(A, n, w, V); else sym_eig_ql(A, n, w, V); }

/* ------------------------------------------------------------------ factors --------------------- */
/* ProjectionTwoFrameOneCamFactor::Evaluate (projectionTwoFrameOneCamFactor.cpp:43-151).
 * Jacobians are row-major num_residuals x global_size, any may be NULL. */
GFO void gfo_eval_visual(const gf_ba_visual_factor* f, double sqrt_info, const double* pose_i, const double* pose_j,
                         const double* ex, double inv_dep, double td, double* res, double* Ji, double* Jj, double* Jex,
                         double* Jf, double* Jtd)
{
    const double *Pi = pose_i, *Qi = pose_i + 3, *Pj = pose_j, *Qj = pose_j + 3, *tic = ex, *qic = ex + 3;
    v3 vi = {f->vel_i[0], f->vel_i[1], 0}, vj = {f->vel_j[0], f->vel_j[1], 0};
    v3 pts_i_td, pts_j_td, pc_i, pimu_i, pw, pimu_j, pc_j, t;
    for (int k = 0; k < 3; k++) { pts_i_td[k] = f->pts_i[k] - (td - f->td_i) * vi[k]; pts_j_td[k] = f->pts_j[k] - (td - f->td_j) * vj[k]; }
    for (int k = 0; k < 3; k++) pc_i[k] = pts_i_td[k] / inv_dep;
    m3 Ri, Rj, ric, RjT, ricT;
    q_to_R(Qi, Ri); q_to_R(Qj, Rj); q_to_R(qic, ric); m3_T(Rj, RjT); m3_T(ric, ricT);
    m3_v(ric, pc_i, pimu_i); for (int k = 0; k < 3; k++) pimu_i[k] += tic[k];
    m3_v(Ri, pimu_i, pw); for (int k = 0; k < 3; k++) pw[k] += Pi[k];
    for (int k = 0; k < 3; k++) t[k] = pw[k] - Pj[k];
    m3_v(RjT, t, pimu_j);           /* Qj.inverse() * (pts_w - Pj) (unit quaternion) */
    for (int k = 0; k < 3; k++) t[k] = pimu_j[k] - tic[k];
    m3_v(ricT, t, pc_j);
    double dep_j = pc_j[2];
    res[0] = sqrt_info * (pc_j[0] / dep_j - pts_j_td[0]);
    res[1] = sqrt_info * (pc_j[1] / dep_j - pts_j_td[1]);
    if (!Ji && !Jj && !Jex && !Jf && !Jtd) return;
    double reduce[6] = {1. / dep_j, 0, -pc_j[0] / (dep_j * dep_j), 0, 1. / dep_j, -pc_j[1] / (dep_j * dep_j)};
    for (int k = 0; k < 6; k++) reduce[k] *= sqrt_info;
    m3 A, B, S; /* A = ric^T Rj^T */
    m3_mul(ricT, RjT, A);
    if (Ji) {
        double jaco[18];
        m3_mul(A, Ri, B); skew(pimu_i, S); m3 C; m3_mul(B, S, C);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { jaco[r * 6 + c] = A[r * 3 + c]; jaco[r * 6 + 3 + c] = -C[r * 3 + c]; }
        for (int r = 0; r < 2; r++) { for (int c = 0; c < 6; c++) Ji[r * 7 + c] = reduce[r * 3] * jaco[c] + reduce[r * 3 + 1] * jaco[6 + c] + reduce[r * 3 + 2] * jaco[12 + c]; Ji[r * 7 + 6] = 0; }
    }
    if (Jj) {
        double jaco[18];
        skew(pimu_j, S); m3 C; m3_mul(ricT, S, C);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { jaco[r * 6 + c] = -A[r * 3 + c]; jaco[r * 6 + 3 + c] = C[r * 3 + c]; }
        for (int r = 0; r < 2; r++) { for (int c = 0; c < 6; c++) Jj[r * 7 + c] = reduce[r * 3] * jaco[c] + reduce[r * 3 + 1] * jaco[6 + c] + reduce[r * 3 + 2] * jaco[12 + c]; Jj[r * 7 + 6] = 0; }
    }
    m3 tmp_r; /* ric^T Rj^T Ri ric */
    m3_mul(A, Ri, B); m3_mul(B, ric, tmp_r);
    if (Jex) {
        double jaco[18];
        m3 RjTRi, M, L;
        m3_mul(RjT, Ri, RjTRi);
        for (int k = 0; k < 9; k++) M[k] = RjTRi[k]; M[0] -= 1; M[4] -= 1; M[8] -= 1;
        m3_mul(ricT, M, L);
        m3 S1, T1, S2, S3; v3 u, w2, x;
        skew(pc_i, S1); m3_mul(tmp_r, S1, T1);
        m3_v(tmp_r, pc_i, u); skew(u, S2);
        m3_v(Ri, tic, w2); for (int k = 0; k < 3; k++) w2[k] += Pi[k] - Pj[k];
        m3_v(RjT, w2, x); for (int k = 0; k < 3; k++) x[k] -= tic[k];
        m3_v(ricT, x, w2); skew(w2, S3);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { jaco[r * 6 + c] = L[r * 3 + c]; jaco[r * 6 + 3 + c] = -T1[r * 3 + c] + S2[r * 3 + c] + S3[r * 3 + c]; }
        for (int r = 0; r < 2; r++) { for (int c = 0; c < 6; c++) Jex[r * 7 + c] = reduce[r * 3] * jaco[c] + reduce[r * 3 + 1] * jaco[6 + c] + reduce[r * 3 + 2] * jaco[12 + c]; Jex[r * 7 + 6] = 0; }
    }
    if (Jf) {
        v3 u; m3_v(tmp_r, pts_i_td, u);
        for (int r = 0; r < 2; r++) Jf[r] = (reduce[r * 3] * u[0] + reduce[r * 3 + 1] * u[1] + reduce[r * 3 + 2] * u[2]) * -1.0 / (inv_dep * inv_dep);
    }
    if (Jtd) {
        v3 u; m3_v(tmp_r, vi, u);
        for (int r = 0; r < 2; r++) Jtd[r] = (reduce[r * 3] * u[0] + reduce[r * 3 + 1] * u[1] + reduce[r * 3 + 2] * u[2]) / inv_dep * -1.0 + sqrt_info * vj[r];
    }
}

/* IMUFactor::Evaluate (imu_factor.h:28-191) + IntegrationBase::evaluate (integration_base.h:169-195).
 * sqrt_info (15x15 upper) is passed in (gfo_sqrt_info of the covariance; constant during a solve). */
enum { O_P = 0, O_R = 3, O_V = 6, O_BA = 9, O_BG = 12 };
static void blk(const double* J, int r0, int c0, m3 out) { for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) out[r * 3 + c] = J[(r0 + r) * 15 + c0 + c]; }
static void set_blk(double* J, int ld, int r0, int c0, const m3 M, double s) { for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) J[(r0 + r) * ld + c0 + c] = s * M[r * 3 + c]; }
static void left_mul_sqrt(const double* U, int n, double* J, int cols)
{ /* J <- U * J, J is n x cols */
    double* T = (double*)malloc(sizeof(double) * n * cols);
    for (int i = 0; i < n; i++) for (int c = 0; c < cols; c++) { double s = 0; for (int k = 0; k < n; k++) s += U[i * n + k] * J[k * cols + c]; T[i * cols + c] = s; }
    memcpy(J, T, sizeof(double) * n * cols);
    free(T);
}
GFO void gfo_eval_imu(const gf_ba_imu_factor* f, const double* sqrt_info, const double* G, const double* pose_i, const double* sb_i,
                      const double* pose_j, const double* sb_j, double* res, double* J0, double* J1, double* J2, double* J3)
{
    const double *Pi = pose_i, *Qi = pose_i + 3, *Vi = sb_i, *Bai = sb_i + 3, *Bgi = sb_i + 6;
    const double *Pj = pose_j, *Qj = pose_j + 3, *Vj = sb_j, *Baj = sb_j + 3, *Bgj = sb_j + 6;
    m3 dp_dba, dp_dbg, dq_dbg, dv_dba, dv_dbg;
    blk(f->jacobian, O_P, O_BA, dp_dba); blk(f->jacobian, O_P, O_BG, dp_dbg); blk(f->jacobian, O_R, O_BG, dq_dbg);
    blk(f->jacobian, O_V, O_BA, dv_dba); blk(f->jacobian, O_V, O_BG, dv_dbg);
    v3 dba, dbg, t, u;
    for (int k = 0; k < 3; k++) { dba[k] = Bai[k] - f->linearized_ba[k]; dbg[k] = Bgi[k] - f->linearized_bg[k]; }
    q4 dq, corr_q, Qi_inv, tq, tq2;
    m3_v(dq_dbg, dbg, t); delta_q(t, dq); q_mul(f->delta_q, dq, corr_q);
    v3 corr_v, corr_p;
    m3_v(dv_dba, dba, t); m3_v(dv_dbg, dbg, u); for (int k = 0; k < 3; k++) corr_v[k] = f->delta_v[k] + t[k] + u[k];
    m3_v(dp_dba, dba, t); m3_v(dp_dbg, dbg, u); for (int k = 0; k < 3; k++) corr_p[k] = f->delta_p[k] + t[k] + u[k];
    q_inv(Qi, Qi_inv);
    double dt = f->sum_dt;
    double r[15];
    v3 a, b;
    for (int k = 0; k < 3; k++) a[k] = 0.5 * G[k] * dt * dt + Pj[k] - Pi[k] - Vi[k] * dt;
    q_rot(Qi_inv, a, t); for (int k = 0; k < 3; k++) r[O_P + k] = t[k] - corr_p[k];
    q_inv(corr_q, tq); q_mul(Qi_inv, Qj, tq2); q_mul(tq, tq2, tq);
    for (int k = 0; k < 3; k++) r[O_R + k] = 2 * tq[k];
    for (int k = 0; k < 3; k++) b[k] = G[k] * dt + Vj[k] - Vi[k];
    q_rot(Qi_inv, b, u); for (int k = 0; k < 3; k++) r[O_V + k] = u[k] - corr_v[k];
    for (int k = 0; k < 3; k++) { r[O_BA + k] = Baj[k] - Bai[k]; r[O_BG + k] = Bgj[k] - Bgi[k]; }
    for (int i = 0; i < 15; i++) { double s = 0; for (int k = 0; k < 15; k++) s += sqrt_info[i * 15 + k] * r[k]; res[i] = s; }
    if (!J0 && !J1 && !J2 && !J3) return;
    m3 RiT, S, M, N;
    q_to_R(Qi_inv, RiT);
    if (J0) {
        memset(J0, 0, sizeof(double) * 15 * 7);
        set_blk(J0, 7, O_P, O_P, RiT, -1.0);
        skew(t, S); /* t = Qi^-1 * (0.5 G dt^2 + Pj - Pi - Vi dt) */
        set_blk(J0, 7, O_P, O_R, S, 1.0);
        q4 qji; q_inv(Qj, tq); q_mul(tq, Qi, qji);
        q_left_br(qji, M); q_right_br(corr_q, N);
        /* -(Qleft(Qj^-1 Qi) * Qright(corrected_delta_q)).bottomRightCorner<3,3>(): the 4x4 product's lower-right block */
        {
            double L4[16], R4[16], P4[16];
            /* Qleft */
            L4[0] = qji[3]; L4[1] = -qji[0]; L4[2] = -qji[1]; L4[3] = -qji[2];
            for (int rr = 0; rr < 3; rr++) { L4[(rr + 1) * 4] = qji[rr]; for (int cc = 0; cc < 3; cc++) L4[(rr + 1) * 4 + 1 + cc] = M[rr * 3 + cc]; }
            R4[0] = corr_q[3]; R4[1] = -corr_q[0]; R4[2] = -corr_q[1]; R4[3] = -corr_q[2];
            for (int rr = 0; rr < 3; rr++) { R4[(rr + 1) * 4] = corr_q[rr]; for (int cc = 0; cc < 3; cc++) R4[(rr + 1) * 4 + 1 + cc] = N[rr * 3 + cc]; }
            for (int rr = 0; rr < 4; rr++) for (int cc = 0; cc < 4; cc++) { double s = 0; for (int k = 0; k < 4; k++) s += L4[rr * 4 + k] * R4[k * 4 + cc]; P4[rr * 4 + cc] = s; }
            for (int rr = 0; rr < 3; rr++) for (int cc = 0; cc < 3; cc++) J0[(O_R + rr) * 7 + O_R + cc] = -P4[(rr + 1) * 4 + 1 + cc];
        }
        skew(u, S); /* u = Qi^-1 * (G dt + Vj - Vi) */
        set_blk(J0, 7, O_V, O_R, S, 1.0);
        left_mul_sqrt(sqrt_info, 15, J0, 7);
    }
    if (J1) {
        memset(J1, 0, sizeof(double) * 15 * 9);
        set_blk(J1, 9, O_P, O_V - O_V, RiT, -dt);
        set_blk(J1, 9, O_P, O_BA - O_V, dp_dba, -1.0);
        set_blk(J1, 9, O_P, O_BG - O_V, dp_dbg, -1.0);
        q4 q3; q_inv(Qj, tq); q_mul(tq, Qi, q3); q_mul(q3, f->delta_q, q3);
        q_left_br(q3, M); m3_mul(M, dq_dbg, N);
        set_blk(J1, 9, O_R, O_BG - O_V, N, -1.0);
        set_blk(J1, 9, O_V, O_V - O_V, RiT, -1.0);
        set_blk(J1, 9, O_V, O_BA - O_V, dv_dba, -1.0);
        set_blk(J1, 9, O_V, O_BG - O_V, dv_dbg, -1.0);
        for (int k = 0; k < 3; k++) { J1[(O_BA + k) * 9 + O_BA - O_V + k] = -1.0; J1[(O_BG + k) * 9 + O_BG - O_V + k] = -1.0; }
        left_mul_sqrt(sqrt_info, 15, J1, 9);
    }
    if (J2) {
        memset(J2, 0, sizeof(double) * 15 * 7);
        m3 Ri_inv; q_to_R(Qi_inv, Ri_inv);
        set_blk(J2, 7, O_P, O_P, Ri_inv, 1.0);
        q4 q3; q_inv(corr_q, tq); q_mul(tq, Qi_inv, q3); q_mul(q3, Qj, q3);
        q_left_br(q3, M);
        set_blk(J2, 7, O_R, O_R, M, 1.0);
        left_mul_sqrt(sqrt_info, 15, J2, 7);
    }
    if (J3) {
        memset(J3, 0, sizeof(double) * 15 * 9);
        set_blk(J3, 9, O_V, O_V - O_V, RiT, 1.0);
        for (int k = 0; k < 3; k++) { J3[(O_BA + k) * 9 + O_BA - O_V + k] = 1.0; J3[(O_BG + k) * 9 + O_BG - O_V + k] = 1.0; }
        left_mul_sqrt(sqrt_info, 15, J3, 9);
    }
}

/* ------------------------------------------------------------------ wheel odometry factor ------- */
/* Sophus (upstream, un-vendored; the reference's CMake finds it as a system package) SO3<double>::exp / log and the
 * right Jacobians vendored in utility/sophus_utils.hpp:155-236, restated.  epsilon = 1e-10 (Sophus::Constants<double>). */
#define SOPHUS_EPS 1e-10
static void so3_exp_q(const v3 w, q4 q)     /* so3.hpp expAndTheta: quaternion (x,y,z,w) */
{
    double t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], imag, real;
    if (t2 < SOPHUS_EPS * SOPHUS_EPS) {
        double t4 = t2 * t2;
        imag = 0.5 - (1.0 / 48.0) * t2 + (1.0 / 3840.0) * t4;
        real = 1.0 - (1.0 / 8.0) * t2 + (1.0 / 384.0) * t4;
    } else {
        double t = sqrt(t2), h = 0.5 * t;
        imag = sin(h) / t; real = cos(h);
    }
    q[0] = imag * w[0]; q[1] = imag * w[1]; q[2] = imag * w[2]; q[3] = real;
}
static void so3_log_q(const q4 qin, v3 out)  /* so3.hpp logAndTheta on the normalised quaternion */
{
    q4 q; memcpy(q, qin, sizeof(q4)); q_normalize(q);
    double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2], w = q[3], f;
    if (n2 < SOPHUS_EPS * SOPHUS_EPS) {
        f = 2.0 / w - (2.0 / 3.0) * n2 / (w * w * w);
    } else {
        double n = sqrt(n2);
        if (fabs(w) < SOPHUS_EPS) f = (w > 0 ? M_PI : -M_PI) / n;
        else f = 2.0 * atan(n / w) / n;
    }
    out[0] = f * q[0]; out[1] = f * q[1]; out[2] = f * q[2];
}
static void so3_exp_R(const v3 w, m3 R) { q4 q; so3_exp_q(w, q); q_to_R(q, R); }
static void so3_Jr(const v3 phi, m3 J)       /* sophus_utils.hpp:155-184 */
{
    double n2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
    m3 h, h2; skew(phi, h); m3_mul(h, h, h2);
    double a, b;
    if (n2 > SOPHUS_EPS) { double n = sqrt(n2); a = (1.0 - cos(n)) / n2; b = (n - sin(n)) / (n2 * n); }
    else { a = 0.5; b = 1.0 / 6.0; }
    for (int k = 0; k < 9; k++) J[k] = ((k % 4 == 0) ? 1.0 : 0.0) - a * h[k] + b * h2[k];
}
static void so3_Jr_inv(const v3 phi, m3 J)   /* sophus_utils.hpp:195-236 */
{
    double n2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
    m3 h, h2; skew(phi, h); m3_mul(h, h, h2);
    double b;
    if (n2 > SOPHUS_EPS) {
        double n = sqrt(n2);
        if (n < M_PI - 1e-5) b = 1.0 / n2 - (1.0 + cos(n)) / (2.0 * n * sin(n));   /* epsilonSqrt = 1e-5 */
        else b = 1.0 / (M_PI * M_PI);
    } else b = 1.0 / 12.0;
    for (int k = 0; k < 9; k++) J[k] = ((k % 4 == 0) ? 1.0 : 0.0) + 0.5 * h[k] + b * h2[k];
}

/* WheelFactor::Evaluate (wheel_factor.h:28-247) + WheelIntegrationBase::evaluate (wheel_integration_base.h:179-219).
 * Residual rows: 0-2 position, 3-5 rotation.  Jacobians row-major in the GLOBAL block sizes (6x7 for poses with a zero
 * last column, 6x1 for sx, sy, sw, td), already multiplied by sqrt_info = LLT(cov^-1).L^T (recomputed per call as in
 * the reference).  The formulas -- including exp(forward_compensate_v) in the sx/sy blocks -- are the reference's. */
GFO int gfo_eval_wheel(const gf_ba_wheel_factor* f, const double* pose_i, const double* pose_j, const double* exw,
                       double sx, double sy, double sw, double td, double* res,
                       double* J0, double* J1, double* J2, double* Jsx, double* Jsy, double* Jsw, double* Jtd)
{
    const double* Pi = pose_i; const double* Qi = pose_i + 3; const double* Pj = pose_j; const double* Qj = pose_j + 3;
    const double* tio = exw; const double* qio = exw + 3;
    v3 dp_dsx, dp_dsy, dp_dsw, dq_dsw;
    for (int k = 0; k < 3; k++) { dp_dsx[k] = f->jacobian[k * 3 + 0]; dp_dsy[k] = f->jacobian[k * 3 + 1]; dp_dsw[k] = f->jacobian[k * 3 + 2]; dq_dsw[k] = f->jacobian[(3 + k) * 3 + 2]; }
    const double dsx = sx - f->linearized_sx, dsy = sy - f->linearized_sy, dsw = sw - f->linearized_sw, dtd = td - f->linearized_td;
    const double sv[3] = {sx, sy, 1.0};
    m3 Ri, Rj, rio; q_to_R(Qi, Ri); q_to_R(Qj, Rj); q_to_R(qio, rio);
    v3 cp; for (int k = 0; k < 3; k++) cp[k] = f->delta_p[k] + dp_dsx[k] * dsx + dp_dsy[k] * dsy + dp_dsw[k] * dsw;
    q4 dq0, e, cq; memcpy(dq0, f->delta_q, sizeof(q4)); q_normalize(dq0);
    v3 t3; for (int k = 0; k < 3; k++) t3[k] = dq_dsw[k] * dsw;
    so3_exp_q(t3, e); q_mul(dq0, e, cq); q_normalize(cq);
    m3 Rcq; q_to_R(cq, Rcq);
    v3 fcw, fcv, bcv, bcw, nbcw;
    for (int k = 0; k < 3; k++) { fcw[k] = sw * f->linearized_gyr[k] * dtd; fcv[k] = sv[k] * f->linearized_vel[k] * dtd; bcv[k] = sv[k] * f->vel_1[k] * dtd; bcw[k] = sw * f->gyr_1[k] * dtd; nbcw[k] = -bcw[k]; }
    q4 E1, E2, qt, dqt; so3_exp_q(fcw, E1); so3_exp_q(nbcw, E2);
    q_mul(E1, cq, qt); q_mul(qt, E2, dqt); q_normalize(dqt);
    m3 RE1; q_to_R(E1, RE1);
    v3 u, inner, dpt; m3_v(Rcq, bcv, u);
    for (int k = 0; k < 3; k++) inner[k] = fcv[k] + cp[k] - u[k];
    m3_v(RE1, inner, dpt);
    /* (Ri rio)^T (Rj tio + Pj - Ri tio - Pi) */
    m3 Rio, RioT; m3_mul(Ri, rio, Rio); m3_T(Rio, RioT);
    v3 a1, a2, dw, dpos; m3_v(Rj, tio, a1); m3_v(Ri, tio, a2);
    for (int k = 0; k < 3; k++) dw[k] = a1[k] + Pj[k] - a2[k] - Pi[k];
    m3_v(RioT, dw, dpos);
    double raw[6];
    for (int k = 0; k < 3; k++) raw[k] = dpos[k] - dpt[k];
    q4 qiqio, inv1, inv2, qjqio, t1, t2; q_mul(Qi, qio, qiqio); q_inv(qiqio, inv1); q_inv(dqt, inv2); q_mul(Qj, qio, qjqio);
    q_mul(inv2, inv1, t1); q_mul(t1, qjqio, t2);
    v3 rq; so3_log_q(t2, rq);
    for (int k = 0; k < 3; k++) raw[3 + k] = rq[k];
    double U[36];
    if (gfo_sqrt_info(f->covariance, 6, U)) return -1;
    for (int i = 0; i < 6; i++) { double v = 0; for (int k = 0; k < 6; k++) v += U[i * 6 + k] * raw[k]; res[i] = v; }
    if (!J0 && !J1 && !J2 && !Jsx && !Jsy && !Jsw && !Jtd) return 0;
    m3 Jri; so3_Jr_inv(rq, Jri);
    v3 drdsw; for (int k = 0; k < 3; k++) drdsw[k] = dq_dsw[k] * dsw;
    m3 Jr_drdsw; so3_Jr(drdsw, Jr_drdsw);
    m3 S, A, B, C, RiT, rioT; m3_T(Ri, RiT); m3_T(rio, rioT);
    if (J0) {
        memset(J0, 0, sizeof(double) * 42);
        set_blk(J0, 7, 0, 0, RioT, -1.0);
        skew(tio, S); m3_mul(Ri, S, A); m3_mul(RioT, A, B);                 /* (Ri rio)^T (Ri [tio]x) */
        v3 w1; m3_v(RiT, dw, w1); skew(w1, S); m3_mul(rioT, S, C);          /* rio^T [Ri^T dw]x */
        for (int k = 0; k < 9; k++) B[k] += C[k];
        set_blk(J0, 7, 0, 3, B, 1.0);
        q4 qa, qb; q_inv(qjqio, qa); q_mul(qa, Qi, qb); q_to_R(qb, A); m3_mul(Jri, A, B);
        set_blk(J0, 7, 3, 3, B, -1.0);
        left_mul_sqrt(U, 6, J0, 7);
    }
    if (J1) {
        memset(J1, 0, sizeof(double) * 42);
        set_blk(J1, 7, 0, 0, RioT, 1.0);
        skew(tio, S); m3_mul(RioT, Rj, A); m3_mul(A, S, B);
        set_blk(J1, 7, 0, 3, B, -1.0);
        m3_mul(Jri, rioT, B);
        set_blk(J1, 7, 3, 3, B, 1.0);
        left_mul_sqrt(U, 6, J1, 7);
    }
    if (J2) {
        memset(J2, 0, sizeof(double) * 42);
        for (int k = 0; k < 9; k++) A[k] = Rj[k] - Ri[k];
        m3_mul(RioT, A, B);
        set_blk(J2, 7, 0, 0, B, 1.0);
        skew(dpos, S);
        set_blk(J2, 7, 0, 3, S, 1.0);
        q4 qa, qb, qc; q_inv(qjqio, qa); q_mul(qa, Qi, qb); q_mul(qb, qio, qc); q_to_R(qc, A);
        for (int k = 0; k < 9; k++) A[k] = ((k % 4 == 0) ? 1.0 : 0.0) - A[k];
        m3_mul(Jri, A, B);
        set_blk(J2, 7, 3, 3, B, 1.0);
        left_mul_sqrt(U, 6, J2, 7);
    }
    m3 Jrtd, Jrmtd, Rfcv, Rfcw, Rnr, Rbcw, RcqT;
    v3 nfcw, nrq; for (int k = 0; k < 3; k++) { nfcw[k] = -fcw[k]; nrq[k] = -rq[k]; }
    so3_Jr(fcw, Jrtd); so3_Jr(nfcw, Jrmtd);
    so3_exp_R(fcv, Rfcv); so3_exp_R(fcw, Rfcw); so3_exp_R(nrq, Rnr); so3_exp_R(bcw, Rbcw); m3_T(Rcq, RcqT);
    for (int axis = 0; axis < 2; axis++) {
        double* Jo = axis == 0 ? Jsx : Jsy;
        if (!Jo) continue;
        const double* dpds = axis == 0 ? dp_dsx : dp_dsy;
        v3 e1 = {0, 0, 0}, e2 = {0, 0, 0}, w1, w2, w3;
        e1[axis] = f->linearized_vel[axis] * dtd;            /* I_axis * linearized_vel * dtd */
        e2[axis] = f->vel_1[axis] * dtd;                     /* I_axis * vel_1 * dtd */
        m3_v(Rcq, e2, w1);
        for (int k = 0; k < 3; k++) w2[k] = e1[k] + dpds[k] - w1[k];
        m3_v(Rfcv, w2, w3);
        for (int k = 0; k < 3; k++) { Jo[k] = -w3[k]; Jo[3 + k] = 0.0; }
        left_mul_sqrt(U, 6, Jo, 1);
    }
    v3 common;   /* forward_compensate_v + corrected_delta_p - corrected_delta_q * back_compensate_v */
    for (int k = 0; k < 3; k++) common[k] = inner[k];
    if (Jsw) {
        v3 w1, w2, w3, w4, w5, lg;
        m3_v(Jr_drdsw, dq_dsw, w1); skew(w1, S);
        v3 svv1; for (int k = 0; k < 3; k++) svv1[k] = sv[k] * f->vel_1[k] * dtd;
        m3_v(S, svv1, w2); m3_v(Rcq, w2, w3);                                /* Rcq [Jr dq_dsw]x sv vel_1 dtd */
        for (int k = 0; k < 3; k++) lg[k] = f->linearized_gyr[k] * dtd;
        m3_v(Jrtd, lg, w4); skew(w4, S); m3_v(S, common, w5);                /* [Jrtd gyr dtd]x common */
        v3 tot; for (int k = 0; k < 3; k++) tot[k] = dp_dsw[k] - w3[k] + w5[k];
        v3 outp; m3_v(Rfcw, tot, outp);
        v3 r1, r2, r3, r4, r5;
        m3_v(RcqT, w4, r1);                                                   /* Rcq^T Jrtd gyr dtd */
        for (int k = 0; k < 3; k++) r2[k] = r1[k] + w1[k];
        m3_v(Rbcw, r2, r3); m3_v(Rnr, r3, r4); m3_v(Jri, r4, r5);
        for (int k = 0; k < 3; k++) { Jsw[k] = -outp[k]; Jsw[3 + k] = -r5[k]; }
        left_mul_sqrt(U, 6, Jsw, 1);
    }
    if (Jtd) {
        v3 w1, w2, w3, w4, w5, svl, svv, swg;
        for (int k = 0; k < 3; k++) { svl[k] = sv[k] * f->linearized_vel[k]; svv[k] = sv[k] * f->vel_1[k]; swg[k] = sw * f->linearized_gyr[k]; }
        m3_v(Rcq, svv, w1);
        m3_v(Jrtd, swg, w2); skew(w2, S); m3_v(S, common, w3);
        for (int k = 0; k < 3; k++) w4[k] = svl[k] - w1[k] + w3[k];
        m3_v(Rfcw, w4, w5);
        v3 r1, r2, r3, r4, r5, swg1;
        for (int k = 0; k < 3; k++) swg1[k] = sw * f->gyr_1[k];
        m3_v(RcqT, w2, r1); m3_v(Rbcw, r1, r2);
        m3_v(Jrmtd, swg1, r3);
        for (int k = 0; k < 3; k++) r4[k] = r2[k] - r3[k];
        m3_v(Rnr, r4, r5); v3 r6; m3_v(Jri, r5, r6);
        for (int k = 0; k < 3; k++) { Jtd[k] = -w5[k]; Jtd[3 + k] = -r6[k]; }
        left_mul_sqrt(U, 6, Jtd, 1);
    }
    return 0;
}

/* PlaneFactor::Evaluate (reference factor/plane_factor.h:24-118): roll/pitch of the ground-plane normal seen from the
 * odometer frame and the height of the odometer origin above the plane.  Jacobians row-major in the global block sizes
 * (3x7 pose, 3x7 wheel extrinsic, 3x4 plane rotation, 3x1 plane height), multiplied by diag(sqrt_info). */
GFO void gfo_eval_plane(const double* pose_i, const double* exw, const double* qpw_in, double zpw, const double* sinfo,
                        double* res, double* J0, double* J1, double* J2, double* J3)
{
    const double* Pi = pose_i; const double* Qi = pose_i + 3; const double* tio = exw; const double* qio = exw + 3;
    q4 qpw = {qpw_in[0], qpw_in[1], qpw_in[2], qpw_in[3]};
    m3 Ri, rio, Rpw, RiT, rioT, RpwT; q_to_R(Qi, Ri); q_to_R(qio, rio); q_to_R(qpw, Rpw); m3_T(Ri, RiT); m3_T(rio, rioT); m3_T(Rpw, RpwT);
    const v3 e3 = {0, 0, 1};
    v3 a, b, c, t, u;
    m3_v(RpwT, e3, a); m3_v(RiT, a, b); m3_v(rioT, b, c);      /* rio^T Ri^T Rpw^T e3 */
    m3_v(Ri, tio, t); for (int k = 0; k < 3; k++) t[k] += Pi[k]; /* Pi + Qi tio */
    m3_v(Rpw, t, u);
    res[0] = sinfo[0] * c[0]; res[1] = sinfo[1] * c[1]; res[2] = sinfo[2] * (zpw + u[2]);
    m3 S, A, B;
    if (J0) {
        memset(J0, 0, sizeof(double) * 21);
        skew(b, S); m3_mul(rioT, S, A);                           /* rio^T [Qi^-1 qpw^-1 e3]x : rows 0,1 -> rotation block */
        for (int r = 0; r < 2; r++) for (int k = 0; k < 3; k++) J0[r * 7 + 3 + k] = sinfo[r] * A[r * 3 + k];
        for (int k = 0; k < 3; k++) J0[2 * 7 + k] = sinfo[2] * Rpw[2 * 3 + k];                 /* e3^T Rpw */
        skew(tio, S); m3_mul(Rpw, Ri, A); m3_mul(A, S, B);
        for (int k = 0; k < 3; k++) J0[2 * 7 + 3 + k] = -sinfo[2] * B[2 * 3 + k];               /* -e3^T Rpw Ri [tio]x */
    }
    if (J1) {
        memset(J1, 0, sizeof(double) * 21);
        skew(c, S);
        for (int r = 0; r < 2; r++) for (int k = 0; k < 3; k++) J1[r * 7 + 3 + k] = sinfo[r] * S[r * 3 + k];
        m3_mul(Rpw, Ri, A);
        for (int k = 0; k < 3; k++) J1[2 * 7 + k] = sinfo[2] * A[2 * 3 + k];
    }
    if (J2) {
        memset(J2, 0, sizeof(double) * 12);
        skew(a, S); m3_mul(RiT, S, A); m3_mul(rioT, A, B);        /* rio^T Ri^T [qpw^-1 e3]x */
        for (int r = 0; r < 2; r++) for (int k = 0; k < 3; k++) J2[r * 4 + k] = sinfo[r] * B[r * 3 + k];
        skew(t, S); m3_mul(Rpw, S, A);
        for (int k = 0; k < 3; k++) J2[2 * 4 + k] = -sinfo[2] * A[2 * 3 + k];
    }
    if (J3) { J3[0] = 0; J3[1] = 0; J3[2] = sinfo[2]; }
}

/* ------------------------------------------------------------------ program layout -------------- */
typedef struct {
    int F, nfeat;
    int col_pose[GF_BA_MAX_FRAMES], col_sb[GF_BA_MAX_FRAMES], col_ex, col_td;
    int col_exw, col_ix[3], col_tdw;   /* wheel extrinsic, sx sy sw, wheel time offset (only with wheel factors) */
    int col_pr, col_pz, row_plane;     /* plane rotation (local 3) and height (USE_PLANE) */
    int* col_feat;   /* -1: constant or unused */
    int n_cam, n_lm, n_cols;
    int row_prior, row_imu, row_wheel, row_vis, n_rows;
    int use_sb;
} layout_t;

typedef struct {
    double pose[GF_BA_MAX_FRAMES][7], sb[GF_BA_MAX_FRAMES][9], ex[7], td;
    double exw[7], ix[3], tdw;
    double pr[4], pz;
    double* feat;
} state_t;

static void state_load(const gf_ba_problem* p, state_t* s)
{
    memcpy(s->pose, p->para_pose, sizeof(double) * 7 * p->n_frames);
    if (p->para_speed_bias) memcpy(s->sb, p->para_speed_bias, sizeof(double) * 9 * p->n_frames);
    memcpy(s->ex, p->para_ex_pose, sizeof(double) * 7);
    s->td = p->para_td[0];
    memset(s->exw, 0, sizeof(s->exw)); s->exw[6] = 1.0; s->ix[0] = s->ix[1] = s->ix[2] = 1.0; s->tdw = 0.0;
    if (p->n_wheel > 0) { memcpy(s->exw, p->para_ex_wheel, sizeof(double) * 7); memcpy(s->ix, p->para_ix_wheel, sizeof(double) * 3); s->tdw = p->para_td_wheel[0]; }
    s->pr[0] = s->pr[1] = s->pr[2] = 0; s->pr[3] = 1; s->pz = 0;
    if (p->n_plane > 0) { memcpy(s->exw, p->para_ex_wheel, sizeof(double) * 7); memcpy(s->pr, p->para_plane_R, sizeof(double) * 4); s->pz = p->para_plane_Z[0]; }
    s->feat = (double*)malloc(sizeof(double) * (p->n_features > 0 ? p->n_features : 1));
    memcpy(s->feat, p->para_feature, sizeof(double) * p->n_features);
}
static void state_copy(const gf_ba_problem* p, const state_t* a, state_t* b)
{
    double* f = b->feat;
    *b = *a;
    b->feat = f;
    memcpy(b->feat, a->feat, sizeof(double) * p->n_features);
}
static void state_store(const gf_ba_problem* p, const state_t* s)
{
    memcpy(p->para_pose, s->pose, sizeof(double) * 7 * p->n_frames);
    if (p->para_speed_bias) memcpy(p->para_speed_bias, s->sb, sizeof(double) * 9 * p->n_frames);
    memcpy(p->para_ex_pose, s->ex, sizeof(double) * 7);
    p->para_td[0] = s->td;
    if (p->n_wheel > 0) { memcpy(p->para_ex_wheel, s->exw, sizeof(double) * 7); memcpy(p->para_ix_wheel, s->ix, sizeof(double) * 3); p->para_td_wheel[0] = s->tdw; }
    if (p->n_plane > 0) { memcpy(p->para_ex_wheel, s->exw, sizeof(double) * 7); memcpy(p->para_plane_R, s->pr, sizeof(double) * 4); p->para_plane_Z[0] = s->pz; }
    memcpy(p->para_feature, s->feat, sizeof(double) * p->n_features);
}

/* A residual block may not list one parameter block twice (ceres::Problem refuses it; the reference builds the visual factor
 * only for imu_i != imu_j): such a window is an argument error. */
static int same_frame_visual(const gf_ba_problem* p)
{
    for (int v = 0; v < p->n_visual; v++) if (p->visual[v].imu_i == p->visual[v].imu_j) return 1;
    return 0;
}

static void make_layout(const gf_ba_problem* p, layout_t* L)
{
    int c = 0;
    L->F = p->n_frames; L->nfeat = p->n_features;
    L->use_sb = (p->para_speed_bias != NULL) && !p->pose0_const;   /* USE_IMU */
    for (int f = 0; f < L->F; f++) {
        int is_const = p->frames_const || (f == 0 && p->pose0_const);
        L->col_pose[f] = is_const ? -1 : c; if (!is_const) c += 6;
    }
    for (int f = 0; f < L->F; f++) {
        int is_const = p->frames_const || !L->use_sb;
        L->col_sb[f] = is_const ? -1 : c; if (!is_const) c += 9;
    }
    L->col_ex = p->ex_pose_const ? -1 : c; if (!p->ex_pose_const) c += 6;
    L->col_td = p->td_const ? -1 : c; if (!p->td_const) c += 1;
    L->col_exw = -1; L->col_ix[0] = L->col_ix[1] = L->col_ix[2] = -1; L->col_tdw = -1;
    if (p->n_wheel > 0 || p->n_plane > 0) {      /* estimator.cpp:3008-3056: the wheel blocks only exist with USE_WHEEL (PlaneFactor reads the extrinsic too) */
        if (!p->ex_wheel_const) { L->col_exw = c; c += 6; }
        if (p->n_wheel > 0 && !p->ix_wheel_const) for (int k = 0; k < 3; k++) L->col_ix[k] = c++;
        if (p->n_wheel > 0 && !p->td_wheel_const) L->col_tdw = c++;
    }
    L->col_pr = L->col_pz = -1;
    if (p->n_plane > 0 && !p->plane_const) { L->col_pr = c; c += 3; L->col_pz = c++; }
    L->n_cam = c;
    L->col_feat = (int*)malloc(sizeof(int) * (L->nfeat > 0 ? L->nfeat : 1));
    for (int k = 0; k < L->nfeat; k++) L->col_feat[k] = -1;
    for (int v = 0; v < p->n_visual; v++) {
        int k = p->visual[v].feature;
        if (!p->feature_const[k] && L->col_feat[k] < 0) L->col_feat[k] = -2;
    }
    for (int k = 0; k < L->nfeat; k++) if (L->col_feat[k] == -2) L->col_feat[k] = c++;
    L->n_lm = c - L->n_cam; L->n_cols = c;
    int r = 0;
    L->row_prior = r; r += (p->prior ? p->prior->n : 0);
    L->row_imu = r; r += 15 * p->n_imu;
    L->row_wheel = r; r += 6 * p->n_wheel;
    L->row_plane = r; r += 3 * p->n_plane;
    L->row_vis = r; r += 2 * p->n_visual;
    L->n_rows = r;
}

static const double* prior_block_ptr(const state_t* s, int kind, int index)
{
    switch (kind) {
    case GF_BA_BLOCK_POSE: return s->pose[index];
    case GF_BA_BLOCK_SPEEDBIAS: return s->sb[index];
    case GF_BA_BLOCK_EX_POSE: return s->ex;
    case GF_BA_BLOCK_TD: return &s->td;
    case GF_BA_BLOCK_EX_WHEEL: return s->exw;
    case GF_BA_BLOCK_SX: return &s->ix[0];
    case GF_BA_BLOCK_SY: return &s->ix[1];
    case GF_BA_BLOCK_SW: return &s->ix[2];
    case GF_BA_BLOCK_TD_WHEEL: return &s->tdw;
    case GF_BA_BLOCK_PLANE_R: return s->pr;
    case GF_BA_BLOCK_PLANE_Z: return &s->pz;
    default: return NULL;
    }
}
static int block_global_size(int kind)
{
    switch (kind) {
    case GF_BA_BLOCK_POSE: case GF_BA_BLOCK_EX_POSE: case GF_BA_BLOCK_EX_WHEEL: return 7;
    case GF_BA_BLOCK_SPEEDBIAS: return 9;
    case GF_BA_BLOCK_PLANE_R: return 4;
    default: return 1;
    }
}
static int block_col(const layout_t* L, int kind, int index)
{
    switch (kind) {
    case GF_BA_BLOCK_POSE: return L->col_pose[index];
    case GF_BA_BLOCK_SPEEDBIAS: return L->col_sb[index];
    case GF_BA_BLOCK_EX_POSE: return L->col_ex;
    case GF_BA_BLOCK_TD: return L->col_td;
    case GF_BA_BLOCK_EX_WHEEL: return L->col_exw;
    case GF_BA_BLOCK_SX: return L->col_ix[0];
    case GF_BA_BLOCK_SY: return L->col_ix[1];
    case GF_BA_BLOCK_SW: return L->col_ix[2];
    case GF_BA_BLOCK_TD_WHEEL: return L->col_tdw;
    case GF_BA_BLOCK_PLANE_R: return L->col_pr;
    case GF_BA_BLOCK_PLANE_Z: return L->col_pz;
    default: return -1;
    }
}

/* MarginalizationFactor::Evaluate residual part (marginalization_factor.cpp:344-376) */
static void prior_dx(const gf_ba_prior* pr, const state_t* s, double* dx)
{
    const double* x0 = pr->x0;
    for (int b = 0; b < pr->n_blocks; b++) {
        int size = block_global_size(pr->block_kind[b]), idx = pr->block_idx[b];
        const double* x = prior_block_ptr(s, pr->block_kind[b], pr->block_index[b]);
        if (size != 7) for (int k = 0; k < size; k++) dx[idx + k] = x[k] - x0[k];
        else {
            for (int k = 0; k < 3; k++) dx[idx + k] = x[k] - x0[k];
            q4 qi, dq; q_inv(x0 + 3, qi); q_mul(qi, x + 3, dq);
            double sgn = (dq[3] >= 0) ? 1.0 : -1.0;    /* if (!(w >= 0)) flip */
            for (int k = 0; k < 3; k++) dx[idx + 3 + k] = 2.0 * sgn * dq[k];
        }
        x0 += size;
    }
}

/* Evaluate all residual blocks: cost = 1/2 sum rho(|r|^2); r, J already loss-corrected (Ceres Corrector with
 * rho'' <= 0, restated in-tree at marginalization_factor.cpp:46-77) and projected on the local parameterisation
 * (first 6 of 7 columns for poses).  J (n_rows x n_cols, row-major) may be NULL. */
static double evaluate(const gf_ba_problem* p, const layout_t* L, const state_t* s, const double* imu_sqrt_info, double* r, double* J)
{
    double cost = 0;
    const int nc = L->n_cols;
    if (J) memset(J, 0, sizeof(double) * (size_t)L->n_rows * nc);
    if (p->prior && p->prior->n > 0) {
        const gf_ba_prior* pr = p->prior;
        int n = pr->n;
        double* dx = (double*)malloc(sizeof(double) * n);
        prior_dx(pr, s, dx);
        for (int i = 0; i < n; i++) {
            double v = pr->linearized_residuals[i];
            for (int k = 0; k < n; k++) v += pr->linearized_jacobians[(size_t)i * n + k] * dx[k];
            r[L->row_prior + i] = v;
            cost += 0.5 * v * v;
        }
        if (J)
            for (int b = 0; b < pr->n_blocks; b++) {
                int col = block_col(L, pr->block_kind[b], pr->block_index[b]);
                if (col < 0) continue;
                int ls = block_global_size(pr->block_kind[b]); if (ls == 7) ls = 6; if (pr->block_kind[b] == GF_BA_BLOCK_PLANE_R) ls = 3;   /* 4 prior columns, the local parameterisation keeps 3 */
                for (int i = 0; i < n; i++) for (int k = 0; k < ls; k++) J[(size_t)(L->row_prior + i) * nc + col + k] = pr->linearized_jacobians[(size_t)i * n + pr->block_idx[b] + k];
            }
        free(dx);
    }
    for (int m = 0; m < p->n_imu; m++) {
        const gf_ba_imu_factor* f = &p->imu[m];
        double res[15], J0[105], J1[135], J2[105], J3[135];
        gfo_eval_imu(f, imu_sqrt_info + 225 * m, p->gravity, s->pose[f->i], s->sb[f->i], s->pose[f->j], s->sb[f->j], res, J ? J0 : NULL, J ? J1 : NULL, J ? J2 : NULL, J ? J3 : NULL);
        int row = L->row_imu + 15 * m;
        for (int i = 0; i < 15; i++) { r[row + i] = res[i]; cost += 0.5 * res[i] * res[i]; }
        if (J) {
            int c0 = L->col_pose[f->i], c1 = L->col_sb[f->i], c2 = L->col_pose[f->j], c3 = L->col_sb[f->j];
            for (int i = 0; i < 15; i++) {
                if (c0 >= 0) for (int k = 0; k < 6; k++) J[(size_t)(row + i) * nc + c0 + k] = J0[i * 7 + k];
                if (c1 >= 0) for (int k = 0; k < 9; k++) J[(size_t)(row + i) * nc + c1 + k] = J1[i * 9 + k];
                if (c2 >= 0) for (int k = 0; k < 6; k++) J[(size_t)(row + i) * nc + c2 + k] = J2[i * 7 + k];
                if (c3 >= 0) for (int k = 0; k < 9; k++) J[(size_t)(row + i) * nc + c3 + k] = J3[i * 9 + k];
            }
        }
    }
    for (int m = 0; m < p->n_wheel; m++) {
        const gf_ba_wheel_factor* f = &p->wheel[m];
        double res[6], J0[42], J1[42], J2[42], Jsx[6], Jsy[6], Jsw[6], Jtw[6];
        gfo_eval_wheel(f, s->pose[f->i], s->pose[f->j], s->exw, s->ix[0], s->ix[1], s->ix[2], s->tdw, res,
                       J ? J0 : NULL, J ? J1 : NULL, J ? J2 : NULL, J ? Jsx : NULL, J ? Jsy : NULL, J ? Jsw : NULL, J ? Jtw : NULL);
        int row = L->row_wheel + 6 * m;
        for (int i = 0; i < 6; i++) { r[row + i] = res[i]; cost += 0.5 * res[i] * res[i]; }
        if (J) {
            int c0 = L->col_pose[f->i], c1 = L->col_pose[f->j];
            for (int i = 0; i < 6; i++) {
                double* Jr = J + (size_t)(row + i) * nc;
                if (c0 >= 0) for (int k = 0; k < 6; k++) Jr[c0 + k] = J0[i * 7 + k];
                if (c1 >= 0) for (int k = 0; k < 6; k++) Jr[c1 + k] = J1[i * 7 + k];
                if (L->col_exw >= 0) for (int k = 0; k < 6; k++) Jr[L->col_exw + k] = J2[i * 7 + k];
                if (L->col_ix[0] >= 0) { Jr[L->col_ix[0]] = Jsx[i]; Jr[L->col_ix[1]] = Jsy[i]; Jr[L->col_ix[2]] = Jsw[i]; }
                if (L->col_tdw >= 0) Jr[L->col_tdw] = Jtw[i];
            }
        }
    }
    for (int m = 0; m < p->n_plane; m++) {
        const int fi = p->plane_frames[m];
        double res[3], J0[21], J1[21], J2[12], J3[3];
        gfo_eval_plane(s->pose[fi], s->exw, s->pr, s->pz, p->plane_sqrt_info, res, J ? J0 : NULL, J ? J1 : NULL, J ? J2 : NULL, J ? J3 : NULL);
        int row = L->row_plane + 3 * m;
        for (int i = 0; i < 3; i++) { r[row + i] = res[i]; cost += 0.5 * res[i] * res[i]; }
        if (J)
            for (int i = 0; i < 3; i++) {
                double* Jr = J + (size_t)(row + i) * nc;
                if (L->col_pose[fi] >= 0) for (int k = 0; k < 6; k++) Jr[L->col_pose[fi] + k] = J0[i * 7 + k];
                if (L->col_exw >= 0) for (int k = 0; k < 6; k++) Jr[L->col_exw + k] = J1[i * 7 + k];
                if (L->col_pr >= 0) { for (int k = 0; k < 3; k++) Jr[L->col_pr + k] = J2[i * 4 + k]; Jr[L->col_pz] = J3[i]; }
            }
    }
    for (int v = 0; v < p->n_visual; v++) {
        const gf_ba_visual_factor* f = &p->visual[v];
        double res[2], Ji[14], Jj[14], Jex[14], Jf[2], Jtd[2];
        gfo_eval_visual(f, p->visual_sqrt_info, s->pose[f->imu_i], s->pose[f->imu_j], s->ex, s->feat[f->feature], s->td, res,
                        J ? Ji : NULL, J ? Jj : NULL, J ? Jex : NULL, J ? Jf : NULL, J ? Jtd : NULL);
        /* HuberLoss(1.0): rho(s) = s (s <= 1) | 2 sqrt(s) - 1 ; rho' = 1 | 1/sqrt(s) ; rho'' <= 0 -> scale by sqrt(rho') */
        double sq = res[0] * res[0] + res[1] * res[1], rho0, rho1;
        if (sq > 1.0) { double rr = sqrt(sq); rho0 = 2.0 * rr - 1.0; rho1 = 1.0 / rr; if (rho1 < 2.2250738585072014e-308) rho1 = 2.2250738585072014e-308; }
        else { rho0 = sq; rho1 = 1.0; }
        cost += 0.5 * rho0;
        double sc = sqrt(rho1);
        int row = L->row_vis + 2 * v;
        r[row] = sc * res[0]; r[row + 1] = sc * res[1];
        if (J) {
            int ci = L->col_pose[f->imu_i], cj = L->col_pose[f->imu_j], cf = L->col_feat[f->feature];
            for (int i = 0; i < 2; i++) {
                double* Jr = J + (size_t)(row + i) * nc;
                if (ci >= 0) for (int k = 0; k < 6; k++) Jr[ci + k] += sc * Ji[i * 7 + k];
                if (cj >= 0) for (int k = 0; k < 6; k++) Jr[cj + k] += sc * Jj[i * 7 + k];
                if (L->col_ex >= 0) for (int k = 0; k < 6; k++) Jr[L->col_ex + k] = sc * Jex[i * 7 + k];
                if (cf >= 0) Jr[cf] = sc * Jf[i];
                if (L->col_td >= 0) Jr[L->col_td] = sc * Jtd[i];
            }
        }
    }
    return cost;
}

/* Block-sparse linearisation: H = J^T J (n x n, unscaled), g = J^T r, cost, without materialising J.  This is
 * what a production CPU solver does (Ceres' block-sparse Jacobian + Schur eliminator); the dense evaluate() above is
 * kept for the finite-difference tests.  Hp = J0^T J0 of the prior mapped to the layout is passed in (constant). */
static void add_blocks(double* H, double* g, int n, int nres, const double* res, int nb, const int* cols, const int* sizes, const int* lds, double* const* Js)
{
    for (int a = 0; a < nb; a++) {
        if (cols[a] < 0) continue;
        for (int b = 0; b < nb; b++) {
            if (cols[b] < 0) continue;
            for (int i = 0; i < sizes[a]; i++)
                for (int j = 0; j < sizes[b]; j++) {
                    double v = 0;
                    for (int k = 0; k < nres; k++) v += Js[a][k * lds[a] + i] * Js[b][k * lds[b] + j];
                    H[(size_t)(cols[a] + i) * n + cols[b] + j] += v;
                }
        }
        for (int i = 0; i < sizes[a]; i++) { double v = 0; for (int k = 0; k < nres; k++) v += Js[a][k * lds[a] + i] * res[k]; g[cols[a] + i] += v; }
    }
}
static double linearize_blocks(const gf_ba_problem* p, const layout_t* L, const state_t* s, const double* imu_sqrt_info, const double* Hp, double* H, double* g)
{
    const int n = L->n_cols;
    double cost = 0;
    memcpy(H, Hp, sizeof(double) * (size_t)n * n);
    memset(g, 0, sizeof(double) * n);
    if (p->prior && p->prior->n > 0) {
        const gf_ba_prior* pr = p->prior;
        int pn = pr->n;
        double* dx = (double*)malloc(sizeof(double) * pn); double* r = (double*)malloc(sizeof(double) * pn);
        prior_dx(pr, s, dx);
        for (int i = 0; i < pn; i++) { double v = pr->linearized_residuals[i]; for (int k = 0; k < pn; k++) v += pr->linearized_jacobians[(size_t)i * pn + k] * dx[k]; r[i] = v; cost += 0.5 * v * v; }
        for (int b = 0; b < pr->n_blocks; b++) {
            int col = block_col(L, pr->block_kind[b], pr->block_index[b]);
            if (col < 0) continue;
            int ls = block_global_size(pr->block_kind[b]); if (ls == 7) ls = 6; if (pr->block_kind[b] == GF_BA_BLOCK_PLANE_R) ls = 3;   /* 4 prior columns, the local parameterisation keeps 3 */
            for (int k = 0; k < ls; k++) { double v = 0; for (int i = 0; i < pn; i++) v += pr->linearized_jacobians[(size_t)i * pn + pr->block_idx[b] + k] * r[i]; g[col + k] += v; }
        }
        free(dx); free(r);
    }
    for (int m = 0; m < p->n_imu; m++) {
        const gf_ba_imu_factor* f = &p->imu[m];
        double res[15], J0[105], J1[135], J2[105], J3[135];
        gfo_eval_imu(f, imu_sqrt_info + 225 * m, p->gravity, s->pose[f->i], s->sb[f->i], s->pose[f->j], s->sb[f->j], res, J0, J1, J2, J3);
        for (int i = 0; i < 15; i++) cost += 0.5 * res[i] * res[i];
        int cols[4] = {L->col_pose[f->i], L->col_sb[f->i], L->col_pose[f->j], L->col_sb[f->j]}, sizes[4] = {6, 9, 6, 9}, lds[4] = {7, 9, 7, 9};
        double* Js[4] = {J0, J1, J2, J3};
        add_blocks(H, g, n, 15, res, 4, cols, sizes, lds, Js);
    }
    for (int m = 0; m < p->n_wheel; m++) {
        const gf_ba_wheel_factor* f = &p->wheel[m];
        double res[6], J0[42], J1[42], J2[42], Jsx[6], Jsy[6], Jsw[6], Jtw[6];
        gfo_eval_wheel(f, s->pose[f->i], s->pose[f->j], s->exw, s->ix[0], s->ix[1], s->ix[2], s->tdw, res, J0, J1, J2, Jsx, Jsy, Jsw, Jtw);
        for (int i = 0; i < 6; i++) cost += 0.5 * res[i] * res[i];
        int cols[7] = {L->col_pose[f->i], L->col_pose[f->j], L->col_exw, L->col_ix[0], L->col_ix[1], L->col_ix[2], L->col_tdw};
        int sizes[7] = {6, 6, 6, 1, 1, 1, 1}, lds[7] = {7, 7, 7, 1, 1, 1, 1};
        double* Js[7] = {J0, J1, J2, Jsx, Jsy, Jsw, Jtw};
        add_blocks(H, g, n, 6, res, 7, cols, sizes, lds, Js);
    }
    for (int m = 0; m < p->n_plane; m++) {
        const int fi = p->plane_frames[m];
        double res[3], J0[21], J1[21], J2[12], J3[3];
        gfo_eval_plane(s->pose[fi], s->exw, s->pr, s->pz, p->plane_sqrt_info, res, J0, J1, J2, J3);
        for (int i = 0; i < 3; i++) cost += 0.5 * res[i] * res[i];
        int cols[4] = {L->col_pose[fi], L->col_exw, L->col_pr, L->col_pz}, sizes[4] = {6, 6, 3, 1}, lds[4] = {7, 7, 4, 1};
        double* Js[4] = {J0, J1, J2, J3};
        add_blocks(H, g, n, 3, res, 4, cols, sizes, lds, Js);
    }
    for (int v = 0; v < p->n_visual; v++) {
        const gf_ba_visual_factor* f = &p->visual[v];
        double res[2], Ji[14], Jj[14], Jex[14], Jf[2], Jtd[2];
        gfo_eval_visual(f, p->visual_sqrt_info, s->pose[f->imu_i], s->pose[f->imu_j], s->ex, s->feat[f->feature], s->td, res, Ji, Jj, Jex, Jf, Jtd);
        double sq = res[0] * res[0] + res[1] * res[1], rho0, rho1;
        if (sq > 1.0) { double rr = sqrt(sq); rho0 = 2.0 * rr - 1.0; rho1 = 1.0 / rr; if (rho1 < 2.2250738585072014e-308) rho1 = 2.2250738585072014e-308; }
        else { rho0 = sq; rho1 = 1.0; }
        cost += 0.5 * rho0;
        double sc = sqrt(rho1);
        for (int k = 0; k < 14; k++) { Ji[k] *= sc; Jj[k] *= sc; Jex[k] *= sc; }
        for (int k = 0; k < 2; k++) { Jf[k] *= sc; Jtd[k] *= sc; res[k] *= sc; }
        int cols[5] = {L->col_pose[f->imu_i], L->col_pose[f->imu_j], L->col_ex, L->col_feat[f->feature], L->col_td}, sizes[5] = {6, 6, 6, 1, 1}, lds[5] = {7, 7, 7, 1, 1};
        double* Js[5] = {Ji, Jj, Jex, Jf, Jtd};
        add_blocks(H, g, n, 2, res, 5, cols, sizes, lds, Js);
    }
    return cost;
}
static double cost_only(const gf_ba_problem* p, const layout_t* L, const state_t* s, const double* imu_sqrt_info)
{
    double cost = 0;
    if (p->prior && p->prior->n > 0) {
        const gf_ba_prior* pr = p->prior;
        int pn = pr->n;
        double* dx = (double*)malloc(sizeof(double) * pn);
        prior_dx(pr, s, dx);
        for (int i = 0; i < pn; i++) { double v = pr->linearized_residuals[i]; for (int k = 0; k < pn; k++) v += pr->linearized_jacobians[(size_t)i * pn + k] * dx[k]; cost += 0.5 * v * v; }
        free(dx);
    }
    for (int m = 0; m < p->n_imu; m++) {
        const gf_ba_imu_factor* f = &p->imu[m];
        double res[15];
        gfo_eval_imu(f, imu_sqrt_info + 225 * m, p->gravity, s->pose[f->i], s->sb[f->i], s->pose[f->j], s->sb[f->j], res, NULL, NULL, NULL, NULL);
        for (int i = 0; i < 15; i++) cost += 0.5 * res[i] * res[i];
    }
    for (int m = 0; m < p->n_wheel; m++) {
        const gf_ba_wheel_factor* f = &p->wheel[m];
        double res[6];
        gfo_eval_wheel(f, s->pose[f->i], s->pose[f->j], s->exw, s->ix[0], s->ix[1], s->ix[2], s->tdw, res, NULL, NULL, NULL, NULL, NULL, NULL, NULL);
        for (int i = 0; i < 6; i++) cost += 0.5 * res[i] * res[i];
    }
    for (int m = 0; m < p->n_plane; m++) {
        double res[3];
        gfo_eval_plane(s->pose[p->plane_frames[m]], s->exw, s->pr, s->pz, p->plane_sqrt_info, res, NULL, NULL, NULL, NULL);
        for (int i = 0; i < 3; i++) cost += 0.5 * res[i] * res[i];
    }
    for (int v = 0; v < p->n_visual; v++) {
        const gf_ba_visual_factor* f = &p->visual[v];
        double res[2];
        gfo_eval_visual(f, p->visual_sqrt_info, s->pose[f->imu_i], s->pose[f->imu_j], s->ex, s->feat[f->feature], s->td, res, NULL, NULL, NULL, NULL, NULL);
        double sq = res[0] * res[0] + res[1] * res[1];
        cost += 0.5 * (sq > 1.0 ? 2.0 * sqrt(sq) - 1.0 : sq);
    }
    return cost;
}

/* Evaluator::Plus: PoseLocalParameterization::Plus (pose_local_parameterization.cpp:12-26) for 7-blocks */
static void pose_plus(const double* x, const double* d, double* out)
{
    for (int k = 0; k < 3; k++) out[k] = x[k] + d[k];
    q4 dq, q; delta_q(d + 3, dq); q_mul(x + 3, dq, q); q_normalize(q);
    memcpy(out + 3, q, sizeof(q4));
}
static void state_plus(const gf_ba_problem* p, const layout_t* L, const state_t* x, const double* delta, state_t* out)
{
    state_copy(p, x, out);
    for (int f = 0; f < L->F; f++) {
        if (L->col_pose[f] >= 0) pose_plus(x->pose[f], delta + L->col_pose[f], out->pose[f]);
        if (L->col_sb[f] >= 0) for (int k = 0; k < 9; k++) out->sb[f][k] = x->sb[f][k] + delta[L->col_sb[f] + k];
    }
    if (L->col_ex >= 0) pose_plus(x->ex, delta + L->col_ex, out->ex);
    if (L->col_td >= 0) out->td = x->td + delta[L->col_td];
    if (L->col_exw >= 0) {   /* PoseLocalParameterization, or PoseSubsetParameterization (pose_subset_parameterization.cpp:29-33):
                              * the masked components are zeroed inside Plus only, the Jacobian keeps its columns */
        double dd[6];
        for (int k = 0; k < 6; k++) dd[k] = ((p->ex_wheel_subset_mask >> k) & 1) ? 0.0 : delta[L->col_exw + k];
        pose_plus(x->exw, dd, out->exw);
    }
    for (int k = 0; k < 3; k++) if (L->col_ix[k] >= 0) out->ix[k] = x->ix[k] + delta[L->col_ix[k]];
    if (L->col_tdw >= 0) out->tdw = x->tdw + delta[L->col_tdw];
    if (L->col_pr >= 0) {     /* OrientationSubsetParameterization::Plus (orientation_subset_parameterization.cpp:21-37) */
        v3 dd; q4 dq, q;
        for (int k = 0; k < 3; k++) dd[k] = ((p->plane_r_subset_mask >> k) & 1) ? 0.0 : delta[L->col_pr + k];
        delta_q(dd, dq); q_mul(x->pr, dq, q); q_normalize(q); memcpy(out->pr, q, sizeof(q4));
        out->pz = x->pz + delta[L->col_pz];
    }
    for (int k = 0; k < L->nfeat; k++) if (L->col_feat[k] >= 0) out->feat[k] = x->feat[k] + delta[L->col_feat[k]];
}
/* ambient-space difference norms over the non-constant blocks (x_norm, step_norm, gradient_max_norm) */
static void state_diff_norms(const layout_t* L, const state_t* a, const state_t* b, double* l2, double* linf)
{
    double s2 = 0, mx = 0;
#define ACC(v) do { double d_ = (v); s2 += d_ * d_; if (fabs(d_) > mx) mx = fabs(d_); } while (0)
    for (int f = 0; f < L->F; f++) {
        if (L->col_pose[f] >= 0) for (int k = 0; k < 7; k++) ACC(a->pose[f][k] - (b ? b->pose[f][k] : 0));
        if (L->col_sb[f] >= 0) for (int k = 0; k < 9; k++) ACC(a->sb[f][k] - (b ? b->sb[f][k] : 0));
    }
    if (L->col_ex >= 0) for (int k = 0; k < 7; k++) ACC(a->ex[k] - (b ? b->ex[k] : 0));
    if (L->col_td >= 0) ACC(a->td - (b ? b->td : 0));
    if (L->col_exw >= 0) for (int k = 0; k < 7; k++) ACC(a->exw[k] - (b ? b->exw[k] : 0));
    for (int k = 0; k < 3; k++) if (L->col_ix[k] >= 0) ACC(a->ix[k] - (b ? b->ix[k] : 0));
    if (L->col_tdw >= 0) ACC(a->tdw - (b ? b->tdw : 0));
    if (L->col_pr >= 0) { for (int k = 0; k < 4; k++) ACC(a->pr[k] - (b ? b->pr[k] : 0)); ACC(a->pz - (b ? b->pz : 0)); }
    for (int k = 0; k < L->nfeat; k++) if (L->col_feat[k] >= 0) ACC(a->feat[k] - (b ? b->feat[k] : 0));
#undef ACC
    if (l2) *l2 = sqrt(s2);
    if (linf) *linf = mx;
}

/* ------------------------------------------------------------------ the solve ------------------- */
/* Solve (J^T J + D^2) y = J^T r with the landmark columns (n_cam..n_cols) eliminated first (DENSE_SCHUR). */
static int schur_solve(const layout_t* L, const double* H, const double* g, const double* D, double* y)
{
    const int nc = L->n_cam, nl = L->n_lm, n = L->n_cols;
    double* S = (double*)malloc(sizeof(double) * (nc > 0 ? nc : 1) * (nc > 0 ? nc : 1));
    double* b = (double*)malloc(sizeof(double) * (n > 0 ? n : 1));
    double* el = (double*)malloc(sizeof(double) * (nl > 0 ? nl : 1));
    for (int i = 0; i < nc; i++) { for (int j = 0; j < nc; j++) S[i * nc + j] = H[(size_t)i * n + j]; S[i * nc + i] += D[i] * D[i]; b[i] = g[i]; }
    for (int l = 0; l < nl; l++) {
        int c = nc + l;
        double hll = H[(size_t)c * n + c] + D[c] * D[c];
        if (!(hll > 0)) { free(S); free(b); free(el); return -1; }
        el[l] = 1.0 / hll;
        for (int i = 0; i < nc; i++) {
            double w = H[(size_t)i * n + c];
            if (w == 0.0) continue;
            double f = w * el[l];
            b[i] -= f * g[c];
            for (int j = 0; j < nc; j++) S[i * nc + j] -= f * H[(size_t)c * n + j];
        }
    }
    if (nc > 0) { if (chol_lower(S, nc)) { free(S); free(b); free(el); return -1; } chol_solve(S, nc, b); }
    for (int i = 0; i < nc; i++) y[i] = b[i];
    for (int l = 0; l < nl; l++) {
        int c = nc + l;
        double s = g[c];
        for (int j = 0; j < nc; j++) s -= H[(size_t)c * n + j] * y[j];
        y[c] = s * el[l];
    }
    free(S); free(b); free(el);
    for (int i = 0; i < n; i++) if (!isfinite(y[i])) return -1;
    return 0;
}

/* Test aid: override Ceres' default tolerances (function 1e-6, gradient 1e-10, parameter 1e-8) to drive the
 * same loop to the exact optimum when it is compared with an independent solver. */
static double g_func_tol = 1e-6, g_grad_tol = 1e-10, g_param_tol = 1e-8;
GFO void gfo_ba_set_tolerances(double f, double g, double x) { g_func_tol = f; g_grad_tol = g; g_param_tol = x; }

GFO int gfo_ba_solve(const gf_ba_problem* p, gf_ba_summary* sum)
{
    if (same_frame_visual(p)) return GF_ERR_INVALID_ARG;
    layout_t L; make_layout(p, &L);
    const int n = L.n_cols, m = L.n_rows;
    memset(sum, 0, sizeof(*sum));
    sum->reduced_dim = L.n_cam; sum->n_free_landmarks = L.n_lm; sum->n_residuals = m;
    double* imu_sqrt = (double*)malloc(sizeof(double) * 225 * (p->n_imu > 0 ? p->n_imu : 1));
    for (int k = 0; k < p->n_imu; k++) if (gfo_sqrt_info(p->imu[k].covariance, 15, imu_sqrt + 225 * k)) { free(imu_sqrt); free(L.col_feat); return -10; }
    state_t x, cand, tmp; state_load(p, &x); state_load(p, &cand); state_load(p, &tmp);
    double* r = (double*)malloc(sizeof(double) * (m + 1));
    double* rc = (double*)malloc(sizeof(double) * (m + 1));
    double* H = (double*)malloc(sizeof(double) * ((size_t)n * n + 1));
    double* Hp = (double*)calloc((size_t)n * n + 1, 8);      /* J0^T J0 of the prior, constant during the solve */
    if (p->prior && p->prior->n > 0) {
        const gf_ba_prior* pr = p->prior; int pn = pr->n;
        int* pc = (int*)malloc(sizeof(int) * pn);
        for (int k = 0; k < pn; k++) pc[k] = -1;
        for (int b = 0; b < pr->n_blocks; b++) { int col = block_col(&L, pr->block_kind[b], pr->block_index[b]); if (col < 0) continue;
            int ls = block_global_size(pr->block_kind[b]); if (ls == 7) ls = 6; if (pr->block_kind[b] == GF_BA_BLOCK_PLANE_R) ls = 3;   /* 4 prior columns, the local parameterisation keeps 3 */ for (int k = 0; k < ls; k++) pc[pr->block_idx[b] + k] = col + k; }
        for (int a = 0; a < pn; a++) { if (pc[a] < 0) continue; for (int b = 0; b < pn; b++) { if (pc[b] < 0) continue; double v = 0;
            for (int k = 0; k < pn; k++) v += pr->linearized_jacobians[(size_t)k * pn + a] * pr->linearized_jacobians[(size_t)k * pn + b]; Hp[(size_t)pc[a] * n + pc[b]] = v; } }
        free(pc);
    }
    double *g = (double*)calloc(n + 1, 8), *scale = (double*)calloc(n + 1, 8), *diag = (double*)calloc(n + 1, 8), *lmd = (double*)calloc(n + 1, 8);
    double *gs = (double*)calloc(n + 1, 8), *gn = (double*)calloc(n + 1, 8), *step = (double*)calloc(n + 1, 8), *delta = (double*)calloc(n + 1, 8), *tv = (double*)calloc(n + 1, 8);
    /* Ceres defaults (solver.h) + the reference's options (estimator.cpp:3305-3315; the wall-clock cap is disabled) */
    double radius = 1e4, mu = 1e-8; const double min_mu = 1e-8, max_mu = 1.0, mu_inc = 10.0;
    const double min_diag = 1e-6, max_diag = 1e32, func_tol = g_func_tol, grad_tol = g_grad_tol, param_tol = g_param_tol, min_rel_dec = 1e-3;
    int reuse = 0, termination = GF_BA_NO_CONVERGENCE, n_success = 0, invalid_streak = 0;
    double alpha = 0, dogleg_norm = 0, x_norm, grad_max;
    double x_cost;

#define LINEARIZE(first) do {                                                                                 \
        x_cost = linearize_blocks(p, &L, &x, imu_sqrt, Hp, H, g);                                              \
        if (first) for (int c = 0; c < n; c++) scale[c] = 1.0 / (1.0 + sqrt(H[(size_t)c * n + c]));            \
        /* gradient of the unscaled problem -> gradient_max_norm = |x - Plus(x, -g)|_inf */                   \
        for (int c = 0; c < n; c++) tv[c] = -g[c];                                                             \
        state_plus(p, &L, &x, tv, &tmp); state_diff_norms(&L, &x, &tmp, NULL, &grad_max);                      \
        for (int a = 0; a < n; a++) { for (int b = 0; b < n; b++) H[(size_t)a * n + b] *= scale[a] * scale[b]; g[a] *= scale[a]; } \
    } while (0)

    LINEARIZE(1);
    state_diff_norms(&L, &x, NULL, &x_norm, NULL);
    sum->initial_cost = x_cost; sum->cost[0] = x_cost; sum->radius[0] = radius;
    int it = 0;
    if (n == 0 || grad_max <= grad_tol) { termination = GF_BA_CONVERGENCE_GRADIENT; goto done; }
    while (1) {
        if (it >= p->max_num_iterations || it >= GF_BA_MAX_ITERATIONS) { termination = GF_BA_NO_CONVERGENCE; break; }
        if (radius < 1e-32) { termination = GF_BA_NO_CONVERGENCE; break; }
        it++;
        /* ---- DoglegStrategy::ComputeStep ---- */
        int solver_failed = 0;
        if (!reuse) {
            reuse = 1;
            for (int c = 0; c < n; c++) { double d = H[(size_t)c * n + c]; d = d < min_diag ? min_diag : (d > max_diag ? max_diag : d); diag[c] = sqrt(d); }
            for (int c = 0; c < n; c++) gs[c] = g[c] / diag[c];                     /* ComputeGradient */
            { double num = 0, den = 0;                                              /* ComputeCauchyPoint: |J (g/D^2)|^2 = v^T H v */
              for (int c = 0; c < n; c++) { num += gs[c] * gs[c]; tv[c] = gs[c] / diag[c]; }
              for (int a = 0; a < n; a++) { double s = 0; for (int b = 0; b < n; b++) s += H[(size_t)a * n + b] * tv[b]; den += tv[a] * s; }
              alpha = num / den; }
            solver_failed = 1;
            while (mu < max_mu) {                                                   /* ComputeGaussNewtonStep */
                for (int c = 0; c < n; c++) lmd[c] = diag[c] * sqrt(mu);
                if (schur_solve(&L, H, g, lmd, gn) == 0) { solver_failed = 0; break; }
                mu *= mu_inc;
            }
            if (!solver_failed) for (int c = 0; c < n; c++) gn[c] *= -diag[c];
        }
        int step_valid = 0; double model_change = 0;
        if (!solver_failed) {                                                       /* ComputeTraditionalDoglegStep */
            double gnorm = 0, gnn = 0;
            for (int c = 0; c < n; c++) { gnorm += gs[c] * gs[c]; gnn += gn[c] * gn[c]; }
            gnorm = sqrt(gnorm); gnn = sqrt(gnn);
            if (gnn <= radius) { for (int c = 0; c < n; c++) step[c] = gn[c]; dogleg_norm = gnn; }
            else if (gnorm * alpha >= radius) { for (int c = 0; c < n; c++) step[c] = -(radius / gnorm) * gs[c]; dogleg_norm = radius; }
            else {
                double b_dot_a = 0; for (int c = 0; c < n; c++) b_dot_a += gs[c] * gn[c]; b_dot_a *= -alpha;
                double a2 = pow(alpha * gnorm, 2.0);
                double bma2 = a2 - 2 * b_dot_a + pow(gnn, 2);
                double cc = b_dot_a - a2;
                double dd = sqrt(cc * cc + bma2 * (pow(radius, 2.0) - a2));
                double beta = (cc <= 0) ? (dd - cc) / bma2 : (radius * radius - a2) / (dd + cc);
                double nn = 0;
                for (int c = 0; c < n; c++) { step[c] = (-alpha * (1.0 - beta)) * gs[c] + beta * gn[c]; nn += step[c] * step[c]; }
                dogleg_norm = sqrt(nn);
            }
            for (int c = 0; c < n; c++) step[c] /= diag[c];
            /* model_cost_change = -(J s)^T (r + J s / 2) = -(s^T g + s^T H s / 2) */
            double sg = 0, sHs = 0;
            for (int a = 0; a < n; a++) { sg += step[a] * g[a]; double s = 0; for (int b = 0; b < n; b++) s += H[(size_t)a * n + b] * step[b]; sHs += step[a] * s; }
            model_change = -(sg + 0.5 * sHs);
            step_valid = model_change > 0.0;
        }
        if (!step_valid) {                                                          /* HandleInvalidStep */
            if (++invalid_streak >= 5) { termination = GF_BA_FAILURE; sum->cost[it] = x_cost; sum->radius[it] = radius; break; }
            mu *= mu_inc; reuse = 0;
            sum->cost[it] = x_cost; sum->radius[it] = radius;
            continue;
        }
        invalid_streak = 0;
        for (int c = 0; c < n; c++) delta[c] = step[c] * scale[c];
        state_plus(p, &L, &x, delta, &cand);
        double cand_cost = cost_only(p, &L, &cand, imu_sqrt);
        double step_norm; state_diff_norms(&L, &x, &cand, &step_norm, NULL);
        if (step_norm <= param_tol * (x_norm + param_tol)) { termination = GF_BA_CONVERGENCE_PARAMETER; sum->cost[it] = x_cost; sum->radius[it] = radius; break; }
        if (fabs(x_cost - cand_cost) <= func_tol * x_cost) { termination = GF_BA_CONVERGENCE_FUNCTION; sum->cost[it] = x_cost; sum->radius[it] = radius; break; }
        double rel = (x_cost - cand_cost) / model_change;
        if (rel > min_rel_dec) {                                                    /* HandleSuccessfulStep */
            state_copy(p, &cand, &x);
            state_diff_norms(&L, &x, NULL, &x_norm, NULL);
            LINEARIZE(0);
            n_success++;
            if (rel < 0.25) radius *= 0.5;                                          /* DoglegStrategy::StepAccepted */
            if (rel > 0.75) radius = fmax(radius, 3.0 * dogleg_norm);
            mu = fmax(min_mu, 2.0 * mu / mu_inc);
            reuse = 0;
            sum->cost[it] = x_cost; sum->radius[it] = radius;
            if (grad_max <= grad_tol) { termination = GF_BA_CONVERGENCE_GRADIENT; break; }
        } else {                                                                    /* HandleUnsuccessfulStep */
            radius *= 0.5; reuse = 1;
            sum->cost[it] = x_cost; sum->radius[it] = radius;
        }
    }
done:
    sum->iterations = it; sum->num_successful_steps = n_success; sum->termination = termination; sum->final_cost = x_cost;
    state_store(p, &x);
    free(x.feat); free(cand.feat); free(tmp.feat); free(imu_sqrt); free(r); free(rc); free(H); free(Hp);
    free(g); free(scale); free(diag); free(lmd); free(gs); free(gn); free(step); free(delta); free(tv); free(L.col_feat);
    return 0;
}

/* cost at the current parameter values (1/2 sum rho) -- test aid */
GFO double gfo_ba_cost(const gf_ba_problem* p)
{
    if (same_frame_visual(p)) return NAN;
    layout_t L; make_layout(p, &L);
    double* imu_sqrt = (double*)malloc(sizeof(double) * 225 * (p->n_imu > 0 ? p->n_imu : 1));
    for (int k = 0; k < p->n_imu; k++) gfo_sqrt_info(p->imu[k].covariance, 15, imu_sqrt + 225 * k);
    state_t x; state_load(p, &x);
    double* r = (double*)malloc(sizeof(double) * (L.n_rows + 1));
    double c = evaluate(p, &L, &x, imu_sqrt, r, NULL);
    free(r); free(x.feat); free(imu_sqrt); free(L.col_feat);
    return c;
}

/* Dense linearisation at the current values: J (rows x cols, loss-corrected, local), r, column map.  Test aid
 * (finite differences, SciPy cross-check).  Returns rows; cols via *n_cols. */
GFO int gfo_ba_linearize(const gf_ba_problem* p, double* r_out, double* J_out, int* n_cols, int cap_rows, int cap_cols)
{
    if (same_frame_visual(p)) return GF_ERR_INVALID_ARG;
    layout_t L; make_layout(p, &L);
    *n_cols = L.n_cols;
    if (L.n_rows > cap_rows || L.n_cols > cap_cols) { free(L.col_feat); return GF_ERR_CAPACITY; }
    double* imu_sqrt = (double*)malloc(sizeof(double) * 225 * (p->n_imu > 0 ? p->n_imu : 1));
    for (int k = 0; k < p->n_imu; k++) gfo_sqrt_info(p->imu[k].covariance, 15, imu_sqrt + 225 * k);
    state_t x; state_load(p, &x);
    evaluate(p, &L, &x, imu_sqrt, r_out, J_out);
    int rows = L.n_rows;
    free(x.feat); free(imu_sqrt); free(L.col_feat);
    return rows;
}
/* x <- Plus(x, delta) in the oracle's column order (test aid for finite differences) */
GFO void gfo_ba_plus(const gf_ba_problem* p, const double* delta)
{
    layout_t L; make_layout(p, &L);
    state_t x, y; state_load(p, &x); state_load(p, &y);
    state_plus(p, &L, &x, delta, &y);
    state_store(p, &y);
    free(x.feat); free(y.feat); free(L.col_feat);
}

/* ------------------------------------------------------------------ marginalisation ------------- */
/* MARGIN_OLD (estimator.cpp:3334-3535) + MarginalizationInfo::{preMarginalize, marginalize}
 * (marginalization_factor.cpp:115-308).  Factors: last prior (drop pose0, speedbias0), IMU(0->1) (drop 0,1),
 * every visual factor whose landmark starts in frame 0 (drop pose0 and the landmark).  Kept blocks are ordered
 * pose[1..], speedbias[1..], ex_pose, td (the reference orders by heap address; only J0^T J0 and J0^T r0 are
 * order-independent and those are what the tests compare).  After addr_shift the kept pose/speedbias indices are
 * decremented by one.  With wheel factors the WheelFactor(0->1) joins (pose 0 dropped) and the wheel extrinsic, sx, sy,
 * sw and the wheel time offset follow as kept blocks.  out_x0 / out_J / out_r must hold 16F+19, n*n, n doubles. */
static int marg_run(const gf_ba_problem* p, int second_new, gf_ba_prior* out, double* out_x0, double* out_J, double* out_r)
{
    if (same_frame_visual(p)) return GF_ERR_INVALID_ARG;
    const int F = p->n_frames;
    const int use_sb = (p->para_speed_bias != NULL) && !p->pose0_const;
    state_t s; state_load(p, &s);
    /* marginalised block layout: pose0 (6), sb0 (9), landmarks starting in frame 0 (1 each) */
    int* lm_col = (int*)malloc(sizeof(int) * (p->n_features + 1));
    for (int k = 0; k < p->n_features; k++) lm_col[k] = -1;
    int pos = 0;
    const int old_ = !second_new, fdrop = old_ ? 0 : F - 2;     /* MARGIN_SECOND_NEW drops para_Pose[WINDOW_SIZE - 1] (estimator.cpp:3549-3551) */
    if (!old_) {
        int has = 0;
        if (p->prior && p->prior->n > 0) for (int b = 0; b < p->prior->n_blocks; b++) if (p->prior->block_kind[b] == GF_BA_BLOCK_POSE && p->prior->block_index[b] == fdrop) has = 1;
        if (!has) { free(lm_col); free(s.feat); return 0; }
    }
    const int col_p0 = pos; pos += 6;
    int col_sb0 = -1;
    if (old_ && use_sb) { col_sb0 = pos; pos += 9; }
    for (int v = 0; old_ && v < p->n_visual; v++) if (p->visual[v].imu_i == 0 && lm_col[p->visual[v].feature] < 0) lm_col[p->visual[v].feature] = pos++;
    const int m = pos;
    /* kept blocks: every other block the factors touch */
    int used_pose[GF_BA_MAX_FRAMES] = {0}, used_sb[GF_BA_MAX_FRAMES] = {0}, used_ex = 0, used_td = 0, used_exw = 0, used_ix[3] = {0, 0, 0}, used_tdw = 0, used_pr = 0, used_pz = 0;
    if (p->prior && p->prior->n > 0)
        for (int b = 0; b < p->prior->n_blocks; b++) {
            int k = p->prior->block_kind[b], i = p->prior->block_index[b];
            if (k == GF_BA_BLOCK_POSE) used_pose[i] = 1; else if (k == GF_BA_BLOCK_SPEEDBIAS) used_sb[i] = 1;
            else if (k == GF_BA_BLOCK_EX_POSE) used_ex = 1; else if (k == GF_BA_BLOCK_TD) used_td = 1;
            else if (k == GF_BA_BLOCK_EX_WHEEL) used_exw = 1; else if (k >= GF_BA_BLOCK_SX && k <= GF_BA_BLOCK_SW) used_ix[k - GF_BA_BLOCK_SX] = 1;
            else if (k == GF_BA_BLOCK_TD_WHEEL) used_tdw = 1;
            else if (k == GF_BA_BLOCK_PLANE_R) used_pr = 1; else if (k == GF_BA_BLOCK_PLANE_Z) used_pz = 1;
        }
    int have_imu01 = 0; const gf_ba_imu_factor* imu01 = NULL;
    for (int k = 0; old_ && k < p->n_imu; k++) if (p->imu[k].i == 0 && p->imu[k].j == 1 && p->imu[k].sum_dt < 10.0) { have_imu01 = 1; imu01 = &p->imu[k]; used_pose[1] = 1; used_sb[1] = 1; }
    for (int v = 0; old_ && v < p->n_visual; v++) if (p->visual[v].imu_i == 0) { used_pose[p->visual[v].imu_j] = 1; used_ex = 1; used_td = 1; }
    /* WheelFactor(pre_integrations_wheel[1]) with para_Pose[0] dropped (estimator.cpp:3367-3377) */
    const gf_ba_wheel_factor* wheel01 = NULL;
    for (int k = 0; old_ && k < p->n_wheel; k++) if (p->wheel[k].i == 0 && p->wheel[k].j == 1 && p->wheel[k].sum_dt < 10.0) { wheel01 = &p->wheel[k]; used_pose[1] = 1; used_exw = 1; used_ix[0] = used_ix[1] = used_ix[2] = 1; used_tdw = 1; }
    /* PlaneFactor(para_Pose[0], para_Ex_Pose_wheel, para_plane_R, para_plane_Z), para_Pose[0] dropped (estimator.cpp:3379-3390) */
    int plane0 = 0;
    for (int k = 0; old_ && k < p->n_plane; k++) if (p->plane_frames[k] == 0) plane0 = 1;
    if (plane0) { used_exw = 1; used_pr = 1; used_pz = 1; }
    int col_pose[GF_BA_MAX_FRAMES], col_sb[GF_BA_MAX_FRAMES], col_ex = -1, col_td = -1, col_exw = -1, col_ix[3] = {-1, -1, -1}, col_tdw = -1, col_pr = -1, col_pz = -1;
    for (int f = 0; f < F; f++) { col_pose[f] = -1; col_sb[f] = -1; }
    col_pose[fdrop] = col_p0; if (old_) col_sb[0] = col_sb0;
    for (int f = 0; f < F; f++) if (f != fdrop && used_pose[f]) { col_pose[f] = pos; pos += 6; }
    for (int f = 0; f < F; f++) if (!(old_ && f == 0) && used_sb[f] && use_sb) { col_sb[f] = pos; pos += 9; }
    if (used_ex) { col_ex = pos; pos += 6; }
    if (used_td) { col_td = pos; pos += 1; }
    if (used_exw) { col_exw = pos; pos += 6; }
    for (int k = 0; k < 3; k++) if (used_ix[k]) col_ix[k] = pos++;
    if (used_tdw) col_tdw = pos++;
    /* the plane rotation keeps its 4 global columns: MarginalizationInfo::localSize only maps 7 -> 6 (marginalization_factor.h) */
    if (used_pr) { col_pr = pos; pos += 4; }
    if (used_pz) col_pz = pos++;
    const int N = pos, n = N - m;
    double* A = (double*)calloc((size_t)N * N + 1, 8);
    double* bvec = (double*)calloc(N + 1, 8);
#define ADD_BLOCKS(nres, res, nb, cols, sizes, lds, Js)                                                             \
    for (int a_ = 0; a_ < nb; a_++) { if (cols[a_] < 0) continue;                                                  \
        for (int b_ = 0; b_ < nb; b_++) { if (cols[b_] < 0) continue;                                              \
            for (int i_ = 0; i_ < sizes[a_]; i_++) for (int j_ = 0; j_ < sizes[b_]; j_++) { double s_ = 0;         \
                for (int k_ = 0; k_ < nres; k_++) s_ += Js[a_][k_ * lds[a_] + i_] * Js[b_][k_ * lds[b_] + j_];     \
                A[(size_t)(cols[a_] + i_) * N + cols[b_] + j_] += s_; } }                                          \
        for (int i_ = 0; i_ < sizes[a_]; i_++) { double s_ = 0; for (int k_ = 0; k_ < nres; k_++) s_ += Js[a_][k_ * lds[a_] + i_] * res[k_]; bvec[cols[a_] + i_] += s_; } }
    /* last prior */
    if (p->prior && p->prior->n > 0) {
        const gf_ba_prior* pr = p->prior;
        int pn = pr->n;
        double* dx = (double*)malloc(sizeof(double) * pn);
        double* res = (double*)malloc(sizeof(double) * pn);
        prior_dx(pr, &s, dx);
        for (int i = 0; i < pn; i++) { double v = pr->linearized_residuals[i]; for (int k = 0; k < pn; k++) v += pr->linearized_jacobians[(size_t)i * pn + k] * dx[k]; res[i] = v; }
        for (int a = 0; a < pr->n_blocks; a++) {
            int ka = pr->block_kind[a], ia = pr->block_index[a];
#define MARG_COL(k_, i_) ((k_) == GF_BA_BLOCK_POSE ? col_pose[i_] : (k_) == GF_BA_BLOCK_SPEEDBIAS ? col_sb[i_] : (k_) == GF_BA_BLOCK_EX_POSE ? col_ex : (k_) == GF_BA_BLOCK_TD ? col_td : \
                          (k_) == GF_BA_BLOCK_EX_WHEEL ? col_exw : (k_) == GF_BA_BLOCK_TD_WHEEL ? col_tdw : (k_) == GF_BA_BLOCK_PLANE_R ? col_pr : (k_) == GF_BA_BLOCK_PLANE_Z ? col_pz : col_ix[(k_) - GF_BA_BLOCK_SX])
            int ca = MARG_COL(ka, ia);
            int sa = block_global_size(ka); if (sa == 7) sa = 6;
            for (int b2 = 0; b2 < pr->n_blocks; b2++) {
                int kb = pr->block_kind[b2], ib = pr->block_index[b2];
                int cb = MARG_COL(kb, ib);
                int sb2 = block_global_size(kb); if (sb2 == 7) sb2 = 6;
                for (int i = 0; i < sa; i++) for (int j = 0; j < sb2; j++) { double v = 0; for (int k = 0; k < pn; k++) v += pr->linearized_jacobians[(size_t)k * pn + pr->block_idx[a] + i] * pr->linearized_jacobians[(size_t)k * pn + pr->block_idx[b2] + j]; A[(size_t)(ca + i) * N + cb + j] += v; }
            }
            for (int i = 0; i < sa; i++) { double v = 0; for (int k = 0; k < pn; k++) v += pr->linearized_jacobians[(size_t)k * pn + pr->block_idx[a] + i] * res[k]; bvec[ca + i] += v; }
        }
        free(dx); free(res);
    }
    if (have_imu01) {
        double sq[225], res[15], J0[105], J1[135], J2[105], J3[135];
        gfo_sqrt_info(imu01->covariance, 15, sq);
        gfo_eval_imu(imu01, sq, p->gravity, s.pose[0], s.sb[0], s.pose[1], s.sb[1], res, J0, J1, J2, J3);
        int cols[4] = {col_pose[0], col_sb[0], col_pose[1], col_sb[1]}, sizes[4] = {6, 9, 6, 9}, lds[4] = {7, 9, 7, 9};
        double* Js[4] = {J0, J1, J2, J3};
        ADD_BLOCKS(15, res, 4, cols, sizes, lds, Js)
    }
    if (wheel01) {
        double res[6], J0[42], J1[42], J2[42], Jsx[6], Jsy[6], Jsw[6], Jtw[6];
        gfo_eval_wheel(wheel01, s.pose[0], s.pose[1], s.exw, s.ix[0], s.ix[1], s.ix[2], s.tdw, res, J0, J1, J2, Jsx, Jsy, Jsw, Jtw);
        int cols[7] = {col_pose[0], col_pose[1], col_exw, col_ix[0], col_ix[1], col_ix[2], col_tdw}, sizes[7] = {6, 6, 6, 1, 1, 1, 1}, lds[7] = {7, 7, 7, 1, 1, 1, 1};
        double* Js[7] = {J0, J1, J2, Jsx, Jsy, Jsw, Jtw};
        ADD_BLOCKS(6, res, 7, cols, sizes, lds, Js)
    }
    if (plane0) {
        double res[3], J0[21], J1[21], J2[12], J3[3];
        gfo_eval_plane(s.pose[0], s.exw, s.pr, s.pz, p->plane_sqrt_info, res, J0, J1, J2, J3);
        int cols[4] = {col_pose[0], col_exw, col_pr, col_pz}, sizes[4] = {6, 6, 4, 1}, lds[4] = {7, 7, 4, 1};
        double* Js[4] = {J0, J1, J2, J3};
        ADD_BLOCKS(3, res, 4, cols, sizes, lds, Js)
    }
    for (int v = 0; old_ && v < p->n_visual; v++) {
        const gf_ba_visual_factor* f = &p->visual[v];
        if (f->imu_i != 0) continue;
        double res[2], Ji[14], Jj[14], Jex[14], Jf[2], Jtd[2];
        gfo_eval_visual(f, p->visual_sqrt_info, s.pose[0], s.pose[f->imu_j], s.ex, s.feat[f->feature], s.td, res, Ji, Jj, Jex, Jf, Jtd);
        double sq = res[0] * res[0] + res[1] * res[1], rho1 = 1.0;
        if (sq > 1.0) rho1 = 1.0 / sqrt(sq);
        double sc = sqrt(rho1);   /* ResidualBlockInfo::Evaluate, marginalization_factor.cpp:46-77 (alpha = 0 since rho'' <= 0) */
        for (int k = 0; k < 14; k++) { Ji[k] *= sc; Jj[k] *= sc; Jex[k] *= sc; }
        for (int k = 0; k < 2; k++) { Jf[k] *= sc; Jtd[k] *= sc; res[k] *= sc; }
        int cols[5] = {col_pose[0], col_pose[f->imu_j], col_ex, lm_col[f->feature], col_td}, sizes[5] = {6, 6, 6, 1, 1}, lds[5] = {7, 7, 7, 1, 1};
        double* Js[5] = {Ji, Jj, Jex, Jf, Jtd};
        ADD_BLOCKS(2, res, 5, cols, sizes, lds, Js)
    }
    /* Schur complement with eigen-truncated inverse (eps = 1e-8), then J0 = sqrt(S) V^T, r0 = sqrt(S^-1) V^T b */
    const double eps = 1e-8;
    double* Amm = (double*)malloc(sizeof(double) * m * m);
    for (int i = 0; i < m; i++) for (int j = 0; j < m; j++) Amm[i * m + j] = 0.5 * (A[(size_t)i * N + j] + A[(size_t)j * N + i]);
    double* w = (double*)malloc(sizeof(double) * (N + 1)); double* V = (double*)malloc(sizeof(double) * ((size_t)N * N + 1));
    sym_eig(Amm, m, w, V);
    double* Ainv = (double*)calloc((size_t)m * m, 8);
    for (int k = 0; k < m; k++) if (w[k] > eps) { double iw = 1.0 / w[k]; for (int i = 0; i < m; i++) for (int j = 0; j < m; j++) Ainv[i * m + j] += V[i * m + k] * iw * V[j * m + k]; }
    double* T = (double*)malloc(sizeof(double) * ((size_t)n * m + 1));   /* Arm * Amm_inv */
    for (int i = 0; i < n; i++) for (int j = 0; j < m; j++) { double v = 0; for (int k = 0; k < m; k++) v += A[(size_t)(m + i) * N + k] * Ainv[k * m + j]; T[(size_t)i * m + j] = v; }
    double* Ar = (double*)malloc(sizeof(double) * ((size_t)n * n + 1)); double* br = (double*)malloc(sizeof(double) * (n + 1));
    for (int i = 0; i < n; i++) {
        for (int j = 0; j < n; j++) { double v = A[(size_t)(m + i) * N + m + j]; for (int k = 0; k < m; k++) v -= T[(size_t)i * m + k] * A[(size_t)k * N + m + j]; Ar[(size_t)i * n + j] = v; }
        double v = bvec[m + i]; for (int k = 0; k < m; k++) v -= T[(size_t)i * m + k] * bvec[k]; br[i] = v;
    }
    /* Eigen's SelfAdjointEigenSolver reads the lower triangle; symmetrise for the Jacobi stand-in */
    for (int i = 0; i < n; i++) for (int j = 0; j < i; j++) Ar[(size_t)j * n + i] = Ar[(size_t)i * n + j];
    sym_eig(Ar, n, w, V);
    for (int k = 0; k < n; k++) {
        double S = w[k] > eps ? w[k] : 0.0, Si = w[k] > eps ? 1.0 / w[k] : 0.0;
        double ss = sqrt(S), sis = sqrt(Si), vb = 0;
        for (int i = 0; i < n; i++) { out_J[(size_t)k * n + i] = ss * V[(size_t)i * n + k]; vb += V[(size_t)i * n + k] * br[i]; }
        out_r[k] = sis * vb;
    }
    /* kept blocks after addr_shift (estimator.cpp:3500-3534 / 3583-3621): MARGIN_OLD shifts every frame down by one,
     * MARGIN_SECOND_NEW moves frame F-1 into the slot of the dropped frame F-2 */
    memset(out, 0, sizeof(*out));
    out->n = n;
    int nb = 0; double* xp = out_x0;
#define SHIFTED(f_) (old_ ? (f_) - 1 : ((f_) == F - 1 ? F - 2 : (f_)))
    for (int f = 0; f < F; f++) if (f != fdrop && col_pose[f] >= 0) { out->block_kind[nb] = GF_BA_BLOCK_POSE; out->block_index[nb] = SHIFTED(f); out->block_idx[nb] = col_pose[f] - m; memcpy(xp, s.pose[f], 56); xp += 7; nb++; }
    for (int f = 0; f < F; f++) if (!(old_ && f == 0) && col_sb[f] >= 0) { out->block_kind[nb] = GF_BA_BLOCK_SPEEDBIAS; out->block_index[nb] = SHIFTED(f); out->block_idx[nb] = col_sb[f] - m; memcpy(xp, s.sb[f], 72); xp += 9; nb++; }
    if (col_ex >= 0) { out->block_kind[nb] = GF_BA_BLOCK_EX_POSE; out->block_index[nb] = 0; out->block_idx[nb] = col_ex - m; memcpy(xp, s.ex, 56); xp += 7; nb++; }
    if (col_td >= 0) { out->block_kind[nb] = GF_BA_BLOCK_TD; out->block_index[nb] = 0; out->block_idx[nb] = col_td - m; xp[0] = s.td; xp += 1; nb++; }
    if (col_exw >= 0) { out->block_kind[nb] = GF_BA_BLOCK_EX_WHEEL; out->block_index[nb] = 0; out->block_idx[nb] = col_exw - m; memcpy(xp, s.exw, 56); xp += 7; nb++; }
    for (int k = 0; k < 3; k++) if (col_ix[k] >= 0) { out->block_kind[nb] = GF_BA_BLOCK_SX + k; out->block_index[nb] = 0; out->block_idx[nb] = col_ix[k] - m; xp[0] = s.ix[k]; xp += 1; nb++; }
    if (col_tdw >= 0) { out->block_kind[nb] = GF_BA_BLOCK_TD_WHEEL; out->block_index[nb] = 0; out->block_idx[nb] = col_tdw - m; xp[0] = s.tdw; xp += 1; nb++; }
    if (col_pr >= 0) { out->block_kind[nb] = GF_BA_BLOCK_PLANE_R; out->block_index[nb] = 0; out->block_idx[nb] = col_pr - m; memcpy(xp, s.pr, 32); xp += 4; nb++; }
    if (col_pz >= 0) { out->block_kind[nb] = GF_BA_BLOCK_PLANE_Z; out->block_index[nb] = 0; out->block_idx[nb] = col_pz - m; xp[0] = s.pz; xp += 1; nb++; }
    out->n_blocks = nb; out->x0 = out_x0; out->linearized_jacobians = out_J; out->linearized_residuals = out_r;
    free(lm_col); free(A); free(bvec); free(Amm); free(w); free(V); free(Ainv); free(T); free(Ar); free(br); free(s.feat);
    return n;
}
GFO int gfo_ba_marginalize_old(const gf_ba_problem* p, gf_ba_prior* out, double* out_x0, double* out_J, double* out_r)
{
    return marg_run(p, 0, out, out_x0, out_J, out_r);
}
/* MARGIN_SECOND_NEW (estimator.cpp:3536-3631): the last prior is the only factor (MarginalizationFactor evaluated at the current
 * state, no loss function), para_Pose[WINDOW_SIZE - 1] is marginalised; returns 0 when the prior does not hold that pose. */
GFO int gfo_ba_marginalize_second_new(const gf_ba_problem* p, gf_ba_prior* out, double* out_x0, double* out_J, double* out_r)
{
    return marg_run(p, 1, out, out_x0, out_J, out_r);
}
