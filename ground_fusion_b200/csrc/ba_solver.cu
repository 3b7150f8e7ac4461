// ba_solver.cu -- gf_ba_* (C ABI): Estimator::optimization()'s ceres::Solve (DENSE_SCHUR + DOGLEG,
// estimator.cpp:3303-3318) on one GPU, FP64.  Algorithm and constants: oracle/ba_oracle.c (restatement of
// Ceres 1.14's trust_region_minimizer.cc / dogleg_strategy.cc; parity with Ceres itself is unpinned, see DESIGN.md).
//
// Data flow of one solve (everything stays on the device between the upload and the final download):
//   (host)          initial solver state and candidate := x travel with the problem upload; H_prior and the accumulators are memset
//   k_ba_prior_hessian  H_prior = J0^T J0
//   k_ba_eval       mode 0 "linearise": one CTA per pose pair (i,j) evaluates its visual factors, stages the
//                   Huber-corrected Jacobian slab [Ji|Jj|Jex|Jtd] in shared memory and reduces it to block
//                   Hessians; one CTA per IMU factor; one CTA for the marginalisation prior.  Landmark terms
//                   (h_ll, g_l, W = H_landmark,camera) go to their own arrays: J is never materialised.
//                   mode 1 "candidate cost": residuals only at x (+) delta.
//   k_ba_step       single CTA: Jacobi scaling, Schur complement of the free landmarks into the packed reduced
//                   system, Cholesky (rhs carried as an extra row), traditional dogleg, model cost change,
//                   candidate x (+) delta.
//   (ba_decide)     step acceptance, trust-region / mu update, convergence tests (the Ceres state machine): run by the
//                   last CTA of k_ba_eval(1) to finish.
// All four are enqueued for every iteration up front; kernels return immediately once the state says "done",
// so the host synchronises exactly once per solve.
#include <stdlib.h>
#include <new>
#include <type_traits>
#include <vector>

#include "ba_factors.cuh"
#include "ba_chol.cuh"

using namespace gf;
using namespace gfba;

namespace gfba {

constexpr int MAXF = GF_BA_MAX_FRAMES;
constexpr int X_POSE = 0, X_SB = 7 * MAXF, X_EX = X_SB + 9 * MAXF, X_TD = X_EX + 7, X_EXW = X_TD + 1, X_IX = X_EXW + 7, X_TDW = X_IX + 3,
              X_PR = X_TDW + 1, X_PZ = X_PR + 4, X_FEAT = X_PZ + 1;
constexpr int PAIR_THREADS = 256, PAIR_CHUNK = 64;   // factors staged per pass (2*64 rows x 20 cols in smem)
constexpr int RB_THREADS = ST_THREADS;               // k_ba_step block size (ba_chol.cuh)
constexpr int SCHUR_WARPS = 8;                       // k_ba_schur: one warp per 8x8 tile of the reduced system
// k_ba_schur's dynamic shared memory at the largest window: cl[L] | ss[nc+1] | sv[nc] (above the 48 KB default from L ~ 5,800)
constexpr size_t SCHUR_SMEM_MAX = sizeof(double) * (GF_BA_MAX_FREE_LANDMARKS + 2 * MAX_NC + 2);
// k_ba_step's dynamic shared memory at nc = MAX_NC (factor tiles | diagonal inverses | 3 tiles | y, z), 219.5 KB: with the
// kernel's static shared memory (the window descriptor among it) within the 227 KB a CTA may have
constexpr size_t STEP_SMEM_MAX = sizeof(double) * (64 * TILE_CAP + 64 * MAX_N8 + 192 + 2 * 8 * MAX_N8);

struct BaState {
    double x_cost, cand_cost, radius, mu, alpha, dogleg_norm, model_change, x_norm, step_norm, grad_max;
    double cost_hist[GF_BA_MAX_ITERATIONS + 1], radius_hist[GF_BA_MAX_ITERATIONS + 1];
    double acc_cost[2];          // cost accumulated by k_ba_eval into buffer 0/1
    double cauchy_num, cauchy_den;   // |gs|^2 and v^T H' v accumulated by k_ba_schur
    double dl_a, dl_b;           // the last dogleg step in D-space: dl_a * gs + dl_b * gn
    int it, reuse, done, termination, n_success, invalid_streak, need_linearize, step_valid, cur, first, max_iter, solver_failed;
    unsigned int eval_ticket;    // CTAs of the current k_ba_eval(1) that have finished: the last one runs the decision
    int setup_failed;            // sticky: an IMU covariance was singular / not positive definite (first k_ba_eval); nothing is solved
    long long prof[32];          // clock64() cycles per phase of k_ba_step, summed over iterations (debug)
};

struct BaDev {
    int F, nfeat, n_vis, n_imu, n_wheel, n_pairs, nc, L, n;
    int col_pose[MAXF], col_sb[MAXF], col_ex, col_td;
    int lm_dense;             // marginalisation: landmark columns are ordinary columns of H (cf < nc), no W / hll arrays
    int col_exw, col_ix[3], col_tdw, exw_mask;     // wheel extrinsic / intrinsics / time offset (-1: constant or absent)
    const gf_ba_wheel_factor* wheel;
    int n_plane, col_pr, col_pz, pr_mask;          // PlaneFactor: frames, plane rotation (local 3) / height columns
    const int* plane_frames;
    double plane_sinfo[3];
    const int* col_feat;
    double *X, *Xc;
    const gf_ba_visual_factor* vis;
    const int *pair_start, *pair_ij;
    const gf_ba_imu_factor* imu;
    double* imu_sqrt;
    int pn, pnb;
    int pkind[64], pindex[64], pidx[64], pxoff[64];
    const double *pJ, *pr0, *px0;
    const int* pcol;          // [pn] prior column -> layout column or -1
    double* Hp;               // [nc*nc]
    double* acc[2];           // accumulators: [H nc*nc | g n | W L*nc | hll L]
    double *scale, *diag, *gs, *gn, *step, *delta;
    double* Sg;               // reduced system written by k_ba_schur: row-major 8x8 tiles tix(I,J) of the (nc+1)-row augmented matrix (row nc = rhs)
    double* Lg;               // factor tiles beyond tile_cap (spill, L2-resident)
    int tile_cap;             // factor tiles kept in shared memory (TILE_CAP; smaller only when GF_BA_TILE_CAP is set, to test the spill path)
    double gravity[3], vis_sqrt_info;
    BaState* st;
    int eval_grid, schur_grid;   // this window's own CTA counts of k_ba_eval / k_ba_schur (a batch launches the largest; the rest exit)
};
static_assert(sizeof(BaDev) % 8 == 0, "BaDev is copied to shared memory in 8-byte words");

// Every kernel of a solve serves a batch of windows (gf_ba_solve_multi; gf_ba_solve is the batch of one): blockIdx.y picks the
// window and its descriptor is copied to shared memory at kernel entry.  The descriptors travel with the upload that precedes the
// whole launch chain, so the copy may run before gf_pdl_wait and overlaps the tail of the predecessor; a __syncthreads must
// follow before the descriptor is read.
__device__ __forceinline__ void load_window(BaDev& sd, const BaDev* __restrict__ src)
{
    const unsigned long long* s = reinterpret_cast<const unsigned long long*>(src);
    unsigned long long* t = reinterpret_cast<unsigned long long*>(&sd);
    for (int e = threadIdx.x; e < (int)(sizeof(BaDev) / 8); e += blockDim.x) t[e] = s[e];
}

__device__ __forceinline__ double* acc_H(const BaDev& d, int b) { return d.acc[b]; }
__device__ __forceinline__ double* acc_g(const BaDev& d, int b) { return d.acc[b] + (size_t)d.nc * d.nc; }
__device__ __forceinline__ double* acc_W(const BaDev& d, int b) { return d.acc[b] + (size_t)d.nc * d.nc + d.n; }
__device__ __forceinline__ double* acc_hll(const BaDev& d, int b) { return d.acc[b] + (size_t)d.nc * d.nc + d.n + (size_t)d.L * d.nc; }
__host__ __device__ inline size_t acc_size(int nc, int L) { return (size_t)nc * nc + (nc + L) + (size_t)L * nc + L; }

__device__ __forceinline__ double block_reduce_sum(double v, double* sh)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    double t = 0;
    if (w == 0) {
        t = (l < nw) ? sh[l] : 0.0;
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (l == 0) sh[0] = t;
    }
    __syncthreads();
    t = sh[0];
    __syncthreads();
    return t;
}

// ------------------------------------------------------------------------------------------------
// IMU sqrt-information matrix  sqrt_info = LLT(cov^-1).L^T  (reference imu_factor.h:73), one warp: the same Gauss-Jordan
// (partial pivoting) + Cholesky as gfba::sqrt_info_from_cov / the oracle, element updates spread over the lanes (identical
// arithmetic per element).  M: 15 x 30 doubles of shared memory.  Run by the IMU CTAs of the first k_ba_eval, next to the
// thread that evaluates the factor; false = the covariance is singular / not positive definite.
__device__ __forceinline__ bool imu_sqrt_info_warp(const double* __restrict__ cov, double* M, double* __restrict__ out, int lane)
{
    const int n = 15, w2 = 30;
    for (int e = lane; e < n * w2; e += 32) { int i = e / w2, j = e - i * w2; M[e] = j < n ? cov[i * n + j] : ((j - n) == i ? 1.0 : 0.0); }
    __syncwarp();
    bool ok = true;
    for (int c = 0; c < n; c++) {
        // partial pivoting: the first row (lowest index) with the largest |M[r][c]|, r >= c, by a warp argmax (same choice as the
        // sequential scan of the oracle)
        double pv = (lane >= c && lane < n) ? fabs(M[lane * w2 + c]) : -1.0;
        int piv = lane;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, pv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, piv, o);
            if (ov > pv || (ov == pv && oi < piv)) { pv = ov; piv = oi; }
        }
        if (M[piv * w2 + c] == 0.0) { ok = false; break; }
        __syncwarp();
        if (piv != c && lane < w2) { double t = M[c * w2 + lane]; M[c * w2 + lane] = M[piv * w2 + lane]; M[piv * w2 + lane] = t; }
        __syncwarp();
        double dpiv = M[c * w2 + c];
        __syncwarp();
        if (lane < w2) M[c * w2 + lane] /= dpiv;
        __syncwarp();
        for (int e = lane; e < n * w2; e += 32) {
            int r = e / w2, j = e - r * w2;
            if (r == c) continue;
            double fct = M[r * w2 + c];
            // every lane of row r must read fct before column c of that row is overwritten: column c itself is updated last
            if (j != c && fct != 0.0) M[e] -= fct * M[c * w2 + j];
        }
        __syncwarp();
        if (lane < n && lane != c) { double fct = M[lane * w2 + c]; if (fct != 0.0) M[lane * w2 + c] -= fct * M[c * w2 + c]; }
        __syncwarp();
    }
    if (ok) {          // Cholesky (lower) of the inverse held in the right half: lane i owns row i (same per-element arithmetic as the oracle)
        double* A = M + n;
        for (int j = 0; j < n; j++) {
            double t = 0.0;
            if (lane >= j && lane < n) {
                t = A[lane * w2 + j];
                for (int k = 0; k < j; k++) t -= A[lane * w2 + k] * A[j * w2 + k];
            }
            double dd = __shfl_sync(0xffffffffu, t, j);
            if (!(dd > 0.0)) { ok = false; break; }
            dd = sqrt(dd);
            if (lane == j) A[j * w2 + j] = dd;
            else if (lane > j && lane < n) A[lane * w2 + j] = t / dd;
            __syncwarp();
        }
        if (ok) for (int e = lane; e < n * n; e += 32) { int i = e / n, j = e - i * n; out[e] = (j >= i) ? A[j * w2 + i] : 0.0; }
    }
    return ok;
}
__global__ void k_ba_prior_hessian(const BaDev* __restrict__ wins)
{
    __shared__ BaDev sd;
    load_window(sd, wins + blockIdx.y);
    __syncthreads();
    const BaDev& d = sd;
    const int nc = d.nc, pn = d.pn;
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= pn * pn) return;
    int pa = e / pn, pb = e - pa * pn;
    int ca = d.pcol[pa], cb = d.pcol[pb];
    if (ca < 0 || cb < 0) return;
    double s = 0;
    for (int k = 0; k < pn; k++) s += d.pJ[(size_t)k * pn + pa] * d.pJ[(size_t)k * pn + pb];
    d.Hp[(size_t)ca * nc + cb] = s;
}

// ------------------------------------------------------------------------------------------------
// TrustRegionMinimizer's step acceptance, radius / mu update and convergence tests; run by the last CTA of k_ba_eval(1)
__device__ void ba_decide(const BaDev& d)
{
    BaState& st = *d.st;
    if (st.done || st.setup_failed) return;
    const int tid = threadIdx.x, nt = blockDim.x;
    __shared__ int accept;
    __syncthreads();
    if (tid == 0) {
        accept = 0;
        const int it = st.it;
        if (!st.step_valid) {
            if (++st.invalid_streak >= 5) { st.done = 1; st.termination = GF_BA_FAILURE; }
            st.mu *= 10.0; st.reuse = 0;
            st.cost_hist[it] = st.x_cost; st.radius_hist[it] = st.radius;
        } else {
            st.invalid_streak = 0;
            const double x_cost = st.x_cost, cand = *(volatile double*)&st.acc_cost[st.cur ^ 1];     // candidate cost, summed by all CTAs of k_ba_eval(1)
            if (st.step_norm <= 1e-8 * (st.x_norm + 1e-8)) { st.done = 1; st.termination = GF_BA_CONVERGENCE_PARAMETER; st.cost_hist[it] = x_cost; st.radius_hist[it] = st.radius; }
            else if (fabs(x_cost - cand) <= 1e-6 * x_cost) { st.done = 1; st.termination = GF_BA_CONVERGENCE_FUNCTION; st.cost_hist[it] = x_cost; st.radius_hist[it] = st.radius; }
            else {
                double rel = (x_cost - cand) / st.model_change;
                if (rel > 1e-3) {
                    accept = 1; st.n_success++;
                    if (rel < 0.25) st.radius *= 0.5;
                    if (rel > 0.75) st.radius = fmax(st.radius, 3.0 * st.dogleg_norm);
                    st.mu = fmax(1e-8, 2.0 * st.mu / 10.0);
                    st.reuse = 0; st.need_linearize = 1;
                    st.radius_hist[it] = st.radius;          // cost_hist[it] is written when the new linearisation is adopted
                } else {
                    st.radius *= 0.5; st.reuse = 1;
                    st.cost_hist[it] = x_cost; st.radius_hist[it] = st.radius;
                }
            }
        }
    }
    __syncthreads();
    if (accept) { const int tot = X_FEAT + d.nfeat; for (int e = tid; e < tot; e += nt) d.X[e] = d.Xc[e]; }
}

// mode 0: linearise at X into the inactive accumulator (first linearisation); mode 1: linearise at the candidate Xc
// into the inactive accumulator (cost in acc_cost[inactive])
__device__ __forceinline__ void ba_eval_body(const BaDev& d, int mode)
{
    __shared__ double sJ[2 * PAIR_CHUNK][20];
    __shared__ double sR[2 * PAIR_CHUNK];
    __shared__ double sred[32];
    __shared__ double simu_J[15 * 30], simu_JU[15 * 30], simu_r[15], simu_ru[15];
    const BaState& st = *d.st;
    if (st.done || st.setup_failed) return;
#ifdef GF_PROFILE
    const long long t_eval0 = clock64();
#define PHMAX(k) do { if (tid == 0) atomicMax((unsigned long long*)&d.st->prof[k], (unsigned long long)(clock64() - t_eval0)); } while (0)
#else
#define PHMAX(k) do { } while (0)
#endif
    const int tid = threadIdx.x;
    const int tgt = st.cur ^ 1;            // inactive buffer
    if (mode == 0) { if (!st.need_linearize) return; }
    else if (!st.step_valid) return;
    // mode 1 linearises at the candidate: if k_ba_decide accepts the step this *is* the next linearisation (the same
    // arithmetic on the same numbers as re-evaluating at X after the copy), if it rejects it the buffer is simply
    // cleared again by the next k_ba_schur.  The target buffer was zeroed by k_ba_schur of this iteration.
    const double* X = mode == 0 ? d.X : d.Xc;
    double* costp = &d.st->acc_cost[tgt];
    const bool jac = true;
    const int b = blockIdx.x;
    if (b < d.n_pairs) {
        // ---------------- visual factors of one pose pair ----------------
        const int f0 = d.pair_start[b], f1 = d.pair_start[b + 1];
        const int pi = d.pair_ij[2 * b], pj = d.pair_ij[2 * b + 1];
        int cols[4] = {d.col_pose[pi], d.col_pose[pj], d.col_ex, d.col_td};
        const int bsz[4] = {6, 6, 6, 1}, boff[4] = {0, 6, 12, 18};
        double out0 = 0, out1 = 0;          // this thread's two entries of the 19x19 (+19 gradient) product
        double cost = 0;
        for (int c0 = f0; c0 < f1; c0 += PAIR_CHUNK) {
            int nf = min(PAIR_CHUNK, f1 - c0);
            if (tid < nf) {
                const gf_ba_visual_factor& f = d.vis[c0 + tid];
                double res[2], J[40];
                eval_visual(f, d.vis_sqrt_info, X + X_POSE + 7 * f.imu_i, X + X_POSE + 7 * f.imu_j, X + X_EX, X[X_FEAT + f.feature], X[X_TD], res, J, jac);
                double sc, rho = huber(res[0] * res[0] + res[1] * res[1], sc);
                cost += 0.5 * rho;
                if (jac) {
                    for (int r = 0; r < 2; r++) { for (int c = 0; c < 20; c++) sJ[2 * tid + r][c] = sc * J[r * 20 + c]; sR[2 * tid + r] = sc * res[r]; }
                    int cf = d.col_feat[f.feature];
                    if (cf >= 0 && d.lm_dense) {      // marginalisation: the landmark is a column of the dense matrix
                        double j0 = sc * J[19], j1 = sc * J[39], r0 = sc * res[0], r1 = sc * res[1];
                        double* H = acc_H(d, tgt);
                        atomicAdd(&H[(size_t)cf * d.nc + cf], j0 * j0 + j1 * j1);
                        atomicAdd(&acc_g(d, tgt)[cf], j0 * r0 + j1 * r1);
                        for (int q = 0; q < 4; q++) if (cols[q] >= 0)
                            for (int k = 0; k < bsz[q]; k++) {
                                const double w_ = j0 * sc * J[boff[q] + k] + j1 * sc * J[20 + boff[q] + k];
                                atomicAdd(&H[(size_t)cf * d.nc + cols[q] + k], w_);
                                atomicAdd(&H[(size_t)(cols[q] + k) * d.nc + cf], w_);
                            }
                    } else if (cf >= 0) {      // landmark terms: h_ll, g_l, W[l][camera cols]
                        int l = cf - d.nc;
                        double j0 = sc * J[19], j1 = sc * J[39], r0 = sc * res[0], r1 = sc * res[1];
                        atomicAdd(&acc_hll(d, tgt)[l], j0 * j0 + j1 * j1);
                        atomicAdd(&acc_g(d, tgt)[cf], j0 * r0 + j1 * r1);
                        double* Wl = acc_W(d, tgt) + (size_t)l * d.nc;
                        for (int q = 0; q < 4; q++) if (cols[q] >= 0)
                            for (int k = 0; k < bsz[q]; k++) atomicAdd(&Wl[cols[q] + k], j0 * sc * J[boff[q] + k] + j1 * sc * J[20 + boff[q] + k]);
                    }
                }
            }
            if (jac) {
                __syncthreads();
                // 19x19 J^T J entries + 19 J^T r entries = 380 outputs, two per thread
                for (int o = tid, slot = 0; o < 380; o += PAIR_THREADS, slot++) {
                    double s = 0;
                    if (o < 361) { int a = o / 19, c = o - a * 19; for (int r = 0; r < 2 * nf; r++) s += sJ[r][a] * sJ[r][c]; }
                    else { int a = o - 361; for (int r = 0; r < 2 * nf; r++) s += sJ[r][a] * sR[r]; }
                    if (slot == 0) out0 += s; else out1 += s;
                }
                __syncthreads();
            }
        }
        if (jac) {
            auto col_of = [&](int a) { int q = a < 6 ? 0 : a < 12 ? 1 : a < 18 ? 2 : 3; return cols[q] < 0 ? -1 : cols[q] + (a - boff[q]); };
            for (int o = tid, slot = 0; o < 380; o += PAIR_THREADS, slot++) {
                double v = slot == 0 ? out0 : out1;
                if (o < 361) { int a = o / 19, c = o - a * 19; int ca = col_of(a), cc = col_of(c); if (ca >= 0 && cc >= 0) atomicAdd(&acc_H(d, tgt)[(size_t)ca * d.nc + cc], v); }
                else { int ca = col_of(o - 361); if (ca >= 0) atomicAdd(&acc_g(d, tgt)[ca], v); }
            }
        }
        cost = block_reduce_sum(cost, sred);
        if (tid == 0 && cost != 0.0) atomicAdd(costp, cost);
        PHMAX(14);
    } else if (b < d.n_pairs + d.n_imu) {
        // ---------------- one IMU factor ----------------
        const int m = b - d.n_pairs;
        const gf_ba_imu_factor& f = d.imu[m];
        const double* U = d.imu_sqrt + 225 * m;
        if (tid == 0) eval_imu_raw(f, d.gravity, X + X_POSE + 7 * f.i, X + X_SB + 9 * f.i, X + X_POSE + 7 * f.j, X + X_SB + 9 * f.j, simu_r, simu_J, jac);
        if (mode == 0 && (tid >> 5) == 1) {          // first linearisation: the sqrt-information matrix of this factor, once per solve, on a second warp
            const bool ok = imu_sqrt_info_warp(f.covariance, simu_JU, d.imu_sqrt + 225 * m, tid & 31);
            if (!ok && (tid & 31) == 0) d.st->setup_failed = 1;      // sticky; zeroed by the host; every later kernel returns at once
        }
        __syncthreads();
        if (tid < 15) { double s = 0; for (int k = 0; k < 15; k++) s += U[tid * 15 + k] * simu_r[k]; simu_ru[tid] = s; }
        if (jac) for (int o = tid; o < 450; o += PAIR_THREADS) { int r = o / 30, c = o - r * 30; double s = 0; for (int k = 0; k < 15; k++) s += U[r * 15 + k] * simu_J[k * 30 + c]; simu_JU[o] = s; }
        __syncthreads();
        if (tid == 0) { double c = 0; for (int k = 0; k < 15; k++) c += 0.5 * simu_ru[k] * simu_ru[k]; atomicAdd(costp, c); }
        if (jac) {
            int cols[4] = {d.col_pose[f.i], d.col_sb[f.i], d.col_pose[f.j], d.col_sb[f.j]};
            const int boff[4] = {0, 6, 15, 21};
            auto col_of = [&](int a) { int q = a < 6 ? 0 : a < 15 ? 1 : a < 21 ? 2 : 3; return cols[q] < 0 ? -1 : cols[q] + (a - boff[q]); };
            for (int o = tid; o < 930; o += PAIR_THREADS) {
                if (o < 900) {
                    int a = o / 30, c = o - a * 30; int ca = col_of(a), cc = col_of(c);
                    if (ca < 0 || cc < 0) continue;
                    double s = 0; for (int r = 0; r < 15; r++) s += simu_JU[r * 30 + a] * simu_JU[r * 30 + c];
                    atomicAdd(&acc_H(d, tgt)[(size_t)ca * d.nc + cc], s);
                } else {
                    int a = o - 900, ca = col_of(a);
                    if (ca < 0) continue;
                    double s = 0; for (int r = 0; r < 15; r++) s += simu_JU[r * 30 + a] * simu_ru[r];
                    atomicAdd(&acc_g(d, tgt)[ca], s);
                }
            }
        }
        __syncthreads();
        PHMAX(15);
    } else if (b < d.n_pairs + d.n_imu + d.n_wheel) {
        // ---------------- one wheel factor (6 residuals, 22 local columns) ----------------
        const gf_ba_wheel_factor& f = d.wheel[b - d.n_pairs - d.n_imu];
        double* wJ = simu_J;          // [6][WHEEL_COLS]
        double* wr = simu_r;          // [6]
        if (tid == 0) {
            const bool ok = eval_wheel(f, X + X_POSE + 7 * f.i, X + X_POSE + 7 * f.j, X + X_EXW, X[X_IX], X[X_IX + 1], X[X_IX + 2], X[X_TDW], wr, wJ, jac, simu_JU);
            if (!ok) for (int k = 0; k < 6; k++) { wr[k] = 0.0; for (int c = 0; c < WHEEL_COLS; c++) wJ[k * WHEEL_COLS + c] = 0.0; }
            double c = 0; for (int k = 0; k < 6; k++) c += 0.5 * wr[k] * wr[k];
            atomicAdd(costp, c);
        }
        __syncthreads();
        auto col_of = [&](int a) {
            if (a < 6) return d.col_pose[f.i] < 0 ? -1 : d.col_pose[f.i] + a;
            if (a < 12) return d.col_pose[f.j] < 0 ? -1 : d.col_pose[f.j] + a - 6;
            if (a < 18) return d.col_exw < 0 ? -1 : d.col_exw + a - 12;
            if (a < 21) return d.col_ix[a - 18];
            return d.col_tdw;
        };
        for (int o = tid; o < WHEEL_COLS * (WHEEL_COLS + 1); o += PAIR_THREADS) {
            if (o < WHEEL_COLS * WHEEL_COLS) {
                const int a = o / WHEEL_COLS, c = o - a * WHEEL_COLS, ca = col_of(a), cc = col_of(c);
                if (ca < 0 || cc < 0) continue;
                double s = 0; for (int r = 0; r < 6; r++) s += wJ[r * WHEEL_COLS + a] * wJ[r * WHEEL_COLS + c];
                atomicAdd(&acc_H(d, tgt)[(size_t)ca * d.nc + cc], s);
            } else {
                const int a = o - WHEEL_COLS * WHEEL_COLS, ca = col_of(a);
                if (ca < 0) continue;
                double s = 0; for (int r = 0; r < 6; r++) s += wJ[r * WHEEL_COLS + a] * wr[r];
                atomicAdd(&acc_g(d, tgt)[ca], s);
            }
        }
    } else if (d.n_plane > 0 && b == d.n_pairs + d.n_imu + d.n_wheel) {
        // ---------------- all plane factors (3 residuals, 16 local columns each): one thread per factor ----------------
        if (tid < d.n_plane) {
            const int fi = d.plane_frames[tid];
            double r3[3], Jp[3 * PLANE_COLS];
            eval_plane(X + X_POSE + 7 * fi, X + X_EXW, X + X_PR, X[X_PZ], d.plane_sinfo, r3, Jp, jac);
            atomicAdd(costp, 0.5 * (r3[0] * r3[0] + r3[1] * r3[1] + r3[2] * r3[2]));
            auto col_of = [&](int a) {
                if (a < 6) return d.col_pose[fi] < 0 ? -1 : d.col_pose[fi] + a;
                if (a < 12) return d.col_exw < 0 ? -1 : d.col_exw + a - 6;
                if (a < 15) return d.col_pr < 0 ? -1 : d.col_pr + a - 12;
                return d.col_pz;
            };
            for (int a = 0; a < PLANE_COLS; a++) {
                const int ca = col_of(a);
                if (ca < 0) continue;
                double gsum = 0; for (int r = 0; r < 3; r++) gsum += Jp[r * PLANE_COLS + a] * r3[r];
                atomicAdd(&acc_g(d, tgt)[ca], gsum);
                for (int c = 0; c < PLANE_COLS; c++) {
                    const int cc = col_of(c);
                    if (cc < 0) continue;
                    double hsum = 0; for (int r = 0; r < 3; r++) hsum += Jp[r * PLANE_COLS + a] * Jp[r * PLANE_COLS + c];
                    if (hsum != 0.0) atomicAdd(&acc_H(d, tgt)[(size_t)ca * d.nc + cc], hsum);
                }
            }
        }
    } else if (b == d.n_pairs + d.n_imu + d.n_wheel + (d.n_plane > 0 ? 1 : 0) && d.pn > 0) {
        // ---------------- marginalisation prior: r = r0 + J0 dx, g += J0^T r (H_prior is constant) ----------------
        extern __shared__ double sdyn[];    // dx[pn], r[pn]
        double* dx = sdyn; double* rr = sdyn + d.pn;
        const int pn = d.pn;
        for (int blk = tid; blk < d.pnb; blk += PAIR_THREADS) {
            int kind = d.pkind[blk], idx = d.pidx[blk];
            const double* x0 = d.px0 + d.pxoff[blk];
            const double* x = kind == GF_BA_BLOCK_POSE ? X + X_POSE + 7 * d.pindex[blk] : kind == GF_BA_BLOCK_SPEEDBIAS ? X + X_SB + 9 * d.pindex[blk]
                              : kind == GF_BA_BLOCK_EX_POSE ? X + X_EX : kind == GF_BA_BLOCK_TD ? X + X_TD : kind == GF_BA_BLOCK_EX_WHEEL ? X + X_EXW
                              : kind == GF_BA_BLOCK_SX ? X + X_IX : kind == GF_BA_BLOCK_SY ? X + X_IX + 1 : kind == GF_BA_BLOCK_SW ? X + X_IX + 2
                              : kind == GF_BA_BLOCK_TD_WHEEL ? X + X_TDW : kind == GF_BA_BLOCK_PLANE_R ? X + X_PR : X + X_PZ;
            int size = (kind == GF_BA_BLOCK_POSE || kind == GF_BA_BLOCK_EX_POSE || kind == GF_BA_BLOCK_EX_WHEEL) ? 7 : kind == GF_BA_BLOCK_SPEEDBIAS ? 9 : kind == GF_BA_BLOCK_PLANE_R ? 4 : 1;
            if (size != 7) for (int k = 0; k < size; k++) dx[idx + k] = x[k] - x0[k];
            else {
                for (int k = 0; k < 3; k++) dx[idx + k] = x[k] - x0[k];
                double qi[4], dq[4]; q_inv(x0 + 3, qi); q_mul(qi, x + 3, dq);
                double sgn = (dq[3] >= 0) ? 1.0 : -1.0;
                for (int k = 0; k < 3; k++) dx[idx + 3 + k] = 2.0 * sgn * dq[k];
            }
        }
        __syncthreads();
        double cost = 0;
        for (int i = tid; i < pn; i += PAIR_THREADS) {
            double v = d.pr0[i];
            for (int k = 0; k < pn; k++) v += d.pJ[(size_t)i * pn + k] * dx[k];
            rr[i] = v; cost += 0.5 * v * v;
        }
        cost = block_reduce_sum(cost, sred);
        if (tid == 0) atomicAdd(costp, cost);
        if (jac)
            for (int c = tid; c < pn; c += PAIR_THREADS) {
                int lc = d.pcol[c];
                if (lc < 0) continue;
                double s = 0;
                for (int k = 0; k < pn; k++) s += d.pJ[(size_t)k * pn + c] * rr[k];
                atomicAdd(&acc_g(d, tgt)[lc], s);
            }
        __syncthreads();
        PHMAX(13);
    }
}

__global__ void __launch_bounds__(PAIR_THREADS) k_ba_eval(const BaDev* __restrict__ wins, int mode)
{
    __shared__ BaDev sd;
    gf::gf_pdl_trigger();      // no-ops unless launched with a programmatic dependency (gf_ba_solve)
    load_window(sd, wins + blockIdx.y);
    gf::gf_pdl_wait();
    __syncthreads();
    const BaDev& d = sd;
    if ((int)blockIdx.x >= d.eval_grid) return;
    ba_eval_body(d, mode);
    if (mode == 1) {
        // the last of the window's CTAs to finish takes the decision (accept / reject, radius, mu, convergence): no separate launch
        __shared__ int s_last;
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            const unsigned int t = atomicAdd(&d.st->eval_ticket, 1u);
            s_last = (t == (unsigned)d.eval_grid - 1);
        }
        __syncthreads();
        if (s_last) {
            __threadfence();
            if (threadIdx.x == 0) d.st->eval_ticket = 0u;
            ba_decide(d);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// ambient-space helpers over the non-constant blocks
// Y = X (+) delta on the FREE blocks only (constant blocks of Y already equal X: the host uploads the candidate as a copy of X and nothing else
// ever writes them) and, in the same pass, this thread's share of |X - Y|^2 and max |X - Y| over the ambient coordinates.
__device__ inline void plus_free(const BaDev& d, const double* X, const double* delta, double* Y, int tid, int nt, double& s2, double& mx)
{
    s2 = 0; mx = 0;
    auto put = [&](int off, int size, const double* nv) {      // Y := nv and |X - nv| from the registers (Y is not read back)
        for (int k = 0; k < size; k++) { Y[off + k] = nv[k]; const double v = X[off + k] - nv[k]; s2 += v * v; mx = fmax(mx, fabs(v)); }
    };
    for (int f = tid; f < d.F; f += nt) {
        if (d.col_pose[f] >= 0) { double o[7]; pose_plus(X + X_POSE + 7 * f, delta + d.col_pose[f], o); put(X_POSE + 7 * f, 7, o); }
        if (d.col_sb[f] >= 0) { double o[9]; for (int k = 0; k < 9; k++) o[k] = X[X_SB + 9 * f + k] + delta[d.col_sb[f] + k]; put(X_SB + 9 * f, 9, o); }
    }
    if (tid == nt - 1) {
        if (d.col_ex >= 0) { double o[7]; pose_plus(X + X_EX, delta + d.col_ex, o); put(X_EX, 7, o); }
        if (d.col_td >= 0) { const double o = X[X_TD] + delta[d.col_td]; put(X_TD, 1, &o); }
    }
    if (tid == nt - 2) {
        if (d.col_exw >= 0) {    // PoseSubsetParameterization: masked components are zeroed inside Plus only
            double dd[6], o[7];
            for (int k = 0; k < 6; k++) dd[k] = ((d.exw_mask >> k) & 1) ? 0.0 : delta[d.col_exw + k];
            pose_plus(X + X_EXW, dd, o); put(X_EXW, 7, o);
        }
        for (int k = 0; k < 3; k++) if (d.col_ix[k] >= 0) { const double o = X[X_IX + k] + delta[d.col_ix[k]]; put(X_IX + k, 1, &o); }
        if (d.col_tdw >= 0) { const double o = X[X_TDW] + delta[d.col_tdw]; put(X_TDW, 1, &o); }
    }
    if (tid == nt - 3 && d.col_pr >= 0) {     // OrientationSubsetParameterization::Plus
        double dd[3], dq[4], qn[4];
        for (int k = 0; k < 3; k++) dd[k] = ((d.pr_mask >> k) & 1) ? 0.0 : delta[d.col_pr + k];
        delta_q(dd, dq); q_mul(X + X_PR, dq, qn); q_normalize(qn);
        put(X_PR, 4, qn);
        const double o = X[X_PZ] + delta[d.col_pz]; put(X_PZ, 1, &o);
    }
    for (int k = tid; k < d.nfeat; k += nt) { const int c = d.col_feat[k]; if (c >= 0) { const double o = X[X_FEAT + k] + delta[c]; put(X_FEAT + k, 1, &o); } }
}
// sum of squares of A over the ambient coordinates of the free blocks
__device__ inline double free_norm2(const BaDev& d, const double* A, int tid, int nt)
{
    double s2 = 0;
    auto acc = [&](int off, int size) { for (int k = 0; k < size; k++) s2 += A[off + k] * A[off + k]; };
    for (int f = tid; f < d.F; f += nt) { if (d.col_pose[f] >= 0) acc(X_POSE + 7 * f, 7); if (d.col_sb[f] >= 0) acc(X_SB + 9 * f, 9); }
    if (tid == nt - 1) {
        if (d.col_ex >= 0) acc(X_EX, 7);
        if (d.col_td >= 0) acc(X_TD, 1);
        if (d.col_exw >= 0) acc(X_EXW, 7);
        for (int k = 0; k < 3; k++) if (d.col_ix[k] >= 0) acc(X_IX + k, 1);
        if (d.col_tdw >= 0) acc(X_TDW, 1);
        if (d.col_pr >= 0) { acc(X_PR, 4); acc(X_PZ, 1); }
    }
    for (int k = tid; k < d.nfeat; k += nt) if (d.col_feat[k] >= 0) acc(X_FEAT + k, 1);
    return s2;
}
__device__ __forceinline__ double block_reduce_max(double v, double* sh)
{
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    double t = 0;
    if (w == 0) {
        t = (l < nw) ? sh[l] : 0.0;
        for (int o = 16; o > 0; o >>= 1) t = fmax(t, __shfl_xor_sync(0xffffffffu, t, o));
        if (l == 0) sh[0] = t;
    }
    __syncthreads();
    t = sh[0];
    __syncthreads();
    return t;
}
// N sums at once over a CTA of <= 8 warps: two barriers in total; every thread ends up with all N totals.  sh: N * 8 doubles.
template <int N>
__device__ __forceinline__ void block_reduce_sums(double (&v)[N], double* sh)
{
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int k = 0; k < N; k++)
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    __syncthreads();
    if (l == 0) {
#pragma unroll
        for (int k = 0; k < N; k++) sh[k * 8 + w] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; k++) { double t = 0; for (int q = 0; q < nw; q++) t += sh[k * 8 + q]; v[k] = t; }
}

// ------------------------------------------------------------------------------------------------
// Reduced camera system for the Gauss-Newton solve, (H' + mu D^2) with the free landmarks eliminated (Ceres' SchurEliminator):
//   S[a][b] = H'[a][b] + [a==b] mu D_a^2 - s_a s_b sum_l c_l W[l][a] W[l][b],   c_l = s_l^2 / (h'_ll + mu D_l^2)
//   rhs[b]  = g'[b] - s_b sum_l c_l W[l][b] g_l                (primes = Jacobi-scaled; stored as row nc of the system)
// One warp per 8x8 tile (I,J), I >= J, of the (nc+1)-row augmented system: the rank-L update sum_l c_l w_la w_lb is a chain
// of DMMA.8x8x4 over the landmarks (A[m][k] = c_l W[l0+k][8I+m], B[k][n] = W[l0+k][8J+n]; the right-hand side is the same
// product with "column nc" of W := g_l).  The tile is written row-major to Sg[tix(I,J)*64], which k_ba_step's left-looking
// Cholesky streams.  ss / sv / cl: Jacobi scale, Cauchy direction v_c = g_c s_c^2 / D_c^2 (null: no Cauchy terms) and c_l.
__device__ __forceinline__ void schur_tile(const BaDev& d, const double* __restrict__ H, const double* __restrict__ g, const double* __restrict__ W,
                                           const double* __restrict__ ss, const double* __restrict__ sv, const double* __restrict__ cl, double mu,
                                           int I, int J, int lane, double& num, double& den)
{
    const int nc = d.nc, L = d.L;
    const double* Hp = d.Hp;
    const int ka = lane & 3, ia = 8 * I + (lane >> 2), ib = 8 * J + (lane >> 2);
    auto wx = [&](int l, int c) { return c < nc ? W[(size_t)l * nc + c] : (c == nc ? g[nc + l] : 0.0); };
    double acc0[2] = {0.0, 0.0}, acc1[2] = {0.0, 0.0};
    for (int l0 = 0; l0 < L; l0 += 64) {           // 32 loads from L2 in flight per lane, then sixteen MMAs on two accumulators
        double av[16], bv[16];
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const int l = l0 + 4 * k + ka;
            av[k] = 0.0; bv[k] = 0.0;
            if (l < L) { av[k] = wx(l, ia); bv[k] = wx(l, ib); }
        }
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const int l = l0 + 4 * k + ka;
            const double ak = l < L ? cl[l] * av[k] : 0.0;
            if (k & 1) dmma884(acc1[0], acc1[1], ak, bv[k]); else dmma884(acc0[0], acc0[1], ak, bv[k]);
        }
    }
    const int a = 8 * I + (lane >> 2);
    double out[2];
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const int b = 8 * J + 2 * (lane & 3) + e;
        const double acc = acc0[e] + acc1[e];
        double v;
        if (a > nc || b > nc) v = (a == b) ? 1.0 : 0.0;                      // padding rows of the last tile row
        else if (a == nc) v = (b == nc) ? 1.0 : (g[b] - acc) * ss[b];       // right-hand side (s_nc = 1)
        else if (b == nc) v = 0.0;                                           // above the diagonal of the last tile: unused
        else {
            const double sa = ss[a], sb = ss[b];
            const double hab = H[(size_t)a * nc + b] + Hp[(size_t)a * nc + b];
            v = hab * sa * sb;
            if (a == b) {
                double hd = v; hd = hd < 1e-6 ? 1e-6 : (hd > 1e32 ? 1e32 : hd); v += mu * hd;
                if (sv) { const double gsa = g[a] * sa / sqrt(hd); num += gsa * gsa; }
            }
            v -= acc * sa * sb;
            if (sv && b <= a) den += (a == b ? 1.0 : 2.0) * sv[a] * hab * sv[b];
        }
        out[e] = v;
    }
    *reinterpret_cast<double2*>(d.Sg + (size_t)tix(I, J) * 64 + (lane >> 2) * 8 + 2 * (lane & 3)) = make_double2(out[0], out[1]);
}

__global__ void __launch_bounds__(SCHUR_WARPS * 32) k_ba_schur(const BaDev* __restrict__ wins)
{
    extern __shared__ double ssm[];                // tile CTAs: cl[L] | ss[nc+1] | sv[nc];  last CTA: delta[n]
    __shared__ double sred2[2 * SCHUR_WARPS];
    __shared__ BaDev sd;
    gf::gf_pdl_trigger();
    load_window(sd, wins + blockIdx.y);
    gf::gf_pdl_wait();
    __syncthreads();
    const BaDev& d = sd;
    const int grid = d.schur_grid;                 // this window's CTAs: the tile CTAs, then the one that prepares the vectors
    if ((int)blockIdx.x >= grid) return;
    const BaState& st = *d.st;
    if (st.done || st.setup_failed) return;
    const bool fresh = st.need_linearize != 0;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nt = blockDim.x;
    {   // clear the accumulator that is free during this iteration: k_ba_eval(1) linearises the candidate into it
        const int freeb = fresh ? st.cur : (st.cur ^ 1);
        const size_t tot = acc_size(d.nc, d.L);
        const size_t nthr = (size_t)grid * blockDim.x;
        const size_t me = (size_t)blockIdx.x * blockDim.x + tid;
        for (size_t e = me; e < tot; e += nthr) d.acc[freeb][e] = 0.0;
        if (me == 0) d.st->acc_cost[freeb] = 0.0;
    }
    if (!fresh && st.reuse) return;               // the previous Gauss-Newton step is still valid
    const int cur = fresh ? (st.cur ^ 1) : st.cur;
    const int nc = d.nc, L = d.L, n = d.n;
    const double* H = acc_H(d, cur); const double* Hp = d.Hp; const double* g = acc_g(d, cur);
    const double* W = acc_W(d, cur); const double* hll = acc_hll(d, cur);
    const bool first = st.first != 0;
    const double mu = st.mu;
    // everything (scale, D, c_l) is recomputed locally from the accumulators so that this kernel can run before k_ba_step adopts them
    auto scale_of = [&](int c) { return first ? 1.0 / (1.0 + sqrt(c < nc ? H[(size_t)c * nc + c] + Hp[(size_t)c * nc + c] : hll[c - nc])) : d.scale[c]; };
    if ((int)blockIdx.x == grid - 1) {
        // ---- the last CTA prepares what k_ba_step needs before it can factor: D, gs = g'/D, e_l = 1 / (h'_ll + mu D_l^2), the
        // Jacobi scale (iteration 0) and, for a fresh linearisation, |x| and the gradient max-norm |x - Plus(x, -g)|_inf
        // (TrustRegionMinimizer's gradient tolerance test) -- off the single-CTA critical path of k_ba_step ----
        double* dl = ssm;
        for (int c = tid; c < n; c += nt) {
            const double sc_ = scale_of(c);
            double hd = (c < nc ? H[(size_t)c * nc + c] + Hp[(size_t)c * nc + c] : hll[c - nc]) * sc_ * sc_;
            const double hraw = hd;
            hd = hd < 1e-6 ? 1e-6 : (hd > 1e32 ? 1e32 : hd);
            const double D = sqrt(hd), gc = g[c];
            if (first) d.scale[c] = sc_;
            d.diag[c] = D;
            d.gs[c] = gc * sc_ / D;
            if (c >= nc) d.gn[c] = 1.0 / (hraw + mu * hd);
            dl[c] = -gc;
        }
        if (fresh) {
            __syncthreads();
            double s2, mx;
            plus_free(d, d.X, dl, d.Xc, tid, nt, s2, mx);            // Xc is free scratch here: the accepted candidate has become X
            mx = block_reduce_max(mx, sred2);
            double xs2 = free_norm2(d, d.X, tid, nt);
            xs2 = block_reduce_sum(xs2, sred2);
            if (tid == 0) { d.st->grad_max = mx; d.st->x_norm = sqrt(xs2); }
        }
        return;
    }
    if (st.it >= st.max_iter) return;             // the closing launch only needs the norms
    double* cl = ssm; double* ss = ssm + L; double* sv = ss + nc + 1;
    for (int l = tid; l < L; l += nt) {
        const double sl = scale_of(nc + l), hd = hll[l] * sl * sl;
        const double hc = hd < 1e-6 ? 1e-6 : (hd > 1e32 ? 1e32 : hd);     // D_l^2
        cl[l] = sl * sl / (hd + mu * hc);
    }
    for (int c = tid; c <= nc; c += nt) {
        if (c == nc) { ss[c] = 1.0; continue; }
        const double sc_ = scale_of(c);
        double hd = (H[(size_t)c * nc + c] + Hp[(size_t)c * nc + c]) * sc_ * sc_;
        hd = hd < 1e-6 ? 1e-6 : (hd > 1e32 ? 1e32 : hd);
        ss[c] = sc_; sv[c] = g[c] * sc_ * sc_ / hd;        // v = gs / D (times the Jacobi scale, because H is unscaled)
    }
    __syncthreads();
    const int n8 = (nc + 8) >> 3, ntiles = n8 * (n8 + 1) / 2;
    double num = 0, den = 0;
    const int gw = blockIdx.x * SCHUR_WARPS + warp, nw = (grid - 1) * SCHUR_WARPS;
    for (int t = gw; t < ntiles; t += nw) {
        int I = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
        while (tix(I + 1, 0) <= t) I++;
        while (tix(I, 0) > t) I--;
        schur_tile(d, H, g, W, ss, sv, cl, mu, I, t - tix(I, 0), lane, num, den);
    }
    // landmark part of the Cauchy quadratic form: 2 v_l (W v_c)_l + h_ll v_l^2, warp per landmark (taken from the back of the
    // warp list: the front warps own a tile each)
    for (int l = nw - 1 - gw; l < L; l += nw) {
        double t = 0;
        for (int c0 = 0; c0 < nc; c0 += 256) {
            double wv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) { const int c = c0 + 32 * k + lane; wv[k] = c < nc ? W[(size_t)l * nc + c] : 0.0; }
#pragma unroll
            for (int k = 0; k < 8; k++) { const int c = c0 + 32 * k + lane; if (c < nc) t = fma(wv[k], sv[c], t); }
        }
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) {
            const double sl = scale_of(nc + l), hd = hll[l] * sl * sl;
            const double hc = hd < 1e-6 ? 1e-6 : (hd > 1e32 ? 1e32 : hd);
            const double vl = g[nc + l] * sl * sl / hc;
            den += 2.0 * vl * t + hll[l] * vl * vl;
            const double gsl = g[nc + l] * sl / sqrt(hc); num += gsl * gsl;
        }
    }
    for (int o = 16; o > 0; o >>= 1) { num += __shfl_xor_sync(0xffffffffu, num, o); den += __shfl_xor_sync(0xffffffffu, den, o); }
    if (lane == 0) { sred2[warp] = den; sred2[SCHUR_WARPS + warp] = num; }
    __syncthreads();
    if (tid == 0) {
        double t = 0, u = 0;
        for (int k = 0; k < SCHUR_WARPS; k++) { t += sred2[k]; u += sred2[SCHUR_WARPS + k]; }
        if (t != 0.0) atomicAdd(&d.st->cauchy_den, t);
        if (u != 0.0) atomicAdd(&d.st->cauchy_num, u);
    }
}

// DoglegStrategy::ComputeStep + TrustRegionMinimizer::ComputeTrustRegionStep + candidate point, one CTA.
// Dynamic shared memory: factor tiles (<= tile_cap; first filled with the reduced system by a TMA bulk copy) | inverses of the
// diagonal tiles | 2 scratch tiles | last diagonal tile | y.  After the back substitution the tile area is dead and holds delta.
// One CTA per window of `list` (the windows of a batch that take this instantiation).
template <int R, bool SPILL>
__global__ void __launch_bounds__(RB_THREADS) k_ba_step(const BaDev* __restrict__ wins, const int* __restrict__ list)
{
    extern __shared__ __align__(128) double S[];
    __shared__ double sred[64];
    __shared__ __align__(8) unsigned long long mbar;
    __shared__ int s_fail, s_go;
    __shared__ BaDev sd;
    gf::gf_pdl_trigger();
    load_window(sd, wins + list[blockIdx.y]);
    gf::gf_pdl_wait();
    __syncthreads();
    const BaDev& d = sd;
    BaState& st = *d.st;
    if (st.done || st.setup_failed) return;
    const int tid = threadIdx.x, nt = blockDim.x, warp = tid >> 5, lane = tid & 31, nwarp = nt >> 5;
    const int nc = d.nc, L = d.L, n = d.n;
    const int n8 = (nc + 8) >> 3, ntiles = n8 * (n8 + 1) / 2, ntl = min(ntiles, d.tile_cap);
    TileStoreT<SPILL> T; T.sb = ch_tiles_u32(); T.Lg = d.Lg; T.cap = d.tile_cap;
    double* Linv = S + (size_t)64 * ntl;
    double* S8 = Linv + 64 * n8; double* Ld = S8 + 128; double* yc = Ld + 64; double* zz = yc + ((nc + 8) & ~7);
    const long long t_kernel0 = clock64();      // always on (two clock reads per launch): SM cycles of the launches that took a step
#ifdef GF_PROFILE
    long long t_last = clock64();
#define PH(k) do { if (tid == 0) { long long t_ = clock64(); st.prof[k] += t_ - t_last; t_last = t_; } } while (0)
#else
#define PH(k) do { } while (0)
#endif
    if (tid == 0) {
        // ---- adoption of a fresh linearisation (its vectors and norms were prepared by k_ba_schur) + iteration bookkeeping ----
        int go = 1;
        if (st.need_linearize) {
            st.cur ^= 1; st.need_linearize = 0; st.x_cost = st.acc_cost[st.cur];
            if (st.first) { st.cost_hist[0] = st.x_cost; st.radius_hist[0] = st.radius; st.first = 0; }
            else st.cost_hist[st.it] = st.x_cost;          // cost after the accepted step of iteration `it`
            if (st.grad_max <= 1e-10 || n == 0) { st.done = 1; st.termination = GF_BA_CONVERGENCE_GRADIENT; go = 0; }
            st.reuse = 0;
        }
        if (go && (st.it >= st.max_iter || st.radius < 1e-32)) { st.done = 1; st.termination = GF_BA_NO_CONVERGENCE; go = 0; }
        if (go) {
            st.it++; st.step_valid = 0; st.solver_failed = 0;
            ch_mbar_init(&mbar, 1);
            if (!st.reuse) chol_issue_load(d.Sg, S, ntl, &mbar);      // the copy engine streams the reduced system in while the CTA gets going
        }
        s_go = go; s_fail = 0;
    }
    __syncthreads();
    if (!s_go) return;
    PH(0);   // adoption + bookkeeping
    const int cur = st.cur;
    const double* g = acc_g(d, cur); const double* W = acc_W(d, cur); const double* hll = acc_hll(d, cur);
    const double* H = acc_H(d, cur);
    const double* sc = d.scale;
    if (!st.reuse) {
        if (tid == 0) { st.alpha = st.cauchy_num / st.cauchy_den; st.cauchy_num = 0.0; st.cauchy_den = 0.0; }   // accumulated by k_ba_schur
        // ---- ComputeGaussNewtonStep: (H' + mu D^2) y = g' by Schur complement on the landmarks + Cholesky ----
        unsigned ld_phase = 0;
        bool first_try = true;
        while (true) {
            const double mu = st.mu;
            if (!first_try) {
                // retry with a larger mu (rare): e_l and the reduced system are rebuilt here, by this CTA alone
                __syncthreads();
                if (tid == 0) s_fail = 0;
                for (int l = tid; l < L; l += nt) {
                    const double v = hll[l] * sc[nc + l] * sc[nc + l] + mu * d.diag[nc + l] * d.diag[nc + l];
                    d.gn[nc + l] = 1.0 / v;
                    d.step[nc + l] = sc[nc + l] * sc[nc + l] / v;                               // c_l (scratch)
                }
                __syncthreads();
                double dummy0 = 0, dummy1 = 0;
                for (int t = warp; t < ntiles; t += nwarp) {
                    int I = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
                    while (tix(I + 1, 0) <= t) I++;
                    while (tix(I, 0) > t) I--;
                    schur_tile(d, H, g, W, sc, nullptr, d.step + nc, mu, I, t - tix(I, 0), lane, dummy0, dummy1);
                }
                __threadfence();
                asm volatile("fence.proxy.async;" ::: "memory");                                // generic writes (dead factor, new Sg) before the async-proxy refill
                __syncthreads();
                if (tid == 0) chol_issue_load(d.Sg, S, ntl, &mbar);
            }
            first_try = false;
            if (ntl > 0) ch_mbar_wait(&mbar, ld_phase & 1);
            ld_phase++;
            PH(2);   // reduced system in shared memory
            const bool ok_f = chol_factor<R, SPILL>(d.Sg, T, Linv, S8, Ld, nc, n8, &s_fail);
            PH(3);   // Cholesky
            bool ok = ok_f;
            if (ok) {
                chol_backsubst(T, Linv, Ld, yc, zz, nc);
                __syncthreads();
                int bad = 0;
                for (int c = tid; c < nc; c += nt) if (!isfinite(yc[c])) bad = 1;
                ok = __syncthreads_or(bad) == 0;
            }
            PH(4);   // back substitution
            if (ok) {
                // y_l = e_l (g'_l - w'_l . y_c) ; gn = -D y.  v = s .* y_c staged once; four landmarks per warp pass keep 4 x nc/32 loads in flight
                double* vbuf = nc <= 64 * ntl ? S : d.step;                                      // the factor is dead: the tile area holds v
                for (int c = tid; c < nc; c += nt) vbuf[c] = sc[c] * yc[c];
                __syncthreads();
                for (int l0 = 4 * warp; l0 < L; l0 += 4 * nwarp) {
                    double t[4] = {0, 0, 0, 0};
                    for (int b0 = 0; b0 < nc; b0 += 192) {            // 6 x 4 loads from L2 in flight per lane, then the FMAs
                        double wv[6][4];
#pragma unroll
                        for (int k = 0; k < 6; k++) {
                            const int b = b0 + 32 * k + lane;
#pragma unroll
                            for (int q = 0; q < 4; q++) wv[k][q] = (b < nc && l0 + q < L) ? W[(size_t)(l0 + q) * nc + b] : 0.0;
                        }
#pragma unroll
                        for (int k = 0; k < 6; k++) {
                            const int b = b0 + 32 * k + lane;
                            const double vb = b < nc ? vbuf[b] : 0.0;
#pragma unroll
                            for (int q = 0; q < 4; q++) t[q] = fma(wv[k][q], vb, t[q]);
                        }
                    }
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        for (int o = 16; o > 0; o >>= 1) t[q] += __shfl_xor_sync(0xffffffffu, t[q], o);
                        const int l = l0 + q;
                        if (lane == 0 && l < L) d.gn[nc + l] = -d.diag[nc + l] * (d.gn[nc + l] * (g[nc + l] * sc[nc + l] - t[q] * sc[nc + l]));
                    }
                }
                for (int c = tid; c < nc; c += nt) d.gn[c] = -d.diag[c] * yc[c];
                __syncthreads();
                PH(5);   // landmark back substitution
                break;
            }
            __syncthreads();
            if (tid == 0) st.mu *= 10.0;
            __syncthreads();
            if (!(st.mu < 1.0)) { if (tid == 0) st.solver_failed = 1; break; }
        }
        __syncthreads();
        if (tid == 0) st.reuse = 1;
        __syncthreads();
    }
    if (!st.solver_failed) {
        // ---- ComputeTraditionalDoglegStep: one pass over the vectors, one 7-way reduction ----
        //   u = gs / D, y = -gn / D (the Gauss-Newton solution of (H' + mu D^2) y = g'), g' = scaled gradient
        double r7[7] = {0, 0, 0, 0, 0, 0, 0};      // |gs|^2, |gn|^2, gs.gn, y.g', y.D^2.y, u.g', u.D^2.y
        for (int c = tid; c < n; c += nt) {
            const double gs_ = d.gs[c], gn_ = d.gn[c], D = d.diag[c], gp = g[c] * sc[c], u = gs_ / D, y = -gn_ / D;
            r7[0] += gs_ * gs_; r7[1] += gn_ * gn_; r7[2] += gs_ * gn_;
            r7[3] += y * gp; r7[4] += y * D * D * y; r7[5] += u * gp; r7[6] += u * D * D * y;
        }
        block_reduce_sums<7>(r7, sred);
        const double g2 = r7[0], n2 = r7[1], ga = r7[2], ygp = r7[3], yDy = r7[4], ugp = r7[5], uDy = r7[6];
        const double gnorm = sqrt(g2), gnn = sqrt(n2), radius = st.radius, alpha = st.alpha;
        double ca, cb, dn;                      // step = ca * gs + cb * gn  (D-space)
        if (gnn <= radius) { ca = 0; cb = 1; dn = gnn; }
        else if (gnorm * alpha >= radius) { ca = -(radius / gnorm); cb = 0; dn = radius; }
        else {
            double b_dot_a = -alpha * ga;
            double a2 = (alpha * gnorm) * (alpha * gnorm);
            double bma2 = a2 - 2 * b_dot_a + gnn * gnn;
            double cc = b_dot_a - a2;
            double dd = sqrt(cc * cc + bma2 * (radius * radius - a2));
            double beta = (cc <= 0) ? (dd - cc) / bma2 : (radius * radius - a2) / (dd + cc);
            ca = -alpha * (1.0 - beta); cb = beta; dn = -1.0;
        }
        if (dn < 0) dn = sqrt(fmax(ca * ca * g2 + 2.0 * ca * cb * ga + cb * cb * n2, 0.0));      // |ca gs + cb gn|
        // model_cost_change = -(s^T g' + s^T H' s / 2) with s = (ca gs + cb gn) / D = ca u - cb y.  No mat-vec is needed:
        //   u^T H' u = |gs|^2 / alpha (Cauchy),  H' y = g' - mu D^2 y  =>  y^T H' y = y^T g' - mu y^T D^2 y,  u^T H' y = u^T g' - mu u^T D^2 y
        const double mu_used = st.mu;
        const double uHu = g2 / alpha, wHw = ygp - mu_used * yDy, uHw = -(ugp - mu_used * uDy);
        const double sg = ca * ugp - cb * ygp;
        const double sHs = ca * ca * uHu + 2.0 * ca * cb * uHw + cb * cb * wHw;
        const double model_change = -(sg + 0.5 * sHs);
        PH(6);   // dogleg + model cost change
        // ---- candidate point x (+) delta, delta = s .* scale ----
        double* dl = (n <= 64 * ntl) ? S : d.delta;               // the factor is dead: delta lives in the tile area when it fits
        __syncthreads();
        for (int c = tid; c < n; c += nt) dl[c] = (ca * d.gs[c] + cb * d.gn[c]) / d.diag[c] * sc[c];
        __syncthreads();
        double s2, mx;
        plus_free(d, d.X, dl, d.Xc, tid, nt, s2, mx);
        s2 = block_reduce_sum(s2, sred);
        if (tid == 0) {
            st.dogleg_norm = dn; st.model_change = model_change; st.step_norm = sqrt(s2); st.dl_a = ca; st.dl_b = cb;
            st.step_valid = model_change > 0.0 ? 1 : 0;
            st.cand_cost = 0.0;
        }
        PH(7);   // candidate point
    }
    if (tid == 0) { st.prof[30] += clock64() - t_kernel0; st.prof[31] += 1; }
}

// TrustRegionMinimizer: HandleInvalidStep / tolerances / IsStepSuccessful / HandleSuccessfulStep / HandleUnsuccessfulStep

// ------------------------------------------------------------------------------------------------
// Marginalisation (MarginalizationInfo::marginalize, reference factor/marginalization_factor.cpp:183-308)
// ------------------------------------------------------------------------------------------------
// Symmetric eigendecomposition by cyclic Jacobi in a parallel ordering, one CTA, matrix in global memory (L2).
// A round pairs every index with exactly one other (round-robin tournament), so the n/2 rotations of a round commute
// as a similarity A <- J^T A J with J = product of the plane rotations: the matrix splits into disjoint 2x2 blocks
// (row pair x column pair), each updated independently from the two rotations involved.  V accumulates the rotations
// (columns = eigenvectors), w = diagonal at convergence (off-norm <= 1e-30 * diag-norm, like the oracle's sweep test).
__global__ void __launch_bounds__(1024) k_jacobi_eig(double* A, double* V, double* w, int n, int* sweeps_out)
{
    extern __shared__ double jsm[];           // c[np/2], s[np/2]; then int pr[np/2], qr[np/2]
    __shared__ double sred[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int np = (n + 1) & ~1, hp = np / 2;
    double* cs_c = jsm; double* cs_s = jsm + hp;
    int* pp = reinterpret_cast<int*>(jsm + 2 * hp); int* qq = pp + hp;
    for (int e = tid; e < n * n; e += nt) V[e] = (e / n == e % n) ? 1.0 : 0.0;
    __syncthreads();
    int sweep = 0;
    double prev_off = 1e300;
    for (; sweep < 60; sweep++) {
        double off = 0, dg = 0;
        for (int e = tid; e < n * n; e += nt) { int i = e / n, j = e - i * n; double v = A[e]; if (i == j) dg += v * v; else if (j > i) off += v * v; }
        off = block_reduce_sum(off, sred); dg = block_reduce_sum(dg, sred);
        if (off <= 1e-30 * dg || off == 0.0) break;
        // rounding floor: with entries of 1e9 next to (numerically) zero eigenvalues the off-norm stalls around
        // n * eps * |A| and never meets the test above; once it stops shrinking there further sweeps only reshuffle noise.
        // The floor is (10 n eps)^2 of the squared diagonal norm: a fixed 1e-20 let a slow sweep among clustered small
        // eigenvalues end the decomposition with off-diagonal entries of 1e-10 |A|, 400x double's accuracy at n = 198
        const double floor_ = 10.0 * n * 2.220446049250313e-16;
        if (sweep >= 4 && off <= floor_ * floor_ * dg && off >= 0.25 * prev_off) break;
        prev_off = off;
        for (int round = 0; round < np - 1; round++) {
            for (int k = tid; k < hp; k += nt) {      // n > 2048: more pairs than threads
                int a = k == 0 ? np - 1 : (round + k) % (np - 1);
                int b = k == 0 ? round : (round + np - 1 - k) % (np - 1);
                int p_ = min(a, b), q_ = max(a, b);
                double c = 1.0, sn = 0.0;
                if (q_ < n) {
                    const double apq = A[(size_t)p_ * n + q_];
                    if (apq != 0.0) {
                        const double theta = (A[(size_t)q_ * n + q_] - A[(size_t)p_ * n + p_]) / (2.0 * apq);
                        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                        c = 1.0 / sqrt(t * t + 1.0); sn = t * c;
                    }
                }
                cs_c[k] = c; cs_s[k] = sn; pp[k] = p_; qq[k] = q_;
            }
            __syncthreads();
            // A <- J^T A J on the 2x2 blocks (row pair r, column pair k).  The blocks are disjoint, so a thread first
            // issues the loads of four of its blocks (L2 latency paid once per batch), then rotates and stores them.
            for (int base = tid; base < hp * hp; base += 4 * nt) {
                double a11[4], a12[4], a21[4], a22[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int task = base + u * nt;
                    a11[u] = a12[u] = a21[u] = a22[u] = 0.0;
                    if (task < hp * hp) {
                        const int r = task / hp, k = task - r * hp;
                        const int p1 = pp[r], q1 = qq[r], p2 = pp[k], q2 = qq[k];
                        const bool hq1 = q1 < n, hq2 = q2 < n;          // q == n is the padding index of an odd n
                        a11[u] = A[(size_t)p1 * n + p2];
                        if (hq2) a12[u] = A[(size_t)p1 * n + q2];
                        if (hq1) a21[u] = A[(size_t)q1 * n + p2];
                        if (hq1 && hq2) a22[u] = A[(size_t)q1 * n + q2];
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int task = base + u * nt;
                    if (task < hp * hp) {
                        const int r = task / hp, k = task - r * hp;
                        const int p1 = pp[r], q1 = qq[r], p2 = pp[k], q2 = qq[k];
                        const double c1 = cs_c[r], s1 = cs_s[r], c2 = cs_c[k], s2 = cs_s[k];
                        const bool hq1 = q1 < n, hq2 = q2 < n;
                        // columns: [a.1 a.2] <- [c2 a.1 - s2 a.2, s2 a.1 + c2 a.2]
                        const double b11 = c2 * a11[u] - s2 * a12[u], b12 = s2 * a11[u] + c2 * a12[u];
                        const double b21 = c2 * a21[u] - s2 * a22[u], b22 = s2 * a21[u] + c2 * a22[u];
                        // rows: [b1.; b2.] <- [c1 b1. - s1 b2.; s1 b1. + c1 b2.]
                        A[(size_t)p1 * n + p2] = c1 * b11 - s1 * b21;
                        if (hq2) A[(size_t)p1 * n + q2] = c1 * b12 - s1 * b22;
                        if (hq1) A[(size_t)q1 * n + p2] = s1 * b11 + c1 * b21;
                        if (hq1 && hq2) A[(size_t)q1 * n + q2] = s1 * b12 + c1 * b22;
                    }
                }
            }
            for (int base = tid; base < n * hp; base += 4 * nt) {     // V <- V J, same batching
                double vp[4], vq[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int task = base + u * nt;
                    vp[u] = vq[u] = 0.0;
                    if (task < n * hp) {
                        const int row = task / hp, k = task - row * hp;
                        if (qq[k] < n) { vp[u] = V[(size_t)row * n + pp[k]]; vq[u] = V[(size_t)row * n + qq[k]]; }
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int task = base + u * nt;
                    if (task < n * hp) {
                        const int row = task / hp, k = task - row * hp;
                        if (qq[k] < n) {
                            const double c2 = cs_c[k], s2 = cs_s[k];
                            V[(size_t)row * n + pp[k]] = c2 * vp[u] - s2 * vq[u];
                            V[(size_t)row * n + qq[k]] = s2 * vp[u] + c2 * vq[u];
                        }
                    }
                }
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < n; i += nt) w[i] = A[(size_t)i * n + i];
    if (tid == 0 && sweeps_out) *sweeps_out = sweep;
}

// Symmetric eigendecomposition for the reduced system of the marginalisation (n <= 128): Householder tridiagonalisation +
// implicit-shift QL (EISPACK tred2 / tql2, the algorithm family of Eigen's SelfAdjointEigenSolver; same restatement as
// oracle/ba_oracle.c sym_eig_ql).  One CTA of 128 threads, V column-major in shared memory.  The Householder steps are
// thread-parallel over rows/columns; in the QL phase thread 0 runs the scalar recurrence of a sweep and publishes the plane
// rotations, then every thread applies them to its own row of V.
constexpr int QL_T = 128;
__global__ void __launch_bounds__(QL_T) k_sym_eig_ql(const double* __restrict__ Ag, double* __restrict__ Vg, double* __restrict__ wg, int n)
{
    extern __shared__ double qsm[];          // V[n*n] | d[n] | e[n+1] | rc[n] | rs[n]
    __shared__ double sred[32];
    __shared__ double sh_h, sh_scale, sh_hh;
    __shared__ int sh_m, sh_more;
    double* V = qsm; double* d = V + (size_t)n * n; double* e = d + n; double* rc = e + n + 1; double* rs = rc + n;
    const int tid = threadIdx.x;
#define VV(i, j) V[(size_t)(j) * n + (i)]
    for (int t = tid; t < n * n; t += QL_T) V[t] = Ag[t];              // symmetric: row-major == column-major
    __syncthreads();
    for (int j = tid; j < n; j += QL_T) d[j] = VV(n - 1, j);
    __syncthreads();
    for (int i = n - 1; i > 0; i--) {                                   // ---- tred2 ----
        double sc = 0.0;
        for (int k = tid; k < i; k += QL_T) sc += fabs(d[k]);
        sc = block_reduce_sum(sc, sred);
        if (sc == 0.0) {
            if (tid == 0) e[i] = d[i - 1];
            __syncthreads();
            for (int j = tid; j < i; j += QL_T) { d[j] = VV(i - 1, j); VV(i, j) = 0.0; VV(j, i) = 0.0; }
            __syncthreads();
        } else {
            double hs = 0.0;
            for (int k = tid; k < i; k += QL_T) { const double t = d[k] / sc; d[k] = t; hs += t * t; }
            hs = block_reduce_sum(hs, sred);
            if (tid == 0) {
                double f = d[i - 1], g = sqrt(hs);
                if (f > 0) g = -g;
                e[i] = sc * g; sh_h = hs - f * g; d[i - 1] = f - g;
            }
            __syncthreads();
            const double h = sh_h;
            // e = (symmetric matrix held in the lower triangle) * d, V[j][i] = d[j]
            for (int j = tid; j < i; j += QL_T) {
                double g = 0.0;
                for (int k = 0; k <= j; k++) g += VV(j, k) * d[k];
                for (int k = j + 1; k < i; k++) g += VV(k, j) * d[k];
                rc[j] = g / h;                                       // e[j] / h (kept aside: VV(j, i) aliases nothing of e)
                VV(j, i) = d[j];
            }
            __syncthreads();
            double fs = 0.0;
            for (int j = tid; j < i; j += QL_T) fs += rc[j] * d[j];
            fs = block_reduce_sum(fs, sred);
            const double hh = fs / (h + h);
            for (int j = tid; j < i; j += QL_T) e[j] = rc[j] - hh * d[j];
            __syncthreads();
            for (int t = tid; t < i * i; t += QL_T) {                    // rank-2 update of the lower triangle
                const int j = t / i, k = t - j * i;
                if (k >= j) VV(k, j) -= (d[j] * e[k] + e[j] * d[k]);
            }
            __syncthreads();
            for (int j = tid; j < i; j += QL_T) { d[j] = VV(i - 1, j); VV(i, j) = 0.0; }
            if (tid == 0) d[i] = h;
            __syncthreads();
            continue;
        }
        if (tid == 0) d[i] = 0.0;
        __syncthreads();
    }
    for (int i = 0; i < n - 1; i++) {                                   // ---- accumulate the transformations ----
        if (tid == 0) { VV(n - 1, i) = VV(i, i); VV(i, i) = 1.0; }
        __syncthreads();
        const double h = d[i + 1];
        if (h != 0.0) {
            for (int k = tid; k <= i; k += QL_T) rc[k] = VV(k, i + 1) / h;
            __syncthreads();
            for (int j = tid; j <= i; j += QL_T) {
                double g = 0.0;
                for (int k = 0; k <= i; k++) g += VV(k, i + 1) * VV(k, j);
                for (int k = 0; k <= i; k++) VV(k, j) -= g * rc[k];
            }
            __syncthreads();
        }
        for (int k = tid; k <= i; k += QL_T) VV(k, i + 1) = 0.0;
        __syncthreads();
    }
    for (int j = tid; j < n; j += QL_T) { d[j] = VV(n - 1, j); VV(n - 1, j) = 0.0; }
    __syncthreads();
    if (tid == 0) { VV(n - 1, n - 1) = 1.0; for (int i = 1; i < n; i++) e[i - 1] = e[i]; e[n - 1] = 0.0; }
    __syncthreads();
    // ---- tql2 ----
    double f = 0.0, tst1 = 0.0;                                          // thread 0's scalars
    const double eps = 2.220446049250313e-16;
    for (int l = 0; l < n; l++) {
        if (tid == 0) {
            const double t = fabs(d[l]) + fabs(e[l]);
            if (t > tst1) tst1 = t;
            int m = l;
            while (m < n) { if (fabs(e[m]) <= eps * tst1) break; m++; }
            sh_m = m;
        }
        __syncthreads();
        const int m = sh_m;
        if (m > l) {
            int iter = 0;
            while (true) {
                if (tid == 0) {
                    iter++;
                    double g = d[l], p = (d[l + 1] - g) / (2.0 * e[l]), r = hypot(p, 1.0);
                    if (p < 0) r = -r;
                    d[l] = e[l] / (p + r); d[l + 1] = e[l] * (p + r);
                    const double dl1 = d[l + 1];
                    double h = g - d[l];
                    for (int i = l + 2; i < n; i++) d[i] -= h;
                    f += h;
                    p = d[m];
                    double c = 1.0, c2 = c, c3 = c, s_ = 0.0, s2 = 0.0;
                    const double el1 = e[l + 1];
                    for (int i = m - 1; i >= l; i--) {
                        c3 = c2; c2 = c; s2 = s_;
                        g = c * e[i]; h = c * p; r = hypot(p, e[i]);
                        e[i + 1] = s_ * r; s_ = e[i] / r; c = p / r; p = c * d[i] - s_ * g; d[i + 1] = h + s_ * (c * g + s_ * d[i]);
                        rc[i] = c; rs[i] = s_;
                    }
                    p = -s_ * s2 * c3 * el1 * e[l] / dl1; e[l] = s_ * p; d[l] = c * p;
                    sh_more = (fabs(e[l]) > eps * tst1 && iter < 200) ? 1 : 0;
                }
                __syncthreads();
                if (tid < n) {                                           // this thread's row of V
                    const int k = tid;
                    double hi = VV(k, m);
                    for (int i = m - 1; i >= l; i--) {
                        const double c = rc[i], s_ = rs[i], lo = VV(k, i);
                        VV(k, i + 1) = s_ * lo + c * hi;
                        hi = c * lo - s_ * hi;
                    }
                    VV(k, l) = hi;
                }
                __syncthreads();
                if (!sh_more) break;
            }
        }
        if (tid == 0) { d[l] = d[l] + f; e[l] = 0.0; }
        __syncthreads();
    }
    for (int t = tid; t < n * n; t += QL_T) { const int i = t / n, j = t - i * n; Vg[t] = VV(i, j); }     // row-major out, columns = eigenvectors
    for (int j = tid; j < n; j += QL_T) wg[j] = d[j];
#undef VV
}

struct MargDev {
    int N, m, n;
    const double *H, *Hp, *g;     // accumulated by k_ba_eval (N x N, N)
    double *A, *b;                // N x N, N
    double *Amm, *Vm, *wm, *Ainv; // m x m ...
    double *T;                    // n x m
    double *Ar, *Vr, *wr, *br;    // n x n ...
    double *J0, *r0;
};

__global__ void k_marg_pack(MargDev q)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x, N = q.N;
    if (e < N * N) q.A[e] = q.H[e] + q.Hp[e];
    if (e < N) q.b[e] = q.g[e];
}
__global__ void k_marg_amm(MargDev q)      // Amm = 0.5 (Amm + Amm^T)   (marginalization_factor.cpp:278)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x, m = q.m, N = q.N;
    if (e >= m * m) return;
    const int i = e / m, j = e - i * m;
    q.Amm[e] = 0.5 * (q.A[(size_t)i * N + j] + q.A[(size_t)j * N + i]);
}
__global__ void k_marg_ainv(MargDev q)     // Amm_inv = V diag(w > eps ? 1/w : 0) V^T     (:279-283)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x, m = q.m;
    if (e >= m * m) return;
    const int i = e / m, j = e - i * m;
    double v = 0;
    for (int k = 0; k < m; k++) { const double wk = q.wm[k]; if (wk > 1e-8) v += q.Vm[(size_t)i * m + k] * (1.0 / wk) * q.Vm[(size_t)j * m + k]; }
    q.Ainv[e] = v;
}
__global__ void k_marg_T(MargDev q)        // T = Arm Amm_inv
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x, m = q.m, n = q.n, N = q.N;
    if (e >= n * m) return;
    const int i = e / m, j = e - i * m;
    double v = 0;
    for (int k = 0; k < m; k++) v += q.A[(size_t)(m + i) * N + k] * q.Ainv[(size_t)k * m + j];
    q.T[e] = v;
}
__global__ void k_marg_reduce(MargDev q)   // A = Arr - Arm Amm_inv Amr, b = brr - Arm Amm_inv bmm   (:286-292); lower triangle mirrored
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x, m = q.m, n = q.n, N = q.N;
    if (e < n * n) {
        const int i = e / n, j = e - i * n;
        if (j <= i) {
            double v = q.A[(size_t)(m + i) * N + m + j];
            for (int k = 0; k < m; k++) v -= q.T[(size_t)i * m + k] * q.A[(size_t)k * N + m + j];
            q.Ar[(size_t)i * n + j] = v; q.Ar[(size_t)j * n + i] = v;
        }
    }
    if (e < n) { double v = q.b[m + e]; for (int k = 0; k < m; k++) v -= q.T[(size_t)e * m + k] * q.b[k]; q.br[e] = v; }
}
// ---- structured path: Amm = [[C, B], [B^T, D]] with D the diagonal landmark block --------------------------------------
// When Amm - eps I is positive definite every eigenvalue passes the reference's eps test, the eigen-truncated inverse IS
// the inverse, and Arr - Arm Amm^-1 Amr is the ordinary two-stage Schur complement: landmarks (1x1 pivots) first, then
// the c x c block of pose0 / speedbias0.  Q is the (c+n) x (c+n) system left after the landmarks, order [c | kept].
// flag[0] is set when the positive-definiteness test fails (the generic Jacobi path is run instead).  Launched with at least
// max(R^2, m) threads: thread e < R^2 forms Q[e], thread c <= e < m tests landmark pivot e.
__global__ void k_marg_lm_elim(MargDev q, int c, double* Q, double* qb, double* Ceps, int* flag)
{
    const int R = c + q.n, m = q.m, N = q.N;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    auto gi = [&](int i) { return i < c ? i : m + (i - c); };       // compact index -> column of A
    if (e < R * R) {
        const int i = e / R, j = e - i * R, ai = gi(i), aj = gi(j);
        double v = 0.5 * (q.A[(size_t)ai * N + aj] + q.A[(size_t)aj * N + ai]), ve = v;
        for (int l = c; l < m; l++) {
            const double d = q.A[(size_t)l * N + l];
            const double t = 0.5 * (q.A[(size_t)ai * N + l] + q.A[(size_t)l * N + ai]) * 0.5 * (q.A[(size_t)l * N + aj] + q.A[(size_t)aj * N + l]);
            v -= t / d;
            if (i < c && j < c) ve -= t / (d - 1e-8);
        }
        Q[e] = v;
        if (i < c && j < c) Ceps[i * c + j] = ve - (i == j ? 1e-8 : 0.0);
    }
    if (e < R) {
        const int ai = gi(e);
        double v = q.b[ai];
        for (int l = c; l < m; l++) v -= 0.5 * (q.A[(size_t)ai * N + l] + q.A[(size_t)l * N + ai]) * q.b[l] / q.A[(size_t)l * N + l];
        qb[e] = v;
    }
    if (e >= c && e < m && !(q.A[(size_t)e * N + e] - 1e-8 > 0.0)) atomicExch(flag, 1);
}
// single CTA: Cholesky of the c x c block (and of its eps-shifted twin for the test), X = S^-1 [Q_cr | q_c], reduced system
__global__ void __launch_bounds__(256) k_marg_c_elim(MargDev q, int c, const double* Q, const double* qb, const double* Ceps, int* flag)
{
    __shared__ double Lc[15 * 15], Le[15 * 15];
    __shared__ double X[15 * 128];            // c x (n + 1), n <= 127
    const int tid = threadIdx.x, n = q.n, R = c + n;
    if (tid == 0) {
        bool ok = true;
        for (int pass = 0; pass < 2 && ok; pass++) {
            double* L = pass == 0 ? Lc : Le;
            for (int i = 0; i < c; i++) for (int j = 0; j < c; j++) L[i * c + j] = pass == 0 ? Q[(size_t)i * R + j] : Ceps[i * c + j];
            for (int j = 0; j < c && ok; j++) {
                double d = L[j * c + j];
                for (int k = 0; k < j; k++) d -= L[j * c + k] * L[j * c + k];
                if (!(d > 0.0)) { ok = false; break; }
                d = sqrt(d); L[j * c + j] = d;
                for (int i = j + 1; i < c; i++) { double t = L[i * c + j]; for (int k = 0; k < j; k++) t -= L[i * c + k] * L[j * c + k]; L[i * c + j] = t / d; }
            }
        }
        if (!ok) atomicExch(flag, 1);
    }
    __syncthreads();
    if (*(volatile int*)flag) return;
    for (int col = tid; col <= n; col += blockDim.x) {          // S x = rhs for the n kept columns and the rhs vector
        double y[15];
        for (int i = 0; i < c; i++) { double t = col < n ? Q[(size_t)i * R + c + col] : qb[i]; for (int k = 0; k < i; k++) t -= Lc[i * c + k] * y[k]; y[i] = t / Lc[i * c + i]; }
        for (int i = c - 1; i >= 0; i--) { double t = y[i]; for (int k = i + 1; k < c; k++) t -= Lc[k * c + i] * y[k]; y[i] = t / Lc[i * c + i]; }
        for (int i = 0; i < c; i++) X[i * (n + 1) + col] = y[i];
    }
    __syncthreads();
    for (int e = tid; e < n * n; e += blockDim.x) {
        const int i = e / n, j = e - i * n;
        if (j > i) continue;
        double v = Q[(size_t)(c + i) * R + c + j];
        for (int k = 0; k < c; k++) v -= Q[(size_t)(c + i) * R + k] * X[k * (n + 1) + j];
        q.Ar[(size_t)i * n + j] = v; q.Ar[(size_t)j * n + i] = v;
    }
    for (int i = tid; i < n; i += blockDim.x) {
        double v = qb[c + i];
        for (int k = 0; k < c; k++) v -= Q[(size_t)(c + i) * R + k] * X[k * (n + 1) + n];
        q.br[i] = v;
    }
}

__global__ void k_marg_out(MargDev q)      // J0 = sqrt(S) V^T, r0 = sqrt(S^-1) V^T b     (:294-302)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x, n = q.n;
    if (e < n * n) {
        const int k = e / n, i = e - k * n;
        const double S = q.wr[k] > 1e-8 ? q.wr[k] : 0.0;
        q.J0[e] = sqrt(S) * q.Vr[(size_t)i * n + k];
    }
    if (e < n) {
        const double Si = q.wr[e] > 1e-8 ? 1.0 / q.wr[e] : 0.0;
        double vb = 0; for (int i = 0; i < n; i++) vb += q.Vr[(size_t)i * n + e] * q.br[i];
        q.r0[e] = sqrt(Si) * vb;
    }
}

}  // namespace gfba

// ------------------------------------------------------------------------------------------------
struct gf_ba {
    int device;
    cudaStream_t s;
    cudaEvent_t e0, e1;
    // growable device buffers
    void* dbuf; size_t dcap;
    void* hbuf; size_t hcap;     // pinned staging
    long long prof[32];
    int tile_cap;
    int marg_info[3];            // last marginalisation: GF_MARG_PATH_* bits, Jacobi sweeps on Amm, on the reduced system
};

static int ensure(gf_ba* s, size_t dbytes)
{
    if (dbytes > s->dcap) {
        if (s->dbuf) cudaFree(s->dbuf);
        if (s->hbuf) cudaFreeHost(s->hbuf);
        s->dcap = dbytes * 2;
        GF_CUDA(cudaMalloc(&s->dbuf, s->dcap));
        GF_CUDA(cudaHostAlloc(&s->hbuf, s->dcap, cudaHostAllocDefault));
        s->hcap = s->dcap;
    }
    return GF_OK;
}

extern "C" {

int gf_ba_create(gf_ba** out, int device)
{
    if (!out) return set_err(GF_ERR_INVALID_ARG, "null argument");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) { snprintf(g_err, sizeof(g_err), "no CUDA device visible (%s); libgf_b200 has no CPU fallback", cudaGetErrorString(e)); return GF_ERR_NO_DEVICE; }
    if (device < 0 || device >= n) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    gf_ba* s = new (std::nothrow) gf_ba();
    if (!s) return set_err(GF_ERR_CUDA, "out of host memory");
    memset(s, 0, sizeof(*s));
    s->device = device;
    GF_CUDA(cudaStreamCreateWithFlags(&s->s, cudaStreamNonBlocking));
    GF_CUDA(cudaEventCreate(&s->e0)); GF_CUDA(cudaEventCreate(&s->e1));
    s->tile_cap = TILE_CAP;
    if (const char* e_ = getenv("GF_BA_TILE_CAP")) { const int v = atoi(e_); if (v >= 0 && v < TILE_CAP) s->tile_cap = v; }
    GF_CUDA(cudaFuncSetAttribute(k_ba_step<MAXR / 2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)STEP_SMEM_MAX));
    GF_CUDA(cudaFuncSetAttribute(k_ba_step<MAXR, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)STEP_SMEM_MAX));
    GF_CUDA(cudaFuncSetAttribute(k_jacobi_eig, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    GF_CUDA(cudaFuncSetAttribute(k_sym_eig_ql, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    GF_CUDA(cudaFuncSetAttribute(k_ba_schur, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SCHUR_SMEM_MAX));
    *out = s;
    return GF_OK;
}

void gf_ba_destroy(gf_ba* s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    cudaStreamSynchronize(s->s);
    if (s->dbuf) cudaFree(s->dbuf);
    if (s->hbuf) cudaFreeHost(s->hbuf);
    cudaEventDestroy(s->e0); cudaEventDestroy(s->e1);
    cudaStreamDestroy(s->s);
    delete s;
}

}  // extern "C" (reopened below)

// ------------------------------------------------------------------------------------------------
// One solve in four parts, shared by gf_ba_solve (the batch of one) and gf_ba_solve_multi:
//   ba_layout   argument checks and the column layout of one window (host only: nothing is written anywhere)
//   ba_pack     the window's upload image in its handle's pinned buffer, and its descriptor
//   ba_batch    the uploads, the launch chain of the whole batch on the first handle's stream, the downloads
//   ba_finish   write-back of one window's blocks and summary
struct BaWindow {
    BaDev d;                                   // device pointers are set by ba_pack
    std::vector<int> col_feat, pair_id, pair_start, work_start, work_ij, pcol;
    size_t px0_len;
    int n_work, pn, n8, ntiles, eval_blocks;
    bool spill;                                // k_ba_step<MAXR, true>: the factor does not fit the shared-memory tiles
    size_t prior_smem, step_smem, schur_smem;
    size_t o_X, o_vis, o_imu, o_whl, o_plf, o_ps, o_pij, o_cf, o_pJ, o_pr0, o_px0, o_pcol, o_Xc, o_st, upload_bytes;
    size_t o_sq, o_Hp, o_a0, o_a1, o_vec, o_Sg, o_Lg, bytes;
    size_t base;                               // offset of the window in its handle's buffers (the batch table comes first in the lead handle's)
};

static size_t al16(size_t v) { return (v + 15) / 16 * 16; }

static int ba_layout(const gf_ba* s, const gf_ba_problem* p, BaWindow& w)
{
    if (!p) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (p->n_frames < 1 || p->n_frames > GF_BA_MAX_FRAMES) return set_err(GF_ERR_INVALID_ARG, "n_frames out of range");
    if (p->n_visual < 0 || p->n_imu < 0 || p->n_features < 0) return set_err(GF_ERR_INVALID_ARG, "negative factor / feature count");
    if (!p->para_pose || !p->para_ex_pose || !p->para_td) return set_err(GF_ERR_INVALID_ARG, "null parameter block");
    if ((p->n_features > 0 && (!p->para_feature || !p->feature_const)) || (p->n_visual > 0 && !p->visual) || (p->n_imu > 0 && (!p->imu || !p->para_speed_bias)))
        return set_err(GF_ERR_INVALID_ARG, "factor table or parameter block missing");
    if (p->n_wheel < 0 || (p->n_wheel > 0 && (!p->wheel || !p->para_ex_wheel || !p->para_ix_wheel || !p->para_td_wheel))) return set_err(GF_ERR_INVALID_ARG, "wheel factors without their parameter blocks");
    if (p->n_plane < 0 || p->n_plane > PAIR_THREADS || (p->n_plane > 0 && (!p->plane_frames || !p->para_ex_wheel || !p->para_plane_R || !p->para_plane_Z))) return set_err(GF_ERR_INVALID_ARG, "plane factors without their parameter blocks");
    if (p->max_num_iterations < 0 || p->max_num_iterations > GF_BA_MAX_ITERATIONS) return set_err(GF_ERR_INVALID_ARG, "max_num_iterations out of range");
    const int F = p->n_frames, nfeat = p->n_features;
    // ---- layout (same rules as ceres::Problem construction, estimator.cpp:2950-3100, 3233-3246, 3291) ----
    BaDev& d = w.d; memset(&d, 0, sizeof(d));
    d.F = F; d.nfeat = nfeat; d.n_vis = p->n_visual; d.n_imu = p->n_imu; d.n_wheel = p->n_wheel; d.n_plane = p->n_plane;
    d.pr_mask = p->plane_r_subset_mask; for (int k = 0; k < 3; k++) d.plane_sinfo[k] = p->plane_sqrt_info[k];
    const bool use_sb = p->para_speed_bias && !p->pose0_const;
    int c = 0;
    for (int f = 0; f < MAXF; f++) { d.col_pose[f] = -1; d.col_sb[f] = -1; }
    for (int f = 0; f < F; f++) { bool k = p->frames_const || (f == 0 && p->pose0_const); if (!k) { d.col_pose[f] = c; c += 6; } }
    for (int f = 0; f < F; f++) { bool k = p->frames_const || !use_sb; if (!k) { d.col_sb[f] = c; c += 9; } }
    d.col_ex = p->ex_pose_const ? -1 : c; if (!p->ex_pose_const) c += 6;
    d.col_td = p->td_const ? -1 : c; if (!p->td_const) c += 1;
    d.col_exw = -1; d.col_ix[0] = d.col_ix[1] = d.col_ix[2] = -1; d.col_tdw = -1; d.exw_mask = p->ex_wheel_subset_mask;
    if (p->n_wheel > 0 || p->n_plane > 0) {      // estimator.cpp:3008-3056: these blocks only exist with USE_WHEEL (PlaneFactor reads the extrinsic too)
        if (!p->ex_wheel_const) { d.col_exw = c; c += 6; }
        if (p->n_wheel > 0 && !p->ix_wheel_const) for (int k = 0; k < 3; k++) d.col_ix[k] = c++;
        if (p->n_wheel > 0 && !p->td_wheel_const) d.col_tdw = c++;
    }
    d.col_pr = d.col_pz = -1;
    if (p->n_plane > 0 && !p->plane_const) { d.col_pr = c; c += 3; d.col_pz = c++; }
    for (int k = 0; k < p->n_plane; k++) if (p->plane_frames[k] < 0 || p->plane_frames[k] >= F) return set_err(GF_ERR_INVALID_ARG, "plane factor frame out of range");
    d.nc = c;
    std::vector<int>& col_feat = w.col_feat;
    col_feat.assign(nfeat > 0 ? nfeat : 1, -1);
    for (int v = 0; v < p->n_visual; v++) {
        int k = p->visual[v].feature;
        if (k < 0 || k >= nfeat || p->visual[v].imu_i < 0 || p->visual[v].imu_i >= F || p->visual[v].imu_j < 0 || p->visual[v].imu_j >= F)
            return set_err(GF_ERR_INVALID_ARG, "visual factor index out of range");
        if (p->visual[v].imu_i == p->visual[v].imu_j) return set_err(GF_ERR_INVALID_ARG, "visual factor with imu_i == imu_j");
        if (!p->feature_const[k] && col_feat[k] == -1) col_feat[k] = -2;
    }
    for (int k = 0; k < nfeat; k++) if (col_feat[k] == -2) col_feat[k] = c++;
    d.L = c - d.nc; d.n = c;
    if (d.nc > MAX_NC) return set_err(GF_ERR_CAPACITY, "reduced system larger than 383 unknowns");
    if (d.L > GF_BA_MAX_FREE_LANDMARKS) return set_err(GF_ERR_CAPACITY, "more than GF_BA_MAX_FREE_LANDMARKS (8192) free landmarks");
    // ---- sort visual factors by pose pair ----
    std::vector<int>& pair_id = w.pair_id;
    pair_id.assign(F * F, -1);
    std::vector<int> pair_cnt, pair_ij;
    for (int v = 0; v < p->n_visual; v++) {
        int key = p->visual[v].imu_i * F + p->visual[v].imu_j;
        if (pair_id[key] < 0) { pair_id[key] = (int)pair_cnt.size(); pair_cnt.push_back(0); pair_ij.push_back(p->visual[v].imu_i); pair_ij.push_back(p->visual[v].imu_j); }
        pair_cnt[pair_id[key]]++;
    }
    const int n_pairs = (int)pair_cnt.size();
    std::vector<int>& pair_start = w.pair_start;
    pair_start.assign(n_pairs + 1, 0);
    for (int k = 0; k < n_pairs; k++) pair_start[k + 1] = pair_start[k] + pair_cnt[k];
    // one CTA of k_ba_eval per (pair, chunk of <= PAIR_CHUNK factors): long pairs are cut so that the CTAs are balanced
    w.work_start.assign(1, 0); w.work_ij.clear();
    for (int k = 0; k < n_pairs; k++)
        for (int c0 = pair_start[k]; c0 < pair_start[k + 1]; c0 += PAIR_CHUNK) {
            w.work_ij.push_back(pair_ij[2 * k]); w.work_ij.push_back(pair_ij[2 * k + 1]);
            w.work_start.push_back(std::min(c0 + PAIR_CHUNK, pair_start[k + 1]));
        }
    const int n_work = (int)w.work_ij.size() / 2;
    w.n_work = n_work;
    d.n_pairs = n_work;
    const gf_ba_prior* pr = (p->prior && p->prior->n > 0) ? p->prior : nullptr;
    const int pn = pr ? pr->n : 0;
    w.pn = pn;
    w.pcol.assign(pn > 0 ? pn : 1, -1);
    size_t px0_len = 0;
    if (pr) {
        if (pr->n_blocks > 64) return set_err(GF_ERR_CAPACITY, "more than 64 prior blocks");
        d.pn = pn; d.pnb = pr->n_blocks;
        for (int b = 0; b < pr->n_blocks; b++) {
            int kind = pr->block_kind[b], idx = pr->block_index[b];
            d.pkind[b] = kind; d.pindex[b] = idx; d.pidx[b] = pr->block_idx[b]; d.pxoff[b] = (int)px0_len;
            int gs = (kind == GF_BA_BLOCK_POSE || kind == GF_BA_BLOCK_EX_POSE || kind == GF_BA_BLOCK_EX_WHEEL) ? 7 : kind == GF_BA_BLOCK_SPEEDBIAS ? 9 : kind == GF_BA_BLOCK_PLANE_R ? 4 : 1;
            int ls = gs == 7 ? 6 : gs == 4 ? 3 : gs;      // plane rotation: 4 prior columns, the local parameterisation keeps 3
            if (kind < 0 || kind > GF_BA_BLOCK_PLANE_Z || kind == GF_BA_BLOCK_FEATURE) return set_err(GF_ERR_INVALID_ARG, "unknown prior block kind");
            if ((kind == GF_BA_BLOCK_POSE || kind == GF_BA_BLOCK_SPEEDBIAS) && (idx < 0 || idx >= F)) return set_err(GF_ERR_INVALID_ARG, "prior block index out of range");
            int lc = kind == GF_BA_BLOCK_POSE ? d.col_pose[idx] : kind == GF_BA_BLOCK_SPEEDBIAS ? d.col_sb[idx] : kind == GF_BA_BLOCK_EX_POSE ? d.col_ex : kind == GF_BA_BLOCK_TD ? d.col_td
                     : kind == GF_BA_BLOCK_EX_WHEEL ? d.col_exw : kind == GF_BA_BLOCK_SX ? d.col_ix[0] : kind == GF_BA_BLOCK_SY ? d.col_ix[1] : kind == GF_BA_BLOCK_SW ? d.col_ix[2]
                     : kind == GF_BA_BLOCK_TD_WHEEL ? d.col_tdw : kind == GF_BA_BLOCK_PLANE_R ? d.col_pr : d.col_pz;
            if (lc >= 0) for (int k = 0; k < ls; k++) w.pcol[pr->block_idx[b] + k] = lc + k;
            px0_len += gs;
        }
    }
    w.px0_len = px0_len;
    for (int k = 0; k < p->n_wheel; k++) if (p->wheel[k].i < 0 || p->wheel[k].i >= F || p->wheel[k].j < 0 || p->wheel[k].j >= F) return set_err(GF_ERR_INVALID_ARG, "wheel factor index out of range");
    for (int k = 0; k < p->n_imu; k++) if (p->imu[k].i < 0 || p->imu[k].i >= F || p->imu[k].j < 0 || p->imu[k].j >= F) return set_err(GF_ERR_INVALID_ARG, "imu factor index out of range");
    // ---- offsets in the handle's buffers (relative to w.base) ----
    const int nc = d.nc, L = d.L, n = d.n;
    const int n8 = (nc + 8) / 8, ntiles = n8 * (n8 + 1) / 2;      // 8x8 tiles of the (nc+1)-row augmented reduced system
    w.n8 = n8; w.ntiles = ntiles;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += al16(bytes); return o; };
    w.o_X = take(sizeof(double) * (X_FEAT + nfeat)); w.o_vis = take(sizeof(gf_ba_visual_factor) * (size_t)p->n_visual);
    w.o_imu = take(sizeof(gf_ba_imu_factor) * (size_t)p->n_imu); w.o_whl = take(sizeof(gf_ba_wheel_factor) * (size_t)p->n_wheel);
    w.o_plf = take(sizeof(int) * (size_t)(p->n_plane > 0 ? p->n_plane : 1)); w.o_ps = take(sizeof(int) * (n_work + 1));
    w.o_pij = take(sizeof(int) * 2 * (size_t)(n_work > 0 ? n_work : 1)); w.o_cf = take(sizeof(int) * (size_t)(nfeat > 0 ? nfeat : 1));
    w.o_pJ = take(sizeof(double) * (size_t)pn * pn); w.o_pr0 = take(sizeof(double) * pn);
    w.o_px0 = take(sizeof(double) * px0_len); w.o_pcol = take(sizeof(int) * (size_t)(pn > 0 ? pn : 1));
    w.o_Xc = take(sizeof(double) * (X_FEAT + nfeat)); w.o_st = take(sizeof(BaState));     // uploaded too: candidate := x, initial solver state
    w.upload_bytes = off;
    w.o_sq = take(sizeof(double) * 225 * (size_t)(p->n_imu > 0 ? p->n_imu : 1));
    w.o_Hp = take(sizeof(double) * (size_t)nc * nc); w.o_a0 = take(sizeof(double) * acc_size(nc, L)); w.o_a1 = take(sizeof(double) * acc_size(nc, L));
    w.o_vec = take(sizeof(double) * 6 * (size_t)(n > 0 ? n : 1)); w.o_Sg = take(sizeof(double) * 64 * (size_t)ntiles);
    w.o_Lg = take(sizeof(double) * 64 * (size_t)(ntiles > s->tile_cap ? ntiles - s->tile_cap : 1));
    w.bytes = off;
    // ---- launch shapes ----
    w.eval_blocks = n_work + p->n_imu + p->n_wheel + (p->n_plane > 0 ? 1 : 0) + (pn ? 1 : 0);
    d.eval_grid = w.eval_blocks > 0 ? w.eval_blocks : 1;
    d.schur_grid = (ntiles + SCHUR_WARPS - 1) / SCHUR_WARPS + 1;      // + the CTA that prepares k_ba_step's vectors and norms
    d.tile_cap = s->tile_cap;
    w.spill = !(ntiles <= s->tile_cap && n8 <= (MAXR / 2) * CH_BULK);
    w.prior_smem = sizeof(double) * 2 * (size_t)pn;
    w.step_smem = sizeof(double) * (64 * (size_t)std::min(ntiles, s->tile_cap) + 64 * (size_t)n8 + 192 + 2 * (size_t)((nc + 8) & ~7));
    w.schur_smem = sizeof(double) * (size_t)std::max(L + 2 * nc + 2, n + 1);
    return GF_OK;
}

// radius, mu: the initial trust-region state (Ceres' defaults 1e4, 1e-8 for a solve); max_iter: BaState::max_iter
static void ba_pack(gf_ba* s, const gf_ba_problem* p, BaWindow& w, double radius, double mu, int max_iter)
{
    const int F = p->n_frames, nfeat = p->n_features, n = w.d.n, pn = w.pn;
    const gf_ba_prior* pr = pn ? p->prior : nullptr;
    char* hb = (char*)s->hbuf + w.base; char* db = (char*)s->dbuf + w.base;
    double* hX = (double*)(hb + w.o_X);
    memset(hX, 0, sizeof(double) * (X_FEAT + nfeat));
    memcpy(hX + X_POSE, p->para_pose, sizeof(double) * 7 * F);
    if (p->para_speed_bias) memcpy(hX + X_SB, p->para_speed_bias, sizeof(double) * 9 * F);
    memcpy(hX + X_EX, p->para_ex_pose, sizeof(double) * 7);
    hX[X_TD] = p->para_td[0];
    hX[X_EXW + 6] = 1.0; hX[X_IX] = hX[X_IX + 1] = hX[X_IX + 2] = 1.0;
    if (p->n_wheel > 0) { memcpy(hX + X_EXW, p->para_ex_wheel, sizeof(double) * 7); memcpy(hX + X_IX, p->para_ix_wheel, sizeof(double) * 3); hX[X_TDW] = p->para_td_wheel[0]; }
    hX[X_PR + 3] = 1.0;
    if (p->n_plane > 0) { memcpy(hX + X_EXW, p->para_ex_wheel, sizeof(double) * 7); memcpy(hX + X_PR, p->para_plane_R, sizeof(double) * 4); hX[X_PZ] = p->para_plane_Z[0]; memcpy(hb + w.o_plf, p->plane_frames, sizeof(int) * p->n_plane); }
    memcpy(hX + X_FEAT, p->para_feature, sizeof(double) * nfeat);
    memcpy(hb + w.o_Xc, hX, sizeof(double) * (X_FEAT + nfeat));           // the candidate starts as a copy: its constant blocks never change
    {   // TrustRegionMinimizer / DoglegStrategy initial state; the first linearisation goes to buffer 0
        BaState* h0 = (BaState*)(hb + w.o_st);
        memset(h0, 0, sizeof(BaState));
        h0->radius = radius; h0->mu = mu; h0->need_linearize = 1; h0->cur = 1; h0->first = 1; h0->max_iter = max_iter;
    }
    {   // factors sorted by pair
        gf_ba_visual_factor* hv = (gf_ba_visual_factor*)(hb + w.o_vis);
        std::vector<int> fill(w.pair_start.begin(), w.pair_start.end() - 1);
        for (int v = 0; v < p->n_visual; v++) { int k = w.pair_id[p->visual[v].imu_i * F + p->visual[v].imu_j]; hv[fill[k]++] = p->visual[v]; }
    }
    if (p->n_imu) memcpy(hb + w.o_imu, p->imu, sizeof(gf_ba_imu_factor) * (size_t)p->n_imu);
    if (p->n_wheel) memcpy(hb + w.o_whl, p->wheel, sizeof(gf_ba_wheel_factor) * (size_t)p->n_wheel);
    memcpy(hb + w.o_ps, w.work_start.data(), sizeof(int) * (w.n_work + 1));
    if (w.n_work) memcpy(hb + w.o_pij, w.work_ij.data(), sizeof(int) * 2 * w.n_work);
    memcpy(hb + w.o_cf, w.col_feat.data(), sizeof(int) * (size_t)(nfeat > 0 ? nfeat : 1));
    if (pr) {
        memcpy(hb + w.o_pJ, pr->linearized_jacobians, sizeof(double) * (size_t)pn * pn);
        memcpy(hb + w.o_pr0, pr->linearized_residuals, sizeof(double) * pn);
        memcpy(hb + w.o_px0, pr->x0, sizeof(double) * w.px0_len);
        memcpy(hb + w.o_pcol, w.pcol.data(), sizeof(int) * pn);
    }
    BaDev& d = w.d;
    d.col_feat = (const int*)(db + w.o_cf); d.X = (double*)(db + w.o_X); d.Xc = (double*)(db + w.o_Xc);
    d.vis = (const gf_ba_visual_factor*)(db + w.o_vis); d.pair_start = (const int*)(db + w.o_ps); d.pair_ij = (const int*)(db + w.o_pij);
    d.imu = (const gf_ba_imu_factor*)(db + w.o_imu); d.imu_sqrt = (double*)(db + w.o_sq);
    d.wheel = (const gf_ba_wheel_factor*)(db + w.o_whl); d.plane_frames = (const int*)(db + w.o_plf);
    d.pJ = (const double*)(db + w.o_pJ); d.pr0 = (const double*)(db + w.o_pr0); d.px0 = (const double*)(db + w.o_px0); d.pcol = (const int*)(db + w.o_pcol);
    d.Hp = (double*)(db + w.o_Hp); d.acc[0] = (double*)(db + w.o_a0); d.acc[1] = (double*)(db + w.o_a1);
    double* vec = (double*)(db + w.o_vec);
    const size_t nn = (size_t)(n > 0 ? n : 1);
    d.scale = vec; d.diag = vec + nn; d.gs = vec + 2 * nn; d.gn = vec + 3 * nn; d.step = vec + 4 * nn; d.delta = vec + 5 * nn;
    d.Sg = (double*)(db + w.o_Sg); d.Lg = (double*)(db + w.o_Lg);
    d.st = (BaState*)(db + w.o_st);
    for (int k = 0; k < 3; k++) d.gravity[k] = p->gravity[k];
    d.vis_sqrt_info = p->visual_sqrt_info;
}

static void ba_finish(gf_ba* s, const gf_ba_problem* p, const BaWindow& w, gf_ba_summary* sum, float ms)
{
    const char* hb = (const char*)s->hbuf + w.base;
    const double* hX = (const double*)(hb + w.o_X);
    const BaState* hs = (const BaState*)(hb + w.o_st);
    const int F = p->n_frames;
    memcpy(p->para_pose, hX + X_POSE, sizeof(double) * 7 * F);
    if (p->para_speed_bias) memcpy(p->para_speed_bias, hX + X_SB, sizeof(double) * 9 * F);
    memcpy(p->para_ex_pose, hX + X_EX, sizeof(double) * 7);
    p->para_td[0] = hX[X_TD];
    if (p->n_wheel > 0) { memcpy(p->para_ex_wheel, hX + X_EXW, sizeof(double) * 7); memcpy(p->para_ix_wheel, hX + X_IX, sizeof(double) * 3); p->para_td_wheel[0] = hX[X_TDW]; }
    if (p->n_plane > 0) { memcpy(p->para_ex_wheel, hX + X_EXW, sizeof(double) * 7); memcpy(p->para_plane_R, hX + X_PR, sizeof(double) * 4); p->para_plane_Z[0] = hX[X_PZ]; }
    memcpy(p->para_feature, hX + X_FEAT, sizeof(double) * p->n_features);
    sum->iterations = hs->it; sum->num_successful_steps = hs->n_success; sum->termination = hs->termination;
    sum->reduced_dim = w.d.nc; sum->n_free_landmarks = w.d.L; sum->n_residuals = w.pn + 15 * p->n_imu + 6 * p->n_wheel + 3 * p->n_plane + 2 * p->n_visual;
    sum->initial_cost = hs->cost_hist[0]; sum->final_cost = hs->x_cost;
    for (int k = 0; k <= GF_BA_MAX_ITERATIONS; k++) { sum->cost[k] = hs->cost_hist[k]; sum->radius[k] = hs->radius_hist[k]; }
    sum->device_ms = ms;
    memcpy(s->prof, hs->prof, sizeof(s->prof));
}

// prefixes the error text with the window it belongs to (gf_ba_solve_multi)
static int window_err(int k, int rc)
{
    char t[sizeof(g_err)];
    snprintf(t, sizeof(t), "window %d: %s", k, g_err);
    memcpy(g_err, t, sizeof(t));
    return rc;
}

static void capture_window(const gf_ba* s, const gf_ba_problem* p, const BaWindow& w, gf_ba_step_capture* c);

// gf_ba_first_step: the solve's chain stopped after the first k_ba_step, with every intermediate downloaded
struct BaCapture {
    double radius, mu;
    gf_ba_step_capture* out;      // one per window
};

// Windows k = 0..n-1 (problem ps[k] on handle hs[k]), every one validated before anything is written or enqueued.  All work goes to
// hs[0]'s stream; hs[0]'s buffers also hold the batch table: the n descriptors and the two lists of windows per k_ba_step
// instantiation.  Launch count: that of the window with the most iterations, plus one k_ba_step per iteration when both
// instantiations are needed.  cap (non-null): the same chain up to the first k_ba_step (k_ba_prior_hessian, k_ba_eval(0),
// k_ba_schur, k_ba_step), the window's whole device image copied back after k_ba_schur and after k_ba_step, nothing written back.
static int ba_batch(gf_ba* const* hs, int n, const gf_ba_problem* ps, gf_ba_summary* sums, int32_t* status, bool multi,
                    const BaCapture* cap = nullptr)
{
    std::vector<BaWindow> W(n);
    for (int k = 0; k < n; k++) { const int rc = ba_layout(hs[k], &ps[k], W[k]); if (rc) return multi ? window_err(k, rc) : rc; }
    gf_ba* lead = hs[0];
    GF_CUDA(cudaSetDevice(lead->device));
    const size_t table = al16((sizeof(BaDev) + 2 * sizeof(int)) * (size_t)n);
    for (int k = 0; k < n; k++) {
        W[k].base = k == 0 ? table : 0;
        const int rc = ensure(hs[k], W[k].base + W[k].bytes * (cap ? 2 : 1));      // a capture stages two images of the window
        if (rc) return rc;
    }
    for (int k = 0; k < n; k++) {
        if (sums) memset(&sums[k], 0, sizeof(sums[k]));
        if (status) status[k] = GF_OK;
        if (cap) ba_pack(hs[k], &ps[k], W[k], cap->radius, cap->mu, 1);
        else ba_pack(hs[k], &ps[k], W[k], 1e4, 1e-8, ps[k].max_num_iterations);
    }
    BaDev* hdesc = (BaDev*)lead->hbuf;
    int* hlist = (int*)(hdesc + n);                 // [0, n_small): k_ba_step<MAXR / 2, false>;  [n, n + n_spill): k_ba_step<MAXR, true>
    int n_small = 0, n_spill = 0, iters = 0, eval_grid = 1, schur_grid = 1, prior_grid = 0;
    bool any_eval = false;
    size_t prior_smem = 0, schur_smem = 0, step_smem[2] = {0, 0};
    for (int k = 0; k < n; k++) {
        const BaWindow& w = W[k];
        hdesc[k] = w.d;
        if (w.spill) hlist[n + n_spill++] = k; else hlist[n_small++] = k;
        iters = cap ? 0 : std::max(iters, ps[k].max_num_iterations);
        eval_grid = std::max(eval_grid, w.d.eval_grid); schur_grid = std::max(schur_grid, w.d.schur_grid);
        if (w.pn) prior_grid = std::max(prior_grid, (w.pn * w.pn + 255) / 256);
        any_eval = any_eval || w.eval_blocks > 0;
        prior_smem = std::max(prior_smem, w.prior_smem); schur_smem = std::max(schur_smem, w.schur_smem);
        step_smem[w.spill] = std::max(step_smem[w.spill], w.step_smem);
    }
    const BaDev* wins = (const BaDev*)lead->dbuf;
    const int* dlist = (const int*)(wins + n);
    cudaStream_t st = lead->s;
    GF_CUDA(cudaEventRecord(lead->e0, st));
    for (int k = 0; k < n; k++) {     // the first handle's upload carries the batch table in front of its window
        char* db = (char*)hs[k]->dbuf;
        GF_CUDA(cudaMemcpyAsync(db, hs[k]->hbuf, W[k].base + W[k].upload_bytes, cudaMemcpyHostToDevice, st));
        GF_CUDA(cudaMemsetAsync(db + W[k].base + W[k].o_Hp, 0, al16(sizeof(double) * (size_t)W[k].d.nc * W[k].d.nc) + al16(sizeof(double) * acc_size(W[k].d.nc, W[k].d.L)) * 2, st));   // H_prior, both accumulators
    }
    if (prior_grid) { k_ba_prior_hessian<<<dim3(prior_grid, n), 256, 0, st>>>(wins); GF_LAUNCHED(); }
    if (any_eval) { k_ba_eval<<<dim3(eval_grid, n), PAIR_THREADS, prior_smem, st>>>(wins, 0); GF_LAUNCHED(); }
    // Every kernel of the loop is launched with a programmatic dependency on its predecessor: its CTAs become resident while the
    // predecessor still runs and sit in griddepcontrol.wait, which hides the launch latency at the 26 kernel boundaries of a solve
    // (measured on one H100 SXM at 700 W, C2 window: 0.79-0.80 -> 0.77 ms per solve; GF_BA_NO_PDL=1 restores plain stream order for A/B runs)
    static const bool pdl = getenv("GF_BA_NO_PDL") == nullptr;
    auto launch = [&](auto kern, dim3 grid, int block, size_t smem, auto... args) -> cudaError_t {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = grid; cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
        return cudaLaunchKernelEx(&cfg, kern, args...);
    };
    // Windows with a smaller max_num_iterations are stopped by their own state (BaState::max_iter): their kernels return at once
    for (int it = 0; it <= iters; it++) {
        GF_CUDA(launch(k_ba_schur, dim3(schur_grid, n), SCHUR_WARPS * 32, schur_smem, wins)); GF_LAUNCHED();      // (the closing launch only prepares the norms)
        for (int k = 0; cap && k < n; k++) {      // the reduced system, e_l and the Cauchy sums before k_ba_step consumes them
            const size_t o = W[k].base;
            GF_CUDA(cudaMemcpyAsync((char*)hs[k]->hbuf + o + W[k].bytes, (char*)hs[k]->dbuf + o, W[k].bytes, cudaMemcpyDeviceToHost, st));
        }
        if (n_small) { GF_CUDA(launch(k_ba_step<MAXR / 2, false>, dim3(1, n_small), RB_THREADS, step_smem[0], wins, dlist)); GF_LAUNCHED(); }
        if (n_spill) { GF_CUDA(launch(k_ba_step<MAXR, true>, dim3(1, n_spill), RB_THREADS, step_smem[1], wins, dlist + n)); GF_LAUNCHED(); }
        if (it == iters) break;                  // the extra k_ba_step adopts the last linearisation and closes the run (a capture: the first step)
        GF_CUDA(launch(k_ba_eval, dim3(eval_grid, n), PAIR_THREADS, prior_smem, wins, 1)); GF_LAUNCHED();   // + decision (last CTA of each window)
    }
    GF_CUDA(cudaGetLastError());
    for (int k = 0; k < n; k++) {
        char* hb = (char*)hs[k]->hbuf + W[k].base; char* db = (char*)hs[k]->dbuf + W[k].base;
        if (cap) { GF_CUDA(cudaMemcpyAsync(hb, db, W[k].bytes, cudaMemcpyDeviceToHost, st)); continue; }
        GF_CUDA(cudaMemcpyAsync(hb + W[k].o_X, db + W[k].o_X, sizeof(double) * (X_FEAT + ps[k].n_features), cudaMemcpyDeviceToHost, st));
        GF_CUDA(cudaMemcpyAsync(hb + W[k].o_st, db + W[k].o_st, sizeof(BaState), cudaMemcpyDeviceToHost, st));
    }
    GF_CUDA(cudaEventRecord(lead->e1, st));
    GF_CUDA(cudaStreamSynchronize(st));
    float ms = 0;
    GF_CUDA(cudaEventElapsedTime(&ms, lead->e0, lead->e1));
    int rc = GF_OK;
    for (int k = n - 1; k >= 0; k--) {           // backwards: the error text names the first failing window
        const BaState* h = (const BaState*)((const char*)hs[k]->hbuf + W[k].base + W[k].o_st);
        if (h->setup_failed) {
            rc = set_err(GF_ERR_INVALID_ARG, "an IMU covariance is singular or not positive definite; parameter blocks left untouched");
            if (multi) window_err(k, rc);
            if (status) status[k] = GF_ERR_INVALID_ARG;
            continue;
        }
        if (cap) capture_window(hs[k], &ps[k], W[k], &cap->out[k]);
        else ba_finish(hs[k], &ps[k], W[k], &sums[k], ms);
    }
    return rc;
}

// 1 <= n <= GF_BA_MAX_MULTI distinct handles on one device
static int check_batch(gf_ba* const* solvers, int n)
{
    if (n < 1) return set_err(GF_ERR_INVALID_ARG, "n must be at least 1");
    if (n > GF_BA_MAX_MULTI) return set_err(GF_ERR_CAPACITY, "more than GF_BA_MAX_MULTI (256) windows");
    for (int k = 0; k < n; k++) {
        if (!solvers[k]) return window_err(k, set_err(GF_ERR_INVALID_ARG, "null handle"));
        if (solvers[k]->device != solvers[0]->device) return window_err(k, set_err(GF_ERR_INVALID_ARG, "handle bound to another device than window 0's"));
        for (int j = 0; j < k; j++)
            if (solvers[j] == solvers[k]) { snprintf(g_err, sizeof(g_err), "window %d: handle already used by window %d", k, j); return GF_ERR_INVALID_ARG; }
    }
    return GF_OK;
}

// Unpacks one window's two device images (after k_ba_schur: hbuf + base + bytes; after k_ba_step: hbuf + base) into *c
static void capture_window(const gf_ba* s, const gf_ba_problem* p, const BaWindow& w, gf_ba_step_capture* c)
{
    const char* hb = (const char*)s->hbuf + w.base;          // after k_ba_step
    const char* ha = hb + w.bytes;                           // after k_ba_schur
    const BaDev& d = w.d;
    const int nc = d.nc, L = d.L, n = d.n, F = p->n_frames;
    const size_t nn = (size_t)(n > 0 ? n : 1);
    const BaState* sa = (const BaState*)(ha + w.o_st);
    const BaState* sb = (const BaState*)(hb + w.o_st);
    c->nc = nc; c->L = L; c->n = n; c->spill = w.spill ? 1 : 0;
    for (int f = 0; f < GF_BA_MAX_FRAMES; f++) { c->col_pose[f] = d.col_pose[f]; c->col_sb[f] = d.col_sb[f]; }
    c->col_ex = d.col_ex; c->col_td = d.col_td; c->col_exw = d.col_exw; c->col_tdw = d.col_tdw; c->col_pr = d.col_pr; c->col_pz = d.col_pz;
    for (int k = 0; k < 3; k++) c->col_ix[k] = d.col_ix[k];
    c->initial_cost = sb->x_cost; c->cauchy_num = sa->cauchy_num; c->cauchy_den = sa->cauchy_den; c->alpha = sb->alpha;
    c->dogleg_a = sb->dl_a; c->dogleg_b = sb->dl_b; c->dogleg_norm = sb->dogleg_norm; c->model_change = sb->model_change;
    c->step_norm = sb->step_norm; c->grad_max = sb->grad_max; c->x_norm = sb->x_norm; c->mu = sb->mu; c->radius = sb->radius;
    c->solver_failed = sb->solver_failed; c->step_valid = sb->step_valid; c->done = sb->done; c->termination = sb->termination;
    c->iterations = sb->it;
    // the first linearisation went to accumulator 0 (the host uploads cur = 1)
    const double* acc = (const double*)(hb + w.o_a0);
    const double* vb = (const double*)(hb + w.o_vec);        // scale | D | gs | gn | step | delta
    const double* va = (const double*)(ha + w.o_vec);
    if (c->col_feat) memcpy(c->col_feat, w.col_feat.data(), sizeof(int) * (size_t)p->n_features);
    if (c->imu_sqrt) memcpy(c->imu_sqrt, hb + w.o_sq, sizeof(double) * 225 * (size_t)p->n_imu);
    if (c->H) memcpy(c->H, acc, sizeof(double) * (size_t)nc * nc);
    if (c->Hp) memcpy(c->Hp, hb + w.o_Hp, sizeof(double) * (size_t)nc * nc);
    if (c->g) memcpy(c->g, acc + (size_t)nc * nc, sizeof(double) * n);
    if (c->W) memcpy(c->W, acc + (size_t)nc * nc + n, sizeof(double) * (size_t)L * nc);
    if (c->hll) memcpy(c->hll, acc + (size_t)nc * nc + n + (size_t)L * nc, sizeof(double) * L);
    if (c->scale) memcpy(c->scale, vb, sizeof(double) * n);
    if (c->D) memcpy(c->D, vb + nn, sizeof(double) * n);
    if (c->gs) memcpy(c->gs, vb + 2 * nn, sizeof(double) * n);
    if (c->e_l) memcpy(c->e_l, va + 3 * nn + nc, sizeof(double) * L);      // gn[nc + l] holds e_l until k_ba_step overwrites it
    if (c->gn) memcpy(c->gn, vb + 3 * nn, sizeof(double) * n);
    if (c->S) {          // tiles tix(I, J) (row-major 8x8) of the (nc+1)-row augmented system -> dense lower triangle
        const double* Sg = (const double*)(ha + w.o_Sg);
        const int m = nc + 1;
        for (int a = 0; a < m; a++)
            for (int b = 0; b < m; b++)
                c->S[(size_t)a * m + b] = b > a ? 0.0 : Sg[(size_t)tix(a >> 3, b >> 3) * 64 + (a & 7) * 8 + (b & 7)];
    }
    if (c->delta)        // k_ba_step's own formula on the vectors it used (delta itself may live in shared memory only)
        for (int k = 0; k < n; k++) c->delta[k] = (sb->dl_a * vb[2 * nn + k] + sb->dl_b * vb[3 * nn + k]) / vb[nn + k] * vb[k];
    if (c->Xc) {         // pose | speed-bias | ex | td | ex_wheel | sx sy sw | td_wheel | plane R | plane Z | features
        const double* X = (const double*)(hb + w.o_Xc);
        double* o = c->Xc;
        memcpy(o, X + X_POSE, sizeof(double) * 7 * F); o += 7 * F;
        memcpy(o, X + X_SB, sizeof(double) * 9 * F); o += 9 * F;
        memcpy(o, X + X_EX, sizeof(double) * (X_FEAT - X_EX)); o += X_FEAT - X_EX;
        memcpy(o, X + X_FEAT, sizeof(double) * (size_t)p->n_features);
    }
}

extern "C" {

int gf_ba_step_dims(gf_ba* s, const gf_ba_problem* p, int* dims3)
{
    if (!s || !p || !dims3) return set_err(GF_ERR_INVALID_ARG, "null argument");
    BaWindow w;
    const int rc = ba_layout(s, p, w);
    if (rc) return rc;
    dims3[0] = w.d.nc; dims3[1] = w.d.L; dims3[2] = w.d.n;
    return GF_OK;
}

int gf_ba_first_step(gf_ba* const* solvers, int n, const gf_ba_problem* problems, double radius, double mu, gf_ba_step_capture* out)
{
    if (!solvers || !problems || !out) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (const int rc = check_batch(solvers, n)) return rc;
    // mu >= 1 skips the Gauss-Newton solve and mu = 0 would never leave k_ba_step's retry loop
    if (!(radius > 0.0) || !(mu > 0.0 && mu < 1.0)) return set_err(GF_ERR_INVALID_ARG, "radius must be > 0 and mu in (0, 1)");
    const BaCapture cap = {radius, mu, out};
    return ba_batch(solvers, n, problems, nullptr, nullptr, n > 1, &cap);
}

int gf_ba_solve(gf_ba* s, const gf_ba_problem* p, gf_ba_summary* sum)
{
    if (!s || !p || !sum) return set_err(GF_ERR_INVALID_ARG, "null argument");
    return ba_batch(&s, 1, p, sum, nullptr, false);
}

int gf_ba_solve_multi(gf_ba* const* solvers, int n, const gf_ba_problem* problems, gf_ba_summary* summaries, int32_t* status)
{
    if (!solvers || !problems || !summaries) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (const int rc = check_batch(solvers, n)) return rc;
    return ba_batch(solvers, n, problems, summaries, status, true);
}

/* MARGIN_OLD (estimator.cpp:3334-3535) + MarginalizationInfo::{preMarginalize, marginalize}
 * (marginalization_factor.cpp:115-308) on the GPU: the factors that touch frame 0 -- last prior, IMU(0->1), every visual
 * factor whose landmark starts in frame 0 -- are linearised by the same kernels as the solve into one dense system over
 * [pose0, speedbias0, those landmarks | kept blocks]; the marginalised part is eliminated with the eigen-truncated
 * inverse (eps 1e-8) and the result is re-factored into J0 = sqrt(S) V^T, r0 = sqrt(S^-1) V^T b, exactly the reference's
 * two SelfAdjointEigenSolver calls (here: parallel-ordered Jacobi).  Kept blocks are ordered pose[1..], speedbias[1..],
 * ex_pose, td and their indices are already shifted by one frame (addr_shift, estimator.cpp:3500-3534).
 * The WheelFactor(0->1) joins when the window has wheel factors (its extrinsic / sx / sy / sw / time offset become kept
 * blocks); plane / GNSS factors are not implemented.  out_x0 / out_J / out_r must hold 16*n_frames+19, n*n, n doubles.
 * Returns n (> 0) or a negative error code. */
}  // extern "C" (reopened below)

// MarginalizationInfo::marginalize (marginalization_factor.cpp:272-302) on the dense system q.A, q.b already on the device,
// columns [c dense | m - c diagonal landmarks | n kept]: the structured fast path when it applies, else the literal
// eigen-truncated inverse of Amm; then the eigendecomposition of the reduced system and J0, r0.  d_sw: int[3] on the device
// ([0], [1] Jacobi sweeps of Amm and of the reduced system, [2] the fast path's flag), h_flag: one host int (pinned in marg_run).  Host
// synchronisation: one, to read the fast path's flag.  *path: GF_MARG_PATH_* bits.
static int marg_schur_eig(const MargDev& q, int cdim, bool force_generic, double* Q, double* qb, double* Ceps, int* d_sw, int* h_flag,
                          cudaStream_t st, int* path)
{
    const int m = q.m, n = q.n, Rdim = cdim + n;
    const size_t mm = (size_t)m * m, nn = (size_t)n * n;
    auto jac_smem = [](int nn_) { int hp = ((nn_ + 1) & ~1) / 2; return (size_t)hp * (2 * sizeof(double) + 2 * sizeof(int)) + 8; };
    int* d_flag = d_sw + 2;
    int p = n > 127 ? GF_MARG_PATH_GENERIC | GF_MARG_PATH_WIDE                 // k_marg_c_elim's shared buffer
          : force_generic ? GF_MARG_PATH_GENERIC | GF_MARG_PATH_FORCED : 0;
    if (!p) {
        // regular case: Amm - eps I positive definite => eigen-truncated inverse == inverse => two-stage Schur complement
        GF_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        k_marg_lm_elim<<<(std::max(Rdim * Rdim, m) + 255) / 256, 256, 0, st>>>(q, cdim, Q, qb, Ceps, d_flag); GF_LAUNCHED();
        k_marg_c_elim<<<1, 256, 0, st>>>(q, cdim, Q, qb, Ceps, d_flag); GF_LAUNCHED();
        GF_CUDA(cudaMemcpyAsync(h_flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
        GF_CUDA(cudaStreamSynchronize(st));
        if (*h_flag != 0) p = GF_MARG_PATH_GENERIC | GF_MARG_PATH_NOT_PD;
    }
    if (p & GF_MARG_PATH_GENERIC) {   // some eigenvalue of Amm may be below eps: the reference's eigen-truncated inverse, literally
        k_marg_amm<<<(int)((mm + 255) / 256), 256, 0, st>>>(q); GF_LAUNCHED();
        k_jacobi_eig<<<1, 1024, jac_smem(m), st>>>(q.Amm, q.Vm, q.wm, m, d_sw); GF_LAUNCHED();
        k_marg_ainv<<<(int)((mm + 255) / 256), 256, 0, st>>>(q); GF_LAUNCHED();
        k_marg_T<<<(int)(((size_t)n * m + 255) / 256), 256, 0, st>>>(q); GF_LAUNCHED();
        k_marg_reduce<<<(int)((nn + 255) / 256), 256, 0, st>>>(q); GF_LAUNCHED();
    }
    if (n <= 128) {   // tridiagonalisation + implicit QL in shared memory (what the reference's Eigen solver does)
        k_sym_eig_ql<<<1, QL_T, sizeof(double) * ((size_t)n * n + 4 * (size_t)n + 8), st>>>(q.Ar, q.Vr, q.wr, n); GF_LAUNCHED();
    } else {
        k_jacobi_eig<<<1, 1024, jac_smem(n), st>>>(q.Ar, q.Vr, q.wr, n, d_sw + 1); GF_LAUNCHED();
        p |= GF_MARG_PATH_REDUCED_JACOBI;
    }
    k_marg_out<<<(int)((nn + 255) / 256), 256, 0, st>>>(q); GF_LAUNCHED();
    GF_CUDA(cudaGetLastError());
    *path = p;
    return GF_OK;
}

enum { GF_MARG_OLD = 0, GF_MARG_SECOND_NEW = 1 };
static int marg_run(gf_ba* s, const gf_ba_problem* p, int mode, gf_ba_prior* out, double* out_x0, double* out_J, double* out_r, float* device_ms)
{
    if (!s || !p || !out || !out_x0 || !out_J || !out_r) return set_err(GF_ERR_INVALID_ARG, "null argument");
    if (p->n_frames < 2 || p->n_frames > GF_BA_MAX_FRAMES) return set_err(GF_ERR_INVALID_ARG, "n_frames out of range");
    GF_CUDA(cudaSetDevice(s->device));
    const int F = p->n_frames, nfeat = p->n_features;
    const bool use_sb = p->para_speed_bias && !p->pose0_const;
    // a residual block may not list one parameter block twice (ceres::Problem refuses it; the reference never builds one)
    for (int v = 0; v < p->n_visual; v++) if (p->visual[v].imu_i == p->visual[v].imu_j) return set_err(GF_ERR_INVALID_ARG, "visual factor with imu_i == imu_j");
    // ---- the marginalised and the kept blocks (same rules as the oracle) ----
    std::vector<int> lm_col(nfeat > 0 ? nfeat : 1, -1);
    int pos = 0;
    BaDev d; memset(&d, 0, sizeof(d));
    d.F = F; d.nfeat = nfeat; d.lm_dense = 1;
    for (int f = 0; f < MAXF; f++) { d.col_pose[f] = -1; d.col_sb[f] = -1; }
    d.col_ex = d.col_td = d.col_exw = d.col_tdw = -1; d.col_ix[0] = d.col_ix[1] = d.col_ix[2] = -1; d.col_pr = d.col_pz = -1; d.n_plane = 0;
    const bool old_ = mode == GF_MARG_OLD;
    const int fdrop = old_ ? 0 : F - 2;                        // MARGIN_OLD drops frame 0, MARGIN_SECOND_NEW para_Pose[WINDOW_SIZE - 1]
    const gf_ba_prior* pr = (p->prior && p->prior->n > 0) ? p->prior : nullptr;
    if (!old_) {
        // estimator.cpp:3538-3539: only when the last prior holds para_Pose[WINDOW_SIZE - 1]; otherwise the prior stays as it is
        bool has = false;
        if (pr) for (int b = 0; b < pr->n_blocks; b++) if (pr->block_kind[b] == GF_BA_BLOCK_POSE && pr->block_index[b] == fdrop) has = true;
        if (!has) return 0;
    }
    d.col_pose[fdrop] = pos; pos += 6;
    if (old_ && use_sb) { d.col_sb[0] = pos; pos += 9; }
    std::vector<gf_ba_visual_factor> vis0;
    for (int v = 0; old_ && v < p->n_visual; v++) {
        const gf_ba_visual_factor& f = p->visual[v];
        if (f.feature < 0 || f.feature >= nfeat || f.imu_i < 0 || f.imu_i >= F || f.imu_j < 0 || f.imu_j >= F) return set_err(GF_ERR_INVALID_ARG, "visual factor index out of range");
        if (f.imu_i != 0) continue;
        if (lm_col[f.feature] < 0) lm_col[f.feature] = pos++;
        vis0.push_back(f);
    }
    const int m = pos;
    bool used_pose[MAXF] = {}, used_sb[MAXF] = {}, used_ex = false, used_td = false, used_exw = false, used_ix[3] = {false, false, false}, used_tdw = false, used_pr = false, used_pz = false;
    if (pr) {
        if (pr->n_blocks > 64) return set_err(GF_ERR_CAPACITY, "more than 64 prior blocks");
        for (int b = 0; b < pr->n_blocks; b++) {
            const int k = pr->block_kind[b], i = pr->block_index[b];
            if (k == GF_BA_BLOCK_POSE || k == GF_BA_BLOCK_SPEEDBIAS) { if (i < 0 || i >= F) return set_err(GF_ERR_INVALID_ARG, "prior block index out of range"); (k == GF_BA_BLOCK_POSE ? used_pose : used_sb)[i] = true; }
            else if (k == GF_BA_BLOCK_EX_POSE) used_ex = true;
            else if (k == GF_BA_BLOCK_TD) used_td = true;
            else if (k == GF_BA_BLOCK_EX_WHEEL) used_exw = true;
            else if (k >= GF_BA_BLOCK_SX && k <= GF_BA_BLOCK_SW) used_ix[k - GF_BA_BLOCK_SX] = true;
            else if (k == GF_BA_BLOCK_TD_WHEEL) used_tdw = true;
            else if (k == GF_BA_BLOCK_PLANE_R) used_pr = true;
            else if (k == GF_BA_BLOCK_PLANE_Z) used_pz = true;
            else return set_err(GF_ERR_INVALID_ARG, "unknown prior block kind");
        }
    }
    const gf_ba_imu_factor* imu01 = nullptr;
    for (int k = 0; old_ && k < p->n_imu; k++) if (p->imu[k].i == 0 && p->imu[k].j == 1 && p->imu[k].sum_dt < 10.0) { imu01 = &p->imu[k]; used_pose[1] = true; used_sb[1] = true; }
    for (const auto& f : vis0) { used_pose[f.imu_j] = true; used_ex = true; used_td = true; }
    // WheelFactor(pre_integrations_wheel[1]) with para_Pose[0] dropped (estimator.cpp:3367-3377)
    const gf_ba_wheel_factor* wheel01 = nullptr;
    if (p->n_wheel > 0 && (!p->wheel || !p->para_ex_wheel || !p->para_ix_wheel || !p->para_td_wheel)) return set_err(GF_ERR_INVALID_ARG, "wheel factors without their parameter blocks");
    for (int k = 0; old_ && k < p->n_wheel; k++) if (p->wheel[k].i == 0 && p->wheel[k].j == 1 && p->wheel[k].sum_dt < 10.0) { wheel01 = &p->wheel[k]; used_pose[1] = true; used_exw = true; used_ix[0] = used_ix[1] = used_ix[2] = true; used_tdw = true; }
    // PlaneFactor(para_Pose[0], para_Ex_Pose_wheel, para_plane_R, para_plane_Z) with para_Pose[0] dropped (estimator.cpp:3379-3390)
    bool plane0 = false;
    for (int k = 0; old_ && k < p->n_plane; k++) if (p->plane_frames && p->plane_frames[k] == 0) plane0 = true;
    if (plane0) {
        if (!p->para_ex_wheel || !p->para_plane_R || !p->para_plane_Z) return set_err(GF_ERR_INVALID_ARG, "plane factor without its parameter blocks");
        used_exw = used_pr = used_pz = true;
    }
    if ((used_ix[0] || used_ix[1] || used_ix[2] || used_tdw) && (!p->para_ix_wheel || !p->para_td_wheel)) return set_err(GF_ERR_INVALID_ARG, "prior on wheel blocks without the wheel parameter blocks");
    if (used_exw && !p->para_ex_wheel) return set_err(GF_ERR_INVALID_ARG, "prior on the wheel extrinsic without para_ex_wheel");
    if ((used_pr || used_pz) && (!p->para_plane_R || !p->para_plane_Z)) return set_err(GF_ERR_INVALID_ARG, "prior on the plane blocks without para_plane_R / para_plane_Z");
    for (int f = 0; f < F; f++) if (f != fdrop && used_pose[f]) { d.col_pose[f] = pos; pos += 6; }
    for (int f = 0; f < F; f++) if (!(old_ && f == 0) && used_sb[f] && use_sb) { d.col_sb[f] = pos; pos += 9; }
    if (used_ex) { d.col_ex = pos; pos += 6; }
    if (used_td) { d.col_td = pos; pos += 1; }
    if (used_exw) { d.col_exw = pos; pos += 6; }
    for (int k = 0; k < 3; k++) if (used_ix[k]) d.col_ix[k] = pos++;
    if (used_tdw) d.col_tdw = pos++;
    // the plane rotation has 4 columns here: MarginalizationInfo::localSize only knows the 7 -> 6 case (marginalization_factor.h),
    // PlaneFactor fills the first three (plane_factor.h:95-101), the fourth stays zero
    if (used_pr) { d.col_pr = pos; pos += 4; }
    if (used_pz) d.col_pz = pos++;
    const int N = pos, n = N - m;
    if (n <= 0) return set_err(GF_ERR_INVALID_ARG, "nothing is kept by the marginalisation");
    d.nc = N; d.L = 0; d.n = N; d.n_vis = (int)vis0.size(); d.n_imu = imu01 ? 1 : 0; d.n_wheel = wheel01 ? 1 : 0; d.n_plane = plane0 ? 1 : 0;
    d.pr_mask = 0; for (int k = 0; k < 3; k++) d.plane_sinfo[k] = p->plane_sqrt_info[k];
    // ---- visual factors by pose pair (0, j), cut into chunks ----
    std::vector<int> cnt(F, 0), start(F + 1, 0);
    for (const auto& f : vis0) cnt[f.imu_j]++;
    for (int j = 0; j < F; j++) start[j + 1] = start[j] + cnt[j];
    std::vector<int> work_start(1, 0), work_ij;
    for (int j = 0; j < F; j++)
        for (int c0 = start[j]; c0 < start[j + 1]; c0 += PAIR_CHUNK) { work_ij.push_back(0); work_ij.push_back(j); work_start.push_back(std::min(c0 + PAIR_CHUNK, start[j + 1])); }
    const int n_work = (int)work_ij.size() / 2;
    d.n_pairs = n_work;
    const int pn = pr ? pr->n : 0;
    std::vector<int> pcol(pn > 0 ? pn : 1, -1);
    size_t px0_len = 0;
    if (pr) {
        d.pn = pn; d.pnb = pr->n_blocks;
        for (int b = 0; b < pr->n_blocks; b++) {
            const int kind = pr->block_kind[b], idx = pr->block_index[b];
            d.pkind[b] = kind; d.pindex[b] = idx; d.pidx[b] = pr->block_idx[b]; d.pxoff[b] = (int)px0_len;
            const int gs = (kind == GF_BA_BLOCK_POSE || kind == GF_BA_BLOCK_EX_POSE || kind == GF_BA_BLOCK_EX_WHEEL) ? 7 : kind == GF_BA_BLOCK_SPEEDBIAS ? 9 : kind == GF_BA_BLOCK_PLANE_R ? 4 : 1, ls = gs == 7 ? 6 : gs;
            const int lc = kind == GF_BA_BLOCK_POSE ? d.col_pose[idx] : kind == GF_BA_BLOCK_SPEEDBIAS ? d.col_sb[idx] : kind == GF_BA_BLOCK_EX_POSE ? d.col_ex : kind == GF_BA_BLOCK_TD ? d.col_td
                           : kind == GF_BA_BLOCK_EX_WHEEL ? d.col_exw : kind == GF_BA_BLOCK_TD_WHEEL ? d.col_tdw : kind == GF_BA_BLOCK_PLANE_R ? d.col_pr : kind == GF_BA_BLOCK_PLANE_Z ? d.col_pz
                           : d.col_ix[kind - GF_BA_BLOCK_SX];
            if (lc >= 0) for (int k = 0; k < ls; k++) pcol[pr->block_idx[b] + k] = lc + k;
            px0_len += gs;
        }
    }
    // ---- one upload buffer + work space ----
    auto al = [](size_t v) { return (v + 15) / 16 * 16; };
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += al(bytes); return o; };
    const size_t nv = vis0.size();
    const size_t o_X = take(sizeof(double) * (X_FEAT + nfeat)), o_vis = take(sizeof(gf_ba_visual_factor) * (nv ? nv : 1)), o_imu = take(sizeof(gf_ba_imu_factor)), o_whl = take(sizeof(gf_ba_wheel_factor)), o_plf = take(sizeof(int) * 4),
                 o_ps = take(sizeof(int) * (n_work + 1)), o_pij = take(sizeof(int) * 2 * (size_t)(n_work > 0 ? n_work : 1)), o_cf = take(sizeof(int) * (size_t)(nfeat > 0 ? nfeat : 1)),
                 o_pJ = take(sizeof(double) * (size_t)pn * pn), o_pr0 = take(sizeof(double) * pn), o_px0 = take(sizeof(double) * px0_len), o_pcol = take(sizeof(int) * (size_t)(pn > 0 ? pn : 1));
    const size_t o_st = take(sizeof(BaState)), o_dev = take(sizeof(BaDev));
    const size_t upload_bytes = off;
    const size_t NN = (size_t)N * N, mm = (size_t)m * m, nn = (size_t)n * n;
    const size_t o_sq = take(sizeof(double) * 225), o_Hp = take(sizeof(double) * NN), o_a0 = take(sizeof(double) * acc_size(N, 0)),
                 o_A = take(sizeof(double) * NN), o_b = take(sizeof(double) * N), o_Amm = take(sizeof(double) * mm), o_Vm = take(sizeof(double) * mm), o_wm = take(sizeof(double) * m),
                 o_Ainv = take(sizeof(double) * mm), o_T = take(sizeof(double) * (size_t)n * m), o_Ar = take(sizeof(double) * nn), o_Vr = take(sizeof(double) * nn),
                 o_wr = take(sizeof(double) * n), o_br = take(sizeof(double) * n), o_J0 = take(sizeof(double) * nn), o_r0 = take(sizeof(double) * n), o_sw = take(sizeof(int) * 4),
                 o_Q = take(sizeof(double) * (size_t)(15 + n) * (15 + n)), o_qb = take(sizeof(double) * (15 + n)), o_ce = take(sizeof(double) * 225);
    int rc = ensure(s, off);
    if (rc) return rc;
    char* hb = (char*)s->hbuf; char* db = (char*)s->dbuf;
    double* hX = (double*)(hb + o_X);
    memset(hX, 0, sizeof(double) * (X_FEAT + nfeat));
    memcpy(hX + X_POSE, p->para_pose, sizeof(double) * 7 * F);
    if (p->para_speed_bias) memcpy(hX + X_SB, p->para_speed_bias, sizeof(double) * 9 * F);
    memcpy(hX + X_EX, p->para_ex_pose, sizeof(double) * 7);
    hX[X_TD] = p->para_td[0];
    hX[X_EXW + 6] = 1.0; hX[X_IX] = hX[X_IX + 1] = hX[X_IX + 2] = 1.0;
    if (p->para_ex_wheel) memcpy(hX + X_EXW, p->para_ex_wheel, sizeof(double) * 7);
    if (p->para_ix_wheel && p->para_td_wheel) { memcpy(hX + X_IX, p->para_ix_wheel, sizeof(double) * 3); hX[X_TDW] = p->para_td_wheel[0]; }
    hX[X_PR + 3] = 1.0;
    if (p->para_plane_R && p->para_plane_Z) { memcpy(hX + X_PR, p->para_plane_R, sizeof(double) * 4); hX[X_PZ] = p->para_plane_Z[0]; }
    ((int*)(hb + o_plf))[0] = 0;                               // the one PlaneFactor of the marginalisation sits on frame 0
    memcpy(hX + X_FEAT, p->para_feature, sizeof(double) * nfeat);
    {   // state: linearise into buffer 0 (k_ba_eval mode 0 also forms the sqrt-information of IMU(0->1))
        BaState* h0 = (BaState*)(hb + o_st);
        memset(h0, 0, sizeof(BaState));
        h0->radius = 1e4; h0->mu = 1e-8; h0->need_linearize = 1; h0->cur = 1; h0->first = 1;
    }
    {
        gf_ba_visual_factor* hv = (gf_ba_visual_factor*)(hb + o_vis);
        std::vector<int> fill(start.begin(), start.end() - 1);
        for (const auto& f : vis0) hv[fill[f.imu_j]++] = f;
    }
    if (imu01) memcpy(hb + o_imu, imu01, sizeof(gf_ba_imu_factor));
    if (wheel01) memcpy(hb + o_whl, wheel01, sizeof(gf_ba_wheel_factor));
    memcpy(hb + o_ps, work_start.data(), sizeof(int) * (n_work + 1));
    if (n_work) memcpy(hb + o_pij, work_ij.data(), sizeof(int) * 2 * n_work);
    memcpy(hb + o_cf, lm_col.data(), sizeof(int) * (size_t)(nfeat > 0 ? nfeat : 1));
    if (pr) {
        memcpy(hb + o_pJ, pr->linearized_jacobians, sizeof(double) * (size_t)pn * pn);
        memcpy(hb + o_pr0, pr->linearized_residuals, sizeof(double) * pn);
        memcpy(hb + o_px0, pr->x0, sizeof(double) * px0_len);
        memcpy(hb + o_pcol, pcol.data(), sizeof(int) * pn);
    }
    d.X = (double*)(db + o_X); d.Xc = d.X;
    d.vis = (const gf_ba_visual_factor*)(db + o_vis); d.pair_start = (const int*)(db + o_ps); d.pair_ij = (const int*)(db + o_pij);
    d.imu = (const gf_ba_imu_factor*)(db + o_imu); d.imu_sqrt = (double*)(db + o_sq); d.wheel = (const gf_ba_wheel_factor*)(db + o_whl);
    d.plane_frames = (const int*)(db + o_plf);
    d.col_feat = (const int*)(db + o_cf);
    d.pJ = (const double*)(db + o_pJ); d.pr0 = (const double*)(db + o_pr0); d.px0 = (const double*)(db + o_px0); d.pcol = (const int*)(db + o_pcol);
    d.Hp = (double*)(db + o_Hp); d.acc[0] = (double*)(db + o_a0); d.acc[1] = d.acc[0];
    d.st = (BaState*)(db + o_st);
    memcpy(d.gravity, p->gravity, sizeof(d.gravity)); d.vis_sqrt_info = p->visual_sqrt_info;
    const int eval_blocks = n_work + d.n_imu + d.n_wheel + d.n_plane + (pn ? 1 : 0);
    d.eval_grid = eval_blocks;
    memcpy(hb + o_dev, &d, sizeof(d));                         // the kernels read the descriptor from the device (a batch of one window)
    const BaDev* dd = (const BaDev*)(db + o_dev);
    MargDev q;
    q.N = N; q.m = m; q.n = n; q.H = d.acc[0]; q.Hp = d.Hp; q.g = d.acc[0] + NN;      // acc layout: [H N*N | g N | ...]
    q.A = (double*)(db + o_A); q.b = (double*)(db + o_b); q.Amm = (double*)(db + o_Amm); q.Vm = (double*)(db + o_Vm); q.wm = (double*)(db + o_wm);
    q.Ainv = (double*)(db + o_Ainv); q.T = (double*)(db + o_T); q.Ar = (double*)(db + o_Ar); q.Vr = (double*)(db + o_Vr); q.wr = (double*)(db + o_wr);
    q.br = (double*)(db + o_br); q.J0 = (double*)(db + o_J0); q.r0 = (double*)(db + o_r0);
    cudaStream_t st = s->s;
    GF_CUDA(cudaEventRecord(s->e0, st));
    GF_CUDA(cudaMemcpyAsync(db, hb, upload_bytes, cudaMemcpyHostToDevice, st));
    GF_CUDA(cudaMemsetAsync(db + o_Hp, 0, al(sizeof(double) * NN) + al(sizeof(double) * acc_size(N, 0)), st));     // H_prior and the accumulator
    if (pn) { k_ba_prior_hessian<<<(pn * pn + 255) / 256, 256, 0, st>>>(dd); GF_LAUNCHED(); }
    if (eval_blocks > 0) { k_ba_eval<<<eval_blocks, PAIR_THREADS, sizeof(double) * 2 * (size_t)pn, st>>>(dd, 0); GF_LAUNCHED(); }
    k_marg_pack<<<(int)((NN + 255) / 256), 256, 0, st>>>(q); GF_LAUNCHED();
    const int cdim = (old_ && use_sb) ? 15 : 6;
    int path = 0;
    rc = marg_schur_eig(q, cdim, false, (double*)(db + o_Q), (double*)(db + o_qb), (double*)(db + o_ce), (int*)(db + o_sw), (int*)(hb + o_sw), st, &path);
    if (rc) return rc;
    GF_CUDA(cudaMemcpyAsync(hb + o_J0, db + o_J0, sizeof(double) * nn, cudaMemcpyDeviceToHost, st));
    GF_CUDA(cudaMemcpyAsync(hb + o_r0, db + o_r0, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    GF_CUDA(cudaMemcpyAsync(hb + o_st, db + o_st, sizeof(BaState), cudaMemcpyDeviceToHost, st));
    GF_CUDA(cudaEventRecord(s->e1, st));
    GF_CUDA(cudaMemcpyAsync(hb + o_sw, db + o_sw, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));     // sweep counts (not timed)
    GF_CUDA(cudaStreamSynchronize(st));
    s->marg_info[0] = path;
    s->marg_info[1] = (path & GF_MARG_PATH_GENERIC) ? ((int*)(hb + o_sw))[0] : 0;
    s->marg_info[2] = (path & GF_MARG_PATH_REDUCED_JACOBI) ? ((int*)(hb + o_sw))[1] : 0;
    if (((BaState*)(hb + o_st))->setup_failed) return set_err(GF_ERR_INVALID_ARG, "IMU covariance is not positive definite");
    if (device_ms) GF_CUDA(cudaEventElapsedTime(device_ms, s->e0, s->e1));
    memcpy(out_J, hb + o_J0, sizeof(double) * nn);
    memcpy(out_r, hb + o_r0, sizeof(double) * n);
    // ---- kept blocks after addr_shift (estimator.cpp:3500-3534 / 3583-3621): MARGIN_OLD shifts every frame down by one,
    // MARGIN_SECOND_NEW moves frame F-1 into the slot of the dropped frame F-2 ----
    memset(out, 0, sizeof(*out));
    out->n = n;
    int nb = 0; double* xp = out_x0;
    auto shifted = [&](int f) { return old_ ? f - 1 : (f == F - 1 ? F - 2 : f); };
    for (int f = 0; f < F; f++) if (f != fdrop && d.col_pose[f] >= 0) { out->block_kind[nb] = GF_BA_BLOCK_POSE; out->block_index[nb] = shifted(f); out->block_idx[nb] = d.col_pose[f] - m; memcpy(xp, p->para_pose + 7 * f, 56); xp += 7; nb++; }
    for (int f = 0; f < F; f++) if (!(old_ && f == 0) && d.col_sb[f] >= 0) { out->block_kind[nb] = GF_BA_BLOCK_SPEEDBIAS; out->block_index[nb] = shifted(f); out->block_idx[nb] = d.col_sb[f] - m; memcpy(xp, p->para_speed_bias + 9 * f, 72); xp += 9; nb++; }
    if (d.col_ex >= 0) { out->block_kind[nb] = GF_BA_BLOCK_EX_POSE; out->block_index[nb] = 0; out->block_idx[nb] = d.col_ex - m; memcpy(xp, p->para_ex_pose, 56); xp += 7; nb++; }
    if (d.col_td >= 0) { out->block_kind[nb] = GF_BA_BLOCK_TD; out->block_index[nb] = 0; out->block_idx[nb] = d.col_td - m; xp[0] = p->para_td[0]; xp += 1; nb++; }
    if (d.col_exw >= 0) { out->block_kind[nb] = GF_BA_BLOCK_EX_WHEEL; out->block_index[nb] = 0; out->block_idx[nb] = d.col_exw - m; memcpy(xp, p->para_ex_wheel, 56); xp += 7; nb++; }
    for (int k = 0; k < 3; k++) if (d.col_ix[k] >= 0) { out->block_kind[nb] = GF_BA_BLOCK_SX + k; out->block_index[nb] = 0; out->block_idx[nb] = d.col_ix[k] - m; xp[0] = p->para_ix_wheel[k]; xp += 1; nb++; }
    if (d.col_tdw >= 0) { out->block_kind[nb] = GF_BA_BLOCK_TD_WHEEL; out->block_index[nb] = 0; out->block_idx[nb] = d.col_tdw - m; xp[0] = p->para_td_wheel[0]; xp += 1; nb++; }
    if (d.col_pr >= 0) { out->block_kind[nb] = GF_BA_BLOCK_PLANE_R; out->block_index[nb] = 0; out->block_idx[nb] = d.col_pr - m; memcpy(xp, p->para_plane_R, 32); xp += 4; nb++; }
    if (d.col_pz >= 0) { out->block_kind[nb] = GF_BA_BLOCK_PLANE_Z; out->block_index[nb] = 0; out->block_idx[nb] = d.col_pz - m; xp[0] = p->para_plane_Z[0]; xp += 1; nb++; }
    out->n_blocks = nb; out->x0 = out_x0; out->linearized_jacobians = out_J; out->linearized_residuals = out_r;
    return n;
}

extern "C" {

int gf_ba_marginalize_old(gf_ba* s, const gf_ba_problem* p, gf_ba_prior* out, double* out_x0, double* out_J, double* out_r, float* device_ms)
{
    return marg_run(s, p, GF_MARG_OLD, out, out_x0, out_J, out_r, device_ms);
}

/* MARGIN_SECOND_NEW (estimator.cpp:3536-3631): the only factor is the last prior, evaluated at the current state (r = r0 + J0 dx),
 * para_Pose[WINDOW_SIZE - 1] (frame n_frames - 2) is marginalised by the same eigen-truncated Schur complement and the result is
 * re-factored into J0 / r0; frame n_frames - 1 takes the index of the dropped frame.  Returns n > 0, 0 when the prior does not
 * hold that pose (the reference then keeps the prior untouched), or a negative error code. */
int gf_ba_marginalize_second_new(gf_ba* s, const gf_ba_problem* p, gf_ba_prior* out, double* out_x0, double* out_J, double* out_r, float* device_ms)
{
    return marg_run(s, p, GF_MARG_SECOND_NEW, out, out_x0, out_J, out_r, device_ms);
}

/* Estimator::double2vector (reference estimator.cpp:2440-2494): after the solve the whole window is rotated about z and
 * shifted so that frame 0 keeps the yaw and the position it had before (the 4 unobservable DoF of a VIO window), with the
 * reference's Euler-singularity branch.  Pure host code: Utility::R2ypr / ypr2R (utility/utility.h:78-120) restated. */
static void gf_q_to_R(const double* q, double* R)     /* q = x y z w, normalised first as Quaterniond::normalized() */
{
    double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
    R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
    R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
}
static void gf_R2ypr(const double* R, double* ypr)
{
    const double n0 = R[0], n1 = R[3], n2 = R[6], o0 = R[1], o1 = R[4], a0 = R[2], a1 = R[5];
    const double y = atan2(n1, n0);
    const double p = atan2(-n2, n0 * cos(y) + n1 * sin(y));
    const double r = atan2(a0 * sin(y) - a1 * cos(y), -o0 * sin(y) + o1 * cos(y));
    ypr[0] = y / M_PI * 180.0; ypr[1] = p / M_PI * 180.0; ypr[2] = r / M_PI * 180.0;
}
int gf_ba_double2vector(const gf_ba_problem* p, const double* R0_before, const double* P0_before, int use_imu,
                        double* Rs, double* Ps, double* Vs)
{
    if (!p || !p->para_pose || !Rs || !Ps || (use_imu && (!R0_before || !P0_before))) return set_err(GF_ERR_INVALID_ARG, "null argument");
    const int F = p->n_frames;
    if (F < 1 || F > GF_BA_MAX_FRAMES) return set_err(GF_ERR_INVALID_ARG, "n_frames out of range");
    double rot[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (use_imu) {
        double R00[9], y0[3], y00[3];
        gf_q_to_R(p->para_pose + 3, R00);
        // the reference builds R00 with toRotationMatrix() of the un-normalised quaternion; Ceres keeps it unit-norm
        gf_R2ypr(R0_before, y0); gf_R2ypr(R00, y00);
        const double yd = (y0[0] - y00[0]) / 180.0 * M_PI;
        rot[0] = cos(yd); rot[1] = -sin(yd); rot[3] = sin(yd); rot[4] = cos(yd);          // ypr2R(y_diff, 0, 0)
        if (fabs(fabs(y0[1]) - 90) < 1.0 || fabs(fabs(y00[1]) - 90) < 1.0)                 // euler singular point
            for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { double v = 0; for (int k = 0; k < 3; k++) v += R0_before[r * 3 + k] * R00[c * 3 + k]; rot[r * 3 + c] = v; }
    }
    for (int i = 0; i < F; i++) {
        double Ri[9];
        gf_q_to_R(p->para_pose + 7 * i + 3, Ri);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { double v = 0; for (int k = 0; k < 3; k++) v += rot[r * 3 + k] * Ri[k * 3 + c]; Rs[9 * i + r * 3 + c] = v; }
        double dpos[3];
        for (int k = 0; k < 3; k++) dpos[k] = use_imu ? p->para_pose[7 * i + k] - p->para_pose[k] : p->para_pose[7 * i + k];
        for (int r = 0; r < 3; r++) Ps[3 * i + r] = rot[r * 3] * dpos[0] + rot[r * 3 + 1] * dpos[1] + rot[r * 3 + 2] * dpos[2] + (use_imu ? P0_before[r] : 0.0);
        if (Vs && use_imu && p->para_speed_bias)
            for (int r = 0; r < 3; r++) Vs[3 * i + r] = rot[r * 3] * p->para_speed_bias[9 * i] + rot[r * 3 + 1] * p->para_speed_bias[9 * i + 1] + rot[r * 3 + 2] * p->para_speed_bias[9 * i + 2];
    }
    return GF_OK;
}

int gf_ba_last_marg_info(gf_ba* s, int* info3)
{
    if (!s || !info3) return set_err(GF_ERR_INVALID_ARG, "null argument");
    memcpy(info3, s->marg_info, sizeof(s->marg_info));
    return GF_OK;
}

/* debug: clock64() cycles per phase of k_ba_step of the last solve (see PH() markers) */
int gf_ba_debug_profile(gf_ba* s, long long* out32)
{
    if (!s || !out32) return set_err(GF_ERR_INVALID_ARG, "null argument");
    memcpy(out32, s->prof, sizeof(s->prof));
    return GF_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// Stage-level entry point (tests): the solver's tiled Cholesky + back substitution on an arbitrary SPD system.
namespace gfba {
template <int R, bool SPILL>
__global__ void __launch_bounds__(ST_THREADS) k_stage_chol(const double* Ag, double* Lg, int cap, int nc, double* y, int* fail)
{
    extern __shared__ __align__(128) double S[];
    __shared__ __align__(8) unsigned long long mbar;
    __shared__ int s_fail;
    const int tid = threadIdx.x;
    const int n8 = (nc + 8) >> 3, ntiles = n8 * (n8 + 1) / 2, ntl = min(ntiles, cap);
    TileStoreT<SPILL> T; T.sb = ch_tiles_u32(); T.Lg = Lg; T.cap = cap;
    double* Linv = S + (size_t)64 * ntl;
    double* S8 = Linv + 64 * n8; double* Ld = S8 + 128; double* yc = Ld + 64; double* zz = yc + ((nc + 8) & ~7);
    if (tid == 0) { s_fail = 0; ch_mbar_init(&mbar, 1); chol_issue_load(Ag, S, ntl, &mbar); }
    __syncthreads();
    if (ntl > 0) ch_mbar_wait(&mbar, 0);
    const bool ok = chol_factor<R, SPILL>(Ag, T, Linv, S8, Ld, nc, n8, &s_fail);
    if (ok) chol_backsubst(T, Linv, Ld, yc, zz, nc);
    __syncthreads();
    if (ok) for (int c = tid; c < nc; c += blockDim.x) y[c] = yc[c];
    if (tid == 0) *fail = ok ? 0 : 1;
}
}  // namespace gfba

extern "C" int gf_stage_spd_solve(int device, const double* A, const double* b, int n, double* x, int tile_cap)
{
    if (!A || !b || !x || n < 1 || n > MAX_NC) return set_err(GF_ERR_INVALID_ARG, "bad argument (1 <= n <= 383)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_err(GF_ERR_NO_DEVICE, "no CUDA device visible; libgf_b200 has no CPU fallback");
    if (device < 0 || device >= ndev) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    const int n8 = (n + 8) / 8, ntiles = n8 * (n8 + 1) / 2;
    const int cap = (tile_cap >= 0 && tile_cap < TILE_CAP) ? tile_cap : TILE_CAP;
    std::vector<double> tiles((size_t)ntiles * 64, 0.0);
    for (int I = 0; I < n8; I++)
        for (int J = 0; J <= I; J++)
            for (int r = 0; r < 8; r++)
                for (int c = 0; c < 8; c++) {
                    const int i = 8 * I + r, j = 8 * J + c;
                    double v;
                    if (i > n || j > n) v = (i == j) ? 1.0 : 0.0;
                    else if (i == n) v = (j == n) ? 1.0 : b[j];
                    else if (j == n) v = 0.0;
                    else v = A[(size_t)i * n + j];
                    tiles[(size_t)tix(I, J) * 64 + r * 8 + c] = v;
                }
    double *dA = nullptr, *dL = nullptr, *dy = nullptr; int* df = nullptr;
    const size_t spill = (size_t)(ntiles > cap ? ntiles - cap : 1) * 64;
    GF_CUDA(cudaMalloc(&dA, tiles.size() * sizeof(double)));
    GF_CUDA(cudaMalloc(&dL, spill * sizeof(double)));
    GF_CUDA(cudaMalloc(&dy, (size_t)n * sizeof(double)));
    GF_CUDA(cudaMalloc(&df, sizeof(int)));
    GF_CUDA(cudaMemcpy(dA, tiles.data(), tiles.size() * sizeof(double), cudaMemcpyHostToDevice));
    const size_t smem = sizeof(double) * (64 * (size_t)std::min(ntiles, cap) + 64 * (size_t)n8 + 192 + 2 * (size_t)((n + 8) & ~7));
    GF_CUDA(cudaFuncSetAttribute(k_stage_chol<MAXR / 2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    GF_CUDA(cudaFuncSetAttribute(k_stage_chol<MAXR, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
    if (ntiles <= cap && n8 <= (MAXR / 2) * CH_BULK) k_stage_chol<MAXR / 2, false><<<1, ST_THREADS, smem>>>(dA, dL, cap, n, dy, df);
    else k_stage_chol<MAXR, true><<<1, ST_THREADS, smem>>>(dA, dL, cap, n, dy, df);
    GF_LAUNCHED();
    int fail = 0;
    cudaError_t e = cudaMemcpy(&fail, df, sizeof(int), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && !fail) e = cudaMemcpy(x, dy, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost);
    cudaFree(dA); cudaFree(dL); cudaFree(dy); cudaFree(df);
    if (e != cudaSuccess) { snprintf(g_err, sizeof(g_err), "gf_stage_spd_solve: %s", cudaGetErrorString(e)); return GF_ERR_CUDA; }
    if (fail) return set_err(GF_ERR_INVALID_ARG, "matrix is not positive definite");
    return GF_OK;
}

// Stage-level entry points (tests): the marginalisation's eigensolvers and its Schur complement on a given dense system.
static int stage_device(int device)
{
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_err(GF_ERR_NO_DEVICE, "no CUDA device visible; libgf_b200 has no CPU fallback");
    if (device < 0 || device >= ndev) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    return GF_OK;
}

// Largest Jacobi size the stage entry points take (gf_stage_sym_eig's n, gf_stage_marginalize's m): above 2048 the kernel's
// 1024 threads each set up more than one rotation of a round, and the tests run this bound.
constexpr int STAGE_JACOBI_MAX = 2304;

extern "C" int gf_stage_sym_eig(int device, const double* A, int n, int method, double* w, double* V, int* sweeps)
{
    if (!A || !w || !V || n < 1 || (method == 0 && n > 128) || (method == 1 && n > STAGE_JACOBI_MAX) || (method != 0 && method != 1))
        return set_err(GF_ERR_INVALID_ARG, "bad argument (method 0: 1 <= n <= 128, method 1: 1 <= n <= 2304)");
    int rc = stage_device(device);
    if (rc) return rc;
    const size_t nn = (size_t)n * n;
    std::vector<double> h(nn);
    for (int i = 0; i < n; i++) for (int j = 0; j <= i; j++) h[(size_t)i * n + j] = h[(size_t)j * n + i] = A[(size_t)i * n + j];
    double* dA = nullptr;
    GF_CUDA(cudaMalloc(&dA, sizeof(double) * (3 * nn + n + 1)));           // A | V | w | sweep count
    double* dV = dA + nn; double* dw = dV + nn; int* dsw = (int*)(dw + n);
    cudaError_t e = cudaMemcpy(dA, h.data(), sizeof(double) * nn, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(dsw, 0, sizeof(int));
    if (e == cudaSuccess && method == 0) {
        e = cudaFuncSetAttribute(k_sym_eig_ql, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e == cudaSuccess) { k_sym_eig_ql<<<1, QL_T, sizeof(double) * (nn + 4 * (size_t)n + 8)>>>(dA, dV, dw, n); GF_LAUNCHED(); }
    } else if (e == cudaSuccess) {
        const int hp = ((n + 1) & ~1) / 2;
        e = cudaFuncSetAttribute(k_jacobi_eig, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e == cudaSuccess) { k_jacobi_eig<<<1, 1024, (size_t)hp * (2 * sizeof(double) + 2 * sizeof(int)) + 8>>>(dA, dV, dw, n, dsw); GF_LAUNCHED(); }
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpy(V, dV, sizeof(double) * nn, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(w, dw, sizeof(double) * n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && sweeps) e = cudaMemcpy(sweeps, dsw, sizeof(int), cudaMemcpyDeviceToHost);
    cudaFree(dA);
    if (e != cudaSuccess) { snprintf(g_err, sizeof(g_err), "gf_stage_sym_eig: %s", cudaGetErrorString(e)); return GF_ERR_CUDA; }
    return GF_OK;
}

extern "C" int gf_stage_marginalize(int device, const double* A, const double* b, int N, int c, int L, int force_generic,
                                    double* J0, double* r0, int* path)
{
    const int m = c + L, n = N - m;
    if (!A || !b || !J0 || !r0 || !path || c < 1 || c > 15 || L < 0 || m > STAGE_JACOBI_MAX || n < 1 || n > 16 * GF_BA_MAX_FRAMES + 22)
        return set_err(GF_ERR_INVALID_ARG, "bad argument (1 <= c <= 15, L >= 0, c + L <= 2304, 1 <= N - c - L <= 198)");
    for (int l = c; l < m; l++)
        for (int k = c; k < m; k++)
            if (k != l && A[(size_t)l * N + k] != 0.0) return set_err(GF_ERR_INVALID_ARG, "the landmark block is not diagonal");
    int rc = stage_device(device);
    if (rc) return rc;
    const size_t NN = (size_t)N * N, mm = (size_t)m * m, nn = (size_t)n * n, R = (size_t)c + n;
    const size_t nd = NN + N + 3 * mm + m + (size_t)n * m + 3 * nn + 3 * (size_t)n + R * R + R + 225;
    double* d = nullptr;
    GF_CUDA(cudaMalloc(&d, sizeof(double) * (nd + 2)));                       // ... | int[4] sweeps and flag
    int* dsw = (int*)(d + nd);
    MargDev q;
    memset(&q, 0, sizeof(q));
    q.N = N; q.m = m; q.n = n;
    double* t = d;
    auto take = [&](size_t k) { double* p = t; t += k; return p; };
    q.A = take(NN); q.b = take(N); q.Amm = take(mm); q.Vm = take(mm); q.wm = take(m); q.Ainv = take(mm); q.T = take((size_t)n * m);
    q.Ar = take(nn); q.Vr = take(nn); q.wr = take(n); q.br = take(n); q.J0 = take(nn); q.r0 = take(n);
    double* dQ = take(R * R); double* dqb = take(R); double* dce = take(225);
    int h_flag = 0, p = 0, hsw[2] = {0, 0};
    cudaError_t e = cudaMemcpy(q.A, A, sizeof(double) * NN, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(q.b, b, sizeof(double) * N, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(dsw, 0, sizeof(int) * 4);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_sym_eig_ql, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_jacobi_eig, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e == cudaSuccess) {
        rc = marg_schur_eig(q, c, force_generic != 0, dQ, dqb, dce, dsw, &h_flag, 0, &p);
        if (!rc) e = cudaMemcpy(J0, q.J0, sizeof(double) * nn, cudaMemcpyDeviceToHost);
        if (!rc && e == cudaSuccess) e = cudaMemcpy(r0, q.r0, sizeof(double) * n, cudaMemcpyDeviceToHost);
        if (!rc && e == cudaSuccess) e = cudaMemcpy(hsw, dsw, sizeof(int) * 2, cudaMemcpyDeviceToHost);
    }
    cudaFree(d);
    if (rc) return rc;
    if (e != cudaSuccess) { snprintf(g_err, sizeof(g_err), "gf_stage_marginalize: %s", cudaGetErrorString(e)); return GF_ERR_CUDA; }
    path[0] = p;
    path[1] = (p & GF_MARG_PATH_GENERIC) ? hsw[0] : 0;
    path[2] = (p & GF_MARG_PATH_REDUCED_JACOBI) ? hsw[1] : 0;
    return GF_OK;
}

// ------------------------------------------------------------------------------------------------
// FP64 rate probe (bench.py quotes the back end's roofline against it): dependent-free DFMA and DMMA.8x8x4 loops on every SM.
namespace gfba {
__global__ void __launch_bounds__(256) k_probe_dfma(double* out, int n)
{
    double a0 = out[0] + threadIdx.x, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
    const double b = out[1], c = out[2];
    for (int i = 0; i < n; i++) {
        a0 = fma(a0, b, c); a1 = fma(a1, b, c); a2 = fma(a2, b, c); a3 = fma(a3, b, c);
        a4 = fma(a4, b, c); a5 = fma(a5, b, c); a6 = fma(a6, b, c); a7 = fma(a7, b, c);
    }
    if (a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7 == 12345.678) out[8] = a0;
}
__global__ void __launch_bounds__(256) k_probe_dmma(double* out, int n)
{
    const double a = out[1], b = out[2];
    double c[8][2];
#pragma unroll
    for (int k = 0; k < 8; k++) c[k][0] = c[k][1] = 0.0;
    for (int i = 0; i < n; i++) {
#pragma unroll
        for (int k = 0; k < 8; k++) dmma884(c[k][0], c[k][1], a, b);
    }
    double s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s += c[k][0] + c[k][1];
    if (s == 12345.678) out[8] = s;
}
}  // namespace gfba

extern "C" int gf_probe_fp64(int device, double* dfma_gflops, double* dmma_gflops)
{
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_err(GF_ERR_NO_DEVICE, "no CUDA device visible; libgf_b200 has no CPU fallback");
    if (device < 0 || device >= ndev) return set_err(GF_ERR_INVALID_ARG, "device index out of range");
    GF_CUDA(cudaSetDevice(device));
    cudaDeviceProp pr;
    GF_CUDA(cudaGetDeviceProperties(&pr, device));
    double* d = nullptr;
    GF_CUDA(cudaMalloc(&d, 4096));
    const double h[4] = {1.0000001, 0.9999999, 1e-9, 0.0};
    GF_CUDA(cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice));
    cudaEvent_t e0, e1;
    GF_CUDA(cudaEventCreate(&e0)); GF_CUDA(cudaEventCreate(&e1));
    const int grid = pr.multiProcessorCount * 4, n = 1 << 15;
    double res[2] = {0, 0};
    for (int which = 0; which < 2; which++) {
        float best = 1e30f;
        for (int rep = 0; rep < 4; rep++) {
            GF_CUDA(cudaEventRecord(e0));
            if (which == 0) k_probe_dfma<<<grid, 256>>>(d, n); else k_probe_dmma<<<grid, 256>>>(d, n);
            GF_LAUNCHED();
            GF_CUDA(cudaEventRecord(e1));
            GF_CUDA(cudaEventSynchronize(e1));
            float ms = 0; GF_CUDA(cudaEventElapsedTime(&ms, e0, e1));
            if (rep > 0 && ms < best) best = ms;
        }
        const double fma = which == 0 ? 8.0 * n * 256.0 * grid : 8.0 * n * 256.0 * (256 / 32) * grid;
        res[which] = 2.0 * fma / (best * 1e-3) / 1e9;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d);
    if (dfma_gflops) *dfma_gflops = res[0];
    if (dmma_gflops) *dmma_gflops = res[1];
    return GF_OK;
}
