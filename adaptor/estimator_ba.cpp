// Estimator::optimization() (vins_estimator/src/estimator/estimator.cpp:2884-3631) on libgf_b200.so: vector2double's arrays
// are handed to gf_ba_solve (gf_ba_solve_multi for several estimators) as they are, the AddResidualBlock loops become descriptor rows, and the MARGIN_OLD /
// MARGIN_SECOND_NEW branches become one call each (one gf_ba_marginalize_multi call for several estimators).  Wheel, plane and GNSS blocks follow the same pattern (INTEGRATION.md);
// this file carries the camera + IMU case the reference's default configs run.
#include "estimator_ba.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace {
[[noreturn]] void gf_fatal(const char *what)
{
    std::fprintf(stderr, "gf_b200: %s: %s\n", what, gf_last_error());
    std::abort();                                  // ROS_BREAK() in the reference
}
template <int R, int C> void to_row_major(const Eigen::Matrix<double, R, C> &m, double *out)
{
    for (int i = 0; i < R; i++) for (int j = 0; j < C; j++) out[i * C + j] = m(i, j);   // Eigen stores column-major
}
void copy3(const Eigen::Vector3d &v, double *o) { o[0] = v(0); o[1] = v(1); o[2] = v(2); }
}  // namespace

Estimator::Estimator()
{
    std::memset(para_Pose, 0, sizeof(para_Pose)); std::memset(para_SpeedBias, 0, sizeof(para_SpeedBias));
    std::memset(para_Feature, 0, sizeof(para_Feature)); std::memset(para_Ex_Pose, 0, sizeof(para_Ex_Pose));
    para_Td[0][0] = 0;
}
Estimator::~Estimator()
{
    if (gf_ba_) gf_ba_destroy(gf_ba_);
}

// The ceres::Problem of estimator.cpp:2895-3300 as a gf_ba_problem; rows owns the factor tables P points into
void Estimator::buildProblem(BaRows &rows)
{
    if (!gf_ba_ && gf_ba_create(&gf_ba_, device)) gf_fatal("gf_ba_create");
    gf_ba_problem &P = rows.P;
    P = gf_ba_problem{};
    P.n_frames = frame_count + 1;
    P.max_num_iterations = NUM_ITERATIONS;                                   // estimator.cpp:3308
    P.para_pose = &para_Pose[0][0]; P.para_speed_bias = &para_SpeedBias[0][0];
    P.para_ex_pose = para_Ex_Pose[0]; P.para_feature = &para_Feature[0][0]; P.para_td = para_Td[0];
    P.pose0_const = !USE_IMU;                                                // :2936-2937
    P.frames_const = systemstationary && stationary_detect;                  // :2938-2947
    P.ex_pose_const = !openExEstimation;                                     // :2955-2969 (the caller updates openExEstimation)
    double v0 = 0; for (int k = 0; k < 3; k++) v0 += Vs[0](k) * Vs[0](k);
    P.td_const = !ESTIMATE_TD || v0 < 0.2 * 0.2;                             // :3076-3080
    P.ex_wheel_const = P.ix_wheel_const = P.td_wheel_const = P.plane_const = 1;
    copy3(G, P.gravity);
    P.visual_sqrt_info = FOCAL_LENGTH / 1.5;                                 // :193

    std::vector<gf_ba_imu_factor> &imu = rows.imu;
    imu.clear();
    if (USE_IMU)
        for (int i = 0; i < frame_count; i++) {                              // :3104-3113
            const int j = i + 1;
            const IntegrationBase *pre = pre_integrations[j];
            if (pre->sum_dt > 10.0) continue;
            gf_ba_imu_factor f{};
            f.i = i; f.j = j; f.sum_dt = pre->sum_dt;
            copy3(pre->delta_p, f.delta_p); copy3(pre->delta_v, f.delta_v);
            for (int k = 0; k < 4; k++) f.delta_q[k] = pre->delta_q.coeffs()(k);
            copy3(pre->linearized_ba, f.linearized_ba); copy3(pre->linearized_bg, f.linearized_bg);
            to_row_major(pre->jacobian, f.jacobian); to_row_major(pre->covariance, f.covariance);
            imu.push_back(f);
        }
    std::vector<gf_ba_visual_factor> &vis = rows.vis;
    std::vector<uint8_t> &feature_const = rows.feature_const;
    vis.clear(); feature_const.clear();
    int feature_index = -1;
    for (auto &it_per_id : f_manager.feature) {                              // :3268-3296
        it_per_id.used_num = (int)it_per_id.feature_per_frame.size();
        if (it_per_id.used_num < 4) continue;
        ++feature_index;
        const int imu_i = it_per_id.start_frame;
        int imu_j = imu_i - 1;
        const FeaturePerFrame &fi = it_per_id.feature_per_frame[0];
        for (auto &fj : it_per_id.feature_per_frame) {
            imu_j++;
            if (imu_i == imu_j) continue;
            gf_ba_visual_factor f{};
            f.imu_i = imu_i; f.imu_j = imu_j; f.feature = feature_index;
            copy3(fi.point, f.pts_i); copy3(fj.point, f.pts_j);
            f.vel_i[0] = fi.velocity(0); f.vel_i[1] = fi.velocity(1); f.vel_j[0] = fj.velocity(0); f.vel_j[1] = fj.velocity(1);
            f.td_i = fi.cur_td; f.td_j = fj.cur_td;
            vis.push_back(f);
        }
        feature_const.push_back(it_per_id.estimate_flag == 1);               // :3291-3292
    }
    P.n_features = feature_index + 1;
    P.visual = vis.data(); P.n_visual = (int)vis.size();
    P.imu = imu.data(); P.n_imu = (int)imu.size();
    P.feature_const = feature_const.data();
    P.prior = have_prior_ ? &prior_ : nullptr;                               // :2895-2903
}

void Estimator::optimization()
{
    BaRows rows;
    buildProblem(rows);
    if (gf_ba_solve(gf_ba_, &rows.P, &last_summary)) gf_fatal("gf_ba_solve");     // ceres::Solve, :3318
    marginalize(rows.P);
}

// Several estimators (one per robot / camera rig served by this GPU) at the same point of their processImage: every window is
// built as optimization() builds it, all are solved by one gf_ba_solve_multi call from this thread, then all are marginalised
// by one gf_ba_marginalize_multi call, each as its own marginalization_flag says.  The same blocks and priors as calling
// optimization() on each in turn.
void Estimator::optimizationMulti(Estimator *const *est, int n)
{
    std::vector<BaRows> rows(n);
    std::vector<gf_ba *> handles(n);
    std::vector<gf_ba_problem> P(n);
    std::vector<gf_ba_summary> S(n);
    for (int k = 0; k < n; k++) {
        est[k]->buildProblem(rows[k]);
        P[k] = rows[k].P; handles[k] = est[k]->gf_ba_;
    }
    if (gf_ba_solve_multi(handles.data(), n, P.data(), S.data(), nullptr)) gf_fatal("gf_ba_solve_multi");
    std::vector<int32_t> modes(n), kept(n);
    std::vector<gf_ba_prior> next(n);
    std::vector<std::vector<double>> x0(n), J(n), r(n);
    std::vector<double *> px0(n), pJ(n), pr(n);
    for (int k = 0; k < n; k++) {
        est[k]->last_summary = S[k];
        modes[k] = est[k]->marginalization_flag == MARGIN_OLD ? GF_BA_MARGIN_OLD : GF_BA_MARGIN_SECOND_NEW;
        const size_t cap = 16 * (size_t)P[k].n_frames + 24;
        x0[k].resize(cap); J[k].resize(cap * cap); r[k].resize(cap);
        px0[k] = x0[k].data(); pJ[k] = J[k].data(); pr[k] = r[k].data();
    }
    if (gf_ba_marginalize_multi(handles.data(), n, P.data(), modes.data(), next.data(), px0.data(), pJ.data(), pr.data(), kept.data(), nullptr))
        gf_fatal("gf_ba_marginalize_multi");
    for (int k = 0; k < n; k++) est[k]->adoptPrior(kept[k], next[k], x0[k], J[k], r[k]);
}

// MARGIN_OLD / MARGIN_SECOND_NEW at the end of optimization(): the prior of the next window
void Estimator::marginalize(const gf_ba_problem &P)
{
    const size_t cap = 16 * (size_t)P.n_frames + 24;
    std::vector<double> x0(cap), J(cap * cap), r(cap);
    gf_ba_prior next{};
    int n;
    if (marginalization_flag == MARGIN_OLD)                                  // :3334-3535
        n = gf_ba_marginalize_old(gf_ba_, &P, &next, x0.data(), J.data(), r.data(), nullptr);
    else                                                                     // :3536-3631
        n = gf_ba_marginalize_second_new(gf_ba_, &P, &next, x0.data(), J.data(), r.data(), nullptr);
    if (n < 0) gf_fatal("marginalisation");
    adoptPrior(n, next, x0, J, r);
}

// The marginalisation's result (n = its return value) becomes the prior of the next window; x0, J, r are the buffers `next`
// points into and are taken over
void Estimator::adoptPrior(int n, const gf_ba_prior &next, std::vector<double> &x0, std::vector<double> &J, std::vector<double> &r)
{
    if (n == 0) return;                            // MARGIN_SECOND_NEW with a prior that does not hold the pose -> keep it
    prior_x0_.swap(x0); prior_J_.swap(J); prior_r_.swap(r);
    prior_ = next;
    prior_.x0 = prior_x0_.data(); prior_.linearized_jacobians = prior_J_.data(); prior_.linearized_residuals = prior_r_.data();
    have_prior_ = true;
}
