// Drives the adaptor classes from flat binary dumps written by tests/test_adaptor.py; the outputs go back as flat binaries.
//   harness fe <in> <out>   frames through FeatureTracker::trackImage
//   harness fe-eq <in> <out>  the same with EQUALIZE = 1
//   harness fe-box <in> <out> frames and their detections (int m, m x 4 int64 after each frame) through
//                             FeatureTracker::trackImagebox; after each featureFrame: cur_pts as (n, n x (id, x, y, track_cnt))
//   harness ba <in> <out>   one window through Estimator::optimization()
//   harness ba-multi <in> <out>  several estimators' windows, each round through one Estimator::optimizationMulti call
//   harness ba-seq <in> <out>    the same input through each estimator's optimization() in turn
//   harness dm <in> <out>   keyframes and pose corrections through DenseMap (PoseGraph's octree blocks); after each call the
//                           returned point_rgbd (add only), the cloud and the filtered cloud's indices
//   harness gm <in> <out>   keyframes' point_rgbd and pose corrections through GridMapper (the grid_mapping tool); after each
//                           call bel, the map.png pixels and the OccupancyGrid data
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "dense_map.h"
#include "estimator_ba.h"
#include "feature_tracker.h"
#include "grid_map.h"

int MAX_CNT = 150, MIN_DIST = 30, FLOW_BACK = 1, EQUALIZE = 0;
int USE_IMU = 1, NUM_ITERATIONS = 8, ESTIMATE_TD = 0;
double FOCAL_LENGTH = 600.0;
Eigen::Vector3d G;

static void rd(FILE *f, void *p, size_t n) { if (fread(p, 1, n, f) != n) { std::fprintf(stderr, "short read\n"); std::exit(2); } }
template <class T> static T rd1(FILE *f) { T v; rd(f, &v, sizeof(T)); return v; }

static int run_fe(const char *in, const char *out, bool with_boxes)
{
    FILE *f = fopen(in, "rb"), *o = fopen(out, "wb");
    if (!f || !o) return 2;
    const int n = rd1<int>(f), w = rd1<int>(f), h = rd1<int>(f), with_depth = rd1<int>(f);
    double p[8]; rd(f, p, sizeof(p));
    MAX_CNT = rd1<int>(f); MIN_DIST = rd1<int>(f); FLOW_BACK = rd1<int>(f);
    FeatureTracker tracker;
    tracker.setPinhole(p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7], with_depth);
    std::vector<unsigned char> gray((size_t)w * h); std::vector<unsigned short> depth((size_t)w * h);
    for (int k = 0; k < n; k++) {
        const double t = rd1<double>(f);
        rd(f, gray.data(), gray.size());
        if (with_depth) rd(f, depth.data(), depth.size() * 2);
        cv::Mat img(h, w, CV_8UC1, gray.data()), dimg;
        if (with_depth) dimg = cv::Mat(h, w, CV_16UC1, depth.data());
        std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> frame;
        if (with_boxes) {
            auto msg = std::make_shared<darknet_ros_msgs::BoundingBoxes>();
            msg->bounding_boxes.resize(rd1<int>(f));
            for (auto &b : msg->bounding_boxes) { b.xmin = rd1<int64_t>(f); b.ymin = rd1<int64_t>(f); b.xmax = rd1<int64_t>(f); b.ymax = rd1<int64_t>(f); }
            frame = tracker.trackImagebox(t, msg, img, dimg);
        } else {
            frame = tracker.trackImage(t, img, dimg);
        }
        const int m = (int)frame.size();
        fwrite(&m, 4, 1, o);
        for (auto &kv : frame) {                                   // std::map: ascending feature id, as featureBuf consumers see it
            fwrite(&kv.first, 4, 1, o);
            fwrite(kv.second[0].second.data(), 8, 8, o);
        }
        if (with_boxes) {
            const int np = (int)tracker.cur_pts.size();
            fwrite(&np, 4, 1, o);
            for (int i = 0; i < np; i++) {
                fwrite(&tracker.ids[i], 4, 1, o); fwrite(&tracker.cur_pts[i].x, 4, 1, o); fwrite(&tracker.cur_pts[i].y, 4, 1, o);
                fwrite(&tracker.track_cnt[i], 4, 1, o);
            }
        }
    }
    fclose(f); fclose(o);
    return 0;
}

// one window of the input (the Estimator members optimization() reads) into est
static void read_window(FILE *f, Estimator &est, int n_frames)
{
    est.marginalization_flag = rd1<int>(f) ? Estimator::MARGIN_SECOND_NEW : Estimator::MARGIN_OLD;
    const int n_feat = rd1<int>(f);
    rd(f, est.para_Pose, sizeof(double) * 7 * n_frames);
    rd(f, est.para_SpeedBias, sizeof(double) * 9 * n_frames);
    rd(f, est.para_Ex_Pose[0], 56);
    for (int k = 0; k < n_frames; k++) for (int c = 0; c < 3; c++) est.Vs[k](c) = est.para_SpeedBias[k][c];
    for (int j = 1; j < n_frames; j++) {
        delete est.pre_integrations[j];
        IntegrationBase *b = est.pre_integrations[j] = new IntegrationBase;
        b->sum_dt = rd1<double>(f);
        rd(f, b->delta_p.data(), 24); rd(f, b->delta_q.coeffs().data(), 32); rd(f, b->delta_v.data(), 24);
        rd(f, b->linearized_ba.data(), 24); rd(f, b->linearized_bg.data(), 24);
        double m[225];
        rd(f, m, sizeof(m)); for (int i = 0; i < 15; i++) for (int c = 0; c < 15; c++) b->jacobian(i, c) = m[i * 15 + c];
        rd(f, m, sizeof(m)); for (int i = 0; i < 15; i++) for (int c = 0; c < 15; c++) b->covariance(i, c) = m[i * 15 + c];
    }
    est.f_manager.feature.clear();
    for (int k = 0; k < n_feat; k++) {
        FeaturePerId it;
        it.feature_id = k; it.start_frame = rd1<int>(f);
        const int n_obs = rd1<int>(f);
        it.estimate_flag = rd1<int>(f);
        est.para_Feature[k][0] = rd1<double>(f);
        for (int q = 0; q < n_obs; q++) {
            FeaturePerFrame fr;
            rd(f, fr.point.data(), 24); rd(f, fr.velocity.data(), 16); fr.cur_td = rd1<double>(f);
            it.feature_per_frame.push_back(fr);
        }
        est.f_manager.feature.push_back(it);
    }
}

// the solved window: blocks, then iterations, final cost, prior dimension, termination; with_prior: the next prior's r0 and J0
static void write_window(FILE *o, const Estimator &est, int n_frames, bool with_prior)
{
    fwrite(est.para_Pose, sizeof(double) * 7, n_frames, o);
    fwrite(est.para_SpeedBias, sizeof(double) * 9, n_frames, o);
    fwrite(&est.para_Feature[0][0], sizeof(double), est.f_manager.feature.size(), o);
    const double tail[4] = {(double)est.last_summary.iterations, est.last_summary.final_cost, (double)est.prior_dim(), (double)est.last_summary.termination};
    fwrite(tail, 8, 4, o);
    if (with_prior && est.prior_dim() > 0) {
        const int n = est.prior_dim();
        fwrite(est.prior().linearized_residuals, sizeof(double), n, o);
        fwrite(est.prior().linearized_jacobians, sizeof(double), (size_t)n * n, o);
    }
}

static int run_ba(const char *in, const char *out)
{
    FILE *f = fopen(in, "rb"), *o = fopen(out, "wb");
    if (!f || !o) return 2;
    static Estimator est;
    const int n_frames = rd1<int>(f), n_windows = rd1<int>(f);
    est.frame_count = n_frames - 1;
    NUM_ITERATIONS = rd1<int>(f);
    rd(f, G.data(), 24);
    for (int w = 0; w < n_windows; w++) {
        read_window(f, est, n_frames);
        est.optimization();
        write_window(o, est, n_frames, false);
    }
    fclose(f); fclose(o);
    return 0;
}

// n_est estimators, each with its own chain of windows: int n_est, then the `ba` input with n_windows = n_est * rounds windows in
// round-major order (window r * n_est + e belongs to estimator e).  batched: each round is one Estimator::optimizationMulti call;
// else every estimator's optimization() in turn.  Output: the windows in input order, each followed by the prior it left.
static int run_ba_multi(const char *in, const char *out, bool batched)
{
    FILE *f = fopen(in, "rb"), *o = fopen(out, "wb");
    if (!f || !o) return 2;
    const int n_est = rd1<int>(f), n_frames = rd1<int>(f), n_windows = rd1<int>(f);
    NUM_ITERATIONS = rd1<int>(f);
    rd(f, G.data(), 24);
    std::vector<std::unique_ptr<Estimator>> est;
    std::vector<Estimator *> ptr;
    for (int e = 0; e < n_est; e++) { est.emplace_back(new Estimator); est.back()->frame_count = n_frames - 1; ptr.push_back(est.back().get()); }
    for (int r = 0; r < n_windows / n_est; r++) {
        for (int e = 0; e < n_est; e++) read_window(f, *est[e], n_frames);
        if (batched) Estimator::optimizationMulti(ptr.data(), n_est);
        else for (int e = 0; e < n_est; e++) est[e]->optimization();
        for (int e = 0; e < n_est; e++) write_window(o, *est[e], n_frames, true);
    }
    fclose(f); fclose(o);
    return 0;
}

// Input: w, h, pinhole[8], depth_dist, depth_boundary, qic[9] (row-major), tic[3], max_points, max_keyframes, n_ops; each op is
// int 0 + R[9] (row-major) + P[3] + rgb (h x w x 3) + depth (h x w u16), or int 1 + n + n x (R[9], P[3]).
static int run_dm(const char *in, const char *out)
{
    FILE *f = fopen(in, "rb"), *o = fopen(out, "wb");
    if (!f || !o) return 2;
    const int w = rd1<int>(f), h = rd1<int>(f);
    double p[8], q[9];
    rd(f, p, sizeof(p));
    const int dd = rd1<int>(f), db = rd1<int>(f);
    rd(f, q, sizeof(q));
    Eigen::Matrix3d qic; Eigen::Vector3d tic;
    for (int i = 0; i < 9; i++) qic(i / 3, i % 3) = q[i];
    rd(f, tic.data(), 24);
    const int max_points = rd1<int>(f), max_keyframes = rd1<int>(f), n_ops = rd1<int>(f);
    DenseMap map(w, h, p, dd, db, qic, tic, max_points, max_keyframes);
    auto pose = [&](Eigen::Matrix3d &R, Eigen::Vector3d &P) {
        double r[9]; rd(f, r, sizeof(r));
        for (int i = 0; i < 9; i++) R(i / 3, i % 3) = r[i];
        rd(f, P.data(), 24);
    };
    std::vector<unsigned char> rgb((size_t)w * h * 3);
    std::vector<unsigned short> depth((size_t)w * h);
    for (int op = 0; op < n_ops; op++) {
        if (rd1<int>(f) == 0) {
            Eigen::Matrix3d R; Eigen::Vector3d P;
            pose(R, P);
            rd(f, rgb.data(), rgb.size()); rd(f, depth.data(), depth.size() * 2);
            const auto pts = map.addKeyFrame(R, P, cv::Mat(h, w, CV_8UC3, rgb.data()), cv::Mat(h, w, CV_16UC1, depth.data()));
            const int m = (int)pts.size();
            fwrite(&m, 4, 1, o);
            for (auto &v : pts) fwrite(v.data(), 4, 6, o);
        } else {
            const int n = rd1<int>(f);
            std::vector<Eigen::Matrix3d> Rs(n); std::vector<Eigen::Vector3d> Ps(n);
            for (int k = 0; k < n; k++) pose(Rs[k], Ps[k]);
            map.updatePath(Rs, Ps);
        }
        std::vector<float> xyz; std::vector<unsigned char> col; std::vector<int32_t> idx;
        map.cloud(xyz, col);
        const int n = (int)(xyz.size() / 3);
        fwrite(&n, 4, 1, o); fwrite(xyz.data(), 4, xyz.size(), o); fwrite(col.data(), 1, col.size(), o);
        map.filtered(xyz, col, idx);
        const int nf = (int)idx.size();
        fwrite(&nf, 4, 1, o); fwrite(idx.data(), 4, idx.size(), o);
    }
    fclose(f); fclose(o);
    return 0;
}

// Input: size_x, size_y, init_x, init_y, cell_size, p_occ, p_free, p_prior, qic[9] (row-major), tic[3], max_points,
// max_keyframes, max_records, n_ops; each op is int 0 + R[9] + P[3] + n + n x 6 floats (point_rgbd), or int 1 + n + n x (R[9], P[3]).
static int run_gm(const char *in, const char *out)
{
    FILE *f = fopen(in, "rb"), *o = fopen(out, "wb");
    if (!f || !o) return 2;
    int sz[4];
    rd(f, sz, sizeof(sz));
    double c[4], q[9];
    rd(f, c, sizeof(c));
    rd(f, q, sizeof(q));
    Eigen::Matrix3d qic; Eigen::Vector3d tic;
    for (int i = 0; i < 9; i++) qic(i / 3, i % 3) = q[i];
    rd(f, tic.data(), 24);
    const int max_points = rd1<int>(f), max_keyframes = rd1<int>(f), max_records = rd1<int>(f), n_ops = rd1<int>(f);
    GridMapper map(qic, tic, sz[0], sz[1], sz[2], sz[3], c[0], c[1], c[2], c[3], max_points, max_keyframes, max_records);
    auto pose = [&](Eigen::Matrix3d &R, Eigen::Vector3d &P) {
        double r[9]; rd(f, r, sizeof(r));
        for (int i = 0; i < 9; i++) R(i / 3, i % 3) = r[i];
        rd(f, P.data(), 24);
    };
    for (int op = 0; op < n_ops; op++) {
        if (rd1<int>(f) == 0) {
            Eigen::Matrix3d R; Eigen::Vector3d P;
            pose(R, P);
            std::vector<Eigen::Matrix<float, 6, 1>> pts(rd1<int>(f));
            for (auto &v : pts) rd(f, v.data(), 24);
            map.addKeyFrame(R, P, pts);
        } else {
            const int n = rd1<int>(f);
            std::vector<Eigen::Matrix3d> Rs(n); std::vector<Eigen::Vector3d> Ps(n);
            for (int k = 0; k < n; k++) pose(Rs[k], Ps[k]);
            map.updatePath(Rs, Ps);
        }
        const auto bel = map.bel();
        const auto img = map.image();
        const auto occ = map.occupancy();
        fwrite(bel.data(), 8, bel.size(), o); fwrite(img.data(), 1, img.size(), o); fwrite(occ.data(), 1, occ.size(), o);
    }
    fclose(f); fclose(o);
    return 0;
}

int main(int argc, char **argv)
{
    if (argc != 4) { std::fprintf(stderr, "usage: harness fe|fe-eq|fe-box|ba|ba-multi|ba-seq|dm|gm <in> <out>\n"); return 2; }
    if (!std::strcmp(argv[1], "fe-eq")) EQUALIZE = 1;
    if (!std::strcmp(argv[1], "dm")) return run_dm(argv[2], argv[3]);
    if (!std::strcmp(argv[1], "gm")) return run_gm(argv[2], argv[3]);
    if (!std::strcmp(argv[1], "ba-multi") || !std::strcmp(argv[1], "ba-seq")) return run_ba_multi(argv[2], argv[3], argv[1][3] == 'm');
    return argv[1][0] == 'f' ? run_fe(argv[2], argv[3], !std::strcmp(argv[1], "fe-box")) : run_ba(argv[2], argv[3]);
}
