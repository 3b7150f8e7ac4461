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
//   harness fm <in> <out>   a call script through FeatureManager (the landmark table on the GPU); after each call its return
//                           values and the whole table (FeatureManager::features)
//   harness fm-bench <in> <out>  host time per frame of the FeatureManager stage from C++ alone: the calls one processImage makes
//                           around the solve, once over a std::list on the host with the stateless gf_fm_* calls and once over
//                           gf_fm_window, alternating; <out> is one JSON object (tools/bench_fm_window.py reads it)
//   harness fm-group-bench <in> <out>  the same stage for K windows: through gf_fm_window_group, K windows in sequence, K threads
#include <algorithm>
#include <array>
#include <chrono>
#include <list>
#include <unordered_map>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <thread>
#include <vector>

#include "dense_map.h"
#include "estimator_ba.h"
#include "feature_manager.h"
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

// ops: 0 add (fc, td, n, n x (id, v[8])) -> margin_old, 3 counters, parallax; 1 triangulate (fc, poses); 2 fillProblem -> rows, para, const;
// 3 setDepth (n, x); 4 removeFailures; 5 removeOutlier (n, ids); 6 removeBackShiftDepth (R, P, R, P); 7 removeBack; 8 removeFront (fc);
// 9 outliersRejection (poses) -> ids; 10 movingConsistencyCheckW (poses) -> ids; 11 predictPtsInNextFrame (fc, poses) -> (id, xyz);
// poses: Ps [11][3], Rs [11][9] row-major, tic, ric
static int run_fm(const char *in, const char *out)
{
    FILE *f = fopen(in, "rb"), *o = fopen(out, "wb");
    if (!f || !o) return 2;
    const double min_parallax = rd1<double>(f), depth_threshold = rd1<double>(f), init_depth = rd1<double>(f);
    const int cap = rd1<int>(f), n_ops = rd1<int>(f);
    gf_device::FeatureManager fm(min_parallax, depth_threshold, init_depth, cap);
    Eigen::Vector3d Ps[11], tic; Eigen::Matrix3d Rs[11], ric;
    auto mat = [&](Eigen::Matrix3d &M) { double r[9]; rd(f, r, sizeof(r)); for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) M(i, j) = r[3 * i + j]; };
    auto poses = [&]() {
        for (auto &P : Ps) rd(f, P.data(), 24);
        for (auto &R : Rs) mat(R);
        rd(f, tic.data(), 24); mat(ric);
    };
    auto put_ids = [&](const std::set<int> &s) { const int n = (int)s.size(); fwrite(&n, 4, 1, o); for (int id : s) fwrite(&id, 4, 1, o); };
    for (int k = 0; k < n_ops; k++) {
        const int op = rd1<int>(f);
        if (op == 0) {
            const int fc = rd1<int>(f); const double td = rd1<double>(f); const int n = rd1<int>(f);
            std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> image;
            for (int i = 0; i < n; i++) { const int id = rd1<int>(f); Eigen::Matrix<double, 8, 1> v; rd(f, v.data(), 64); image[id].emplace_back(0, v); }
            const int margin = fm.addFeatureCheckParallax(fc, image, td);
            const int c[4] = {margin, fm.last_track_num, fm.new_feature_num, fm.long_track_num};
            fwrite(c, 4, 4, o); fwrite(&fm.last_average_parallax, 8, 1, o);
        } else if (op == 1) { const int fc = rd1<int>(f); poses(); fm.triangulate(fc, Ps, Rs, tic, ric); }
        else if (op == 2) {
            std::vector<gf_ba_visual_factor> rows; std::vector<double> para; std::vector<uint8_t> cst;
            fm.fillProblem(rows, para, cst);
            const int n[2] = {(int)rows.size(), (int)para.size()};
            fwrite(n, 4, 2, o); fwrite(rows.data(), sizeof(gf_ba_visual_factor), rows.size(), o); fwrite(para.data(), 8, para.size(), o); fwrite(cst.data(), 1, cst.size(), o);
        } else if (op == 3) { std::vector<double> x(rd1<int>(f)); rd(f, x.data(), 8 * x.size()); fm.setDepth(x); }
        else if (op == 4) fm.removeFailures();
        else if (op == 5) { std::set<int> s; for (int n = rd1<int>(f); n > 0; n--) s.insert(rd1<int>(f)); fm.removeOutlier(s); }
        else if (op == 6) { Eigen::Matrix3d R0, R1; Eigen::Vector3d P0, P1; mat(R0); rd(f, P0.data(), 24); mat(R1); rd(f, P1.data(), 24); fm.removeBackShiftDepth(R0, P0, R1, P1); }
        else if (op == 7) fm.removeBack();
        else if (op == 8) fm.removeFront(rd1<int>(f));
        else if (op == 9 || op == 10) {
            poses();
            std::set<int> s;
            if (op == 9) fm.outliersRejection(s, Ps, Rs, tic, ric); else fm.movingConsistencyCheckW(s, Ps, Rs, tic, ric);
            put_ids(s);
        } else if (op == 11) {
            const int fc = rd1<int>(f); poses();
            auto pred = fm.predictPtsInNextFrame(fc, Ps, Rs, tic, ric);
            const int n = (int)pred.size(); fwrite(&n, 4, 1, o);
            for (auto &kv : pred) { fwrite(&kv.first, 4, 1, o); fwrite(kv.second.data(), 8, 3, o); }
        } else return 2;
        const auto tab = fm.features();
        const int n = (int)tab.size(); fwrite(&n, 4, 1, o);
        for (auto &it : tab) {
            const int h[5] = {it.feature_id, it.start_frame, (int)it.feature_per_frame.size(), it.estimate_flag, it.solve_flag};
            fwrite(h, 4, 5, o); fwrite(&it.estimated_depth, 8, 1, o);
            for (auto &r : it.feature_per_frame) fwrite(r.data(), 8, 9, o);
        }
    }
    fclose(f); fclose(o);
    return 0;
}

// ---- fm-bench: the FeatureManager stage in C++, host lists + stateless calls against the resident table ----
namespace fmb {
static void ok(int rc, const char *what) { if (rc != GF_OK) { std::fprintf(stderr, "%s: %s\n", what, gf_last_error()); std::exit(3); } }
struct Obs { int id; double v[8]; };
struct Poses { double P[33], R[99], tic[3], ric[9]; };
struct Lm { int id, start; double est = -1; int eflag = 0, sflag = 0; std::vector<std::array<double, 9>> obs; int end() const { return start + (int)obs.size() - 1; } };
constexpr int W = 10;
constexpr double FOCAL = 600.0, INIT_DEPTH = 5.0;

// FeatureManager as the reference keeps it: a std::list on the host; the per-landmark loops are the stateless library calls
struct HostFM {
    std::list<Lm> feature;
    double min_parallax, depth_threshold;
    std::vector<int32_t> start, nobs, off, flag, cnt; std::vector<double> pts, dep, est, e2, e3;
    void flatten(const std::vector<Lm *> &f, bool with_depth)
    {
        const size_t n = f.size();
        start.resize(n); nobs.resize(n); off.resize(n); est.resize(n); flag.resize(n); pts.clear(); dep.clear();
        int o = 0;
        for (size_t i = 0; i < n; i++) {
            start[i] = f[i]->start; nobs[i] = (int)f[i]->obs.size(); off[i] = o; est[i] = f[i]->est; flag[i] = f[i]->eflag; o += nobs[i];
            for (auto &r : f[i]->obs) { pts.insert(pts.end(), r.begin(), r.begin() + 3); if (with_depth) dep.push_back(r[7]); }
        }
    }
    bool add(int fc, const std::vector<Obs> &image, double td)
    {
        std::unordered_map<int, Lm *> index;
        index.reserve(feature.size() * 2);
        for (auto &it : feature) index[it.id] = &it;
        int last = 0, fresh = 0, lng = 0;
        for (auto &o : image) {
            std::array<double, 9> row;
            std::copy(o.v, o.v + 8, row.begin()); row[8] = td;
            auto f = index.find(o.id);
            if (f == index.end()) { feature.emplace_back(); Lm &l = feature.back(); l.id = o.id; l.start = fc; l.obs.push_back(row); fresh++; }
            else { f->second->obs.push_back(row); last++; lng += f->second->obs.size() >= 4; }
        }
        if (fc < 2 || last < 20 || lng < 40 || fresh > 0.5 * last) return true;
        std::vector<double> pi, pj;
        for (auto &it : feature)
            if (it.start <= fc - 2 && it.end() >= fc - 1) {
                auto &a = it.obs[fc - 2 - it.start]; auto &b = it.obs[fc - 1 - it.start];
                pi.insert(pi.end(), a.begin(), a.begin() + 3); pj.insert(pj.end(), b.begin(), b.begin() + 3);
            }
        if (pi.empty()) return true;
        double sum = 0;
        ok(gf_fm_parallax(0, (int)pi.size() / 3, pi.data(), pj.data(), &sum), "gf_fm_parallax");
        return sum / (pi.size() / 3) >= min_parallax;
    }
    void triangulate(const Poses &p)
    {
        std::vector<Lm *> f;
        for (auto &it : feature) f.push_back(&it);
        if (f.empty()) return;
        flatten(f, true);
        ok(gf_fm_triangulate(0, (int)f.size(), start.data(), nobs.data(), off.data(), (int)dep.size(), pts.data(), dep.data(), est.data(), flag.data(), 11, p.P, p.R,
                             p.tic, p.ric, depth_threshold, INIT_DEPTH), "gf_fm_triangulate");
        for (size_t i = 0; i < f.size(); i++) { f[i]->est = est[i]; f[i]->eflag = flag[i]; }
    }
    void fill(std::vector<gf_ba_visual_factor> &rows, std::vector<double> &para, std::vector<uint8_t> &cst)
    {
        rows.clear(); para.clear(); cst.clear();
        for (auto &it : feature) {
            if (it.obs.size() < 4) continue;
            const int k = (int)para.size();
            para.push_back(1.0 / it.est); cst.push_back(it.eflag == 1);
            for (size_t a = 1; a < it.obs.size(); a++) {
                gf_ba_visual_factor v{};
                v.imu_i = it.start; v.imu_j = it.start + (int)a; v.feature = k;
                for (int c = 0; c < 3; c++) { v.pts_i[c] = it.obs[0][c]; v.pts_j[c] = it.obs[a][c]; }
                for (int c = 0; c < 2; c++) { v.vel_i[c] = it.obs[0][5 + c]; v.vel_j[c] = it.obs[a][5 + c]; }
                v.td_i = it.obs[0][8]; v.td_j = it.obs[a][8];
                rows.push_back(v);
            }
        }
    }
    void setDepth(const std::vector<double> &x)
    {
        size_t k = 0;
        for (auto &it : feature) if (it.obs.size() >= 4) { it.est = 1.0 / x[k++]; it.sflag = it.est < 0 ? 2 : 1; }
    }
    std::vector<int> moving(const Poses &p)
    {
        std::vector<Lm *> f;
        for (auto &it : feature) if (it.obs.size() >= 2 && it.start < W - 2 && !(it.est < 0)) f.push_back(&it);
        std::vector<int> out;
        if (f.empty()) return out;
        flatten(f, false);
        e2.resize(f.size()); e3.resize(f.size()); cnt.resize(f.size());
        ok(gf_fm_reprojection_errors(0, (int)f.size(), start.data(), nobs.data(), off.data(), (int)pts.size() / 3, pts.data(), est.data(), 11, p.P, p.R, p.tic, p.ric,
                                     e2.data(), e3.data(), cnt.data()), "gf_fm_reprojection_errors");
        for (size_t i = 0; i < f.size(); i++) if (cnt[i] > 0 && (FOCAL * e2[i] / cnt[i] > 10 || e3[i] / cnt[i] > 2.0)) out.push_back(f[i]->id);
        return out;
    }
    void removeIds(const std::vector<int> &ids) { feature.remove_if([&](const Lm &l) { return std::find(ids.begin(), ids.end(), l.id) != ids.end(); }); }
    int predict(int fc, const Poses &p, std::vector<double> &xyz)
    {
        std::vector<int32_t> first; std::vector<double> uv, d;
        for (auto &it : feature) if (it.est > 0 && it.obs.size() >= 2 && it.end() == fc) { first.push_back(it.start); uv.insert(uv.end(), it.obs[0].begin(), it.obs[0].begin() + 3); d.push_back(it.est); }
        xyz.resize(3 * first.size());
        if (!first.empty()) ok(gf_fm_predict_next(0, (int)first.size(), first.data(), uv.data(), d.data(), 11, fc, p.P, p.R, p.tic, p.ric, xyz.data()), "gf_fm_predict_next");
        return (int)first.size();
    }
    void removeBackShiftDepth(const Poses &p)
    {
        std::vector<Lm *> moved; std::vector<double> uv, d;
        for (auto it = feature.begin(); it != feature.end();) {
            if (it->start != 0) { it->start--; ++it; continue; }
            const auto first = it->obs.front();
            it->obs.erase(it->obs.begin());
            if (it->obs.size() < 2) { it = feature.erase(it); continue; }
            moved.push_back(&*it); uv.insert(uv.end(), first.begin(), first.begin() + 3); d.push_back(it->est); ++it;
        }
        if (moved.empty()) return;
        ok(gf_fm_back_shift_depth(0, (int)moved.size(), uv.data(), d.data(), p.R, p.P, p.R + 9, p.P + 3, INIT_DEPTH), "gf_fm_back_shift_depth");
        for (size_t i = 0; i < moved.size(); i++) moved[i]->est = d[i];
    }
    void removeFront(int fc)
    {
        for (auto it = feature.begin(); it != feature.end();) {
            if (it->start == fc) { it->start--; ++it; continue; }
            if (it->end() < fc - 1) { ++it; continue; }
            it->obs.erase(it->obs.begin() + (W - 1 - it->start));
            if (it->obs.empty()) it = feature.erase(it); else ++it;
        }
    }
    void removeFailures() { feature.remove_if([](const Lm &l) { return l.sflag == 2; }); }
};

struct Pass { double stage_us, fill_us; long factors; };
static double median(std::vector<double> v) { std::sort(v.begin(), v.end()); return v.empty() ? 0 : v[v.size() / 2]; }
using clk = std::chrono::steady_clock;
static double us(clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count(); }

// one pass of the stream; `win` null: the host list.  The same calls in the same order on both arms; the solve is left out
// (setDepth gets the depth vector back), and at most three of the ids the consistency check flags are removed per frame.
static Pass pass(const std::vector<std::vector<Obs>> &frames, const Poses &p, double min_parallax, double depth_threshold, gf_fm_window *win)
{
    HostFM h; h.min_parallax = min_parallax; h.depth_threshold = depth_threshold;
    if (win) ok(gf_fm_window_clear(win), "clear");
    std::vector<double> t_stage, t_fill, para(8192), xyz(3 * 8192);
    std::vector<gf_ba_visual_factor> rows; std::vector<uint8_t> cst(8192); std::vector<gf_obs> obs; std::vector<int32_t> ids(8192);
    if (win) rows.resize(8192 * 10);
    long factors = 0;
    for (size_t k = 0; k < frames.size(); k++) {
        const int fc = (int)std::min<size_t>(k, W);
        const auto t0 = clk::now();
        int margin = 0;
        if (win) {
            obs.resize(frames[k].size());
            for (size_t i = 0; i < obs.size(); i++) { obs[i].id = frames[k][i].id; obs[i].track_cnt = 0; std::copy(frames[k][i].v, frames[k][i].v + 8, obs[i].v); }
            int32_t c4[4]; double par;
            ok(gf_fm_window_add_frame(win, fc, obs.data(), (int)obs.size(), nullptr, 0.0, &margin, c4, &par), "add_frame");
        } else margin = h.add(fc, frames[k], 0.0);
        if (fc < W) continue;
        int nf = 0, nv = 0, n = 0;
        if (win) ok(gf_fm_window_triangulate(win, fc, p.P, p.R, p.tic, p.ric), "triangulate"); else h.triangulate(p);
        const auto t1 = clk::now();
        if (win) ok(gf_fm_window_fill_problem(win, rows.data(), (int)rows.size(), &nv, para.data(), cst.data(), &nf), "fill_problem");
        else { std::vector<double> pf; std::vector<uint8_t> c; h.fill(rows, pf, c); nv = (int)rows.size(); nf = (int)pf.size(); std::copy(pf.begin(), pf.end(), para.begin()); }
        t_fill.push_back(us(t1, clk::now())); factors = nv;
        std::vector<int> bad;
        if (win) {
            ok(gf_fm_window_set_depth(win, para.data(), nf), "set_depth");
            ok(gf_fm_window_outliers(win, p.P, p.R, p.tic, p.ric, GF_FM_OUTLIERS_MOVING, ids.data(), &n), "outliers");
            bad.assign(ids.begin(), ids.begin() + n);
        } else { h.setDepth(std::vector<double>(para.begin(), para.begin() + nf)); bad = h.moving(p); }
        std::sort(bad.begin(), bad.end());
        if (bad.size() > 3) bad.resize(3);
        if (win) {
            std::vector<int32_t> b(bad.begin(), bad.end());
            ok(gf_fm_window_remove_ids(win, b.data(), (int)b.size()), "remove_ids");
            ok(gf_fm_window_predict_next(win, fc, p.P, p.R, p.tic, p.ric, ids.data(), xyz.data(), &n), "predict_next");
            if (margin || k % 3 == 0) ok(gf_fm_window_remove_back_shift_depth(win, p.R, p.P, p.R + 9, p.P + 3), "remove_back_shift_depth");
            else ok(gf_fm_window_remove_front(win, fc), "remove_front");
            ok(gf_fm_window_remove_failures(win), "remove_failures");
            ok(gf_fm_window_size(win, &n), "size");                 // the frame's work has finished on the device before the clock stops
        } else {
            h.removeIds(bad); h.predict(fc, p, xyz);
            if (margin || k % 3 == 0) h.removeBackShiftDepth(p); else h.removeFront(fc);
            h.removeFailures();
        }
        t_stage.push_back(us(t0, clk::now()));
    }
    return {median(t_stage), median(t_fill), factors};
}
}  // namespace fmb

static int run_fm_bench(const char *in, const char *out)
{
    using namespace fmb;
    FILE *f = fopen(in, "rb"), *o = fopen(out, "w");
    if (!f || !o) return 2;
    const int rounds = rd1<int>(f), n_frames = rd1<int>(f);
    const double min_parallax = rd1<double>(f), depth_threshold = rd1<double>(f);
    Poses p; rd(f, &p, sizeof(p));
    std::vector<std::vector<Obs>> frames(n_frames);
    for (auto &fr : frames) { fr.resize(rd1<int>(f)); for (auto &ob : fr) { ob.id = rd1<int>(f); rd(f, ob.v, 64); } }
    gf_fm_window_cfg c{};
    c.max_features = 8192; c.window_size = 10; c.min_parallax = min_parallax; c.depth_threshold = depth_threshold; c.init_depth = INIT_DEPTH;
    gf_fm_window *win = nullptr;
    ok(gf_fm_window_create(&win, 0, &c), "gf_fm_window_create");
    const Pass wa = pass(frames, p, min_parallax, depth_threshold, nullptr), wb = pass(frames, p, min_parallax, depth_threshold, win);    // warm-up
    std::vector<Pass> a, b;
    for (int r = 0; r < rounds; r++) { a.push_back(pass(frames, p, min_parallax, depth_threshold, nullptr)); b.push_back(pass(frames, p, min_parallax, depth_threshold, win)); }
    gf_fm_window_destroy(win);
    auto put = [&](const char *name, const std::vector<Pass> &v, bool last) {
        std::vector<double> s, fl;
        for (auto &x : v) { s.push_back(x.stage_us); fl.push_back(x.fill_us); }
        std::fprintf(o, "\"%s\": {\"stage_us\": {\"median\": %.3f, \"min\": %.3f, \"max\": %.3f}, \"factor_loop_us\": {\"median\": %.3f, \"min\": %.3f, \"max\": %.3f}}%s",
                     name, median(s), *std::min_element(s.begin(), s.end()), *std::max_element(s.begin(), s.end()), median(fl),
                     *std::min_element(fl.begin(), fl.end()), *std::max_element(fl.begin(), fl.end()), last ? "" : ", ");
    };
    std::fprintf(o, "{\"factors_per_window\": [%ld, %ld], ", wa.factors, wb.factors);
    put("stateless_calls_host_list", a, false); put("gf_fm_window", b, true);
    std::fprintf(o, "}\n");
    fclose(f); fclose(o);
    return 0;
}

// ---- fm-group-bench: the same stage for K windows, through gf_fm_window_group, K windows in sequence, or K threads ----
namespace fmg {
using namespace fmb;
enum Arm { GROUP, SEQUENTIAL, THREADS };

// the stage of one frame on window w alone, as fmb::pass runs it on the resident table
static void single_frame(gf_fm_window *w, const std::vector<gf_obs> &obs, int fc, size_t k, const Poses &p, std::vector<gf_ba_visual_factor> &rows,
                         std::vector<double> &para, std::vector<uint8_t> &cst, std::vector<int32_t> &ids, std::vector<double> &xyz)
{
    int margin = 0, nf = 0, nv = 0, n = 0; int32_t c4[4]; double par;
    ok(gf_fm_window_add_frame(w, fc, obs.data(), (int)obs.size(), nullptr, 0.0, &margin, c4, &par), "add_frame");
    if (fc < W) return;
    ok(gf_fm_window_triangulate(w, fc, p.P, p.R, p.tic, p.ric), "triangulate");
    ok(gf_fm_window_fill_problem(w, rows.data(), (int)rows.size(), &nv, para.data(), cst.data(), &nf), "fill_problem");
    ok(gf_fm_window_set_depth(w, para.data(), nf), "set_depth");
    ok(gf_fm_window_outliers(w, p.P, p.R, p.tic, p.ric, GF_FM_OUTLIERS_MOVING, ids.data(), &n), "outliers");
    std::vector<int32_t> bad(ids.begin(), ids.begin() + n);
    std::sort(bad.begin(), bad.end());
    if (bad.size() > 3) bad.resize(3);
    ok(gf_fm_window_remove_ids(w, bad.data(), (int)bad.size()), "remove_ids");
    ok(gf_fm_window_predict_next(w, fc, p.P, p.R, p.tic, p.ric, ids.data(), xyz.data(), &n), "predict_next");
    if (margin || k % 3 == 0) ok(gf_fm_window_remove_back_shift_depth(w, p.R, p.P, p.R + 9, p.P + 3), "remove_back_shift_depth");
    else ok(gf_fm_window_remove_front(w, fc), "remove_front");
    ok(gf_fm_window_remove_failures(w), "remove_failures");
    ok(gf_fm_window_size(w, &n), "size");                           // the frame's work has finished on the device
}

struct Buf {
    std::vector<gf_ba_visual_factor> rows; std::vector<double> para, xyz; std::vector<uint8_t> cst; std::vector<int32_t> ids;
    explicit Buf(int cap) : rows((size_t)cap * 10), para(cap), xyz(3 * (size_t)cap), cst(cap), ids(cap) {}
};

// one pass of the stream on K windows; returns microseconds of host time per round (one frame of every window)
static double pass_k(Arm arm, const std::vector<std::vector<gf_obs>> &frames, const Poses &p, std::vector<gf_fm_window *> &w, gf_fm_window_group *g,
                     std::vector<Buf> &b, int cap)
{
    const int K = (int)w.size();
    for (auto *x : w) ok(gf_fm_window_clear(x), "clear");
    for (auto *x : w) { int n; ok(gf_fm_window_size(x, &n), "size"); }
    const auto t0 = clk::now();
    if (arm == THREADS) {
        std::vector<std::thread> th;
        for (int i = 0; i < K; i++)
            th.emplace_back([&, i] { for (size_t k = 0; k < frames.size(); k++) single_frame(w[i], frames[k], (int)std::min<size_t>(k, W), k, p, b[i].rows, b[i].para, b[i].cst, b[i].ids, b[i].xyz); });
        for (auto &t : th) t.join();
        return us(t0, clk::now()) / frames.size();
    }
    std::vector<int32_t> fcs(K), ops(K), start(K + 1), nv(K), nf(K), n(K), c4(4 * K), margin(K), caps(K, cap * 10), ids, id_start(K + 1);
    std::vector<double> tds(K, 0.0), par(K), shift(24 * (size_t)K), Ps(33 * (size_t)K), Rs(99 * (size_t)K), tic(3 * (size_t)K), ric(9 * (size_t)K);
    std::vector<gf_obs> all;
    std::vector<gf_ba_visual_factor *> vo(K); std::vector<double *> pf(K), xyz(K); std::vector<uint8_t *> cs(K); std::vector<int32_t *> io(K);
    std::vector<const double *> x(K);
    for (int i = 0; i < K; i++) {
        vo[i] = b[i].rows.data(); pf[i] = b[i].para.data(); cs[i] = b[i].cst.data(); io[i] = b[i].ids.data(); xyz[i] = b[i].xyz.data(); x[i] = b[i].para.data();
        std::copy(p.P, p.P + 33, &Ps[33 * i]); std::copy(p.R, p.R + 99, &Rs[99 * i]); std::copy(p.tic, p.tic + 3, &tic[3 * i]); std::copy(p.ric, p.ric + 9, &ric[9 * i]);
        std::copy(p.R, p.R + 9, &shift[24 * i]); std::copy(p.P, p.P + 3, &shift[24 * i + 9]); std::copy(p.R + 9, p.R + 18, &shift[24 * i + 12]); std::copy(p.P + 3, p.P + 6, &shift[24 * i + 21]);
    }
    for (size_t k = 0; k < frames.size(); k++) {
        const int fc = (int)std::min<size_t>(k, W);
        if (arm == SEQUENTIAL) {
            for (int i = 0; i < K; i++) single_frame(w[i], frames[k], fc, k, p, b[i].rows, b[i].para, b[i].cst, b[i].ids, b[i].xyz);
            continue;
        }
        all.clear();
        for (int i = 0; i < K; i++) { start[i] = (int)all.size(); all.insert(all.end(), frames[k].begin(), frames[k].end()); fcs[i] = fc; }
        start[K] = (int)all.size();
        ok(gf_fm_window_group_add_frame(g, fcs.data(), all.data(), start.data(), nullptr, tds.data(), margin.data(), c4.data(), par.data(), nullptr), "group add_frame");
        if (fc < W) continue;
        ok(gf_fm_window_group_triangulate(g, fcs.data(), Ps.data(), Rs.data(), tic.data(), ric.data()), "group triangulate");
        ok(gf_fm_window_group_fill_problem(g, vo.data(), caps.data(), nv.data(), pf.data(), cs.data(), nf.data(), nullptr), "group fill_problem");
        ok(gf_fm_window_group_set_depth(g, x.data(), nf.data()), "group set_depth");
        ok(gf_fm_window_group_outliers(g, Ps.data(), Rs.data(), tic.data(), ric.data(), GF_FM_OUTLIERS_MOVING, io.data(), n.data()), "group outliers");
        ids.clear(); id_start[0] = 0;
        for (int i = 0; i < K; i++) {
            std::vector<int32_t> bad(b[i].ids.begin(), b[i].ids.begin() + n[i]);
            std::sort(bad.begin(), bad.end());
            if (bad.size() > 3) bad.resize(3);
            ids.insert(ids.end(), bad.begin(), bad.end()); id_start[i + 1] = (int)ids.size();
        }
        ok(gf_fm_window_group_remove_ids(g, ids.data(), id_start.data()), "group remove_ids");
        ok(gf_fm_window_group_predict_next(g, fcs.data(), Ps.data(), Rs.data(), tic.data(), ric.data(), io.data(), xyz.data(), n.data()), "group predict_next");
        for (int i = 0; i < K; i++) ops[i] = (margin[i] || k % 3 == 0) ? GF_FM_REMOVE_BACK_SHIFT_DEPTH : GF_FM_REMOVE_FRONT;
        ok(gf_fm_window_group_remove(g, ops.data(), fcs.data(), shift.data()), "group remove");
        ok(gf_fm_window_group_remove_failures(g), "group remove_failures");
        float ms;
        ok(gf_fm_window_group_last_device_ms(g, &ms), "group last_device_ms");     // waits for the round's work on the device
    }
    return us(t0, clk::now()) / frames.size();
}
}  // namespace fmg

// input: the fm-bench input, then the number of K values and the K values.  Output: per K and arm, the host time per round
// (one frame of all K windows) averaged over a pass, as median and [min, max] over `rounds` passes, arms alternating.
static int run_fm_group_bench(const char *in, const char *out)
{
    using namespace fmb;
    using namespace fmg;
    FILE *f = fopen(in, "rb"), *o = fopen(out, "w");
    if (!f || !o) return 2;
    const int rounds = rd1<int>(f), n_frames = rd1<int>(f);
    const double min_parallax = rd1<double>(f), depth_threshold = rd1<double>(f);
    Poses p; rd(f, &p, sizeof(p));
    std::vector<std::vector<gf_obs>> frames(n_frames);
    for (auto &fr : frames) {
        fr.resize(rd1<int>(f));
        for (auto &ob : fr) { ob.id = rd1<int>(f); ob.track_cnt = 0; rd(f, ob.v, 64); }
    }
    std::vector<int> Ks(rd1<int>(f));
    for (auto &k : Ks) k = rd1<int>(f);
    const int cap = 2048;
    gf_fm_window_cfg c{};
    c.max_features = cap; c.window_size = 10; c.min_parallax = min_parallax; c.depth_threshold = depth_threshold; c.init_depth = INIT_DEPTH;
    std::fprintf(o, "{\"window_capacity\": %d, \"unit\": \"microseconds of host time per round (one frame of every window), mean over a pass\", \"K\": {", cap);
    for (size_t ki = 0; ki < Ks.size(); ki++) {
        const int K = Ks[ki];
        std::vector<gf_fm_window *> w(K);
        std::vector<Buf> b;
        for (int i = 0; i < K; i++) { ok(gf_fm_window_create(&w[i], 0, &c), "gf_fm_window_create"); b.emplace_back(cap); }
        gf_fm_window_group *g = nullptr;
        ok(gf_fm_window_group_create(&g, w.data(), K), "gf_fm_window_group_create");
        const char *names[3] = {"group", "sequential", "threads"};
        std::vector<double> t[3];
        for (int a = 0; a < 3; a++) pass_k((Arm)a, frames, p, w, g, b, cap);                  // warm-up
        for (int r = 0; r < rounds; r++) for (int a = 0; a < 3; a++) t[a].push_back(pass_k((Arm)a, frames, p, w, g, b, cap));
        gf_fm_window_group_destroy(g);
        for (auto *x : w) gf_fm_window_destroy(x);
        std::fprintf(o, "%s\"%d\": {", ki ? ", " : "", K);
        for (int a = 0; a < 3; a++)
            std::fprintf(o, "%s\"%s\": {\"median\": %.3f, \"min\": %.3f, \"max\": %.3f}", a ? ", " : "", names[a], median(t[a]),
                         *std::min_element(t[a].begin(), t[a].end()), *std::max_element(t[a].begin(), t[a].end()));
        std::fprintf(o, "}");
    }
    std::fprintf(o, "}}\n");
    fclose(f); fclose(o);
    return 0;
}

int main(int argc, char **argv)
{
    if (argc != 4) { std::fprintf(stderr, "usage: harness fe|fe-eq|fe-box|ba|ba-multi|ba-seq|dm|gm|fm|fm-bench|fm-group-bench <in> <out>\n"); return 2; }
    if (!std::strcmp(argv[1], "fe-eq")) EQUALIZE = 1;
    if (!std::strcmp(argv[1], "dm")) return run_dm(argv[2], argv[3]);
    if (!std::strcmp(argv[1], "gm")) return run_gm(argv[2], argv[3]);
    if (!std::strcmp(argv[1], "fm")) return run_fm(argv[2], argv[3]);
    if (!std::strcmp(argv[1], "fm-bench")) return run_fm_bench(argv[2], argv[3]);
    if (!std::strcmp(argv[1], "fm-group-bench")) return run_fm_group_bench(argv[2], argv[3]);
    if (!std::strcmp(argv[1], "ba-multi") || !std::strcmp(argv[1], "ba-seq")) return run_ba_multi(argv[2], argv[3], argv[1][3] == 'm');
    return argv[1][0] == 'f' ? run_fe(argv[2], argv[3], !std::strcmp(argv[1], "fe-box")) : run_ba(argv[2], argv[3]);
}
