#include "feature_manager.h"

#include <cstdio>
#include <cstdlib>

#include "feature_tracker.h"

static void check(int rc, const char *what)
{
    if (rc == GF_OK) return;
    // the reference class has no error path here; there is no CPU fallback behind this path
    std::fprintf(stderr, "gf_b200: %s: %s\n", what, gf_last_error());
    std::abort();
}

namespace {
struct Poses { double P[GF_FM_WINDOW_ROWS * 3], R[GF_FM_WINDOW_ROWS * 9], tic[3], ric[9]; };
void row_major(const Eigen::Matrix3d &M, double *out)
{
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) out[3 * i + j] = M(i, j);
}
Poses poses(const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[], const Eigen::Vector3d &tic, const Eigen::Matrix3d &ric)
{
    Poses p;
    for (int f = 0; f < GF_FM_WINDOW_ROWS; f++) { for (int i = 0; i < 3; i++) p.P[3 * f + i] = Ps[f](i); row_major(Rs[f], p.R + 9 * f); }
    for (int i = 0; i < 3; i++) p.tic[i] = tic(i);
    row_major(ric, p.ric);
    return p;
}
}  // namespace

namespace gf_device {

FeatureManager::FeatureManager(double min_parallax, double depth_threshold, double init_depth, int max_features, int device) : cap_(max_features)
{
    gf_fm_window_cfg c{};
    c.max_features = max_features; c.window_size = 10; c.min_parallax = min_parallax; c.depth_threshold = depth_threshold; c.init_depth = init_depth;
    check(gf_fm_window_create(&w_, device, &c), "gf_fm_window_create");
}

FeatureManager::~FeatureManager() { gf_fm_window_destroy(w_); }

void FeatureManager::clearState() { check(gf_fm_window_clear(w_), "gf_fm_window_clear"); }

bool FeatureManager::added(int margin_old, const int32_t *cnt, double parallax)
{
    last_track_num = cnt[0]; new_feature_num = cnt[1]; long_track_num = cnt[2]; last_average_parallax = parallax;
    return margin_old != 0;
}

bool FeatureManager::addFeatureCheckParallax(int frame_count, const std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> &image, double td)
{
    std::vector<gf_obs> obs;
    obs.reserve(image.size());
    for (auto &kv : image) {
        gf_obs o{};
        o.id = kv.first;
        for (int k = 0; k < 8; k++) o.v[k] = kv.second[0].second(k);
        obs.push_back(o);
    }
    int margin = 0; int32_t cnt[4]; double par = 0;
    check(gf_fm_window_add_frame(w_, frame_count, obs.data(), (int)obs.size(), nullptr, td, &margin, cnt, &par), "gf_fm_window_add_frame");
    return added(margin, cnt, par);
}

bool FeatureManager::addFeatureCheckParallax(int frame_count, const FeatureTracker &tracker, double td)
{
    int margin = 0; int32_t cnt[4]; double par = 0;
    check(gf_fm_window_add_frame_from_tracker(w_, tracker.handle(), frame_count, td, &margin, cnt, &par), "gf_fm_window_add_frame_from_tracker");
    return added(margin, cnt, par);
}

void FeatureManager::triangulate(int frameCnt, const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[], const Eigen::Vector3d &tic, const Eigen::Matrix3d &ric)
{
    const Poses p = poses(Ps, Rs, tic, ric);
    check(gf_fm_window_triangulate(w_, frameCnt, p.P, p.R, p.tic, p.ric), "gf_fm_window_triangulate");
}

std::vector<double> FeatureManager::getDepthVector()
{
    std::vector<double> x(cap_);
    int n = 0;
    check(gf_fm_window_fill_problem(w_, nullptr, 0, nullptr, x.data(), nullptr, &n), "gf_fm_window_fill_problem");
    x.resize(n);
    return x;
}

int FeatureManager::getFeatureCount() { return (int)getDepthVector().size(); }

void FeatureManager::setDepth(const std::vector<double> &x) { check(gf_fm_window_set_depth(w_, x.data(), (int)x.size()), "gf_fm_window_set_depth"); }

void FeatureManager::fillProblem(std::vector<gf_ba_visual_factor> &visual, std::vector<double> &para_feature, std::vector<uint8_t> &feature_const)
{
    visual.resize((size_t)cap_ * (GF_FM_WINDOW_ROWS - 1)); para_feature.resize(cap_); feature_const.resize(cap_);
    int nv = 0, nf = 0;
    check(gf_fm_window_fill_problem(w_, visual.data(), (int)visual.size(), &nv, para_feature.data(), feature_const.data(), &nf), "gf_fm_window_fill_problem");
    visual.resize(nv); para_feature.resize(nf); feature_const.resize(nf);
}

void FeatureManager::removeFailures() { check(gf_fm_window_remove_failures(w_), "gf_fm_window_remove_failures"); }
void FeatureManager::clearDepth() { check(gf_fm_window_clear_depth(w_), "gf_fm_window_clear_depth"); }

void FeatureManager::removeOutlier(const std::set<int> &outlierIndex)
{
    std::vector<int32_t> ids(outlierIndex.begin(), outlierIndex.end());
    check(gf_fm_window_remove_ids(w_, ids.data(), (int)ids.size()), "gf_fm_window_remove_ids");
}

void FeatureManager::removeBackShiftDepth(const Eigen::Matrix3d &marg_R, const Eigen::Vector3d &marg_P, const Eigen::Matrix3d &new_R, const Eigen::Vector3d &new_P)
{
    double mr[9], nr[9];
    row_major(marg_R, mr); row_major(new_R, nr);
    check(gf_fm_window_remove_back_shift_depth(w_, mr, marg_P.data(), nr, new_P.data()), "gf_fm_window_remove_back_shift_depth");
}

void FeatureManager::removeBack() { check(gf_fm_window_remove_back(w_), "gf_fm_window_remove_back"); }
void FeatureManager::removeFront(int frame_count) { check(gf_fm_window_remove_front(w_, frame_count), "gf_fm_window_remove_front"); }

void FeatureManager::outliersRejection(std::set<int> &removeIndex, const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[], const Eigen::Vector3d &tic,
                                       const Eigen::Matrix3d &ric)
{
    const Poses p = poses(Ps, Rs, tic, ric);
    std::vector<int32_t> ids(cap_);
    int n = 0;
    check(gf_fm_window_outliers(w_, p.P, p.R, p.tic, p.ric, GF_FM_OUTLIERS_REPROJECTION, ids.data(), &n), "gf_fm_window_outliers");
    removeIndex.insert(ids.begin(), ids.begin() + n);
}

void FeatureManager::movingConsistencyCheckW(std::set<int> &removeIndex, const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[], const Eigen::Vector3d &tic,
                                             const Eigen::Matrix3d &ric)
{
    const Poses p = poses(Ps, Rs, tic, ric);
    std::vector<int32_t> ids(cap_);
    int n = 0;
    check(gf_fm_window_outliers(w_, p.P, p.R, p.tic, p.ric, GF_FM_OUTLIERS_MOVING, ids.data(), &n), "gf_fm_window_outliers");
    removeIndex.insert(ids.begin(), ids.begin() + n);
}

std::map<int, Eigen::Vector3d> FeatureManager::predictPtsInNextFrame(int frame_count, const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[],
                                                                     const Eigen::Vector3d &tic, const Eigen::Matrix3d &ric)
{
    const Poses p = poses(Ps, Rs, tic, ric);
    std::vector<int32_t> ids(cap_);
    std::vector<double> xyz(3 * (size_t)cap_);
    int n = 0;
    check(gf_fm_window_predict_next(w_, frame_count, p.P, p.R, p.tic, p.ric, ids.data(), xyz.data(), &n), "gf_fm_window_predict_next");
    std::map<int, Eigen::Vector3d> out;
    for (int k = 0; k < n; k++) { Eigen::Vector3d v; for (int i = 0; i < 3; i++) v(i) = xyz[3 * k + i]; out[ids[k]] = v; }
    return out;
}

std::vector<FeaturePerId> FeatureManager::features()
{
    const size_t c = cap_, row = GF_FM_WINDOW_ROWS * GF_FM_WINDOW_ROW_DOUBLES;
    std::vector<int32_t> id(c), start(c), nobs(c), eflag(c), sflag(c);
    std::vector<double> est(c), obs(c * row);
    int n = 0;
    check(gf_fm_window_read(w_, id.data(), start.data(), nobs.data(), est.data(), eflag.data(), sflag.data(), obs.data(), cap_, &n), "gf_fm_window_read");
    std::vector<FeaturePerId> out(n);
    for (int i = 0; i < n; i++) {
        out[i].feature_id = id[i]; out[i].start_frame = start[i]; out[i].estimated_depth = est[i]; out[i].estimate_flag = eflag[i]; out[i].solve_flag = sflag[i];
        out[i].feature_per_frame.resize(nobs[i]);
        for (int a = 0; a < nobs[i]; a++)
            for (int k = 0; k < GF_FM_WINDOW_ROW_DOUBLES; k++) out[i].feature_per_frame[a](k) = obs[i * row + a * GF_FM_WINDOW_ROW_DOUBLES + k];
    }
    return out;
}

}  // namespace gf_device
