// FeatureManager: the reference's class (vins_estimator/src/estimator/feature_manager.h:90-150) over gf_fm_window of
// libgf_b200.so.  The std::list<FeaturePerId> it kept is the handle's table on the GPU; the methods keep their names and
// argument meaning, and the three per-landmark loops of the estimator that read that list (estimator.cpp:3853-4011:
// outliersRejection, movingConsistencyCheckW, predictPtsInNextFrame) are methods here, since the list is no longer the caller's.
// Depth vectors are std::vector<double> where the reference has Eigen::VectorXd.
// The classes are in namespace gf_device: estimator_ba.h still declares the reference's host-side FeatureManager, whose list
// Estimator::optimization() reads; an estimator that takes its factors from fillProblem() drops that one for this.
#pragma once
#include <cstdint>
#include <map>
#include <set>
#include <utility>
#include <vector>

#include <eigen3/Eigen/Dense>

#include "gf_b200.h"

class FeatureTracker;

namespace gf_device {

// FeaturePerId with its FeaturePerFrame rows [x y z u v vx vy depth td], as features() returns them (pubPointCloud's view)
struct FeaturePerId
{
    int feature_id, start_frame;
    double estimated_depth;
    int estimate_flag, solve_flag;
    std::vector<Eigen::Matrix<double, 9, 1>> feature_per_frame;
    int endFrame() const { return start_frame + (int)feature_per_frame.size() - 1; }
};

class FeatureManager
{
  public:
    // MIN_PARALLAX as the reference stores it (pixels / FOCAL_LENGTH), DEPTH_THRESHOLD, INIT_DEPTH
    FeatureManager(double min_parallax, double depth_threshold, double init_depth, int max_features = 2048, int device = 0);
    ~FeatureManager();
    FeatureManager(const FeatureManager &) = delete;
    FeatureManager &operator=(const FeatureManager &) = delete;

    void clearState();
    int getFeatureCount();
    bool addFeatureCheckParallax(int frame_count, const std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> &image, double td);
    // the frame `tracker` returned last, taken from where it lies on the device
    bool addFeatureCheckParallax(int frame_count, const FeatureTracker &tracker, double td);
    void triangulate(int frameCnt, const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[], const Eigen::Vector3d &tic, const Eigen::Matrix3d &ric);
    std::vector<double> getDepthVector();
    void setDepth(const std::vector<double> &x);
    // the visual factors of gf_ba_problem with the matching para_Feature / constant flags (estimator.cpp:3268-3297)
    void fillProblem(std::vector<gf_ba_visual_factor> &visual, std::vector<double> &para_feature, std::vector<uint8_t> &feature_const);
    void removeFailures();
    void clearDepth();
    void removeOutlier(const std::set<int> &outlierIndex);
    void removeBackShiftDepth(const Eigen::Matrix3d &marg_R, const Eigen::Vector3d &marg_P, const Eigen::Matrix3d &new_R, const Eigen::Vector3d &new_P);
    void removeBack();
    void removeFront(int frame_count);
    void outliersRejection(std::set<int> &removeIndex, const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[], const Eigen::Vector3d &tic, const Eigen::Matrix3d &ric);
    void movingConsistencyCheckW(std::set<int> &removeIndex, const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[], const Eigen::Vector3d &tic, const Eigen::Matrix3d &ric);
    std::map<int, Eigen::Vector3d> predictPtsInNextFrame(int frame_count, const Eigen::Vector3d Ps[], const Eigen::Matrix3d Rs[], const Eigen::Vector3d &tic,
                                                         const Eigen::Matrix3d &ric);
    std::vector<FeaturePerId> features();

    int last_track_num = 0, new_feature_num = 0, long_track_num = 0;
    double last_average_parallax = 0;

  private:
    bool added(int margin_old, const int32_t *cnt, double parallax);
    gf_fm_window *w_ = nullptr;
    int cap_;
};

}  // namespace gf_device
