// The slice of class Estimator (vins_estimator/src/estimator/estimator.h:147, members :262-330) that
// Estimator::optimization() reads and writes, with optimization() rebuilt on libgf_b200.so.  Member names, array shapes and
// the FeatureManager / IntegrationBase fields are the reference's, so the body below is what a maintainer pastes over
// estimator.cpp:2884-3631; the rest of the class (ROS buffers, initialisation, slideWindow) is untouched and not repeated.
#pragma once
#include <list>
#include <vector>

#include <eigen3/Eigen/Dense>

#include "gf_b200.h"

const int WINDOW_SIZE = 10;          // parameters.h:21
const int NUM_OF_F = 1000;           // parameters.h:23
enum SIZE_PARAMETERIZATION { SIZE_POSE = 7, SIZE_SPEEDBIAS = 9, SIZE_FEATURE = 1 };   // parameters.h:172-178

extern int USE_IMU, NUM_ITERATIONS, ESTIMATE_TD;
extern double FOCAL_LENGTH;
extern Eigen::Vector3d G;

struct IntegrationBase {             // factor/integration_base.h:197-212: the members IMUFactor::Evaluate reads
    double sum_dt = 0;
    Eigen::Vector3d delta_p, delta_v, linearized_ba, linearized_bg;
    Eigen::Quaterniond delta_q;
    Eigen::Matrix<double, 15, 15> jacobian, covariance;
};
struct FeaturePerFrame {             // feature_manager.h:31-72
    Eigen::Vector3d point;
    Eigen::Vector2d velocity;
    double cur_td = 0, depth = 0;
};
struct FeaturePerId {                // feature_manager.h:75-100
    int feature_id = 0, start_frame = 0, used_num = 0, estimate_flag = 0;
    double estimated_depth = -1;
    std::vector<FeaturePerFrame> feature_per_frame;
};
struct FeatureManager {
    std::list<FeaturePerId> feature;
};

class Estimator
{
  public:
    enum MarginalizationFlag { MARGIN_OLD = 0, MARGIN_SECOND_NEW = 1 };
    Estimator();
    ~Estimator();
    void optimization();
    static void optimizationMulti(Estimator *const *est, int n);

    int frame_count = WINDOW_SIZE;
    MarginalizationFlag marginalization_flag = MARGIN_OLD;
    bool openExEstimation = false, systemstationary = false, stationary_detect = false;
    Eigen::Vector3d Vs[WINDOW_SIZE + 1];
    IntegrationBase *pre_integrations[WINDOW_SIZE + 1] = {};
    FeatureManager f_manager;
    double para_Pose[WINDOW_SIZE + 1][SIZE_POSE];
    double para_SpeedBias[WINDOW_SIZE + 1][SIZE_SPEEDBIAS];
    double para_Feature[NUM_OF_F][SIZE_FEATURE];
    double para_Ex_Pose[2][SIZE_POSE];
    double para_Td[1][1];

    gf_ba_summary last_summary{};
    int device = 0;
    int prior_dim() const { return have_prior_ ? prior_.n : 0; }
    const gf_ba_prior &prior() const { return prior_; }

  private:
    struct BaRows {                  // one window's gf_ba_problem and the factor tables it points into
        gf_ba_problem P{};
        std::vector<gf_ba_imu_factor> imu;
        std::vector<gf_ba_visual_factor> vis;
        std::vector<uint8_t> feature_const;
    };
    void buildProblem(BaRows &rows);
    void marginalize(const gf_ba_problem &P);
    void adoptPrior(int n, const gf_ba_prior &next, std::vector<double> &x0, std::vector<double> &J, std::vector<double> &r);
    gf_ba *gf_ba_ = nullptr;
    // last_marginalization_info + last_marginalization_parameter_blocks (estimator.h:318-319)
    bool have_prior_ = false;
    gf_ba_prior prior_{};
    std::vector<double> prior_x0_, prior_J_, prior_r_;
};
