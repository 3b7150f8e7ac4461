// FeatureTracker with the reference's class surface (vins_estimator/src/featureTracker/feature_tracker.h:43-99) whose
// trackImage / setPrediction / removeOutliers bodies call libgf_b200.so.  Callers (Estimator::inputImage,
// estimator.cpp:182-221; sync_process in rosNodeTest.cpp) compile against it unchanged.  The members the reference's other
// code reads after a frame (drawTrack: cur_pts, ids, track_cnt; prev/cur time) are kept and refreshed from the result.
#pragma once
#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include <darknet_ros_msgs/BoundingBoxes.h>
#include <eigen3/Eigen/Dense>
#include <opencv2/opencv.hpp>

#include "gf_b200.h"

// parameters.h:130-134 (read from the YAML by readParameters): defined by the node, declared here as the reference does
extern int MAX_CNT;
extern int MIN_DIST;
extern int FLOW_BACK;
// parameters.h:33: every image goes through cv::createCLAHE() (clip 40, 8 x 8 tiles) before trackImage (rosNodeTest.cpp:256-261)
extern int EQUALIZE;

class FeatureTracker
{
  public:
    FeatureTracker();
    ~FeatureTracker();
    FeatureTracker(const FeatureTracker &) = delete;
    FeatureTracker &operator=(const FeatureTracker &) = delete;

    std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> trackImage(double _cur_time, const cv::Mat &_img, const cv::Mat &_img1 = cv::Mat());
    // USE_YOLO (Estimator::inputImagebox): trackImage, with the features strictly inside a detected box left out of the returned
    // frame only; cur_pts / ids / track_cnt keep them, as the reference's do (feature_tracker.cpp:374-678)
    std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> trackImagebox(double _cur_time, const darknet_ros_msgs::BoundingBoxesConstPtr &_boxes,
                                                                                          const cv::Mat &_img, const cv::Mat &_img1 = cv::Mat());
    // readIntrinsicParameter(calib_file, depth) (feature_tracker.cpp:745-762) parses the camodocal YAML; the parsed PINHOLE
    // parameters are all this path needs.  With camodocal present: m_camera[0]->writeParameters(p) -> setPinhole(p[4..7], p[0..3]).
    void setPinhole(double fx, double fy, double cx, double cy, double k1, double k2, double p1, double p2, int depth);
    void setPrediction(std::map<int, Eigen::Vector3d> &predictPts);
    void removeOutliers(std::set<int> &removePtsIds);
    // the library's tracker (null before the first frame), for FeatureManager::addFeatureCheckParallax(frame_count, tracker, td)
    const gf_tracker *handle() const { return gf_; }

    int row = 0, col = 0;
    std::vector<cv::Point2f> cur_pts;
    std::vector<int> ids;
    std::vector<int> track_cnt;
    double cur_time = 0, prev_time = 0;
    bool stereo_cam = false;
    bool depth_cam = false;
    bool hasPrediction = false;
    int device = 0;          // CUDA device of this camera stream

  private:
    void start(double _cur_time, const cv::Mat &_img);
    std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> publish(int n, const uint8_t *in_box);
    gf_tracker *gf_ = nullptr;          // created on the first frame: needs its size
    gf_tracker_cfg cfg_{};
    std::vector<gf_obs> out_;
    std::vector<uint8_t> in_box_;
    std::vector<gf_box> boxes_;
};
