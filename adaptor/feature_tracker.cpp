// Bodies of FeatureTracker::{trackImage, trackImagebox, setPrediction, removeOutliers} on the GPU library.  Replaces
// feature_tracker.cpp:103-372, 374-678, 1006-1027, 1029-1045 of the reference; nothing here touches OpenCV algorithms.
#include "feature_tracker.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace {
[[noreturn]] void gf_fatal(const char *what)
{
    // the reference aborts through ROS_BREAK() on unrecoverable errors; there is no CPU fallback behind this path
    std::fprintf(stderr, "gf_b200: %s: %s\n", what, gf_last_error());
    std::abort();
}
}  // namespace

FeatureTracker::FeatureTracker() {}
FeatureTracker::~FeatureTracker()
{
    if (gf_) gf_tracker_destroy(gf_);
}

void FeatureTracker::setPinhole(double fx, double fy, double cx, double cy, double k1, double k2, double p1, double p2, int depth)
{
    const double p[8] = {fx, fy, cx, cy, k1, k2, p1, p2};
    std::memcpy(cfg_.pinhole, p, sizeof(p));
    depth_cam = depth != 0;            // feature_tracker.cpp:757-758
}

// The first frame creates the tracker (it needs the image size); every frame advances the time stamps.
void FeatureTracker::start(double _cur_time, const cv::Mat &_img)
{
    if (!gf_) {
        cfg_.max_cnt = MAX_CNT; cfg_.min_dist = MIN_DIST; cfg_.flow_back = FLOW_BACK; cfg_.depth_cam = depth_cam ? 1 : 0;
        row = _img.rows; col = _img.cols;
        if (gf_tracker_create(&gf_, device, col, row, &cfg_)) gf_fatal("gf_tracker_create");
        // the reference equalises in getImageFromMsg before trackImage sees the frame; here the library does it on the GPU
        // from the first frame on, which is the same image for every call (INTEGRATION.md)
        if (EQUALIZE && gf_tracker_set_equalize(gf_, 40.0, 8, 8)) gf_fatal("gf_tracker_set_equalize");
        out_.resize(MAX_CNT > 0 ? MAX_CNT : 1);
        in_box_.resize(out_.size());
    }
    prev_time = cur_time; cur_time = _cur_time;
}

// featureFrame from the n results (without the ones flagged in in_box, when given); cur_pts / ids / track_cnt get all n.
std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> FeatureTracker::publish(int n, const uint8_t *in_box)
{
    hasPrediction = false;             // feature_tracker.cpp:365
    std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> featureFrame;
    cur_pts.resize(n); ids.resize(n); track_cnt.resize(n);
    for (int i = 0; i < n; i++) {
        cur_pts[i] = cv::Point2f((float)out_[i].v[3], (float)out_[i].v[4]);
        ids[i] = out_[i].id; track_cnt[i] = out_[i].track_cnt;
        if (in_box && in_box[i]) continue;
        Eigen::Matrix<double, 8, 1> v;
        std::memcpy(v.data(), out_[i].v, sizeof(out_[i].v));      // x y z p_u p_v velocity_x velocity_y depth (:344-369)
        featureFrame[out_[i].id].emplace_back(0, v);
    }
    return featureFrame;
}

std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> FeatureTracker::trackImage(double _cur_time, const cv::Mat &_img, const cv::Mat &_img1)
{
    start(_cur_time, _img);
    int n = 0;
    const uint16_t *depth = _img1.empty() ? nullptr : _img1.ptr<uint16_t>();
    if (gf_tracker_track(gf_, _cur_time, _img.data, _img.step, depth, _img1.empty() ? 0 : _img1.step, 0, nullptr, 0, out_.data(), &n, nullptr,
                         nullptr, nullptr))
        gf_fatal("gf_tracker_track");
    return publish(n, nullptr);
}

std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 8, 1>>>> FeatureTracker::trackImagebox(double _cur_time, const darknet_ros_msgs::BoundingBoxesConstPtr &_boxes,
                                                                                                     const cv::Mat &_img, const cv::Mat &_img1)
{
    start(_cur_time, _img);
    boxes_.clear();
    for (const darknet_ros_msgs::BoundingBox &b : _boxes->bounding_boxes) boxes_.push_back(gf_box{b.xmin, b.ymin, b.xmax, b.ymax});
    int n = 0;
    const uint16_t *depth = _img1.empty() ? nullptr : _img1.ptr<uint16_t>();
    if (gf_tracker_track(gf_, _cur_time, _img.data, _img.step, depth, _img1.empty() ? 0 : _img1.step, 0, boxes_.data(), (int)boxes_.size(),
                         out_.data(), &n, in_box_.data(), nullptr, nullptr))
        gf_fatal("gf_tracker_track");
    return publish(n, in_box_.data());
}

void FeatureTracker::setPrediction(std::map<int, Eigen::Vector3d> &predictPts)
{
    if (!gf_) return;
    std::vector<int32_t> id; std::vector<double> xyz;
    id.reserve(predictPts.size()); xyz.reserve(3 * predictPts.size());
    for (auto &kv : predictPts) { id.push_back(kv.first); xyz.insert(xyz.end(), kv.second.data(), kv.second.data() + 3); }
    if (gf_tracker_set_prediction(gf_, id.data(), xyz.data(), (int)id.size())) gf_fatal("gf_tracker_set_prediction");
    hasPrediction = true;
}

void FeatureTracker::removeOutliers(std::set<int> &removePtsIds)
{
    if (!gf_) return;
    std::vector<int32_t> id(removePtsIds.begin(), removePtsIds.end());
    if (gf_tracker_remove_ids(gf_, id.data(), (int)id.size())) gf_fatal("gf_tracker_remove_ids");
}
