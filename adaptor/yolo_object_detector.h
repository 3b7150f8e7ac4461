// YoloObjectDetector on libgf_b200's gf_detector: the part of the darknet_ros node (vins_estimator/src/YoloObjectDetector.cpp)
// that the use_yolo front end consumes -- one BGR8 frame in, the darknet_ros_msgs::BoundingBoxes the node would publish for it
// out, ready for FeatureTracker::trackImagebox.  The node's ROS plumbing (topics, action server, three-slot asynchronous buffer,
// display) is not reproduced: detect() is synchronous, so the boxes belong to the frame passed in.
#pragma once
#include <string>
#include <vector>

#include <darknet_ros_msgs/BoundingBoxes.h>
#include <opencv2/opencv.hpp>

#include "gf_b200.h"

class YoloObjectDetector {
public:
    // cfg / weights: the darknet files the node's yaml names; thresh: its detection threshold; class_labels: the names the
    // node's yaml lists (BoundingBox::Class; ids index them), may be empty.  Throws std::runtime_error with gf_detector_last_error().
    YoloObjectDetector(const std::string& cfg, const std::string& weights, float thresh,
                       const std::vector<std::string>& class_labels = {}, int device = 0);
    ~YoloObjectDetector();
    YoloObjectDetector(const YoloObjectDetector&) = delete;
    YoloObjectDetector& operator=(const YoloObjectDetector&) = delete;

    // One frame (CV_8UC3, BGR).  Empty bounding_boxes when the node would publish nothing (no box, or more than 100).
    darknet_ros_msgs::BoundingBoxes detect(const cv::Mat& bgr, double stamp = 0);
    // GF_DETECTOR_EXACT (the default: bit-exact with darknet's CPU build) or GF_DETECTOR_TF32 (tensor-core convolutions with
    // TF32-rounded operands, not bit-exact).  Throws std::runtime_error on another value or a device failure.
    void setPrecision(int precision);

private:
    gf_detector* det_ = nullptr;
    std::vector<std::string> labels_;
};
