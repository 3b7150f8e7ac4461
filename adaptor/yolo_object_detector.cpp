#include "yolo_object_detector.h"

#include <stdexcept>

YoloObjectDetector::YoloObjectDetector(const std::string& cfg, const std::string& weights, float thresh,
                                       const std::vector<std::string>& class_labels, int device)
    : labels_(class_labels)
{
    if (gf_detector_create(&det_, device, cfg.c_str(), weights.c_str(), thresh) != GF_OK)
        throw std::runtime_error(std::string("gf_detector_create: ") + gf_detector_last_error());
}

YoloObjectDetector::~YoloObjectDetector() { gf_detector_destroy(det_); }

void YoloObjectDetector::setPrecision(int precision)
{
    if (gf_detector_set_precision(det_, precision) != GF_OK)
        throw std::runtime_error(std::string("gf_detector_set_precision: ") + gf_detector_last_error());
}

darknet_ros_msgs::BoundingBoxes YoloObjectDetector::detect(const cv::Mat& bgr, double stamp)
{
    gf_box boxes[GF_MAX_BOXES];
    int ids[GF_MAX_BOXES];
    float probs[GF_MAX_BOXES];
    int n = 0;
    if (gf_detector_detect(det_, bgr.data, bgr.step, bgr.cols, bgr.rows, 0, boxes, ids, probs, GF_MAX_BOXES, &n) != GF_OK)
        throw std::runtime_error(std::string("gf_detector_detect: ") + gf_detector_last_error());
    darknet_ros_msgs::BoundingBoxes msg;
    msg.header.stamp = stamp;
    msg.header.frame_id = "detection";
    msg.image_header.stamp = stamp;
    for (int i = 0; i < n; i++) {
        darknet_ros_msgs::BoundingBox b;
        b.Class = ids[i] < (int)labels_.size() ? labels_[ids[i]] : std::to_string(ids[i]);
        b.id = (int16_t)ids[i];
        b.probability = probs[i];
        b.xmin = boxes[i].xmin; b.ymin = boxes[i].ymin; b.xmax = boxes[i].xmax; b.ymax = boxes[i].ymax;
        msg.bounding_boxes.push_back(b);
    }
    return msg;
}
