// DenseMap: the colour map of the reference's mapping node on libgf_b200.so.  It replaces the node's sampling loop
// (dense_map/src/pose_graph_node.cpp:598-623) and PoseGraph's three octree blocks (pose_graph.cpp: the constructor's octree
// at :29-34, addKeyFrame's insertion and RadiusOutlierRemoval at :191-239, updatePath's rebuild at :997-1058).  PoseGraph keeps
// one DenseMap instead of octree / cloud / save_cloud; loop detection and the pose-graph optimisation stay as they are and
// pass their corrected poses in.
#pragma once
#include <vector>

#include <eigen3/Eigen/Dense>
#include <opencv2/opencv.hpp>

#include "gf_b200.h"

class DenseMap
{
  public:
    // COL, ROW, cam0_calib's PINHOLE parameters (fx fy cx cy k1 k2 p1 p2), DEPTH_DIST, DEPTH_BOUNDARY, qic / tic
    DenseMap(int col, int row, const double pinhole[8], int depth_dist, int depth_boundary, const Eigen::Matrix3d &qic, const Eigen::Vector3d &tic,
             int max_points, int max_keyframes, int device = 0);
    ~DenseMap();
    DenseMap(const DenseMap &) = delete;
    DenseMap &operator=(const DenseMap &) = delete;

    // the node's sampling loop on image (RGB8) and depth (16UC1, mm), then addKeyFrame's octree block with the pose after drift
    // correction (R = r_drift * R; P = r_drift * P + t_drift): returns the keyframe's point_rgbd as the reference leaves it
    // (compacted to the inserted points)
    std::vector<Eigen::Matrix<float, 6, 1>> addKeyFrame(const Eigen::Matrix3d &R, const Eigen::Vector3d &P, const cv::Mat &image, const cv::Mat &depth);
    // updatePath's octree block: every keyframe's corrected pose (getPose after optimize4DoF / optimize6DoF) in keyframelist order
    void updatePath(const std::vector<Eigen::Matrix3d> &R, const std::vector<Eigen::Vector3d> &P);
    // what pub_octree publishes (cloud_filtered; idx: each point's index in the cloud) and save_cloud
    void filtered(std::vector<float> &xyz, std::vector<unsigned char> &rgb, std::vector<int32_t> &idx) const;
    void cloud(std::vector<float> &xyz, std::vector<unsigned char> &rgb) const;

  private:
    gf_dense_map *m_ = nullptr;
};
