// GridMapper: the occupancy grid of the reference's grid_mapping tool on libgf_b200.so.  It replaces the tool's GridMap and
// GridMapper (support_files/grid_mapping/grid_map.cpp, grid_mapper.cpp) and the per-keyframe body of main.cpp's loop (:114-120):
// each keyframe's point_rgbd with its corrected pose goes in as it is saved, and the grid is kept online instead of being built
// after the run.  updatePath re-applies every keyframe with new poses, as running the tool again over a new pose_graph.txt does.
#pragma once
#include <cstdint>
#include <vector>

#include <eigen3/Eigen/Dense>

#include "gf_b200.h"

class GridMapper
{
  public:
    // qic / tic: camera to body; the grid (size_x, size_y, init_x, init_y, cell_size) and P_occ, P_free, P_prior as the tool's
    // GridMap and GridMapper constructors take them
    GridMapper(const Eigen::Matrix3d &qic, const Eigen::Vector3d &tic, int size_x, int size_y, int init_x, int init_y, double cell_size,
               double p_occ, double p_free, double p_prior, int max_points, int max_keyframes, int max_records, int device = 0);
    ~GridMapper();
    GridMapper(const GridMapper &) = delete;
    GridMapper &operator=(const GridMapper &) = delete;

    // main.cpp's loop body for one keyframe: PG_R, PG_T and its point_rgbd
    void addKeyFrame(const Eigen::Matrix3d &R, const Eigen::Vector3d &P, const std::vector<Eigen::Matrix<float, 6, 1>> &point_rgbd);
    // every keyframe's corrected pose in the order they were added
    void updatePath(const std::vector<Eigen::Matrix3d> &R, const std::vector<Eigen::Vector3d> &P);
    // bel_data_ (column-major, size_x * size_y); the pixels saveMap writes to map.png (size_x rows of size_y); the OccupancyGrid
    // data the mapping node publishes from that image
    std::vector<double> bel() const;
    std::vector<uint8_t> image() const;
    std::vector<int8_t> occupancy() const;

  private:
    gf_grid_map *m_ = nullptr;
    size_t cells_ = 0;
};
