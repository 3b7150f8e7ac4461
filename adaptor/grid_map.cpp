#include "grid_map.h"

#include <cstdio>
#include <cstdlib>

static void check(int rc, const char *what)
{
    if (rc == GF_OK) return;
    // the reference tool has no error path here; there is no CPU fallback behind this path
    std::fprintf(stderr, "gf_b200: %s: %s\n", what, gf_last_error());
    std::abort();
}

static void row_major(const Eigen::Matrix3d &M, double *out)
{
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) out[3 * i + j] = M(i, j);
}

GridMapper::GridMapper(const Eigen::Matrix3d &qic, const Eigen::Vector3d &tic, int size_x, int size_y, int init_x, int init_y, double cell_size,
                       double p_occ, double p_free, double p_prior, int max_points, int max_keyframes, int max_records, int device)
{
    gf_grid_map_cfg c{};
    c.size_x = size_x; c.size_y = size_y; c.init_x = init_x; c.init_y = init_y; c.cell_size = cell_size;
    c.p_occ = p_occ; c.p_free = p_free; c.p_prior = p_prior;
    row_major(qic, c.ric);
    for (int i = 0; i < 3; i++) c.tic[i] = tic(i);
    c.max_points = max_points; c.max_keyframes = max_keyframes; c.max_records = max_records;
    check(gf_grid_map_create(&m_, device, &c), "gf_grid_map_create");
    cells_ = (size_t)size_x * size_y;
}

GridMapper::~GridMapper() { gf_grid_map_destroy(m_); }

void GridMapper::addKeyFrame(const Eigen::Matrix3d &R, const Eigen::Vector3d &P, const std::vector<Eigen::Matrix<float, 6, 1>> &point_rgbd)
{
    double r[9], p[3] = {P(0), P(1), P(2)};
    row_major(R, r);
    std::vector<float> flat(6 * point_rgbd.size());
    for (size_t i = 0; i < point_rgbd.size(); i++) for (int k = 0; k < 6; k++) flat[6 * i + k] = point_rgbd[i](k);
    check(gf_grid_map_add_keyframe(m_, r, p, flat.data(), (int)point_rgbd.size(), 6, 0), "gf_grid_map_add_keyframe");
}

void GridMapper::updatePath(const std::vector<Eigen::Matrix3d> &R, const std::vector<Eigen::Vector3d> &P)
{
    std::vector<double> r(9 * R.size()), p(3 * P.size());
    for (size_t k = 0; k < R.size(); k++) row_major(R[k], &r[9 * k]);
    for (size_t k = 0; k < P.size(); k++) for (int i = 0; i < 3; i++) p[3 * k + i] = P[k](i);
    check(gf_grid_map_update_poses(m_, (int)R.size(), r.data(), p.data()), "gf_grid_map_update_poses");
}

std::vector<double> GridMapper::bel() const
{
    std::vector<double> out(cells_);
    check(gf_grid_map_read(m_, GF_GRID_MAP_BEL, out.data()), "gf_grid_map_read");
    return out;
}

std::vector<uint8_t> GridMapper::image() const
{
    std::vector<uint8_t> out(cells_);
    check(gf_grid_map_read(m_, GF_GRID_MAP_IMAGE, out.data()), "gf_grid_map_read");
    return out;
}

std::vector<int8_t> GridMapper::occupancy() const
{
    std::vector<int8_t> out(cells_);
    check(gf_grid_map_read(m_, GF_GRID_MAP_OCCUPANCY, out.data()), "gf_grid_map_read");
    return out;
}
