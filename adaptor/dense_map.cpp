#include "dense_map.h"

#include <cstdio>
#include <cstdlib>

static void check(int rc, const char *what)
{
    if (rc == GF_OK) return;
    // the reference has no error path here (PCL throws on allocation failure); there is no CPU fallback behind this path
    std::fprintf(stderr, "gf_b200: %s: %s\n", what, gf_last_error());
    std::abort();
}

static void row_major(const Eigen::Matrix3d &M, double *out)
{
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) out[3 * i + j] = M(i, j);
}

DenseMap::DenseMap(int col, int row, const double pinhole[8], int depth_dist, int depth_boundary, const Eigen::Matrix3d &qic, const Eigen::Vector3d &tic,
                   int max_points, int max_keyframes, int device)
{
    gf_dense_map_cfg c{};
    c.width = col; c.height = row; c.depth_dist = depth_dist; c.depth_boundary = depth_boundary;
    for (int i = 0; i < 8; i++) c.pinhole[i] = pinhole[i];
    row_major(qic, c.ric);
    for (int i = 0; i < 3; i++) c.tic[i] = tic(i);
    c.max_points = max_points; c.max_keyframes = max_keyframes;
    check(gf_dense_map_create(&m_, device, &c), "gf_dense_map_create");
}

DenseMap::~DenseMap() { gf_dense_map_destroy(m_); }

std::vector<Eigen::Matrix<float, 6, 1>> DenseMap::addKeyFrame(const Eigen::Matrix3d &R, const Eigen::Vector3d &P, const cv::Mat &image, const cv::Mat &depth)
{
    double r[9], p[3] = {P(0), P(1), P(2)};
    row_major(R, r);
    int n = 0;
    check(gf_dense_map_add_keyframe(m_, r, p, image.data, image.step, (const uint16_t *)depth.data, depth.step, 0, &n), "gf_dense_map_add_keyframe");
    int n_kf = 0;
    check(gf_dense_map_size(m_, nullptr, nullptr, &n_kf), "gf_dense_map_size");
    std::vector<float> flat(6 * (size_t)n);
    check(gf_dense_map_keyframe_points(m_, n_kf - 1, flat.data(), &n), "gf_dense_map_keyframe_points");
    std::vector<Eigen::Matrix<float, 6, 1>> out(n);
    for (int i = 0; i < n; i++) for (int k = 0; k < 6; k++) out[i](k) = flat[6 * (size_t)i + k];
    return out;
}

void DenseMap::updatePath(const std::vector<Eigen::Matrix3d> &R, const std::vector<Eigen::Vector3d> &P)
{
    std::vector<double> r(9 * R.size()), p(3 * P.size());
    for (size_t k = 0; k < R.size(); k++) row_major(R[k], &r[9 * k]);
    for (size_t k = 0; k < P.size(); k++) for (int i = 0; i < 3; i++) p[3 * k + i] = P[k](i);
    check(gf_dense_map_update_poses(m_, (int)R.size(), r.data(), p.data()), "gf_dense_map_update_poses");
}

void DenseMap::filtered(std::vector<float> &xyz, std::vector<unsigned char> &rgb, std::vector<int32_t> &idx) const
{
    int n = 0;
    check(gf_dense_map_size(m_, nullptr, &n, nullptr), "gf_dense_map_size");
    xyz.resize(3 * (size_t)n); rgb.resize(3 * (size_t)n); idx.resize(n);
    check(gf_dense_map_read(m_, GF_DENSE_MAP_FILTERED, xyz.data(), rgb.data(), idx.data()), "gf_dense_map_read");
}

void DenseMap::cloud(std::vector<float> &xyz, std::vector<unsigned char> &rgb) const
{
    int n = 0;
    check(gf_dense_map_size(m_, &n, nullptr, nullptr), "gf_dense_map_size");
    xyz.resize(3 * (size_t)n); rgb.resize(3 * (size_t)n);
    check(gf_dense_map_read(m_, GF_DENSE_MAP_CLOUD, xyz.data(), rgb.data(), nullptr), "gf_dense_map_read");
}
