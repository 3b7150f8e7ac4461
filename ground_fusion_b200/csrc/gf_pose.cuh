// gf_pose.cuh -- a keyframe point carried into the world frame, shared by the dense map (dm_map.cu) and the occupancy grid
// (gm_grid.cu).  Both build with -fmad=false: every product and sum rounds separately, as Eigen's double products do without
// FMA contraction.
#pragma once
#include "gf_common.cuh"

namespace gf {

struct Pose { double R[9], P[3]; };                // row-major R; world = R x + P
struct Ext { double ric[9], tic[3]; };             // camera to body

__device__ __forceinline__ void mv3(const double* M, const double* x, double* y)
{   // Eigen's Matrix3d * Vector3d without FMA: ((m0 x0 + m1 x1) + m2 x2) per row
    const double y0 = M[0] * x[0] + M[1] * x[1] + M[2] * x[2];
    const double y1 = M[3] * x[0] + M[4] * x[1] + M[5] * x[2];
    const double y2 = M[6] * x[0] + M[7] * x[1] + M[8] * x[2];
    y[0] = y0; y[1] = y1; y[2] = y2;
}
// pointWorld = R * (qic * point + tic) + P of a float camera-frame point promoted to double (dense_map pose_graph.cpp:197,
// grid_mapping main.cpp:114-119)
__device__ __forceinline__ void to_world(const Ext& e, const Pose& T, const float* l, double* w)
{
    const double p[3] = {(double)l[0], (double)l[1], (double)l[2]};
    double a[3], b[3];
    mv3(e.ric, p, a);
    for (int k = 0; k < 3; k++) a[k] = a[k] + e.tic[k];
    mv3(T.R, a, b);
    for (int k = 0; k < 3; k++) w[k] = b[k] + T.P[k];
}

}  // namespace gf
