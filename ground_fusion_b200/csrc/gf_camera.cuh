// gf_camera.cuh -- camodocal's PINHOLE camera (camera_models/src/camera_models/PinholeCamera.cc), shared by the front end
// (fe_tracker.cu) and the dense map (dm_map.cu).  Both build with -fmad=false: every product and sum rounds separately, as
// the reference's double arithmetic does without FMA contraction.
#pragma once
#include "gf_common.cuh"

namespace gf {

struct CamParams { double fx, fy, cx, cy, k1, k2, p1, p2; int no_distortion; };

// pinhole[8] = fx fy cx cy k1 k2 p1 p2 (gf_tracker_cfg / gf_dense_map_cfg)
inline CamParams make_cam(const double* p)
{
    CamParams c;
    c.fx = p[0]; c.fy = p[1]; c.cx = p[2]; c.cy = p[3]; c.k1 = p[4]; c.k2 = p[5]; c.p1 = p[6]; c.p2 = p[7];
    c.no_distortion = (p[4] == 0.0 && p[5] == 0.0 && p[6] == 0.0 && p[7] == 0.0);
    return c;
}

__device__ __forceinline__ void cam_distortion(const CamParams& c, double x, double y, double& dx, double& dy)
{   // PinholeCamera::distortion, camera_models/src/camera_models/PinholeCamera.cc:646-662
    double mx2 = x * x, my2 = y * y, mxy = x * y;
    double rho2 = mx2 + my2;
    double rad = c.k1 * rho2 + c.k2 * rho2 * rho2;
    dx = x * rad + 2.0 * c.p1 * mxy + c.p2 * (rho2 + 2.0 * mx2);
    dy = y * rad + 2.0 * c.p2 * mxy + c.p1 * (rho2 + 2.0 * my2);
}
__device__ __forceinline__ void cam_lift(const CamParams& c, double u, double v, double& ox, double& oy)
{   // PinholeCamera::liftProjective, PinholeCamera.cc:450-510 (recursive distortion model, n = 8)
    double ik11 = 1.0 / c.fx, ik13 = -c.cx / c.fx, ik22 = 1.0 / c.fy, ik23 = -c.cy / c.fy;
    double mx_d = ik11 * u + ik13, my_d = ik22 * v + ik23;
    if (c.no_distortion) { ox = mx_d; oy = my_d; return; }
    double dx, dy;
    cam_distortion(c, mx_d, my_d, dx, dy);
    double mx_u = mx_d - dx, my_u = my_d - dy;
    for (int i = 1; i < 8; i++) {
        cam_distortion(c, mx_u, my_u, dx, dy);
        mx_u = mx_d - dx;
        my_u = my_d - dy;
    }
    ox = mx_u; oy = my_u;
}
__device__ __forceinline__ void cam_project(const CamParams& c, double X, double Y, double Z, double& u, double& v)
{   // PinholeCamera::spaceToPlane, PinholeCamera.cc:520-541
    double x = X / Z, y = Y / Z;
    if (!c.no_distortion) { double dx, dy; cam_distortion(c, x, y, dx, dy); x = x + dx; y = y + dy; }
    u = c.fx * x + c.cx;
    v = c.fy * y + c.cy;
}

}  // namespace gf
