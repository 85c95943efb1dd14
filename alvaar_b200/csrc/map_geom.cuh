// map_geom.cuh -- the device geometry of the map matchers (match.cu: the local map against a keyframe; reacquire.cu: the frozen
// map against a tracked frame's fresh detections).  One copy, so that both gate map points on the same bits:
//   quat_R / world_to_cam   Frame::projWorldToCam (src/slam/src/frame.cpp:447-467): Tcw * X with Tcw = Twc.inverse(), the
//                           rotation from the NORMALISED quaternion (Eigen's toRotationMatrix)
//   project_cam<LENS>       CameraCalibration::projectCamToImageDist (camera_calibration.cpp:34-55): the pinhole through a
//                           cv::Point3f, or the lens models of camera_model.h
// Bit-exact only without FMA contraction: the including files compile with -fmad=false.
#pragma once
#include "camera_model.h"

namespace alva_geom {

// LENS_NONE: the zero-distortion projection; LENS_RADTAN / LENS_FISHEYE: the lens models of camera_model.h (Camera::Lens values)
enum { LENS_NONE = 0, LENS_RADTAN = 1, LENS_FISHEYE = 2 };

__device__ __forceinline__ void quat_R(const double* q, double* R) {
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
// Twc = [t, q(x, y, z, w)]
__device__ __forceinline__ void world_to_cam(const double* Twc, const double* X, double* c) {
    double R[9], ti[3];
    quat_R(Twc + 3, R);
#pragma unroll
    for (int i = 0; i < 3; i++) ti[i] = -(R[i] * Twc[0] + R[3 + i] * Twc[1] + R[6 + i] * Twc[2]);
#pragma unroll
    for (int i = 0; i < 3; i++) c[i] = (R[i] * X[0] + R[3 + i] * X[1] + R[6 + i] * X[2]) + ti[i];
}
// K4 = {fx, fy, cx, cy}; D4: the lens coefficients (unused for LENS_NONE)
template <int LENS>
__device__ __forceinline__ void project_cam(const double* K4, const double* D4, const double* c, float* px) {
    if constexpr (LENS == LENS_RADTAN) {
        alva_cam::project_dist(K4, D4, c, px);
    } else if constexpr (LENS == LENS_FISHEYE) {
        alva_cam::project_dist_fisheye(K4, D4, c, px);
    } else {
        const double iz = 1. / c[2];
        const double x = (double)(float)(c[0] * iz), y = (double)(float)(c[1] * iz);   // cv::Point3f(x, y, 1.0)
        px[0] = (float)(x * K4[0] + K4[2]);
        px[1] = (float)(y * K4[1] + K4[3]);
    }
}

}  // namespace alva_geom
