// camera_model.h -- the radial-tangential lens model (k1, k2, p1, p2) of the reference's CameraCalibration, in one place for
// the host state machine (system_core.h), the kernels (camera.cu, match.cu) and the CPU System backend of the test suite.
//
// The reference stores its coefficients as an Eigen::Vector4d, so its cv::Mat copy is never empty and it always runs OpenCV
// (src/slam/src/camera_calibration.cpp:34-72):
//   undistort_point  CameraCalibration::undistortImagePoint -> cv::undistortPoints(pt, out, K, D, K)
//                    = cvUndistortPointsInternal (opencv calib3d/src/undistort.dispatch.cpp:384-556) with
//                    TermCriteria(COUNT, 5, 0.01) (:574): exactly 5 iterations, no error test; R = K and no P, so RR = K and the
//                    result stays in pixels
//   project_dist     CameraCalibration::projectCamToImageDist -> cv::projectPoints of the FLOAT point (x/z, y/z, 1) with zero
//                    rvec / tvec = cvProjectPoints2Internal (opencv calib3d/src/calibration.cpp:526-810, distortion :780-803)
// Both are restated in OpenCV's expression order, with its 14-coefficient array (the 10 unused entries are zeros that still
// take part in the arithmetic: 0 * inf is NaN, -0 + 0 is +0) and its identity tilt and rotation matrices multiplied out as
// Matx::operator* accumulates (s = 0; s += a(i, k) * b(k), core/matx.hpp:860-870).  Bit-exact only without FMA contraction:
// device users compile with -fmad=false, host users with -ffp-contract=off.
//
// Both take K4 = {fx, fy, cx, cy} and D4 = {k1, k2, p1, p2}.
#pragma once

#if defined(__CUDACC__)
#define ALVA_CAM_FN __host__ __device__ inline
#else
#define ALVA_CAM_FN inline
#endif

namespace alva_cam {

// out = cv::undistortPoints of the float pixel (u, v), rounded to float
ALVA_CAM_FN void undistort_point(const double* K4, const double* D4, float u_in, float v_in, float* out) {
    const double k[14] = {D4[0], D4[1], D4[2], D4[3], 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    const double fx = K4[0], fy = K4[1], cx = K4[2], cy = K4[3];
    const double ifx = 1. / fx, ify = 1. / fy;
    double x = u_in, y = v_in;
    const double u = x, v = y;
    x = (x - cx) * ifx;
    y = (y - cy) * ify;
    // invMatTilt (identity) * (x, y, 1)                                                                            :482-486
    const double t0 = ((0. + 1. * x) + 0. * y) + 0. * 1.;
    const double t1 = ((0. + 0. * x) + 1. * y) + 0. * 1.;
    const double t2 = ((0. + 0. * x) + 0. * y) + 1. * 1.;
    const double invProj = t2 ? 1. / t2 : 1;
    const double x0 = x = invProj * t0;
    const double y0 = y = invProj * t1;
    for (int j = 0; j < 5; j++) {                                                                                   // :490-507
        const double r2 = x * x + y * y;
        const double icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
        if (icdist < 0) {   // the model folds back at this radius: the plain pinhole point               :498-503
            x = (u - cx) * ifx;
            y = (v - cy) * ify;
            break;
        }
        const double deltaX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2;
        const double deltaY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2;
        x = (x0 - deltaX) * icdist;
        y = (y0 - deltaY) * icdist;
    }
    // RR = K                                                                                                       :539-543
    const double xx = fx * x + 0. * y + cx;
    const double yy = 0. * x + fy * y + cy;
    const double ww = 1. / (0. * x + 0. * y + 1.);
    out[0] = (float)(xx * ww);
    out[1] = (float)(yy * ww);
}

// out = cv::projectPoints of the camera-frame point p through cv::Point3f(p.x / p.z, p.y / p.z, 1), rounded to float
ALVA_CAM_FN void project_dist(const double* K4, const double* D4, const double* p, float* out) {
    const double k[14] = {D4[0], D4[1], D4[2], D4[3], 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    const double fx = K4[0], fy = K4[1], cx = K4[2], cy = K4[3];
    const double inverseZ = 1. / p[2];
    const double X = (float)(p[0] * inverseZ), Y = (float)(p[1] * inverseZ), Z = 1.0f;   // camera_calibration.cpp:36-46
    // R = Rodrigues(0) = identity, t = 0                                                                           :777-779
    double x = 1. * X + 0. * Y + 0. * Z + 0.;
    double y = 0. * X + 1. * Y + 0. * Z + 0.;
    double z = 0. * X + 0. * Y + 1. * Z + 0.;
    z = z ? 1. / z : 1;                                                                                             // :786-789
    x *= z; y *= z;
    const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;                                                    // :791-801
    const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
    const double cdist = 1 + k[0] * r2 + k[1] * r4 + k[4] * r6;
    const double icdist2 = 1. / (1 + k[5] * r2 + k[6] * r4 + k[7] * r6);
    const double xd0 = x * cdist * icdist2 + k[2] * a1 + k[3] * a2 + k[8] * r2 + k[9] * r4;
    const double yd0 = y * cdist * icdist2 + k[2] * a3 + k[3] * a1 + k[10] * r2 + k[11] * r4;
    // matTilt (identity) * (xd0, yd0, 1)                                                                           :803-806
    const double t0 = ((0. + 1. * xd0) + 0. * yd0) + 0. * 1.;
    const double t1 = ((0. + 0. * xd0) + 1. * yd0) + 0. * 1.;
    const double t2 = ((0. + 0. * xd0) + 0. * yd0) + 1. * 1.;
    const double invProj = t2 ? 1. / t2 : 1;
    const double xd = invProj * t0, yd = invProj * t1;
    out[0] = (float)(xd * fx + cx);                                                                                 // :808-809, :1010
    out[1] = (float)(yd * fy + cy);
}

}  // namespace alva_cam
