// oracle/ref_camera.cpp -- TEST INFRASTRUCTURE ONLY (never on the product path).
//
// The reference's own CameraCalibration (src/slam/src/camera_calibration.cpp, compiled unmodified with the reference's OpenCV
// 4.5.5 by oracle/build_ref_camera.sh into oracle/_ref/libalva_ref_camera.so) behind a C ABI, one object per call:
//   ref_undistort_points  CameraCalibration::undistortImagePoint of every pixel px [n][2]   (what Frame::computeKeypoint calls)
//   ref_project_points    CameraCalibration::projectCamToImageDist of every camera point Xc [n][3]
// K4 = {fx, fy, cx, cy}, D4 = {k1, k2, p1, p2}: the arguments System::configure hands to it (system.cpp:13-40).
#include "camera_calibration.hpp"
#include <cstdint>

extern "C" {

void ref_undistort_points(const float* px, int n, const double* K4, const double* D4, int w, int h, float* unpx) {
    const CameraCalibration cam(K4[0], K4[1], K4[2], K4[3], D4[0], D4[1], D4[2], D4[3], w, h, 20);
    for (int i = 0; i < n; i++) {
        const cv::Point2f p = cam.undistortImagePoint(cv::Point2f(px[2 * i], px[2 * i + 1]));
        unpx[2 * i] = p.x;
        unpx[2 * i + 1] = p.y;
    }
}

void ref_project_points(const double* Xc, int n, const double* K4, const double* D4, int w, int h, float* uv) {
    const CameraCalibration cam(K4[0], K4[1], K4[2], K4[3], D4[0], D4[1], D4[2], D4[3], w, h, 20);
    for (int i = 0; i < n; i++) {
        const cv::Point2f p = cam.projectCamToImageDist(Eigen::Vector3d(Xc[3 * i], Xc[3 * i + 1], Xc[3 * i + 2]));
        uv[2 * i] = p.x;
        uv[2 * i + 1] = p.y;
    }
}

}  // extern "C"
