// oracle/ref_fisheye.cpp -- TEST INFRASTRUCTURE ONLY (never on the product path).
//
// OpenCV's own equidistant fisheye model (cv::fisheye in the reference's vendored OpenCV 4.5.5, built by oracle/build_ref.sh and
// linked by oracle/build_ref_fisheye.sh into oracle/_ref/libalva_ref_fisheye.so) behind a C ABI, called the way System calls
// the lens where the reference's CameraCalibration calls cv::undistortPoints / cv::projectPoints (camera_calibration.cpp:34-72):
//   ref_fisheye_undistort_points  cv::fisheye::undistortPoints(pt, out, K, D, noArray(), K) of every float pixel px [n][2]
//   ref_fisheye_project_points    cv::fisheye::projectPoints of cv::Point3f(x / z, y / z, 1) for every camera point Xc [n][3],
//                                 zero rvec / tvec (CV_32F, as CameraCalibration passes them), alpha = 0
// K4 = {fx, fy, cx, cy} and D4 = {k1, k2, k3, k4} become a 3x3 and a 4x1 CV_64F Mat, as CameraCalibration's eigen2cv copies are.
// Each call also runs OpenCV once more on the same values as CV_64F points, which gives the double each float result was
// rounded from (out64, may be NULL): the tests use it to tell a rounding-boundary case from a real difference.
#include <opencv2/calib3d.hpp>
#include <opencv2/core.hpp>
#include <vector>

namespace {
void mats(const double* K4, const double* D4, cv::Mat& K, cv::Mat& D) {
    K = (cv::Mat_<double>(3, 3) << K4[0], 0., K4[2], 0., K4[1], K4[3], 0., 0., 1.);
    D = (cv::Mat_<double>(4, 1) << D4[0], D4[1], D4[2], D4[3]);
}
}  // namespace

extern "C" {

void ref_fisheye_undistort_points(const float* px, int n, const double* K4, const double* D4, float* out32, double* out64) {
    cv::Mat K, D;
    mats(K4, D4, K, D);
    for (int i = 0; i < n; i++) {
        std::vector<cv::Point2f> pt{cv::Point2f(px[2 * i], px[2 * i + 1])}, out;
        cv::fisheye::undistortPoints(pt, out, K, D, cv::noArray(), K);
        out32[2 * i] = out[0].x;
        out32[2 * i + 1] = out[0].y;
        if (out64) {
            std::vector<cv::Point2d> pd{cv::Point2d(px[2 * i], px[2 * i + 1])}, od;
            cv::fisheye::undistortPoints(pd, od, K, D, cv::noArray(), K);
            out64[2 * i] = od[0].x;
            out64[2 * i + 1] = od[0].y;
        }
    }
}

void ref_fisheye_project_points(const double* Xc, int n, const double* K4, const double* D4, float* out32, double* out64) {
    cv::Mat K, D;
    mats(K4, D4, K, D);
    const cv::Mat R = cv::Mat::zeros(3, 1, CV_32F);
    for (int i = 0; i < n; i++) {
        const double inverseZ = 1. / Xc[3 * i + 2];
        const double x = Xc[3 * i] * inverseZ, y = Xc[3 * i + 1] * inverseZ;
        const cv::Point3f p(x, y, 1.0);
        std::vector<cv::Point3f> v{p};
        std::vector<cv::Point2f> out;
        cv::fisheye::projectPoints(v, out, R, R, K, D, 0.0);
        out32[2 * i] = out[0].x;
        out32[2 * i + 1] = out[0].y;
        if (out64) {
            std::vector<cv::Point3d> vd{cv::Point3d(p.x, p.y, p.z)};
            std::vector<cv::Point2d> od;
            cv::fisheye::projectPoints(vd, od, R, R, K, D, 0.0);
            out64[2 * i] = od[0].x;
            out64[2 * i + 1] = od[0].y;
        }
    }
}

}  // extern "C"
