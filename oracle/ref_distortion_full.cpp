// oracle/ref_distortion_full.cpp -- TEST INFRASTRUCTURE ONLY (never on the product path).
//
// The reference's vendored OpenCV 4.5.5 (built by oracle/build_ref.sh, linked by oracle/build_ref_distortion_full.sh into
// oracle/_ref/libalva_ref_distortion_full.so) behind a C ABI, called exactly as the reference's CameraCalibration calls the lens
// (camera_calibration.cpp:34-72), with OpenCV's whole distortion vector in place of its four coefficients:
//   ref_full_undistort_points  cv::undistortPoints(pt, out, K, D, K) of every float pixel px [n][2]
//   ref_full_project_points    cv::projectPoints of cv::Point3f(x / z, y / z, 1) for every camera point Xc [n][3], zero rvec /
//                              tvec (CV_32F, as CameraCalibration passes them)
// K4 = {fx, fy, cx, cy} becomes a 3x3 CV_64F Mat and coeffs [ncoeffs] (5, 8, 12 or 14 entries) an ncoeffs x 1 CV_64F Mat.  Each
// call also runs OpenCV on the same values as CV_64F points, which gives the double each float result was rounded from (out64,
// may be NULL): the tests use it to tell a rounding-boundary case from a real difference.
#include <opencv2/calib3d.hpp>
#include <opencv2/core.hpp>
#include <vector>

namespace {
void mats(const double* K4, const double* coeffs, int ncoeffs, cv::Mat& K, cv::Mat& D) {
    K = (cv::Mat_<double>(3, 3) << K4[0], 0., K4[2], 0., K4[1], K4[3], 0., 0., 1.);
    D = cv::Mat(ncoeffs, 1, CV_64F);
    for (int i = 0; i < ncoeffs; i++) D.at<double>(i) = coeffs[i];
}
}  // namespace

extern "C" {

void ref_full_undistort_points(const float* px, int n, const double* K4, const double* coeffs, int ncoeffs, float* out32, double* out64) {
    cv::Mat K, D;
    mats(K4, coeffs, ncoeffs, K, D);
    for (int i = 0; i < n; i++) {
        std::vector<cv::Point2f> pt{cv::Point2f(px[2 * i], px[2 * i + 1])}, out;
        cv::undistortPoints(pt, out, K, D, K);
        out32[2 * i] = out[0].x;
        out32[2 * i + 1] = out[0].y;
        if (out64) {
            std::vector<cv::Point2d> pd{cv::Point2d(px[2 * i], px[2 * i + 1])}, od;
            cv::undistortPoints(pd, od, K, D, K);
            out64[2 * i] = od[0].x;
            out64[2 * i + 1] = od[0].y;
        }
    }
}

void ref_full_project_points(const double* Xc, int n, const double* K4, const double* coeffs, int ncoeffs, float* out32, double* out64) {
    cv::Mat K, D;
    mats(K4, coeffs, ncoeffs, K, D);
    const cv::Mat R = cv::Mat::zeros(3, 1, CV_32F);
    for (int i = 0; i < n; i++) {
        const double inverseZ = 1. / Xc[3 * i + 2];
        const double x = Xc[3 * i] * inverseZ, y = Xc[3 * i + 1] * inverseZ;
        const cv::Point3f p(x, y, 1.0);
        std::vector<cv::Point3f> v{p};
        std::vector<cv::Point2f> out;
        cv::projectPoints(v, R, R, K, D, out);
        out32[2 * i] = out[0].x;
        out32[2 * i + 1] = out[0].y;
        if (out64) {
            std::vector<cv::Point3d> vd{cv::Point3d(p.x, p.y, p.z)};
            std::vector<cv::Point2d> od;
            cv::projectPoints(vd, R, R, K, D, od);
            out64[2 * i] = od[0].x;
            out64[2 * i + 1] = od[0].y;
        }
    }
}

}  // extern "C"
