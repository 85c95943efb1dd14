/* oracle/camera_oracle.c -- CPU restatement of the reference's lens model (OpenCV's radial-tangential k1 k2 p1 p2).
 *
 * TEST INFRASTRUCTURE ONLY (see alva_oracle.c's header).  The product's own statement is alvaar_b200/csrc/camera_model.h; this
 * file is written separately from it so that the tests can hold the two against each other and against the reference.
 *
 * Reference (paths under /root/reference):
 *   CameraCalibration::undistortImagePoint     src/slam/src/camera_calibration.cpp:57-72  cv::undistortPoints(pts, out, K, D, K)
 *   CameraCalibration::projectCamToImageDist   src/slam/src/camera_calibration.cpp:34-55  cv::projectPoints(Point3f, 0, 0, K, D)
 *   cvUndistortPointsInternal                  src/libs/opencv/modules/calib3d/src/undistort.dispatch.cpp:384-556
 *       TermCriteria(COUNT, 5, 0.01) :574 -> exactly 5 iterations, the error test (:509-532) never runs; RR = K (matR = K, no P)
 *   cvProjectPoints2Internal                   src/libs/opencv/modules/calib3d/src/calibration.cpp:526-810 (loop :774-809),
 *       R = Rodrigues(0) = identity (:311-313), t = 0; the double results rounded to float by cvConvert (:1010)
 * The reference's D_ is an Eigen::Vector4d, its cv::Mat never empty: these paths run even with zero coefficients.
 * OpenCV's 14-entry k[] is kept (entries 4..13 zero, still multiplied in), as are its identity matrix products, which Matx
 * accumulates from s = 0 (core/include/opencv2/core/matx.hpp:860-870).
 * PINNED: tests/test_oracle_distortion.py (golden + live reference): bit-identical float outputs.
 */
#include <math.h>
#include <stdint.h>

/* Matx33d::eye() * (a, b, 1), row r */
static double eye_row(int r, double a, double b)
{
    const double e[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    const double v[3] = {a, b, 1};
    double s = 0;
    for (int k = 0; k < 3; k++) s += e[r][k] * v[k];
    return s;
}

static void undistort_one(const double* K4, const double* D4, float pu, float pv, float* out)
{
    double k[14] = {0};
    for (int i = 0; i < 4; i++) k[i] = D4[i];
    const double A[3][3] = {{K4[0], 0, K4[2]}, {0, K4[1], K4[3]}, {0, 0, 1}};
    const double RR[3][3] = {{K4[0], 0, K4[2]}, {0, K4[1], K4[3]}, {0, 0, 1}};   /* matR = K (:438-442) */
    const double fx = A[0][0], fy = A[1][1], ifx = 1. / fx, ify = 1. / fy, cx = A[0][2], cy = A[1][2];   /* :458-463 */
    double x = pu, y = pv, x0, y0, u, v;                                                                  /* :467-479 */
    u = x; v = y;
    x = (x - cx) * ifx;
    y = (y - cy) * ify;
    {   /* :482-486 */
        const double t0 = eye_row(0, x, y), t1 = eye_row(1, x, y), t2 = eye_row(2, x, y);
        const double invProj = t2 ? 1. / t2 : 1;
        x0 = x = invProj * t0;
        y0 = y = invProj * t1;
    }
    for (int j = 0; j < 5; j++) {   /* :490-507 */
        double r2 = x * x + y * y;
        double icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
        if (icdist < 0) {
            x = (u - cx) * ifx;
            y = (v - cy) * ify;
            break;
        }
        double deltaX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2;
        double deltaY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2;
        x = (x0 - deltaX) * icdist;
        y = (y0 - deltaY) * icdist;
    }
    {   /* :539-543 */
        double xx = RR[0][0] * x + RR[0][1] * y + RR[0][2];
        double yy = RR[1][0] * x + RR[1][1] * y + RR[1][2];
        double ww = 1. / (RR[2][0] * x + RR[2][1] * y + RR[2][2]);
        x = xx * ww;
        y = yy * ww;
    }
    out[0] = (float)x;   /* :545-549 */
    out[1] = (float)y;
}

/* CameraCalibration::projectCamToImageDist of one camera-frame point */
void orc_project_cam_dist(const double* K4, const double* D4, const double* p, float* out)
{
    double k[14] = {0};
    for (int i = 0; i < 4; i++) k[i] = D4[i];
    const double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0, 0, 0};
    const double fx = K4[0], fy = K4[1], cx = K4[2], cy = K4[3];
    /* camera_calibration.cpp:36-46: double x = p.x / z, y = p.y / z -> cv::Point3f(x, y, 1.0) -> cvConvert to double (:573) */
    const double inverseZ = 1. / p[2];
    const float fX = (float)(p[0] * inverseZ), fY = (float)(p[1] * inverseZ), fZ = (float)1.0;
    const double X = fX, Y = fY, Z = fZ;
    double x = R[0] * X + R[1] * Y + R[2] * Z + t[0];   /* :777-779 */
    double y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    z = z ? 1. / z : 1;   /* :788-789 */
    x *= z; y *= z;
    const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;   /* :791-801 */
    const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
    const double cdist = 1 + k[0] * r2 + k[1] * r4 + k[4] * r6;
    const double icdist2 = 1. / (1 + k[5] * r2 + k[6] * r4 + k[7] * r6);
    const double xd0 = x * cdist * icdist2 + k[2] * a1 + k[3] * a2 + k[8] * r2 + k[9] * r4;
    const double yd0 = y * cdist * icdist2 + k[2] * a3 + k[3] * a1 + k[10] * r2 + k[11] * r4;
    const double v0 = eye_row(0, xd0, yd0), v1 = eye_row(1, xd0, yd0), v2 = eye_row(2, xd0, yd0);   /* :803-806 */
    const double invProj = v2 ? 1. / v2 : 1;
    const double xd = invProj * v0, yd = invProj * v1;
    out[0] = (float)(xd * fx + cx);   /* :808-809, :1010 */
    out[1] = (float)(yd * fy + cy);
}

/* px [n][2] -> unpx [n][2] */
void orc_undistort_points(const float* px, int n, const double* K4, const double* D4, float* unpx)
{
    for (int i = 0; i < n; i++) undistort_one(K4, D4, px[2 * i], px[2 * i + 1], unpx + 2 * i);
}

/* Xc [n][3] camera-frame points -> uv [n][2] */
void orc_project_points(const double* Xc, int n, const double* K4, const double* D4, float* uv)
{
    for (int i = 0; i < n; i++) orc_project_cam_dist(K4, D4, Xc + 3 * i, uv + 2 * i);
}
