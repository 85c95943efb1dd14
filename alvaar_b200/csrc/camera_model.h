// camera_model.h -- the radial-tangential lens model (k1, k2, p1, p2) of the reference's CameraCalibration, OpenCV's full
// 14-coefficient form of it (k3..k6, the thin prism s1..s4 and the tilt tau_x, tau_y) and its fisheye model, in one place for
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
// Both are restated in OpenCV's expression order, with its 14-coefficient array (entries a four-coefficient lens does not use
// are zeros that still take part in the arithmetic: 0 * inf is NaN, -0 + 0 is +0) and its tilt and rotation matrices multiplied out as
// Matx::operator* accumulates (s = 0; s += a(i, k) * b(k), core/matx.hpp:860-870).  Bit-exact only without FMA contraction:
// device users compile with -fmad=false, host users with -ffp-contract=off.
//
// The 14-coefficient forms (undistort_point_full, project_dist_full) take the whole vector and the two tilt matrices, which the
// host builds once per lens (make_lens_full); undistort_point / project_dist take K4 = {fx, fy, cx, cy} and D4 = {k1, k2, p1, p2}
// and call them with ten zeros and the identity.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define ALVA_CAM_FN __host__ __device__ inline
#else
#define ALVA_CAM_FN inline
#endif

namespace alva_cam {

constexpr double kHalfPi = 1.57079632679489661923;   // CV_PI / 2.

// OpenCV's full pinhole distortion vector: k[14] = {k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4, tau_x, tau_y} (the 4-, 5-, 8-
// and 12-entry vectors of cv::calibrateCamera are its prefixes, zero-padded), with the two tilt matrices of
// detail::computeTiltProjectionMatrix (tilt_matrices below, host only) row-major.  Passed by value into the kernels.
struct LensFull {
    double k[14];
    double tilt[9];    // matTilt, what projectPoints applies
    double itilt[9];   // invMatTilt, what undistortPoints applies
};

// out = cv::undistortPoints of the float pixel (u, v), rounded to float; k: the 14 coefficients, invMatTilt: row-major 3x3
ALVA_CAM_FN void undistort_point_full(const double* K4, const double* k, const double* invMatTilt, float u_in, float v_in, float* out) {
    const double* M = invMatTilt;
    const double fx = K4[0], fy = K4[1], cx = K4[2], cy = K4[3];
    const double ifx = 1. / fx, ify = 1. / fy;
    double x = u_in, y = v_in;
    const double u = x, v = y;
    x = (x - cx) * ifx;
    y = (y - cy) * ify;
    // invMatTilt * (x, y, 1)                                                                                       :482-486
    const double t0 = ((0. + M[0] * x) + M[1] * y) + M[2] * 1.;
    const double t1 = ((0. + M[3] * x) + M[4] * y) + M[5] * 1.;
    const double t2 = ((0. + M[6] * x) + M[7] * y) + M[8] * 1.;
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

// out = cv::projectPoints of the camera-frame point p through cv::Point3f(p.x / p.z, p.y / p.z, 1), rounded to float; k: the 14
// coefficients, matTilt: row-major 3x3
ALVA_CAM_FN void project_dist_full(const double* K4, const double* k, const double* matTilt, const double* p, float* out) {
    const double* M = matTilt;
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
    // matTilt * (xd0, yd0, 1)                                                                                      :803-806
    const double t0 = ((0. + M[0] * xd0) + M[1] * yd0) + M[2] * 1.;
    const double t1 = ((0. + M[3] * xd0) + M[4] * yd0) + M[5] * 1.;
    const double t2 = ((0. + M[6] * xd0) + M[7] * yd0) + M[8] * 1.;
    const double invProj = t2 ? 1. / t2 : 1;
    const double xd = invProj * t0, yd = invProj * t1;
    out[0] = (float)(xd * fx + cx);                                                                                 // :808-809, :1010
    out[1] = (float)(yd * fy + cy);
}

// the four-coefficient model: the 14-entry array with ten literal zeros and the literal identity tilt
ALVA_CAM_FN void undistort_point(const double* K4, const double* D4, float u_in, float v_in, float* out) {
    const double k[14] = {D4[0], D4[1], D4[2], D4[3], 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    const double eye[9] = {1., 0., 0., 0., 1., 0., 0., 0., 1.};
    undistort_point_full(K4, k, eye, u_in, v_in, out);
}
ALVA_CAM_FN void project_dist(const double* K4, const double* D4, const double* p, float* out) {
    const double k[14] = {D4[0], D4[1], D4[2], D4[3], 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    const double eye[9] = {1., 0., 0., 0., 1., 0., 0., 0., 1.};
    project_dist_full(K4, k, eye, p, out);
}

// detail::computeTiltProjectionMatrix<double>(tauX, tauY) (imgproc/src/distortion_model.hpp:75-123) for matTilt and invMatTilt,
// in Matx's accumulation order; both the identity unless tau_x or tau_y is non-zero, as cvUndistortPointsInternal and
// cvProjectPoints2Internal build them.  Host only (no __device__): glibc's cos / sin are OpenCV's, the device's round differently.
inline void matx33_mul(const double* a, const double* b, double* c) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int l = 0; l < 3; l++) s += a[3 * i + l] * b[3 * l + j];
            c[3 * i + j] = s;
        }
}
inline void tilt_matrices(double tauX, double tauY, double* matTilt, double* invMatTilt) {
    for (int i = 0; i < 9; i++) matTilt[i] = invMatTilt[i] = (i % 4 == 0) ? 1. : 0.;
    if (!(tauX != 0 || tauY != 0)) return;
    const double cTauX = cos(tauX), sTauX = sin(tauX), cTauY = cos(tauY), sTauY = sin(tauY);
    const double matRotX[9] = {1, 0, 0, 0, cTauX, sTauX, 0, -sTauX, cTauX};
    const double matRotY[9] = {cTauY, 0, -sTauY, 0, 1, 0, sTauY, 0, cTauY};
    double R[9];
    matx33_mul(matRotY, matRotX, R);
    const double matProjZ[9] = {R[8], 0, -R[2], 0, R[8], -R[5], 0, 0, 1};
    matx33_mul(matProjZ, R, matTilt);
    const double inv = 1. / R[8];
    const double invMatProjZ[9] = {inv, 0, inv * R[2], 0, inv, inv * R[5], 0, 0, 1};
    const double Rt[9] = {R[0], R[3], R[6], R[1], R[4], R[7], R[2], R[5], R[8]};
    matx33_mul(Rt, invMatProjZ, invMatTilt);
}
// the lens of an OpenCV distortion vector of n = 4, 5, 8, 12 or 14 entries, zero-padded to 14.  False (L untouched) for another
// n, a non-finite coefficient, or |tau_x| or |tau_y| >= pi/2, where 1 / matRotXY(2, 2) is no longer a finite tilt.
inline bool make_lens_full(const double* coeffs, int n, LensFull& L) {
    if (!coeffs || !(n == 4 || n == 5 || n == 8 || n == 12 || n == 14)) return false;
    double k[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < n; i++) {
        if (!(coeffs[i] - coeffs[i] == 0.0)) return false;
        k[i] = coeffs[i];
    }
    if (!(fabs(k[12]) < kHalfPi && fabs(k[13]) < kHalfPi)) return false;
    for (int i = 0; i < 14; i++) L.k[i] = k[i];
    tilt_matrices(k[12], k[13], L.tilt, L.itilt);
    return true;
}

// ------------------------------------------------------------------------------------------------ equidistant fisheye
// OpenCV's cv::fisheye model (k1..k4 on theta, calib3d/src/fisheye.cpp), where the radial-tangential lens above calls
// cv::undistortPoints / cv::projectPoints:
//   undistort_point_fisheye  cv::fisheye::undistortPoints(pt, out, K, D, noArray(), K) of a float pixel   (fisheye.cpp:321-449)
//   project_dist_fisheye     cv::fisheye::projectPoints of the float point (x/z, y/z, 1), zero rvec / tvec, alpha 0  (:71-155)
// Both take K4 = {fx, fy, cx, cy} and D4 = {k1, k2, k3, k4}.  atan and tan are det_atan / det_tan below, not the platform's:
// glibc and CUDA's libdevice round them differently, so one plain-arithmetic version keeps the device, the state machine and
// the CPU test backend bit-identical.  Against OpenCV (glibc) they agree to the last double bit on nearly every point; a float
// result can only differ when the double lies within a few ulps of a float rounding boundary (tests/test_oracle_fisheye.py).

// the high half of x with the low 32 bits cleared
ALVA_CAM_FN double hi_word(double x) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double(__double_as_longlong(x) & (long long)0xffffffff00000000ull);
#else
    unsigned long long b;
    __builtin_memcpy(&b, &x, 8);
    b &= 0xffffffff00000000ull;
    __builtin_memcpy(&x, &b, 8);
    return x;
#endif
}

// atan in double: |x| reduced to [0, 7/16] through atan(x) = atan(c) + atan((x - c) / (1 + x c)), c in {1/2, 1, 3/2, inf}, then
// an odd degree-21 minimax polynomial (the coefficients and the split constants of the classic fdlibm algorithm; < 1 ulp)
ALVA_CAM_FN double det_atan(double x) {
    const double hi[4] = {4.63647609000806093515e-01, 7.85398163397448278999e-01, 9.82793723247329054082e-01, 1.57079632679489655800e+00};
    const double lo[4] = {2.26987774529616870924e-17, 3.06161699786838301793e-17, 1.39033110312309984516e-17, 6.12323399573676603587e-17};
    const double aT[11] = {3.33333333333329318027e-01, -1.99999999998764832476e-01, 1.42857142725034663711e-01,
                           -1.11111104054623557880e-01, 9.09088713343650656196e-02, -7.69187620504482999495e-02,
                           6.66107313738753120669e-02, -5.83357013379057348645e-02, 4.97687799461593236017e-02,
                           -3.65315727442169155270e-02, 1.62858201153657823623e-02};
    if (x != x) return x + x;
    double a = x < 0 ? -x : x;
    if (a >= 7.3786976294838206464e19) return x < 0 ? -(hi[3] + lo[3]) : hi[3] + lo[3];   // 2^66
    int id = -1;
    if (a < 0.4375) {
        if (a < 7.450580596923828125e-9) return x;                                             // 2^-27
    } else if (a < 1.1875) {
        if (a < 0.6875) { id = 0; a = (2.0 * a - 1.0) / (2.0 + a); }
        else { id = 1; a = (a - 1.0) / (a + 1.0); }
    } else if (a < 2.4375) { id = 2; a = (a - 1.5) / (1.0 + 1.5 * a); }
    else { id = 3; a = -1.0 / a; }
    const double z = a * a, w = z * z;
    const double s1 = z * (aT[0] + w * (aT[2] + w * (aT[4] + w * (aT[6] + w * (aT[8] + w * aT[10])))));
    const double s2 = w * (aT[1] + w * (aT[3] + w * (aT[5] + w * (aT[7] + w * aT[9]))));
    if (id < 0) return x - x * (s1 + s2);
    const double r = hi[id] - ((a * (s1 + s2) - lo[id]) - a);
    return x < 0 ? -r : r;
}

// tan in double: x = n pi/2 + (y0 + y1) by a three-part Cody-Waite reduction (|x| < 2^19 pi/2), then tan of the remainder by
// the fdlibm kernel (its coefficients; pi/4 - r above 0.6744) and, for odd n, -1 / tan computed with the split-word correction
ALVA_CAM_FN double det_tan(double x) {
    const double T[13] = {3.33333333333334091986e-01, 1.33333333333201242699e-01, 5.39682539762260521377e-02,
                          2.18694882948595424599e-02, 8.86323982359930005737e-03, 3.59207910759131235356e-03,
                          1.45620945432529025516e-03, 5.88041240820264096874e-04, 2.46463134818469906812e-04,
                          7.81794442939557092300e-05, 7.14072491382608190305e-05, -1.85586374855275456654e-05,
                          2.59073051863633712884e-05};
    const double pio4 = 7.85398163397448278999e-01, pio4lo = 3.06161699786838301793e-17;
    const double invpio2 = 6.36619772367581382433e-01, pio2_1 = 1.57079632673412561417e+00, pio2_2 = 6.07710050630396597660e-11,
                 pio2_2t = 2.02226624879595063154e-21;   // pi/2 = pio2_1 + pio2_2 + pio2_2t (33 + 33 + 53 bits)
    if (!(x - x == 0.0)) return x - x;   // inf, NaN -> NaN
    const bool neg = x < 0;
    const double ax = neg ? -x : x;
    double y0 = ax, y1 = 0.0, fn = 0.0;
    if (ax > pio4) {
        fn = floor(ax * invpio2 + 0.5);
        const double r1 = ax - fn * pio2_1;        // fn * pio2_1 and fn * pio2_2 are exact for fn < 2^20
        const double r2 = r1 - fn * pio2_2;
        const double w2 = fn * pio2_2t - ((r1 - r2) - fn * pio2_2);
        y0 = r2 - w2;
        y1 = (r2 - y0) - w2;
    }
    const bool odd = fn - 2.0 * floor(0.5 * fn) != 0.0;
    // kernel: tan(y0 + y1) (odd = false) or -1 / tan(y0 + y1) (odd = true), |y0| <= pi/4
    double kx = y0, ky = y1;
    const bool big = (kx < 0 ? -kx : kx) >= 0.6743316650390625;
    const bool kneg = kx < 0;
    if (big) {
        if (kneg) { kx = -kx; ky = -ky; }
        const double z0 = pio4 - kx, w0 = pio4lo - ky;
        kx = z0 + w0;
        ky = 0.0;
    }
    const double z = kx * kx, w = z * z;
    double r = T[1] + w * (T[3] + w * (T[5] + w * (T[7] + w * (T[9] + w * T[11]))));
    const double v = z * (T[2] + w * (T[4] + w * (T[6] + w * (T[8] + w * (T[10] + w * T[12])))));
    const double s = z * kx;
    r = ky + z * (s * (r + v) + ky);
    r += T[0] * s;
    const double wr = kx + r;
    double t;
    if (big) {
        const double iv = odd ? -1.0 : 1.0;
        t = (kneg ? -1.0 : 1.0) * (iv - 2.0 * (kx - (wr * wr / (wr + iv) - r)));
    } else if (!odd) {
        t = wr;
    } else {   // -1 / (kx + r) with the split-word correction
        const double zz = hi_word(wr);
        const double vv = r - (zz - kx);
        const double a = -1.0 / wr;
        const double tt = hi_word(a);
        const double ss = 1.0 + tt * zz;
        t = tt + a * (ss + tt * vv);
    }
    return neg ? -t : t;
}

// out = cv::fisheye::undistortPoints of the float pixel (u, v), rounded to float.  Returns false, with out = (-1e6, -1e6)
// (OpenCV's failure value), when the Newton iteration did not converge in 10 steps or theta changed sign.
ALVA_CAM_FN bool undistort_point_fisheye(const double* K4, const double* D4, float u_in, float v_in, float* out) {
    const double f0 = K4[0], f1 = K4[1], c0 = K4[2], c1 = K4[3];
    const double k0 = D4[0], k1 = D4[1], k2 = D4[2], k3 = D4[3];
    const double pi0 = u_in, pi1 = v_in;
    const double pw0 = (pi0 - c0) / f0, pw1 = (pi1 - c1) / f1;                                                     // :378
    double theta_d = sqrt(pw0 * pw0 + pw1 * pw1);
    theta_d = (-kHalfPi < theta_d) ? theta_d : -kHalfPi;                                                          // :385 std::max
    theta_d = (kHalfPi < theta_d) ? kHalfPi : theta_d;                                                            //      std::min
    bool converged = false;
    double theta = theta_d, scale = 0.0;
    if (fabs(theta_d) > 1e-8) {                                                                                   // :392-414
        for (int j = 0; j < 10; j++) {
            const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2, theta8 = theta6 * theta2;
            const double k0_theta2 = k0 * theta2, k1_theta4 = k1 * theta4, k2_theta6 = k2 * theta6, k3_theta8 = k3 * theta8;
            const double theta_fix = (theta * (1 + k0_theta2 + k1_theta4 + k2_theta6 + k3_theta8) - theta_d) /
                                     (1 + 3 * k0_theta2 + 5 * k1_theta4 + 7 * k2_theta6 + 9 * k3_theta8);
            theta = theta - theta_fix;
            if (fabs(theta_fix) < 1e-8) { converged = true; break; }
        }
        scale = det_tan(theta) / theta_d;
    } else {
        converged = true;
    }
    const bool theta_flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);                         // :423
    if (converged && !theta_flipped) {
        const double pu0 = pw0 * scale, pu1 = pw1 * scale;
        // RR = K * eye (P = K, no R), multiplied out as Matx accumulates; RR * (pu0, pu1, 1)                     :359-364, :430-431
        const double pr0 = ((0. + f0 * pu0) + 0. * pu1) + c0 * 1.0;
        const double pr1 = ((0. + 0. * pu0) + f1 * pu1) + c1 * 1.0;
        const double pr2 = ((0. + 0. * pu0) + 0. * pu1) + 1. * 1.0;
        out[0] = (float)(pr0 / pr2);
        out[1] = (float)(pr1 / pr2);
        return true;
    }
    out[0] = -1000000.0f;                                                                                         // :441
    out[1] = -1000000.0f;
    return false;
}

// out = cv::fisheye::projectPoints of the camera-frame point p through cv::Point3f(p.x / p.z, p.y / p.z, 1), rounded to float
ALVA_CAM_FN void project_dist_fisheye(const double* K4, const double* D4, const double* p, float* out) {
    const double f0 = K4[0], f1 = K4[1], c0 = K4[2], c1 = K4[3];
    const double inverseZ = 1. / p[2];
    const double X = (float)(p[0] * inverseZ), Y = (float)(p[1] * inverseZ), Z = 1.0f;   // camera_calibration.cpp:36-46
    // Affine3d(rvec 0, tvec 0) * Xi: rotation eye, translation +0                                                affine.hpp:630-638
    const double Y0 = 1. * X + 0. * Y + 0. * Z + 0.;
    const double Y1 = 0. * X + 1. * Y + 0. * Z + 0.;
    double Y2 = 0. * X + 0. * Y + 1. * Z + 0.;
    if (fabs(Y2) < 2.2250738585072014e-308) Y2 = 1;                                                               // :130-131 DBL_MIN
    const double x0 = Y0 / Y2, x1 = Y1 / Y2;
    const double r2 = (0. + x0 * x0) + x1 * x1;                                                                   // :134-135
    const double r = sqrt(r2);
    const double theta = det_atan(r);
    const double theta2 = theta * theta, theta3 = theta2 * theta, theta4 = theta2 * theta2, theta5 = theta4 * theta,
                 theta6 = theta3 * theta3, theta7 = theta6 * theta, theta8 = theta4 * theta4, theta9 = theta8 * theta;
    const double theta_d = theta + D4[0] * theta3 + D4[1] * theta5 + D4[2] * theta7 + D4[3] * theta9;             // :143
    const double inv_r = r > 1e-8 ? 1.0 / r : 1;
    const double cdist = r > 1e-8 ? theta_d * inv_r : 1;
    const double xd1_0 = x0 * cdist, xd1_1 = x1 * cdist;
    const double xd3_0 = xd1_0 + 0.0 * xd1_1;                                                                     // alpha = 0
    out[0] = (float)(xd3_0 * f0 + c0);                                                                            // :150-153
    out[1] = (float)(xd1_1 * f1 + c1);
}

// the pinhole branch of CameraCalibration::projectCamToImageDist as the state machine's Camera takes it: the normalised point
// rounded to float, then scaled by K
ALVA_CAM_FN void project_pinhole(const double* K4, const double* p, float* out) {
    const double iz = 1. / p[2];
    const double x = (double)(float)(p[0] * iz), y = (double)(float)(p[1] * iz);
    out[0] = (float)(x * K4[0] + K4[2]);
    out[1] = (float)(y * K4[1] + K4[3]);
}

// A rotation-compensated KLT prior (System's gyro mode, not in the reference): the bearing bv of a previous-frame keypoint
// turned into the current camera, c = R^T bv (R = the camera's rotation from the previous frame to the current one, row-major),
// and projected through the lens (0 pinhole, 1 radial-tangential, 2 fisheye, 3 the full OpenCV vector F; D4 unused for the
// pinhole and lens 3, F only for lens 3) -- the infinite homography, exact for a pure rotation.  Returns true and writes out[2] only when the ray is in front of the camera (z > 0)
// and its projection lies inside the w x h image (Camera::inImage); otherwise out is left as it was.
ALVA_CAM_FN bool rotate_prior(int lens, const double* K4, const double* D4, int w, int h, const double* R9, const double* bv,
                              float* out, const LensFull* F = nullptr) {
    double c[3];
    for (int i = 0; i < 3; i++) c[i] = (R9[i] * bv[0] + R9[3 + i] * bv[1]) + R9[6 + i] * bv[2];
    if (!(c[2] > 0.0)) return false;
    float o[2];
    if (lens == 3) project_dist_full(K4, F->k, F->tilt, c, o);
    else if (lens == 2) project_dist_fisheye(K4, D4, c, o);
    else if (lens == 1) project_dist(K4, D4, c, o);
    else project_pinhole(K4, c, o);
    if (!(o[0] >= 0 && o[1] >= 0 && o[0] < w && o[1] < h)) return false;
    out[0] = o[0];
    out[1] = o[1];
    return true;
}

}  // namespace alva_cam
