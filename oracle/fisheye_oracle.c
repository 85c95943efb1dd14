/* oracle/fisheye_oracle.c -- CPU restatement of OpenCV's equidistant fisheye lens (cv::fisheye, k1..k4 on theta) as System
 * applies it with alva_system_set_fisheye.
 *
 * TEST INFRASTRUCTURE ONLY (see alva_oracle.c's header).  The product's own statement is alvaar_b200/csrc/camera_model.h; this
 * file is written separately from it so that the tests can hold the two against each other and against OpenCV.
 *
 * OpenCV 4.5.5 (paths under the reference tree, src/libs/opencv/modules/calib3d/src/fisheye.cpp):
 *   cv::fisheye::undistortPoints(pt, out, K, D, noArray(), K)     :321-449  a float pixel; RR = K * eye; at most 10 Newton
 *       steps on theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8), stopping at |fix| < 1e-8; theta_d
 *       clamped to [-pi/2, pi/2]; (-1e6, -1e6) when the iteration did not converge or theta changed sign
 *   cv::fisheye::projectPoints(Point3f(x/z, y/z, 1), 0, 0, K, D, alpha 0)   :71-155  Affine3d(0, 0) is the identity
 *       (core/include/opencv2/core/affine.hpp:630-638); the double results rounded to float
 * atan / tan: OpenCV calls the C library's.  Here (as in camera_model.h) they are one plain-arithmetic double version -- argument
 * reduction and the odd polynomials of the classic fdlibm algorithms -- so that the host, the device and this file agree bit for
 * bit whatever libm or libdevice would round.  Build with -ffp-contract=off.
 * PINNED: tests/test_oracle_fisheye.py (golden + live OpenCV): identical float bits, up to the double-rounding exemption the
 * test states and counts.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

static const double HALF_PI = 1.57079632679489661923;

static double f_clear_low(double x)
{
    uint64_t b;
    memcpy(&b, &x, 8);
    b &= 0xffffffff00000000ull;
    memcpy(&x, &b, 8);
    return x;
}

double orc_atan(double x)
{
    static const double H[4] = {4.63647609000806093515e-01, 7.85398163397448278999e-01, 9.82793723247329054082e-01, 1.57079632679489655800e+00};
    static const double L[4] = {2.26987774529616870924e-17, 3.06161699786838301793e-17, 1.39033110312309984516e-17, 6.12323399573676603587e-17};
    static const double C[11] = {3.33333333333329318027e-01, -1.99999999998764832476e-01, 1.42857142725034663711e-01,
                                 -1.11111104054623557880e-01, 9.09088713343650656196e-02, -7.69187620504482999495e-02,
                                 6.66107313738753120669e-02, -5.83357013379057348645e-02, 4.97687799461593236017e-02,
                                 -3.65315727442169155270e-02, 1.62858201153657823623e-02};
    if (isnan(x)) return x + x;
    const int sgn = x < 0;
    double t = fabs(x);
    if (t >= 0x1p66) return sgn ? -(H[3] + L[3]) : H[3] + L[3];
    int id;
    if (t < 0.4375) {
        if (t < 0x1p-27) return x;
        id = -1;
    } else if (t < 0.6875) { id = 0; t = (2.0 * t - 1.0) / (2.0 + t); }
    else if (t < 1.1875) { id = 1; t = (t - 1.0) / (t + 1.0); }
    else if (t < 2.4375) { id = 2; t = (t - 1.5) / (1.0 + 1.5 * t); }
    else { id = 3; t = -1.0 / t; }
    const double z = t * t, w = z * z;
    const double odd = z * (C[0] + w * (C[2] + w * (C[4] + w * (C[6] + w * (C[8] + w * C[10])))));
    const double even = w * (C[1] + w * (C[3] + w * (C[5] + w * (C[7] + w * C[9]))));
    if (id < 0) return x - x * (odd + even);
    const double r = H[id] - ((t * (odd + even) - L[id]) - t);
    return sgn ? -r : r;
}

double orc_tan(double x)
{
    static const double T[13] = {3.33333333333334091986e-01, 1.33333333333201242699e-01, 5.39682539762260521377e-02,
                                 2.18694882948595424599e-02, 8.86323982359930005737e-03, 3.59207910759131235356e-03,
                                 1.45620945432529025516e-03, 5.88041240820264096874e-04, 2.46463134818469906812e-04,
                                 7.81794442939557092300e-05, 7.14072491382608190305e-05, -1.85586374855275456654e-05,
                                 2.59073051863633712884e-05};
    const double PIO4 = 7.85398163397448278999e-01, PIO4LO = 3.06161699786838301793e-17, INVPIO2 = 6.36619772367581382433e-01;
    const double P1 = 1.57079632673412561417e+00, P2 = 6.07710050630396597660e-11, P2T = 2.02226624879595063154e-21;
    if (!isfinite(x)) return x - x;
    const int sgn = x < 0;
    const double a = fabs(x);
    /* x = n pi/2 + (y + yy) */
    double y = a, yy = 0.0, n = 0.0;
    if (a > PIO4) {
        n = floor(a * INVPIO2 + 0.5);
        const double r = a - n * P1;
        const double r2 = r - n * P2;
        const double e = n * P2T - ((r - r2) - n * P2);
        y = r2 - e;
        yy = (r2 - y) - e;
    }
    const int odd_n = n - 2.0 * floor(0.5 * n) != 0.0;
    /* tan(y + yy), or -1 / tan(y + yy) for odd n */
    const int large = fabs(y) >= 0.6743316650390625, yneg = y < 0;
    if (large) {
        if (yneg) { y = -y; yy = -yy; }
        const double d = PIO4 - y, dl = PIO4LO - yy;
        y = d + dl;
        yy = 0.0;
    }
    const double z = y * y, w = z * z;
    double r = T[1] + w * (T[3] + w * (T[5] + w * (T[7] + w * (T[9] + w * T[11]))));
    const double v = z * (T[2] + w * (T[4] + w * (T[6] + w * (T[8] + w * (T[10] + w * T[12])))));
    const double s = z * y;
    r = yy + z * (s * (r + v) + yy);
    r += T[0] * s;
    const double sum = y + r;
    double out;
    if (large) {
        const double iv = odd_n ? -1.0 : 1.0;
        out = (yneg ? -1.0 : 1.0) * (iv - 2.0 * (y - (sum * sum / (sum + iv) - r)));
    } else if (!odd_n) {
        out = sum;
    } else {
        const double zh = f_clear_low(sum);
        const double vl = r - (zh - y);
        const double q = -1.0 / sum;
        const double qh = f_clear_low(q);
        const double e = 1.0 + qh * zh;
        out = qh + q * (e + qh * vl);
    }
    return sgn ? -out : out;
}

/* cv::fisheye::undistortPoints of one float pixel; returns 1, or 0 with (-1e6, -1e6) */
int orc_fisheye_undistort_one(const double* K4, const double* D4, float pu, float pv, float* out)
{
    const double f[2] = {K4[0], K4[1]}, c[2] = {K4[2], K4[3]};
    const double k[4] = {D4[0], D4[1], D4[2], D4[3]};
    /* RR = P * eye with P = K (:349-364): Matx accumulates each entry from s = 0 */
    const double Km[3][3] = {{K4[0], 0, K4[2]}, {0, K4[1], K4[3]}, {0, 0, 1}}, E[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    double RR[3][3];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int q = 0; q < 3; q++) s += Km[i][q] * E[q][j];
            RR[i][j] = s;
        }
    const double pi[2] = {pu, pv};
    const double pw[2] = {(pi[0] - c[0]) / f[0], (pi[1] - c[1]) / f[1]};   /* :378 */
    double theta_d = sqrt(pw[0] * pw[0] + pw[1] * pw[1]);
    if (!(-HALF_PI < theta_d)) theta_d = -HALF_PI;                        /* :385, std::max then std::min */
    if (HALF_PI < theta_d) theta_d = HALF_PI;
    int converged = 0;
    double theta = theta_d, scale = 0.0;
    if (fabs(theta_d) > 1e-8) {
        for (int j = 0; j < 10; j++) {
            const double t2 = theta * theta, t4 = t2 * t2, t6 = t4 * t2, t8 = t6 * t2;
            const double a = k[0] * t2, b = k[1] * t4, cc = k[2] * t6, d = k[3] * t8;
            const double fix = (theta * (1 + a + b + cc + d) - theta_d) / (1 + 3 * a + 5 * b + 7 * cc + 9 * d);
            theta = theta - fix;
            if (fabs(fix) < 1e-8) { converged = 1; break; }
        }
        scale = orc_tan(theta) / theta_d;
    } else {
        converged = 1;
    }
    const int flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);
    if (converged && !flipped) {
        const double v[3] = {pw[0] * scale, pw[1] * scale, 1.0};
        double pr[3];
        for (int i = 0; i < 3; i++) {
            double s = 0;
            for (int q = 0; q < 3; q++) s += RR[i][q] * v[q];
            pr[i] = s;
        }
        out[0] = (float)(pr[0] / pr[2]);
        out[1] = (float)(pr[1] / pr[2]);
        return 1;
    }
    out[0] = out[1] = (float)-1000000.0;
    return 0;
}

/* cv::fisheye::projectPoints of the camera-frame point p through cv::Point3f(p.x / p.z, p.y / p.z, 1); exact: the result in
 * double before the float rounding (may be NULL) */
void orc_fisheye_project_cam_exact(const double* K4, const double* D4, const double* p, float* out, double* exact)
{
    const double inverseZ = 1. / p[2];
    const float fx = (float)(p[0] * inverseZ), fy = (float)(p[1] * inverseZ), fz = (float)1.0;
    const double Xi[3] = {fx, fy, fz};
    const double M[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};   /* Affine3d(rvec 0, tvec 0): rows of [I | +0] */
    double Y[3];
    for (int i = 0; i < 3; i++) Y[i] = M[4 * i] * Xi[0] + M[4 * i + 1] * Xi[1] + M[4 * i + 2] * Xi[2] + M[4 * i + 3];
    if (fabs(Y[2]) < 2.2250738585072014e-308) Y[2] = 1;
    const double x[2] = {Y[0] / Y[2], Y[1] / Y[2]};
    double r2 = 0;
    for (int i = 0; i < 2; i++) r2 += x[i] * x[i];
    const double r = sqrt(r2);
    const double th = orc_atan(r);
    const double th2 = th * th, th3 = th2 * th, th4 = th2 * th2, th5 = th4 * th, th6 = th3 * th3, th7 = th6 * th, th8 = th4 * th4,
                 th9 = th8 * th;
    const double th_d = th + D4[0] * th3 + D4[1] * th5 + D4[2] * th7 + D4[3] * th9;
    const double inv_r = r > 1e-8 ? 1.0 / r : 1;
    const double cdist = r > 1e-8 ? th_d * inv_r : 1;
    const double xd1[2] = {x[0] * cdist, x[1] * cdist};
    const double xd3[2] = {xd1[0] + 0.0 * xd1[1], xd1[1]};
    const double fin[2] = {xd3[0] * K4[0] + K4[2], xd3[1] * K4[1] + K4[3]};
    out[0] = (float)fin[0];
    out[1] = (float)fin[1];
    if (exact) { exact[0] = fin[0]; exact[1] = fin[1]; }
}

/* the projection the matcher oracle takes (same signature as camera_oracle.c's orc_project_cam_dist) */
void orc_fisheye_project_cam(const double* K4, const double* D4, const double* p, float* out)
{
    orc_fisheye_project_cam_exact(K4, D4, p, out, NULL);
}

/* px [n][2] -> unpx [n][2]; returns the number of failed points */
int orc_fisheye_undistort_points(const float* px, int n, const double* K4, const double* D4, float* unpx)
{
    int failed = 0;
    for (int i = 0; i < n; i++) failed += !orc_fisheye_undistort_one(K4, D4, px[2 * i], px[2 * i + 1], unpx + 2 * i);
    return failed;
}

/* Xc [n][3] camera-frame points -> uv [n][2] */
void orc_fisheye_project_points(const double* Xc, int n, const double* K4, const double* D4, float* uv)
{
    for (int i = 0; i < n; i++) orc_fisheye_project_cam_exact(K4, D4, Xc + 3 * i, uv + 2 * i, NULL);
}
