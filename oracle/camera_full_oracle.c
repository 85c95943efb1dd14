/* oracle/camera_full_oracle.c -- TEST INFRASTRUCTURE ONLY (never on the product path).
 *
 * A plain-C restatement, separate from alvaar_b200/csrc/camera_model.h, of OpenCV's pinhole lens with its whole distortion
 * vector, as the reference's CameraCalibration calls the library (camera_calibration.cpp:34-72):
 *   orc_full_undistort_points  cv::undistortPoints(pt, out, K, D, K) of float pixels   (undistort.dispatch.cpp:384-556, COUNT 5)
 *   orc_full_project_points    cv::projectPoints of the float point (x/z, y/z, 1), zero rvec / tvec   (calibration.cpp:780-810)
 * D = coeffs [n], n = 4, 5, 8, 12 or 14, zero-padded to k[14] = {k1 k2 p1 p2 k3 k4 k5 k6 s1 s2 s3 s4 tau_x tau_y}; the tilt
 * matrices are detail::computeTiltProjectionMatrix's (imgproc/src/distortion_model.hpp:75-123), the identity unless tau_x or
 * tau_y is non-zero.  Every 3x3 product accumulates as cv::Matx does (s = 0; s += a(i, l) * b(l, j)).  Build with
 * -ffp-contract=off.  Returns -1 (nothing written) for a vector OpenCV or the library refuses. */
#include <math.h>
#include <string.h>

static void mul33(const double* a, const double* b, double* c) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int l = 0; l < 3; l++) s += a[3 * i + l] * b[3 * l + j];
            c[3 * i + j] = s;
        }
}

/* Matx33d * Vec3d(x, y, 1) */
static void mulv(const double* M, double x, double y, double* o) {
    for (int i = 0; i < 3; i++) {
        double s = 0;
        s += M[3 * i] * x;
        s += M[3 * i + 1] * y;
        s += M[3 * i + 2] * 1.;
        o[i] = s;
    }
}

static int lens(const double* coeffs, int n, double* k, double* tilt, double* itilt) {
    if (!(n == 4 || n == 5 || n == 8 || n == 12 || n == 14)) return -1;
    memset(k, 0, 14 * sizeof(double));
    for (int i = 0; i < n; i++) {
        if (!isfinite(coeffs[i])) return -1;
        k[i] = coeffs[i];
    }
    if (!(fabs(k[12]) < M_PI / 2 && fabs(k[13]) < M_PI / 2)) return -1;
    for (int i = 0; i < 9; i++) tilt[i] = itilt[i] = (i % 4 == 0) ? 1. : 0.;
    if (k[12] != 0 || k[13] != 0) {
        const double cx = cos(k[12]), sx = sin(k[12]), cy = cos(k[13]), sy = sin(k[13]);
        const double rx[9] = {1, 0, 0, 0, cx, sx, 0, -sx, cx}, ry[9] = {cy, 0, -sy, 0, 1, 0, sy, 0, cy};
        double r[9];
        mul33(ry, rx, r);
        const double pz[9] = {r[8], 0, -r[2], 0, r[8], -r[5], 0, 0, 1};
        mul33(pz, r, tilt);
        const double inv = 1. / r[8];
        const double ipz[9] = {inv, 0, inv * r[2], 0, inv, inv * r[5], 0, 0, 1};
        const double rt[9] = {r[0], r[3], r[6], r[1], r[4], r[7], r[2], r[5], r[8]};
        mul33(rt, ipz, itilt);
    }
    return 0;
}

int orc_full_undistort_points(const float* px, int npts, const double* K4, const double* coeffs, int n, float* out) {
    double k[14], tilt[9], itilt[9];
    if (lens(coeffs, n, k, tilt, itilt)) return -1;
    const double fx = K4[0], fy = K4[1], cx = K4[2], cy = K4[3], ifx = 1. / fx, ify = 1. / fy;
    for (int i = 0; i < npts; i++) {
        const double u = px[2 * i], v = px[2 * i + 1];
        double x = (u - cx) * ifx, y = (v - cy) * ify, t[3];
        mulv(itilt, x, y, t);
        const double invProj = t[2] ? 1. / t[2] : 1;
        const double x0 = invProj * t[0], y0 = invProj * t[1];
        x = x0; y = y0;
        for (int j = 0; j < 5; j++) {
            const double r2 = x * x + y * y;
            const double icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
            if (icdist < 0) { x = (u - cx) * ifx; y = (v - cy) * ify; break; }
            const double dx = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2;
            const double dy = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2;
            x = (x0 - dx) * icdist;
            y = (y0 - dy) * icdist;
        }
        /* RR = K * I (cvMatMul of P = K and R = I) */
        const double xx = fx * x + 0. * y + cx, yy = 0. * x + fy * y + cy, ww = 1. / (0. * x + 0. * y + 1.);
        out[2 * i] = (float)(xx * ww);
        out[2 * i + 1] = (float)(yy * ww);
    }
    return 0;
}

int orc_full_project_points(const double* Xc, int npts, const double* K4, const double* coeffs, int n, float* out) {
    double k[14], tilt[9], itilt[9];
    if (lens(coeffs, n, k, tilt, itilt)) return -1;
    const double fx = K4[0], fy = K4[1], cx = K4[2], cy = K4[3];
    for (int i = 0; i < npts; i++) {
        const double iz = 1. / Xc[3 * i + 2];
        const float pxf = (float)(Xc[3 * i] * iz), pyf = (float)(Xc[3 * i + 1] * iz), pzf = 1.0f;
        const double X = pxf, Y = pyf, Z = pzf;
        double x = 1. * X + 0. * Y + 0. * Z + 0., y = 0. * X + 1. * Y + 0. * Z + 0., z = 0. * X + 0. * Y + 1. * Z + 0.;
        z = z ? 1. / z : 1;
        x *= z; y *= z;
        const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
        const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
        const double cdist = 1 + k[0] * r2 + k[1] * r4 + k[4] * r6;
        const double icdist2 = 1. / (1 + k[5] * r2 + k[6] * r4 + k[7] * r6);
        const double xd0 = x * cdist * icdist2 + k[2] * a1 + k[3] * a2 + k[8] * r2 + k[9] * r4;
        const double yd0 = y * cdist * icdist2 + k[2] * a3 + k[3] * a1 + k[10] * r2 + k[11] * r4;
        double t[3];
        mulv(tilt, xd0, yd0, t);
        const double invProj = t[2] ? 1. / t[2] : 1;
        out[2 * i] = (float)(invProj * t[0] * fx + cx);
        out[2 * i + 1] = (float)(invProj * t[1] * fy + cy);
    }
    return 0;
}

/* the projection of one camera point through the 14-coefficient vector k14 -- the signature of camera_oracle.c's
 * orc_project_cam_dist, so that the matcher and re-acquisition oracles can take it (tests/camera_full_util.py) */
void orc_full_project_cam(const double* K4, const double* k14, const double* p, float* out) {
    orc_full_project_points(p, 1, K4, k14, 14, out);
}

/* orc_full_project_points with the vector already zero-padded to 14 entries */
void orc_full14_project_points(const double* Xc, int npts, const double* K4, const double* k14, float* out) {
    orc_full_project_points(Xc, npts, K4, k14, 14, out);
}
