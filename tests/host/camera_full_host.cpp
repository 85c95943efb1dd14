// tests/host/camera_full_host.cpp -- TEST INFRASTRUCTURE: the host build of OpenCV's whole distortion vector as the product
// runs it -- alvaar_b200/csrc/camera_model.h (what the kernels run, compiled for the device) and the state machine's Camera
// (system_core.h, what System's host side calls) -- behind a C ABI for tests/test_oracle_distortion_full.py.  Build with
// -ffp-contract=off.  Every entry returns -1 (nothing written) for a vector alva_cam::make_lens_full refuses.
#include "../../alvaar_b200/csrc/system_core.h"

extern "C" {

int cpu_full_undistort_points(const float* px, int n, const double* K4, const double* coeffs, int nc, float* out) {
    alva_cam::LensFull L;
    if (!alva_cam::make_lens_full(coeffs, nc, L)) return -1;
    for (int i = 0; i < n; i++) alva_cam::undistort_point_full(K4, L.k, L.itilt, px[2 * i], px[2 * i + 1], out + 2 * i);
    return 0;
}

int cpu_full_project_points(const double* Xc, int n, const double* K4, const double* coeffs, int nc, float* out) {
    alva_cam::LensFull L;
    if (!alva_cam::make_lens_full(coeffs, nc, L)) return -1;
    for (int i = 0; i < n; i++) alva_cam::project_dist_full(K4, L.k, L.tilt, Xc + 3 * i, out + 2 * i);
    return 0;
}

// the tilt matrices make_lens_full builds: tilt [9], itilt [9] row-major
int cpu_full_tilt(const double* coeffs, int nc, double* tilt, double* itilt) {
    alva_cam::LensFull L;
    if (!alva_cam::make_lens_full(coeffs, nc, L)) return -1;
    for (int i = 0; i < 9; i++) { tilt[i] = L.tilt[i]; itilt[i] = L.itilt[i]; }
    return 0;
}

// the state machine's Camera after setDistortionCoeffs: its lens (0 pinhole, 1 radial-tangential, 3 full) and, with mode 0, its
// undistortion of px [n][2] or, with mode 1, its projection of Xc [n][3]
int cpu_cam_full(const void* in, int n, const double* K4, const double* coeffs, int nc, int mode, float* out) {
    alva_sys::Camera c;
    c.fx = K4[0]; c.fy = K4[1]; c.cx = K4[2]; c.cy = K4[3];
    c.prepare();
    if (!c.setDistortionCoeffs(coeffs, nc)) return -1;
    for (int i = 0; i < n; i++) {
        if (mode == 0) c.undistort(((const float*)in)[2 * i], ((const float*)in)[2 * i + 1], out[2 * i], out[2 * i + 1]);
        else c.projCamToImageDist((const double*)in + 3 * i, out[2 * i], out[2 * i + 1]);
    }
    return c.lens;
}

}  // extern "C"
