// camera.cu -- the lens models of System on the device, batched: one thread per point.
//
//   alva_k_undistort_points  CameraCalibration::undistortImagePoint (camera_calibration.cpp:57-72), called by
//                            Frame::computeKeypoint for every tracked and detected keypoint (frame.cpp:101-109)
//   alva_k_project_points    CameraCalibration::projectCamToImageDist (camera_calibration.cpp:34-55)
//   alva_k_undistort_points_fisheye / alva_k_project_points_fisheye   the same two calls through OpenCV's equidistant fisheye
//                            model (cv::fisheye::undistortPoints / projectPoints) instead of the radial-tangential one
//   alva_k_undistort_points_full / alva_k_project_points_full   the same two calls with OpenCV's whole distortion vector (5, 8,
//                            12 or 14 coefficients: k3, the rational, thin-prism and tilted models); the tilt matrices are
//                            built on the host (alva_cam::make_lens_full) and travel in the kernel's parameters
//   alva_k_rotate_priors     System's gyro mode (not in the reference): the KLT prior of a previous-frame keypoint turned by
//                            the gyroscope's rotation and projected through the lens (alva_cam::rotate_prior), per lens
//                            template
// The arithmetic is camera_model.h, shared with the host state machine; this file is compiled with -fmad=false, so every
// result is bit-identical to the host's and to OpenCV's (tests/test_gpu_distortion.py, tests/test_gpu_fisheye.py).
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include "camera_model.h"
#include <math.h>

namespace {

struct CamArgs { double K[4], D[4]; };   // by value: the coefficients live in the kernel's parameter space
struct FullArgs { double K[4]; alva_cam::LensFull L; };   // the same for the 14-coefficient model and its tilt matrices

// FISH = false: the radial-tangential model; true: the equidistant fisheye model
template <bool FISH>
__global__ void __launch_bounds__(256) undistort_points_kernel(const float2* __restrict__ px, const int32_t* __restrict__ counts,
                                                               int cap, long long total, const CamArgs c, float2* __restrict__ unpx) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int f = (int)(i / cap), j = (int)(i - (long long)f * cap);
    if (counts && j >= min(counts[f], cap)) return;
    const float2 p = px[i];
    float o[2];
    if constexpr (FISH) alva_cam::undistort_point_fisheye(c.K, c.D, p.x, p.y, o);
    else alva_cam::undistort_point(c.K, c.D, p.x, p.y, o);
    unpx[i] = make_float2(o[0], o[1]);
}

template <bool FISH>
__global__ void __launch_bounds__(256) project_points_kernel(const double* __restrict__ Xc, int n, const CamArgs c, float2* __restrict__ uv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double p[3] = {Xc[3 * (size_t)i], Xc[3 * (size_t)i + 1], Xc[3 * (size_t)i + 2]};
    float o[2];
    if constexpr (FISH) alva_cam::project_dist_fisheye(c.K, c.D, p, o);
    else alva_cam::project_dist(c.K, c.D, p, o);
    uv[i] = make_float2(o[0], o[1]);
}

__global__ void __launch_bounds__(256) undistort_points_full_kernel(const float2* __restrict__ px, const int32_t* __restrict__ counts,
                                                                    int cap, long long total, const FullArgs c, float2* __restrict__ unpx) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int f = (int)(i / cap), j = (int)(i - (long long)f * cap);
    if (counts && j >= min(counts[f], cap)) return;
    const float2 p = px[i];
    float o[2];
    alva_cam::undistort_point_full(c.K, c.L.k, c.L.itilt, p.x, p.y, o);
    unpx[i] = make_float2(o[0], o[1]);
}

__global__ void __launch_bounds__(256) project_points_full_kernel(const double* __restrict__ Xc, int n, const FullArgs c, float2* __restrict__ uv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double p[3] = {Xc[3 * (size_t)i], Xc[3 * (size_t)i + 1], Xc[3 * (size_t)i + 2]};
    float o[2];
    alva_cam::project_dist_full(c.K, c.L.k, c.L.tilt, p, o);
    uv[i] = make_float2(o[0], o[1]);
}

// System's gyro mode: the rotation-compensated KLT prior of every flagged point (alva_cam::rotate_prior); an unflagged point,
// or one whose rotated ray is behind the camera or projects outside the image, keeps the prior it has
struct RotArgs { double R[9]; };
template <int LENS> struct RotCam { using type = CamArgs; };   // lenses 0..2: K and four coefficients; lens 3: FullArgs
template <> struct RotCam<3> { using type = FullArgs; };
template <int LENS>
__global__ void __launch_bounds__(256) rotate_priors_kernel(const double* __restrict__ bv, const uint8_t* __restrict__ flag, int n, int w,
                                                            int h, const typename RotCam<LENS>::type c, const RotArgs r,
                                                            float2* __restrict__ prior, uint8_t* __restrict__ rotated) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t done = 0;
    if (flag[i]) {
        const double b[3] = {bv[3 * (size_t)i], bv[3 * (size_t)i + 1], bv[3 * (size_t)i + 2]};
        float o[2];
        bool ok;
        if constexpr (LENS == 3) ok = alva_cam::rotate_prior(3, c.K, nullptr, w, h, r.R, b, o, &c.L);
        else ok = alva_cam::rotate_prior(LENS, c.K, c.D, w, h, r.R, b, o);
        if (ok) { prior[i] = make_float2(o[0], o[1]); done = 1; }
    }
    rotated[i] = done;
}

bool cam_args(const char* fn, const double* K4, const double* D4, CamArgs& c) {
    if (!K4 || !D4) { alva_set_error("%s: K4 and D4 are required (host arrays)", fn); return false; }
    for (int i = 0; i < 4; i++) {
        c.K[i] = K4[i]; c.D[i] = D4[i];
        if (!isfinite(K4[i]) || !isfinite(D4[i])) { alva_set_error("%s: non-finite intrinsics or distortion", fn); return false; }
    }
    if (K4[0] == 0.0 || K4[1] == 0.0) { alva_set_error("%s: fx and fy must be non-zero", fn); return false; }
    return true;
}

template <bool FISH>
int undistort_launch(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4, const double* D4,
                     float* unpx) {
    CamArgs c;
    for (int i = 0; i < 4; i++) { c.K[i] = K4[i]; c.D[i] = D4[i]; }
    const long long total = (long long)nframes * cap;
    undistort_points_kernel<FISH><<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>((const float2*)px, counts, cap, total, c, (float2*)unpx);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

template <bool FISH>
int undistort_checked(const char* fn, alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                      const double* D4, float* unpx) {
    CamArgs c;
    if (!ctx || !px || !unpx || nframes < 1 || cap < 1 || (long long)nframes * cap > (1LL << 36)) {
        alva_set_error("%s: bad argument", fn);
        return ALVA_E_INVALID;
    }
    if (!cam_args(fn, K4, D4, c)) return ALVA_E_INVALID;
    if ((((uintptr_t)px) & 7) || (((uintptr_t)unpx) & 7)) { alva_set_error("%s: px / unpx must be 8-byte aligned", fn); return ALVA_E_INVALID; }
    return undistort_launch<FISH>(ctx, px, counts, nframes, cap, c.K, c.D, unpx);
}

template <bool FISH>
int project_checked(const char* fn, alva_ctx* ctx, const double* Xc, int n, const double* K4, const double* D4, float* uv) {
    CamArgs c;
    if (!ctx || !Xc || !uv || n < 1) { alva_set_error("%s: bad argument", fn); return ALVA_E_INVALID; }
    if (!cam_args(fn, K4, D4, c)) return ALVA_E_INVALID;
    if (((uintptr_t)uv) & 7) { alva_set_error("%s: uv must be 8-byte aligned", fn); return ALVA_E_INVALID; }
    project_points_kernel<FISH><<<(n + 255) / 256, 256, 0, ctx->stream>>>(Xc, n, c, (float2*)uv);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

bool full_args(const char* fn, const double* K4, const double* coeffs, int ncoeffs, FullArgs& c) {
    const double zero[4] = {0, 0, 0, 0};
    CamArgs k;
    if (!cam_args(fn, K4, zero, k)) return false;
    for (int i = 0; i < 4; i++) c.K[i] = K4[i];
    if (!alva_cam::make_lens_full(coeffs, ncoeffs, c.L)) {
        alva_set_error("%s: coeffs must hold 4, 5, 8, 12 or 14 finite values with |tau_x|, |tau_y| < pi/2 (got n = %d)", fn, ncoeffs);
        return false;
    }
    return true;
}

// lens 3 reads F (its coefficients and tilt matrices, already built); the other lenses D4
int rotate_launch(alva_ctx* ctx, const double* bv, const uint8_t* flag, int n, int w, int h, const double* K4, const double* D4, int lens,
                  const double* R9, float* prior, uint8_t* rotated, const alva_cam::LensFull* F) {
    if (n < 1) return 0;
    CamArgs c;
    RotArgs r;
    for (int i = 0; i < 4; i++) { c.K[i] = K4[i]; c.D[i] = D4 ? D4[i] : 0.0; }
    for (int i = 0; i < 9; i++) r.R[i] = R9[i];
    const unsigned grid = (unsigned)((n + 255) / 256);
    float2* p = (float2*)prior;
    if (lens == 3) {
        FullArgs fa;
        for (int i = 0; i < 4; i++) fa.K[i] = K4[i];
        fa.L = *F;
        rotate_priors_kernel<3><<<grid, 256, 0, ctx->stream>>>(bv, flag, n, w, h, fa, r, p, rotated);
    } else if (lens == 2) rotate_priors_kernel<2><<<grid, 256, 0, ctx->stream>>>(bv, flag, n, w, h, c, r, p, rotated);
    else if (lens == 1) rotate_priors_kernel<1><<<grid, 256, 0, ctx->stream>>>(bv, flag, n, w, h, c, r, p, rotated);
    else rotate_priors_kernel<0><<<grid, 256, 0, ctx->stream>>>(bv, flag, n, w, h, c, r, p, rotated);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

}  // namespace

// System's gyro mode (system.cu, CudaBackend::klt_rotated): the coefficients are already checked, no argument checks
int alva_rotate_priors_launch(alva_ctx* ctx, const double* bv, const uint8_t* flag, int n, int w, int h, const double* K4, const double* D4,
                              int lens, const double* R9, float* prior, uint8_t* rotated, const alva_cam::LensFull* F) {
    return rotate_launch(ctx, bv, flag, n, w, h, K4, D4, lens, R9, prior, rotated, F);
}

extern "C" int alva_k_rotate_priors(alva_ctx* ctx, const double* bv, const uint8_t* flag, int n, int w, int h, const double* K4,
                                    const double* D4, int lens, const double* R9, float* prior, uint8_t* rotated) { AlvaDeviceGuard guard__(ctx);
    const char* fn = "alva_k_rotate_priors";
    if (!ctx || n < 0 || w < 1 || h < 1 || lens < 0 || lens > 3 || !R9 || (n > 0 && (!bv || !flag || !prior || !rotated))) {
        alva_set_error("%s: bad argument", fn);
        return ALVA_E_INVALID;
    }
    const double zero[4] = {0, 0, 0, 0};
    CamArgs c;
    FullArgs fa;
    if (lens == 3) {
        if (!D4) { alva_set_error("%s: lens 3 reads 14 coefficients from D4", fn); return ALVA_E_INVALID; }
        if (!full_args(fn, K4, D4, 14, fa)) return ALVA_E_INVALID;
    }
    if (!cam_args(fn, K4, (D4 && lens != 3) ? D4 : zero, c)) return ALVA_E_INVALID;
    for (int i = 0; i < 9; i++) if (!isfinite(R9[i])) { alva_set_error("%s: non-finite rotation", fn); return ALVA_E_INVALID; }
    if (((uintptr_t)prior) & 7) { alva_set_error("%s: prior must be 8-byte aligned", fn); return ALVA_E_INVALID; }
    return rotate_launch(ctx, bv, flag, n, w, h, c.K, c.D, lens, R9, prior, rotated, &fa.L);
}

// host-side launches for callers that already hold the coefficients by value (system.cu): no argument checks
int alva_undistort_points_launch(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                 const double* D4, float* unpx) {
    return undistort_launch<false>(ctx, px, counts, nframes, cap, K4, D4, unpx);
}
int alva_undistort_points_fisheye_launch(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                         const double* D4, float* unpx) {
    return undistort_launch<true>(ctx, px, counts, nframes, cap, K4, D4, unpx);
}

int alva_undistort_points_full_launch(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                      const alva_cam::LensFull& L, float* unpx) {
    FullArgs c;
    for (int i = 0; i < 4; i++) c.K[i] = K4[i];
    c.L = L;
    const long long total = (long long)nframes * cap;
    undistort_points_full_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>((const float2*)px, counts, cap, total, c, (float2*)unpx);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_undistort_points(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                       const double* D4, float* unpx) { AlvaDeviceGuard guard__(ctx);
    return undistort_checked<false>("alva_k_undistort_points", ctx, px, counts, nframes, cap, K4, D4, unpx);
}

extern "C" int alva_k_project_points(alva_ctx* ctx, const double* Xc, int n, const double* K4, const double* D4, float* uv) { AlvaDeviceGuard guard__(ctx);
    return project_checked<false>("alva_k_project_points", ctx, Xc, n, K4, D4, uv);
}

extern "C" int alva_k_undistort_points_fisheye(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap,
                                               const double* K4, const double* D4, float* unpx) { AlvaDeviceGuard guard__(ctx);
    return undistort_checked<true>("alva_k_undistort_points_fisheye", ctx, px, counts, nframes, cap, K4, D4, unpx);
}

extern "C" int alva_k_project_points_fisheye(alva_ctx* ctx, const double* Xc, int n, const double* K4, const double* D4, float* uv) { AlvaDeviceGuard guard__(ctx);
    return project_checked<true>("alva_k_project_points_fisheye", ctx, Xc, n, K4, D4, uv);
}

extern "C" int alva_k_undistort_points_full(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                            const double* coeffs, int ncoeffs, float* unpx) { AlvaDeviceGuard guard__(ctx);
    const char* fn = "alva_k_undistort_points_full";
    FullArgs c;
    if (!ctx || !px || !unpx || nframes < 1 || cap < 1 || (long long)nframes * cap > (1LL << 36)) {
        alva_set_error("%s: bad argument", fn);
        return ALVA_E_INVALID;
    }
    if (!full_args(fn, K4, coeffs, ncoeffs, c)) return ALVA_E_INVALID;
    if ((((uintptr_t)px) & 7) || (((uintptr_t)unpx) & 7)) { alva_set_error("%s: px / unpx must be 8-byte aligned", fn); return ALVA_E_INVALID; }
    return alva_undistort_points_full_launch(ctx, px, counts, nframes, cap, c.K, c.L, unpx);
}

extern "C" int alva_k_project_points_full(alva_ctx* ctx, const double* Xc, int n, const double* K4, const double* coeffs, int ncoeffs,
                                          float* uv) { AlvaDeviceGuard guard__(ctx);
    const char* fn = "alva_k_project_points_full";
    FullArgs c;
    if (!ctx || !Xc || !uv || n < 1) { alva_set_error("%s: bad argument", fn); return ALVA_E_INVALID; }
    if (!full_args(fn, K4, coeffs, ncoeffs, c)) return ALVA_E_INVALID;
    if (((uintptr_t)uv) & 7) { alva_set_error("%s: uv must be 8-byte aligned", fn); return ALVA_E_INVALID; }
    project_points_full_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(Xc, n, c, (float2*)uv);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}
