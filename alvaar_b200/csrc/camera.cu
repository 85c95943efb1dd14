// camera.cu -- the lens models of System on the device, batched: one thread per point.
//
//   alva_k_undistort_points  CameraCalibration::undistortImagePoint (camera_calibration.cpp:57-72), called by
//                            Frame::computeKeypoint for every tracked and detected keypoint (frame.cpp:101-109)
//   alva_k_project_points    CameraCalibration::projectCamToImageDist (camera_calibration.cpp:34-55)
//   alva_k_undistort_points_fisheye / alva_k_project_points_fisheye   the same two calls through OpenCV's equidistant fisheye
//                            model (cv::fisheye::undistortPoints / projectPoints) instead of the radial-tangential one
// The arithmetic is camera_model.h, shared with the host state machine; this file is compiled with -fmad=false, so every
// result is bit-identical to the host's and to OpenCV's (tests/test_gpu_distortion.py, tests/test_gpu_fisheye.py).
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include "camera_model.h"
#include <math.h>

namespace {

struct CamArgs { double K[4], D[4]; };   // by value: the coefficients live in the kernel's parameter space

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

}  // namespace

// host-side launches for callers that already hold the coefficients by value (system.cu): no argument checks
int alva_undistort_points_launch(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                 const double* D4, float* unpx) {
    return undistort_launch<false>(ctx, px, counts, nframes, cap, K4, D4, unpx);
}
int alva_undistort_points_fisheye_launch(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                         const double* D4, float* unpx) {
    return undistort_launch<true>(ctx, px, counts, nframes, cap, K4, D4, unpx);
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
