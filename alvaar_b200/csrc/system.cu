// system.cu -- `System`: the reference's public class (src/slam/src/system.hpp:19-56) re-hosted on the H100 hot path, plus its
// C ABI (alva_system_*).  Same method names, argument meaning and return conventions as the reference so that embind.cpp /
// system.js stay source-compatible (INTEGRATION.md):
//
//   configure(w, h, fx, fy, cx, cy, k1, k2, p1, p2)      system.cpp:13-40
//   reset()                                               system.cpp:42-55
//   findCameraPose(rgba, pose16) -> 1 tracking / 2 reset / 3 not initialised     system.cpp:106-121, 156-175
//   findCameraPoseWithIMU(rgba, imu, pose16) -> 1        system.cpp:57-104
//   findPlane(out16, iterations) -> 0 / 1                 system.cpp:123-137
//   getFramePoints(xy) -> count                           system.cpp:139-154
//
// The state machine (keypoints, map points, keyframes, motion model, the reference's gates and status codes) is
// system_core.h; this file is its CUDA Backend -- every pixel and solver stage of a call runs on the device:
//   pyramid      RGBA -> gray + pyramid + Scharr levels           alva_k_frontend, Scharr levels   (system.cpp:112, visual_frontend.cpp:672-698)
//                with CLAHE on: RGBA -> raw gray -> CLAHE -> L0 -> pyrDown levels -> Scharr   alva_k_clahe, alva_k_pyrdown
//   klt          forward-backward pyramidal LK                    alva_k_klt_fb                     (feature_tracker.cpp:5-111)
//   detect       grid Shi-Tomasi + cornerSubPix                   alva_k_detect_grid                (feature_extractor.cpp:11-158)
//   describe     7x7 blur + rBRIEF-256 at -1 degree               alva_k_orb_blur / _describe       (feature_extractor.cpp:160-214)
//   essential    5-point RANSAC + refinement (initialisation)     alva_k_essential_5pt              (multi_view_geometry.cpp:225-318)
//   p3p / pnp    per-frame pose                                   alva_k_p3p_lmeds, alva_k_pnp      (multi_view_geometry.cpp:24-223)
//   triangulate  new map points at keyframes                      alva_k_triangulate                (multi_view_geometry.cpp:12-22)
//   match_to_map local map -> keyframe matching                   alva_k_match_to_map               (mapper.cpp:354-587)
//   ba_local     local bundle adjustment, both solves + flags     alva_k_ba_local                   (optimizer.cpp:251-359)
// There is no CPU fallback: configure() fails without an sm_90 (H100) device.  Lens distortion: the JS shim always passes zeros
// (system.js:84-141) and configure() rejects non-zero coefficients; setDistortion() (alva_system_set_distortion) sets them on a
// configured System.  With distortion on, klt and detect undistort the points they return with alva_k_undistort_points on the
// device, in the same download (camera.cu, camera_model.h).
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include "system_core.h"
#include <chrono>
#include <exception>
#include <thread>
#include <vector>

int alva_scharr_levels_launch(alva_ctx* ctx, int nlev, const uint8_t* const* src, int16_t* const* dst, const int* w, const int* h,
                              int nframes);
int alva_clahe_launch(alva_ctx* ctx, const uint8_t* src, uint8_t* dst, int w, int h, int nframes, double clip_limit, int tiles_x,
                      int tiles_y, uint8_t* lut);
int alva_undistort_points_launch(alva_ctx* ctx, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                 const double* D4, float* unpx);
int alva_pose_chain_launch(alva_ctx* ctx, int n, int cap, const double* bvs, const double* X, const double* uv, const double* K4,
                           float fx, float fy, uint32_t seed, double* T12, double* info, uint8_t* o1, double* uv2, double* X2,
                           int32_t* n2, double* pose7, uint8_t* o2, double* summ, double huber, double chi2);

namespace {

#define SYS_CUDA(call)                                                                            \
    do {                                                                                          \
        cudaError_t e__ = (call);                                                                 \
        if (e__ != cudaSuccess) {                                                                 \
            alva_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return ALVA_E_CUDA;                                                                   \
        }                                                                                         \
    } while (0)

// One page-locked host buffer and its device mirror: a stage packs its small inputs into the host side, uploads them with ONE
// copy, runs its kernels on the mirror and reads the results back with ONE copy.  (The state machine's own containers are
// pageable std::vectors: copying from them directly costs a driver-side staging pass and an implicit synchronisation per call.)
struct Staging {
    uint8_t *h = nullptr, *d = nullptr;
    size_t cap = 0, off = 0;
    int init(size_t bytes) {
        release();
        if (cudaHostAlloc((void**)&h, bytes, cudaHostAllocDefault) != cudaSuccess || cudaMalloc((void**)&d, bytes) != cudaSuccess) {
            alva_set_error("System: staging allocation of %zu bytes failed (%s)", bytes, cudaGetErrorString(cudaGetLastError()));
            release();
            return ALVA_E_CUDA;
        }
        cap = bytes;
        return 0;
    }
    void release() {
        if (h) { cudaFreeHost(h); h = nullptr; }
        if (d) { cudaFree(d); d = nullptr; }
        cap = off = 0;
    }
    void reset() { off = 0; }
    // n elements of T at the next 256-byte boundary: returns the device pointer, *host receives the host-side twin
    template <class T> T* take(size_t n, T** host) {
        off = (off + 255) & ~(size_t)255;
        T* p = (T*)(d + off);
        if (host) *host = (T*)(h + off);
        off += n * sizeof(T);
        return p;
    }
    bool fits(size_t bytes) const { return bytes + 4096 <= cap; }
};

struct CudaBackend {
    alva_ctx* ctx = nullptr;
    Staging stg;
    cudaGraphExec_t pyr_graph[2] = {nullptr, nullptr};   // the pyramid chain of a frame (front end + pyrDown levels + Scharr), per ping-pong side
    bool graphs_ok = true;
    // cell: State::frameMaxCellSize_ of the preset (40 after configure); cap: the keypoint capacity of a frame at that cell size,
    // cap_alloc: what the cap-sized buffers below hold (a preset with smaller cells grows them, a larger one keeps them)
    int device = 0, w = 0, h = 0, nlev = 0, cur = 0, cap = 0, cap_alloc = 0, cell = 40;
    int lw[4] = {0, 0, 0, 0}, lh[4] = {0, 0, 0, 0};
    uint8_t* rgba_dev = nullptr;
    uint8_t* img[2][4] = {{nullptr, nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr, nullptr}};
    int16_t* der[2][4] = {{nullptr, nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr, nullptr}};
    float *pts_dev = nullptr, *pri_dev = nullptr;
    uint8_t *flag_dev = nullptr, *blur_dev = nullptr, *desc_dev = nullptr;
    int32_t* cnt_dev = nullptr;
    double *quality_dev = nullptr, *dbl_dev = nullptr;   // dbl_dev: [A: 3 cap][B: 3 cap][C: 3 cap][small: 64]
    bool blur_valid = false;
    // CLAHE (State::claheEnabled_ / claheContrastLimit_ / claheTileSize_, visual_frontend.cpp:16-18, 678-681).  When on, the gray
    // frame goes to raw_dev, its equalised image is level 0: KLT and the detector read the equalised pyramid, ORB describes the
    // raw frame (map_manager.cpp:204, 218).  Its pyramid chain differs, so it has its own graph pair, re-captured when a
    // parameter changes; with CLAHE off nothing here is allocated and the original chain and graphs run unchanged.
    bool clahe = false;
    float clahe_clip = 3.f;   // a float in State (state.hpp:44)
    int clahe_tx = 0, clahe_ty = 0, clahe_graph_launches = 0;
    uint8_t *raw_dev = nullptr, *clahe_lut = nullptr;
    size_t clahe_lut_bytes = 0;
    cudaGraphExec_t clahe_graph[2] = {nullptr, nullptr};
    // lens distortion (CameraCalibration::D_): when on, klt() and detect() also return the undistorted positions of their points
    // (unpx()); with it off nothing here is allocated or launched
    bool has_dist = false;
    double K4[4] = {0, 0, 0, 0}, D4[4] = {0, 0, 0, 0};
    float* unpx_dev = nullptr;
    std::vector<float> unpx_host;

    int init(int dev, int W, int H) {
        release();
        device = dev; w = W; h = H;
        ctx = alva_ctx_create(device, nullptr);
        if (!ctx) return ALVA_E_CUDA;
        int ww = W, hh = H;
        nlev = 0;
        for (int k = 0; k < 4; k++) {   // buildOpticalFlowPyramid(win 9, maxLevel 3) stops when a level is not larger than the window
            lw[k] = ww; lh[k] = hh; nlev = k + 1;
            ww = (ww + 1) / 2; hh = (hh + 1) / 2;
            if (ww <= 9 || hh <= 9) break;
        }
        SYS_CUDA(cudaMalloc(&rgba_dev, (size_t)W * H * 4));
        for (int s = 0; s < 2; s++)
            for (int k = 0; k < 4; k++) {
                const int kk = k < nlev ? k : nlev - 1;
                const size_t px = (size_t)lw[kk] * lh[kk];
                SYS_CUDA(cudaMalloc(&img[s][k], px));
                SYS_CUDA(cudaMalloc(&der[s][k], px * 4));
            }
        SYS_CUDA(cudaMalloc(&cnt_dev, 16));
        SYS_CUDA(cudaMalloc(&quality_dev, 8));
        SYS_CUDA(cudaMalloc(&blur_dev, (size_t)W * H));
        const double q0 = 0.001;   // State::extractorMaxQuality_ (state.hpp:59); FeatureExtractor keeps adapting it across resets
        SYS_CUDA(cudaMemcpy(quality_dev, &q0, 8, cudaMemcpyHostToDevice));
        return set_cell(40);   // State(w, h, 40) (system.cpp:15)
    }

    // a frame holds at most ~2 keypoints per cell; 4x leaves room for the transient overshoot before prepareFrame
    static int cap_for(int W, int H, int cs) { return 4 * ((W + cs - 1) / cs) * ((H + cs - 1) / cs) + 64; }

    // the grid cell size of the detector and the local-map matcher, and the keypoint capacity it implies.  Every buffer sized
    // from the capacity is reallocated here when it has to grow (after the stream has drained: every stage ends with a
    // synchronisation, this one makes sure).  The pyramid graphs capture only the frame-sized buffers (rgba_dev, img, der,
    // raw_dev, clahe_lut), none of these, so they stay valid.
    int set_cell(int cs) {
        const int want = cap_for(w, h, cs);
        if (want > cap_alloc) {
            SYS_CUDA(cudaStreamSynchronize(ctx->stream));
            void** bufs[] = {(void**)&pts_dev, (void**)&pri_dev, (void**)&flag_dev, (void**)&desc_dev, (void**)&dbl_dev, (void**)&unpx_dev};
            for (void** b : bufs) if (*b) { cudaFree(*b); *b = nullptr; }
            cap_alloc = 0;
            SYS_CUDA(cudaMalloc(&pts_dev, (size_t)want * 8));
            SYS_CUDA(cudaMalloc(&pri_dev, (size_t)want * 8));
            SYS_CUDA(cudaMalloc(&flag_dev, want));
            SYS_CUDA(cudaMalloc(&desc_dev, (size_t)want * 32));
            SYS_CUDA(cudaMalloc(&dbl_dev, ((size_t)want * 9 + 64) * sizeof(double)));
            if (has_dist) SYS_CUDA(cudaMalloc(&unpx_dev, (size_t)want * 8));
            if (int e = stg.init((size_t)want * 160 + 65536)) return e;
            cap_alloc = want;
        }
        cell = cs;
        cap = want;
        return 0;
    }

    void release() {
        if (rgba_dev) { cudaFree(rgba_dev); rgba_dev = nullptr; }
        for (int s = 0; s < 2; s++)
            for (int k = 0; k < 4; k++) {
                if (img[s][k]) { cudaFree(img[s][k]); img[s][k] = nullptr; }
                if (der[s][k]) { cudaFree(der[s][k]); der[s][k] = nullptr; }
            }
        void** bufs[] = {(void**)&pts_dev, (void**)&pri_dev, (void**)&flag_dev, (void**)&cnt_dev, (void**)&quality_dev, (void**)&blur_dev,
                         (void**)&desc_dev, (void**)&dbl_dev};
        for (void** b : bufs) if (*b) { cudaFree(*b); *b = nullptr; }
        if (arena) { cudaFree(arena); arena = nullptr; arena_cap = 0; }
        for (int k = 0; k < 2; k++) if (pyr_graph[k]) { cudaGraphExecDestroy(pyr_graph[k]); pyr_graph[k] = nullptr; }
        drop_clahe_graphs();
        if (raw_dev) { cudaFree(raw_dev); raw_dev = nullptr; }
        if (clahe_lut) { cudaFree(clahe_lut); clahe_lut = nullptr; clahe_lut_bytes = 0; }
        if (unpx_dev) { cudaFree(unpx_dev); unpx_dev = nullptr; }
        has_dist = false;
        cap = cap_alloc = 0;
        cell = 40;
        clahe = false;
        clahe_clip = 3.f;
        clahe_tx = clahe_ty = 0;
        graphs_ok = true;
        stg.release();
        if (ctx) { alva_ctx_destroy(ctx); ctx = nullptr; }
    }

    void drop_clahe_graphs() {
        for (int k = 0; k < 2; k++) if (clahe_graph[k]) { cudaGraphExecDestroy(clahe_graph[k]); clahe_graph[k] = nullptr; }
    }
    // enabled with a tx x ty grid: the buffers are allocated here, outside any capture
    int set_clahe(bool on, float clip, int tx, int ty) {
        if (on) {
            if (!raw_dev) SYS_CUDA(cudaMalloc(&raw_dev, (size_t)w * h));
            const size_t bytes = (size_t)tx * ty * 256;
            if (bytes > clahe_lut_bytes) {
                if (clahe_lut) { SYS_CUDA(cudaStreamSynchronize(ctx->stream)); cudaFree(clahe_lut); clahe_lut = nullptr; clahe_lut_bytes = 0; }
                SYS_CUDA(cudaMalloc(&clahe_lut, bytes));
                clahe_lut_bytes = bytes;
            }
        }
        if (clip != clahe_clip || tx != clahe_tx || ty != clahe_ty) drop_clahe_graphs();   // the graphs bake the parameters in
        clahe = on; clahe_clip = clip; clahe_tx = tx; clahe_ty = ty;
        return 0;
    }
    uint8_t* gray_raw() { return clahe ? raw_dev : img[cur][0]; }   // what ORB describes

    int set_distortion(const double* d) {
        has_dist = d[0] != 0.0 || d[1] != 0.0 || d[2] != 0.0 || d[3] != 0.0;
        for (int i = 0; i < 4; i++) D4[i] = d[i];
        K4[0] = fx; K4[1] = fy; K4[2] = cx; K4[3] = cy;
        if (has_dist && !unpx_dev) SYS_CUDA(cudaMalloc(&unpx_dev, (size_t)cap_alloc * 8));
        return 0;
    }
    const float* unpx() const { return has_dist ? unpx_host.data() : nullptr; }

    int clahe_launches() {
        uint8_t** L = img[cur];
        if (int e = alva_k_frontend(ctx, rgba_dev, w, h, 1, raw_dev, nullptr, nullptr, nullptr, 20, nullptr, nullptr, 0, 0)) return e;
        if (int e = alva_clahe_launch(ctx, raw_dev, L[0], w, h, 1, (double)clahe_clip, clahe_tx, clahe_ty, clahe_lut)) return e;
        for (int k = 1; k < nlev; k++)
            if (int e = alva_k_pyrdown(ctx, L[k - 1], L[k], lw[k - 1], lh[k - 1], 1)) return e;
        const uint8_t* srcs[4] = {L[0], L[1], L[2], L[3]};
        return alva_scharr_levels_launch(ctx, nlev, srcs, der[cur], lw, lh, 1);
    }
    int pyramid_clahe() {
        cudaStream_t st = ctx->stream;
        if (graphs_ok && !clahe_graph[cur]) {
            cudaGraph_t g = nullptr;
            const long long l0 = ctx->launches;
            bool ok = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
            int e = 0;
            if (ok) {
                e = clahe_launches();
                ok = cudaStreamEndCapture(st, &g) == cudaSuccess && e == 0 && g != nullptr;
            }
            if (ok) ok = cudaGraphInstantiate(&clahe_graph[cur], g, 0) == cudaSuccess;
            if (g) cudaGraphDestroy(g);
            clahe_graph_launches = (int)(ctx->launches - l0);
            ctx->launches = l0;
            if (!ok) { cudaGetLastError(); graphs_ok = false; clahe_graph[cur] = nullptr; }
        }
        if (clahe_graph[cur]) {
            SYS_CUDA(cudaGraphLaunch(clahe_graph[cur], st));
            ctx->launches += clahe_graph_launches;
            return 0;
        }
        return clahe_launches();
    }

    int pyramid_launches() {
        uint8_t** L = img[cur];
        if (int e = alva_k_frontend(ctx, rgba_dev, w, h, 1, L[0], nlev > 1 ? L[1] : nullptr, nlev > 2 ? L[2] : nullptr,
                                    nlev > 3 ? L[3] : nullptr, 20, nullptr, nullptr, 0, 0))
            return e;
        const uint8_t* srcs[4] = {L[0], L[1], L[2], L[3]};
        return alva_scharr_levels_launch(ctx, nlev, srcs, der[cur], lw, lh, 1);
    }
    // The chain is the same 4 launches on the same buffers every other frame: captured once per ping-pong side into a CUDA
    // graph and replayed with one call (no per-launch driver work, no tensor-map encode, dependent launches back to back).
    int pyramid(const uint8_t* rgba) {
        cudaStream_t st = ctx->stream;
        cur ^= 1;   // VisualFrontend::preprocessImage swaps prev / cur pyramids (visual_frontend.cpp:672-698)
        blur_valid = false;
        SYS_CUDA(cudaMemcpyAsync(rgba_dev, rgba, (size_t)w * h * 4, cudaMemcpyHostToDevice, st));
        if (clahe) return pyramid_clahe();
        if (graphs_ok && !pyr_graph[cur]) {
            cudaGraph_t g = nullptr;
            const long long l0 = ctx->launches;
            bool ok = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
            int e = 0;
            if (ok) {
                e = pyramid_launches();
                ok = cudaStreamEndCapture(st, &g) == cudaSuccess && e == 0 && g != nullptr;
            }
            if (ok) ok = cudaGraphInstantiate(&pyr_graph[cur], g, 0) == cudaSuccess;
            if (g) cudaGraphDestroy(g);
            ctx->launches = l0;
            if (!ok) { cudaGetLastError(); graphs_ok = false; pyr_graph[cur] = nullptr; }
        }
        if (pyr_graph[cur]) {
            SYS_CUDA(cudaGraphLaunch(pyr_graph[cur], st));
            ctx->launches += 2 + (nlev > 2 ? nlev - 2 : 0);
            return 0;
        }
        return pyramid_launches();
    }

    int detect(const float* cpts, int ncur, std::vector<float>& fresh) {
        cudaStream_t st = ctx->stream;
        if (ncur > cap) { alva_set_error("System: %d keypoints exceed the frame capacity %d", ncur, cap); return ALVA_E_CAPACITY; }
        int32_t nc = ncur;
        if (ncur) SYS_CUDA(cudaMemcpyAsync(pts_dev, cpts, (size_t)ncur * 8, cudaMemcpyHostToDevice, st));
        SYS_CUDA(cudaMemcpyAsync(cnt_dev + 1, &nc, 4, cudaMemcpyHostToDevice, st));
        const int32_t roi[4] = {20, 20, w - 40, h - 40};   // CameraCalibration(..., imgBorder 20): roi_rect_ (camera_calibration.cpp:21)
        if (int e = alva_k_detect_grid(ctx, img[cur][0], w, h, 1, cell, pts_dev, cnt_dev + 1, cap, roi, quality_dev, pri_dev, nullptr, cnt_dev, cap))
            return e;
        if (has_dist)   // Frame::computeKeypoint's undistortImagePoint of every new keypoint (frame.cpp:101-109)
            if (int e = alva_undistort_points_launch(ctx, pri_dev, cnt_dev, 1, cap, K4, D4, unpx_dev)) return e;
        int32_t n = 0;
        SYS_CUDA(cudaMemcpyAsync(&n, cnt_dev, 4, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        if (n > cap) n = cap;
        fresh.resize((size_t)2 * n);
        if (n) {
            SYS_CUDA(cudaMemcpyAsync(fresh.data(), pri_dev, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
            if (has_dist) {
                unpx_host.resize((size_t)2 * n);
                SYS_CUDA(cudaMemcpyAsync(unpx_host.data(), unpx_dev, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
            }
            SYS_CUDA(cudaStreamSynchronize(st));
        }
        return 0;
    }

    // ORB::create(500, 1, 0)->compute at the given points = 7x7 blur (the shipped build's unfused arithmetic) + rBRIEF-256 steered
    // by KeyPoint::convert's -1 degree; kept = 0 for points within 31 px of the border (empty descriptor in the reference)
    int describe(const float* pts, int n, uint8_t* desc, uint8_t* kept) {
        cudaStream_t st = ctx->stream;
        if (n > cap) { alva_set_error("System: %d keypoints exceed the frame capacity %d", n, cap); return ALVA_E_CAPACITY; }
        if (!blur_valid) { if (int e = alva_k_orb_blur(ctx, gray_raw(), blur_dev, w, h, 1, 0)) return e; blur_valid = true; }
        int32_t nn = n;
        SYS_CUDA(cudaMemcpyAsync(pri_dev, pts, (size_t)n * 8, cudaMemcpyHostToDevice, st));
        SYS_CUDA(cudaMemcpyAsync(cnt_dev + 2, &nn, 4, cudaMemcpyHostToDevice, st));
        if (int e = alva_k_orb_describe(ctx, gray_raw(), blur_dev, w, h, 1, pri_dev, cnt_dev + 2, cap, 0, desc_dev, flag_dev, nullptr)) return e;
        SYS_CUDA(cudaMemcpyAsync(desc, desc_dev, (size_t)n * 32, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaMemcpyAsync(kept, flag_dev, n, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        return 0;
    }

    // FeatureTracker::fbKltTracking(prev pyramid, cur pyramid, 9, levels, 30, 0.5, pts, priors, status)
    int klt(const float* pts, float* priors, int n, int levels, uint8_t* good) {
        cudaStream_t st = ctx->stream;
        if (n > cap) { alva_set_error("System: %d keypoints exceed the frame capacity %d", n, cap); return ALVA_E_CAPACITY; }
        stg.reset();
        float *hp, *hq;
        uint8_t* hg;
        float* dp = stg.take<float>((size_t)2 * n, &hp);
        float* dq = stg.take<float>((size_t)2 * n, &hq);
        const size_t q_off = (uint8_t*)dq - stg.d, up_end = stg.off;
        uint8_t* dg = stg.take<uint8_t>(n, &hg);
        float *hu = nullptr, *du = has_dist ? stg.take<float>((size_t)2 * n, &hu) : nullptr;   // the tracked points, undistorted
        memcpy(hp, pts, (size_t)n * 8);
        memcpy(hq, priors, (size_t)n * 8);
        SYS_CUDA(cudaMemcpyAsync(stg.d, stg.h, up_end, cudaMemcpyHostToDevice, st));
        const int prev = cur ^ 1;
        if (int e = alva_k_klt_fb(ctx, img[prev], der[prev], img[cur], der[cur], w, h, 1, nlev - 1, levels, 9, 30.0f, 0.5f, dp, dq, nullptr, n, dg))
            return e;
        if (has_dist)   // Frame::computeKeypoint's undistortImagePoint of every tracked keypoint (frame.cpp:101-109)
            if (int e = alva_undistort_points_launch(ctx, dq, nullptr, 1, n, K4, D4, du)) return e;
        SYS_CUDA(cudaMemcpyAsync(stg.h + q_off, stg.d + q_off, stg.off - q_off, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        memcpy(priors, hq, (size_t)n * 8);
        memcpy(good, hg, n);
        if (has_dist) unpx_host.assign(hu, hu + 2 * (size_t)n);
        return 0;
    }

    // test hook (alva_system_debug_set_initialisation): the result the next 5-point initialisation returns instead of running
    std::vector<double> init_Rt;
    std::vector<uint8_t> init_outlier;
    int essential(const double* b1, const double* b2, int n, float fx, float fy, double* Rt, uint8_t* outl) {
        cudaStream_t st = ctx->stream;
        if (n > cap) { alva_set_error("System: %d correspondences exceed the frame capacity %d", n, cap); return ALVA_E_CAPACITY; }
        if (init_Rt.size() == 12 && (int)init_outlier.size() == n) {
            memcpy(Rt, init_Rt.data(), 12 * sizeof(double));
            memcpy(outl, init_outlier.data(), n);
            init_Rt.clear(); init_outlier.clear();
            return 1;
        }
        double *A = dbl_dev, *Bv = dbl_dev + 3 * (size_t)cap, *S = dbl_dev + 9 * (size_t)cap;
        SYS_CUDA(cudaMemcpyAsync(A, b1, (size_t)n * 24, cudaMemcpyHostToDevice, st));
        SYS_CUDA(cudaMemcpyAsync(Bv, b2, (size_t)n * 24, cudaMemcpyHostToDevice, st));
        // sampler seed: the reference draws from the clock (state.hpp:67, multiViewRandomEnabled_ = true); any seed is a valid
        // behaviour, the pinned one (12345, what doRandom = false selects) makes runs repeatable
        if (int e = alva_k_essential_5pt(ctx, 1, n, A, Bv, nullptr, 100, 3.0f, 1, fx, fy, 12345u, S, flag_dev, S + 16)) return e;
        double host[20];
        SYS_CUDA(cudaMemcpyAsync(host, S, sizeof host, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaMemcpyAsync(outl, flag_dev, n, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        memcpy(Rt, host, 12 * sizeof(double));
        return host[16] != 0.0 ? 1 : 0;
    }

    int p3p(const double* bv, const double* X, int n, float fx, float fy, double* T12, uint8_t* outl) {
        cudaStream_t st = ctx->stream;
        if (n > cap) { alva_set_error("System: %d points exceed the frame capacity %d", n, cap); return ALVA_E_CAPACITY; }
        double *A = dbl_dev, *Bv = dbl_dev + 3 * (size_t)cap, *S = dbl_dev + 9 * (size_t)cap;
        SYS_CUDA(cudaMemcpyAsync(A, bv, (size_t)n * 24, cudaMemcpyHostToDevice, st));
        SYS_CUDA(cudaMemcpyAsync(Bv, X, (size_t)n * 24, cudaMemcpyHostToDevice, st));
        if (int e = alva_k_p3p_lmeds(ctx, 1, n, A, Bv, nullptr, 100, 3.0f, fx, fy, 12345u, S, flag_dev, S + 16)) return e;
        double host[20];
        SYS_CUDA(cudaMemcpyAsync(host, S, sizeof host, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaMemcpyAsync(outl, flag_dev, n, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        memcpy(T12, host, 12 * sizeof(double));
        return host[16] != 0.0 ? 1 : 0;
    }

    // ceresPnP(unpx, wpts, Twc, 5 iterations, chi2 5.9915, robust, L2 refinement, fx, fy, cx, cy) (visual_frontend.cpp:359-375).
    // The pose of a frame tracked without P3P (p3pEnabled_ off: PnP from the motion prior): one upload, one launch, one download
    // and one synchronisation, through the staging buffer.
    int pnp(const double* uv, const double* X, int n, const double* K4, double* pose7, uint8_t* outl) {
        cudaStream_t st = ctx->stream;
        if (n > cap) { alva_set_error("System: %d points exceed the frame capacity %d", n, cap); return ALVA_E_CAPACITY; }
        stg.reset();
        double *hu, *hx, *hs;
        uint8_t* ho;
        double* du = stg.take<double>((size_t)2 * n, &hu);
        double* dx = stg.take<double>((size_t)3 * n, &hx);
        double* ds = stg.take<double>(28, &hs);   // [0,4) K  [4,11) pose in / out  [16,28) summary
        const size_t up_end = stg.off, down_off = (uint8_t*)ds - stg.d;
        uint8_t* dout = stg.take<uint8_t>(n, &ho);
        if (!stg.fits(stg.off)) { alva_set_error("System: staging buffer too small for %d points", n); return ALVA_E_CAPACITY; }
        memcpy(hu, uv, (size_t)n * 16); memcpy(hx, X, (size_t)n * 24);
        memcpy(hs, K4, 32); memcpy(hs + 4, pose7, 56);
        SYS_CUDA(cudaMemcpyAsync(stg.d, stg.h, up_end, cudaMemcpyHostToDevice, st));
        const float chi2 = 5.9915f;   // State::robustCostThreshold_; ceresPnP takes it as float and uses sqrt(chi2) as the Huber width
        if (int e = alva_k_pnp(ctx, 1, n, ds, du, dx, nullptr, ds + 4, (double)sqrtf(chi2), (double)chi2, 5, 1, 1, dout, ds + 16)) return e;
        SYS_CUDA(cudaMemcpyAsync(stg.h + down_off, stg.d + down_off, stg.off - down_off, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        memcpy(pose7, hs + 4, 56);
        memcpy(outl, ho, n);
        return hs[16 + 10] != 0.0 ? 1 : 0;
    }

    // P3P-LMedS + hand-over + PnP of one frame with one upload, one download and ONE synchronisation (system_core.h replays the
    // host-side decisions of VisualFrontend::computePose on the results).  T12 [12] / ok1: P3P; o1 [n]: its outliers; pose7 / ok2:
    // PnP started from the P3P pose on the survivors; o2 [n - #o1]: its outliers, in the survivors' order.
    bool has_pose_chain() const { return true; }
    int pose_chain(const double* bv, const double* X, const double* uv, int n, const double* K4, float fxf, float fyf, double* T12,
                   uint8_t* o1, int& ok1, double* pose7, uint8_t* o2, int& ok2) {
        cudaStream_t st = ctx->stream;
        if (n > cap) { alva_set_error("System: %d points exceed the frame capacity %d", n, cap); return ALVA_E_CAPACITY; }
        stg.reset();
        double *hb, *hx, *hu, *hk, *hs;
        uint8_t *ho1, *ho2;
        double* db = stg.take<double>((size_t)3 * n, &hb);
        double* dx = stg.take<double>((size_t)3 * n, &hx);
        double* du = stg.take<double>((size_t)2 * n, &hu);
        double* dk = stg.take<double>(4, &hk);
        const size_t up_end = stg.off;
        double* ds = stg.take<double>(48, &hs);            // [0,12) T12  [12,16) P3P info  [16,23) pose7  [24,36) PnP summary  [40] n2
        const size_t down_off = (uint8_t*)ds - stg.d;
        uint8_t* d1 = stg.take<uint8_t>(n, &ho1);
        uint8_t* d2 = stg.take<uint8_t>(n, &ho2);
        const size_t down_end = stg.off;
        double* du2 = stg.take<double>((size_t)2 * n, (double**)nullptr);
        double* dx2 = stg.take<double>((size_t)3 * n, (double**)nullptr);
        if (!stg.fits(stg.off)) { alva_set_error("System: staging buffer too small for %d points", n); return ALVA_E_CAPACITY; }
        memcpy(hb, bv, (size_t)n * 24); memcpy(hx, X, (size_t)n * 24); memcpy(hu, uv, (size_t)n * 16); memcpy(hk, K4, 32);
        SYS_CUDA(cudaMemcpyAsync(stg.d, stg.h, up_end, cudaMemcpyHostToDevice, st));
        const float chi2 = 5.9915f;   // State::robustCostThreshold_; ceresPnP: Huber width std::sqrt(float)
        if (int e = alva_pose_chain_launch(ctx, n, n, db, dx, du, dk, fxf, fyf, 12345u, ds, ds + 12, d1, du2, dx2, (int32_t*)(ds + 40), ds + 16, d2,
                                           ds + 24, (double)sqrtf(chi2), (double)chi2))
            return e;
        SYS_CUDA(cudaMemcpyAsync(stg.h + down_off, stg.d + down_off, down_end - down_off, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        memcpy(T12, hs, 96);
        ok1 = hs[12] != 0.0 ? 1 : 0;
        memcpy(pose7, hs + 16, 56);
        ok2 = hs[24 + 10] != 0.0 ? 1 : 0;
        memcpy(o1, ho1, n);
        memcpy(o2, ho2, n);
        return 0;
    }

    // ---- variable-size problems (local BA, local-map matching): one growable device arena, bump-allocated per call
    uint8_t* arena = nullptr;
    size_t arena_cap = 0, arena_off = 0;
    int arena_begin(size_t bytes) {
        bytes += 4096;
        if (bytes > arena_cap) {
            if (arena) { cudaFree(arena); arena = nullptr; arena_cap = 0; }
            const size_t want = bytes + bytes / 2;
            SYS_CUDA(cudaMalloc(&arena, want));
            arena_cap = want;
        }
        arena_off = 0;
        return 0;
    }
    static size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }
    template <class T> T* arena_take(size_t n) { T* p = (T*)(arena + arena_off); arena_off += al256(n * sizeof(T) + 16); return p; }
    template <class T> T* arena_put(const T* host, size_t n) {
        T* p = arena_take<T>(n);
        if (n) cudaMemcpyAsync(p, host, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream);
        return p;
    }

    bool has_ba_local() const { return true; }
    bool has_match_to_map() const { return true; }

    // the numerical body of Optimizer::localBA (optimizer.cpp:251-359): two solves and both outlier passes in one launch sequence
    int ba_local(alva_sys::BaProblem& bp, int32_t* flags) {
        cudaStream_t st = ctx->stream;
        const size_t nkf = bp.nkf, nlm = bp.nlm, nobs = bp.nobs;
        if (int e = arena_begin(al256(32) + al256(nkf * 56) + al256(nkf) + 3 * al256(nlm * 16) + 4 * al256(nobs * 16) + 16 * 256)) return e;
        double* calib = arena_put(bp.calib, 4);
        double* poses = arena_put(bp.poses.data(), nkf * 7);
        uint8_t* pc = arena_put(bp.pose_const.data(), nkf);
        double* invd = arena_put(bp.invd.data(), nlm);
        int32_t* akf = arena_put(bp.anch_kf.data(), nlm);
        double* auv = arena_put(bp.anch_uv.data(), nlm * 2);
        int32_t* okf = arena_put(bp.obs_kf.data(), nobs);
        int32_t* olm = arena_put(bp.obs_lm.data(), nobs);
        double* ouv = arena_put(bp.obs_uv.data(), nobs * 2);
        int32_t* fl = arena_take<int32_t>(nobs);
        SYS_CUDA(cudaMemsetAsync(fl, 0, nobs * 4, st));
        const float chi2 = 5.9915f;   // State::robustCostThreshold_ (float); the Huber width is std::sqrt(float) (optimizer.cpp:22)
        if (int e = alva_k_ba_local(ctx, 1, (int)nkf, (int)nlm, (int)nobs, calib, poses, pc, invd, akf, auv, okf, olm, ouv, (double)sqrtf(chi2),
                                    (double)chi2, 5, fl, nullptr))
            return e;
        SYS_CUDA(cudaMemcpyAsync(bp.poses.data(), poses, nkf * 56, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaMemcpyAsync(bp.invd.data(), invd, nlm * 8, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaMemcpyAsync(flags, fl, nobs * 4, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        return 0;
    }

    // Mapper::matchToMap(frame, 2 px, 0.2, local map) (mapper.cpp:332)
    int match_to_map(const alva_sys::MatchProblem& m, std::vector<int>& kp_match) {
        cudaStream_t st = ctx->stream;
        const size_t n_kp = m.kp_id.size(), n_mp = m.mp_id.size(), n_kf = m.kf_id.size(), n_obs = m.obs_kfid.size(), n_local = m.local_mp.size();
        if (!n_kp || !n_mp || !n_local) return 0;
        std::vector<int32_t> obs_kf(n_obs);   // keyframe id -> index into kf_Twc
        for (size_t o = 0; o < n_obs; o++) { int ki = 0; while (m.kf_id[ki] != m.obs_kfid[o]) ki++; obs_kf[o] = ki; }
        std::vector<uint8_t> desc = m.desc;
        if (desc.empty()) desc.assign(32, 0);
        const double kf0[7] = {0, 0, 0, 0, 0, 0, 1};
        if (int e = arena_begin(al256(56) + 2 * al256(n_kp * 8) + al256(n_kf * 56 + 56) + al256(n_mp * 24) + al256(n_mp) + 2 * al256((n_mp + 1) * 4) +
                                al256(n_obs * 4) + al256(n_obs * 8) + al256(desc.size()) + al256(n_local * 4) + al256(n_kp * 4) + 20 * 256))
            return e;
        double* Tc = arena_put(m.Twc_cur, 7);
        int32_t* kpmp = arena_put(m.kp_mp.data(), n_kp);
        float* kppx = arena_put(m.kp_px.data(), n_kp * 2);
        double* kfT = n_kf ? arena_put(m.kf_Twc.data(), n_kf * 7) : arena_put(kf0, 7);
        double* wpt = arena_put(m.mp_wpt.data(), n_mp * 3);
        uint8_t* is3 = arena_put(m.mp_is3d.data(), n_mp);
        int32_t* os = arena_put(m.obs_start.data(), n_mp + 1);
        int32_t* ok = arena_put(obs_kf.data(), n_obs);
        float* op = arena_put(m.obs_px.data(), n_obs * 2);
        int32_t* ds = arena_put(m.desc_start.data(), n_mp + 1);
        uint8_t* dd = arena_put(desc.data(), desc.size());
        int32_t* lm = arena_put(m.local_mp.data(), n_local);
        int32_t* out = arena_take<int32_t>(n_kp);
        int32_t* nm = arena_take<int32_t>(4);
        if (int e = alva_k_match_to_map_dist(ctx, w, h, cell, fx, fy, cx, cy, Tc, (int)n_kp, kpmp, kppx, m.nkp3d, (int)(n_kf ? n_kf : 1), kfT, (int)n_mp,
                                             wpt, is3, os, ok, op, ds, dd, (int)n_local, lm, 2.0f, 0.2f, out, nullptr, nm, m.has_dist ? m.dist : nullptr))
            return e;
        std::vector<int32_t> host(n_kp);
        SYS_CUDA(cudaMemcpyAsync(host.data(), out, n_kp * 4, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        for (size_t i = 0; i < n_kp; i++) kp_match[i] = host[i];
        return 0;
    }
    double fx = 0, fy = 0, cx = 0, cy = 0;

    int triangulate(const double* T7, const double* bl, const double* br, int n, double* out) {
        cudaStream_t st = ctx->stream;
        if (n > cap) { alva_set_error("System: %d points exceed the frame capacity %d", n, cap); return ALVA_E_CAPACITY; }
        double *A = dbl_dev, *Bv = dbl_dev + 3 * (size_t)cap, *O = dbl_dev + 6 * (size_t)cap, *S = dbl_dev + 9 * (size_t)cap;
        SYS_CUDA(cudaMemcpyAsync(S, T7, 56, cudaMemcpyHostToDevice, st));
        SYS_CUDA(cudaMemcpyAsync(A, bl, (size_t)n * 24, cudaMemcpyHostToDevice, st));
        SYS_CUDA(cudaMemcpyAsync(Bv, br, (size_t)n * 24, cudaMemcpyHostToDevice, st));
        if (int e = alva_k_triangulate(ctx, S, A, Bv, n, O)) return e;
        SYS_CUDA(cudaMemcpyAsync(out, O, (size_t)n * 24, cudaMemcpyDeviceToHost, st));
        SYS_CUDA(cudaStreamSynchronize(st));
        return 0;
    }
};

}  // namespace

class System {
public:
    System() : core_(be_) {}
    ~System() {
        for (void* p : pinned_) { cudaHostUnregister(p); cudaGetLastError(); }
        be_.release();
    }

    int configure(int imageWidth, int imageHeight, double fx, double fy, double cx, double cy, double k1, double k2, double p1,
                  double p2) {
        configured_ = false;
        if (k1 != 0. || k2 != 0. || p1 != 0. || p2 != 0.) {
            alva_set_error("System::configure: non-zero lens distortion is not accepted here (the reference's shim always passes zeros); "
                           "configure with zeros, then set the coefficients with alva_system_set_distortion");
            return ALVA_E_INVALID;
        }
        if (int e = be_.init(device_, imageWidth, imageHeight)) return e;
        be_.fx = fx; be_.fy = fy; be_.cx = cx; be_.cy = cy;
        core_.configure(imageWidth, imageHeight, fx, fy, cx, cy);
        configured_ = true;
        return 0;
    }

    // keeps the preset and the CLAHE setting (State::reset leaves them, state.cpp) and the lens model
    void reset() { if (configured_) core_.reset(); }

    // CameraCalibration's k1 k2 p1 p2 (camera_calibration.cpp:3-24): the tracker and the map restart under the new model;
    // configure() sets them back to zero
    int setDistortion(double k1, double k2, double p1, double p2) {
        if (!configured_) { alva_set_error("System: not configured"); return ALVA_E_STATE; }
        const double d[4] = {k1, k2, p1, p2};
        for (double v : d)
            if (!std::isfinite(v)) { alva_set_error("alva_system_set_distortion: non-finite coefficient"); return ALVA_E_INVALID; }
        if (int e = be_.set_distortion(d)) return e;
        core_.setDistortion(d);
        return 0;
    }

    // State::claheEnabled_ / claheContrastLimit_ / claheTileSize_ and VisualFrontend's grid Size(imgWidth_ / tile, imgHeight_ / tile)
    // (visual_frontend.cpp:16-18: a double division, truncated); configure() turns it off again (system.cpp:17)
    int setClahe(int enabled, double clip_limit, int tile_size) {
        if (!configured_) { alva_set_error("System: not configured"); return ALVA_E_STATE; }
        const int tx = tile_size > 0 ? core_width() / tile_size : 0, ty = tile_size > 0 ? core_height() / tile_size : 0;
        if (tx < 1 || ty < 1 || !(clip_limit >= 0.0)) {
            alva_set_error("alva_system_set_clahe: tile size %d gives a %dx%d grid, clip limit %g", tile_size, tx, ty, clip_limit);
            return ALVA_E_INVALID;
        }
        return be_.set_clahe(enabled != 0, (float)clip_limit, tx, ty);
    }

    // The reference's preset table (state.hpp:9-17): frameMaxCellSize_, claheEnabled_ (with State's clip 3 / tile 50),
    // mapKeyframeFilteringRatio_, p3pEnabled_.  DEFAULT is what configure() sets (system.cpp:15-19).  The frame grid changes, so
    // the tracker and the map restart (as reset()); the lens model stays; a later setClahe() overrides the CLAHE field.
    int setPreset(int preset) {
        struct Row { int cell; float ratio; bool p3p, clahe; };
        static const Row table[4] = {{40, 0.95f, true, false}, {50, 0.9f, true, false}, {45, 0.9f, false, false}, {35, 0.95f, false, true}};
        if (!configured_) { alva_set_error("System: not configured"); return ALVA_E_STATE; }
        if (preset < ALVA_PRESET_DEFAULT || preset > ALVA_PRESET_ACCURATE) {
            alva_set_error("alva_system_set_preset: unknown preset %d", preset);
            return ALVA_E_INVALID;
        }
        const Row& r = table[preset];
        if (int e = be_.set_cell(r.cell)) return e;
        core_.setPreset(r.cell, r.ratio, r.p3p);
        return setClahe(r.clahe ? 1 : 0, 3.0, 50);   // State::claheContrastLimit_ = 3, claheTileSize_ = 50 (state.hpp:44-45)
    }

    // returns the reference's status codes; pose16 layout as Utils::toPoseArray (src/slam/src/utils.cpp:3-27)
    int findCameraPose(const uint8_t* rgba, double t_ms, float* pose16) {
        if (!configured_) { alva_set_error("System: not configured"); return ALVA_E_STATE; }
        const int st = processGuarded(rgba, t_ms);
        if (st < 0) return st;
        writePose(core_.cur.Twc, pose16);   // the current frame's Twc in every case (identity after a reset / before initialisation)
        return st;
    }
    int findCameraPose(const uint8_t* rgba, float* pose16) { return findCameraPose(rgba, nowMs(), pose16); }

    int findCameraPoseWithIMU(const uint8_t* rgba, const double* imu, float* pose16) {
        if (!configured_) { alva_set_error("System: not configured"); return ALVA_E_STATE; }
        const int st = processGuarded(rgba, nowMs());
        if (st < 0) return st;
        // system.cpp:66-104: rotation from the device orientation quaternion (w, -x, y, z), inverted; the translation follows the
        // visual track while its status is 1 (increments of Twc.translation accumulated into currTranslation_)
        const double qw = imu[0], qx = -imu[1], qy = imu[2], qz = imu[3];
        const double n = sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
        const double w = qw / n, x = qx / n, y = qy / n, z = qz / n;
        const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                             2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                             2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
        if (st == 1) {
            for (int i = 0; i < 3; i++) { imu_t_[i] += core_.cur.Twc.t[i] - imu_prev_[i]; imu_prev_[i] = core_.cur.Twc.t[i]; }
        } else {
            imu_prev_[0] = imu_prev_[1] = imu_prev_[2] = 0.;
        }
        for (int i = 0; i < 16; i++) pose16[i] = 0.f;
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++) pose16[4 * r + c] = (float)R[3 * c + r];
        pose16[12] = (float)imu_t_[0]; pose16[13] = (float)imu_t_[1]; pose16[14] = (float)imu_t_[2];
        pose16[15] = 1.f;
        return 1;
    }

    // system.cpp:123-137, 177-342 as intended (system_core.h::findPlane lists what the reference's own code actually does)
    int findPlane(float* out16, int numIterations) { return configured_ ? core_.findPlane(out16, numIterations) : 0; }

    // (x, y) = truncated undistorted position of the frame's 2-D keypoints (Frame::getKeypoints2d order); writes min(n, cap)
    // pairs, returns the true count (the reference overruns its 4096-int buffer here, SURVEY 8b)
    int getFramePoints(int32_t* xy, int cap_pairs) {
        int n = 0;
        for (auto& kv : core_.cur.kps) {
            if (kv.second.is3d) continue;
            if (n < cap_pairs) { xy[2 * n] = (int)kv.second.ux; xy[2 * n + 1] = (int)kv.second.uy; }
            n++;
        }
        return n;
    }
    // every keypoint of the frame, in the frame's own order: track id (== keypoint id == map point id, map_manager.cpp:166-191),
    // pixel position, 3-D flag and (for 3-D keypoints) the map point's world position
    int getTracks(int32_t* ids, float* px, uint8_t* is3d, double* wpt, int cap) {
        int n = 0;
        for (auto& kv : core_.cur.kps) {
            const alva_sys::Keypoint& k = kv.second;
            if (n < cap) {
                ids[n] = k.id; px[2 * n] = k.px; px[2 * n + 1] = k.py;
                if (is3d) is3d[n] = k.is3d ? 1 : 0;
                if (wpt) {
                    auto mp = core_.mappoints.find(k.id);
                    for (int i = 0; i < 3; i++) wpt[3 * n + i] = (mp != core_.mappoints.end() && mp->second.is3d) ? mp->second.p[i] : 0.0;
                }
            }
            n++;
        }
        return n;
    }
    // the keypoints' ORB descriptors (same order as getTracks): FeatureExtractor::describeFeaturePoints at keyframe creation
    // (feature_extractor.cpp:160-214; empty for points within 31 px of the border, orb.cpp:1130)
    int getDescriptors(uint8_t* desc, uint8_t* has, int cap) {
        int n = 0;
        for (auto& kv : core_.cur.kps) {
            if (n < cap) { memcpy(desc + 32 * (size_t)n, kv.second.desc, 32); has[n] = kv.second.has_desc ? 1 : 0; }
            n++;
        }
        return n;
    }
    int getPose(double* Twc7) { core_.cur.Twc.to7(Twc7); return 0; }
    // page-lock a caller-owned frame buffer that is reused from call to call (the reference's shim allocates its image buffer once,
    // system.js:63-67): uploads from it then run at the host link's rate instead of through the driver's pageable staging
    int pinBuffer(void* ptr, size_t bytes) {
        if (cudaHostRegister(ptr, bytes, cudaHostRegisterDefault) != cudaSuccess) {
            alva_set_error("alva_system_pin_buffer: cudaHostRegister -> %s", cudaGetErrorString(cudaGetLastError()));
            return ALVA_E_CUDA;
        }
        pinned_.push_back(ptr);
        return 0;
    }
    int unpinBuffer(void* ptr) {
        for (size_t i = 0; i < pinned_.size(); i++)
            if (pinned_[i] == ptr) { cudaHostUnregister(ptr); cudaGetLastError(); pinned_.erase(pinned_.begin() + i); return 0; }
        return ALVA_E_INVALID;
    }
    void debugSetInitialisation(const double* Rt12, const uint8_t* outlier, int n) {
        be_.init_Rt.assign(Rt12, Rt12 + 12);
        be_.init_outlier.assign(outlier, outlier + n);
    }
    // {frame id, keyframe id, #keypoints, #3-D keypoints, initialised, #keyframes, #occupied cells, #map point ids}
    int getInfo(int32_t* out8) {
        out8[0] = core_.cur.id; out8[1] = core_.cur.kfid; out8[2] = core_.cur.n; out8[3] = core_.cur.n3d;
        out8[4] = core_.ready_for_init ? 1 : 0; out8[5] = core_.n_kf; out8[6] = core_.cur.nocc; out8[7] = core_.n_mp_ids;
        return 0;
    }
    int numMatched() const { return core_.cur.n; }
    int device_ = 0;

private:
    // no exception crosses the C boundary (the reference aborts on its .at() throws; a library must not)
    int processGuarded(const uint8_t* rgba, double t_ms) {
        try {
            return core_.process(rgba, t_ms);
        } catch (const std::exception& e) {
            alva_set_error("System: inconsistent map state (%s); tracker reset", e.what());
            core_.reset();
            return ALVA_E_STATE;
        }
    }
    static double nowMs() {   // system.cpp:114: milliseconds since the epoch
        return (double)std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::system_clock::now().time_since_epoch()).count();
    }
    static void writePose(const alva_sys::Se3& T, float* p) {
        double R[9];
        T.R(R);
        for (int r = 0; r < 3; r++) { for (int c = 0; c < 3; c++) p[4 * r + c] = (float)R[3 * r + c]; p[4 * r + 3] = 0.f; }
        p[12] = (float)T.t[0]; p[13] = (float)T.t[1]; p[14] = (float)T.t[2]; p[15] = 1.f;
    }
    int core_width() const { return be_.w; }
    int core_height() const { return be_.h; }
    std::vector<void*> pinned_;
    CudaBackend be_;
    alva_sys::SystemCore<CudaBackend> core_;
    bool configured_ = false;
    double imu_t_[3] = {0, 0, 0}, imu_prev_[3] = {0, 0, 0};
};

struct alva_system { System sys; };

extern "C" alva_system* alva_system_create(int device) {
    alva_system* s = new alva_system();
    s->sys.device_ = device;
    return s;
}
extern "C" void alva_system_destroy(alva_system* s) {
    if (!s) return;
    AlvaDeviceGuard guard__(s->sys.device_);
    delete s;
}
extern "C" int alva_system_configure(alva_system* s, int w, int h, double fx, double fy, double cx, double cy, double k1,
                                     double k2, double p1, double p2) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || w < 64 || h < 64) { alva_set_error("alva_system_configure: bad argument"); return ALVA_E_INVALID; }
    return s->sys.configure(w, h, fx, fy, cx, cy, k1, k2, p1, p2);
}
extern "C" int alva_system_set_clahe(alva_system* s, int enabled, double clip_limit, int tile_size) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s) { alva_set_error("alva_system_set_clahe: null handle"); return ALVA_E_INVALID; }
    return s->sys.setClahe(enabled, clip_limit, tile_size);
}
extern "C" int alva_system_set_distortion(alva_system* s, double k1, double k2, double p1, double p2) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s) { alva_set_error("alva_system_set_distortion: null handle"); return ALVA_E_INVALID; }
    return s->sys.setDistortion(k1, k2, p1, p2);
}
extern "C" int alva_system_set_preset(alva_system* s, int preset) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s) { alva_set_error("alva_system_set_preset: null handle"); return ALVA_E_INVALID; }
    return s->sys.setPreset(preset);
}
extern "C" int alva_system_reset(alva_system* s) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1); if (!s) return ALVA_E_INVALID; s->sys.reset(); return 0; }
extern "C" int alva_system_find_camera_pose(alva_system* s, const uint8_t* rgba, float* pose16) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !rgba || !pose16) { alva_set_error("alva_system_find_camera_pose: bad argument"); return ALVA_E_INVALID; }
    return s->sys.findCameraPose(rgba, pose16);
}
extern "C" int alva_system_find_camera_pose_ts(alva_system* s, const uint8_t* rgba, double t_ms, float* pose16) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !rgba || !pose16) { alva_set_error("alva_system_find_camera_pose_ts: bad argument"); return ALVA_E_INVALID; }
    return s->sys.findCameraPose(rgba, t_ms, pose16);
}
extern "C" int alva_system_find_camera_pose_imu(alva_system* s, const uint8_t* rgba, const double* imu, float* pose16) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !rgba || !imu || !pose16) { alva_set_error("alva_system_find_camera_pose_imu: bad argument"); return ALVA_E_INVALID; }
    return s->sys.findCameraPoseWithIMU(rgba, imu, pose16);
}
extern "C" int alva_system_find_plane(alva_system* s, float* out16, int iterations) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !out16) return ALVA_E_INVALID;
    return s->sys.findPlane(out16, iterations);
}
extern "C" int alva_system_get_frame_points(alva_system* s, int32_t* xy, int cap_pairs) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !xy || cap_pairs < 0) return ALVA_E_INVALID;
    return s->sys.getFramePoints(xy, cap_pairs);
}
extern "C" int alva_system_num_matched(alva_system* s) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1); return s ? s->sys.numMatched() : ALVA_E_INVALID; }
extern "C" int alva_system_get_tracks(alva_system* s, int32_t* ids, float* px, uint8_t* is3d, double* wpt, int cap) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !ids || !px || cap < 0) return ALVA_E_INVALID;
    return s->sys.getTracks(ids, px, is3d, wpt, cap);
}
extern "C" int alva_system_get_descriptors(alva_system* s, uint8_t* desc, uint8_t* has, int cap) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !desc || !has || cap < 0) return ALVA_E_INVALID;
    return s->sys.getDescriptors(desc, has, cap);
}
extern "C" int alva_system_debug_set_initialisation(alva_system* s, const double* Rt12, const uint8_t* outlier, int n) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !Rt12 || !outlier || n < 8) return ALVA_E_INVALID;
    s->sys.debugSetInitialisation(Rt12, outlier, n);
    return 0;
}
extern "C" int alva_system_pin_buffer(alva_system* s, void* host_ptr, size_t bytes) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1);
    if (!s || !host_ptr || !bytes) return ALVA_E_INVALID;
    return s->sys.pinBuffer(host_ptr, bytes);
}
extern "C" int alva_system_unpin_buffer(alva_system* s, void* host_ptr) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1); return (s && host_ptr) ? s->sys.unpinBuffer(host_ptr) : ALVA_E_INVALID; }
extern "C" int alva_system_get_pose(alva_system* s, double* Twc7) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1); return (s && Twc7) ? s->sys.getPose(Twc7) : ALVA_E_INVALID; }
extern "C" int alva_system_get_info(alva_system* s, int32_t* out8) { AlvaDeviceGuard guard__(s ? s->sys.device_ : -1); return (s && out8) ? s->sys.getInfo(out8) : ALVA_E_INVALID; }

// N independent camera streams in one call: handles[i] processes rgba[i] (time stamp t_ms[i]; t_ms may be NULL = the system
// clock); poses16 [n][16], status [n] = the per-stream return value of alva_system_find_camera_pose_ts.  Every System owns its
// CUDA stream and its state, so the streams run concurrently on the device: the call drives them from n host threads (the last
// one is the caller's) and returns when all are done.  Returns 0, or the first negative status.
extern "C" int alva_system_find_camera_pose_batch(alva_system* const* handles, const uint8_t* const* rgba, const double* t_ms, int n,
                                                  float* poses16, int* status) {
    if (!handles || !rgba || !poses16 || !status || n < 1) { alva_set_error("alva_system_find_camera_pose_batch: bad argument"); return ALVA_E_INVALID; }
    for (int i = 0; i < n; i++)
        if (!handles[i] || !rgba[i]) { alva_set_error("alva_system_find_camera_pose_batch: null handle / frame %d", i); return ALVA_E_INVALID; }
    auto one = [&](int i) {
        AlvaDeviceGuard guard__(handles[i]->sys.device_);
        status[i] = t_ms ? handles[i]->sys.findCameraPose(rgba[i], t_ms[i], poses16 + 16 * (size_t)i) : handles[i]->sys.findCameraPose(rgba[i], poses16 + 16 * (size_t)i);
    };
    std::vector<std::thread> th;
    th.reserve(n - 1);
    for (int i = 0; i + 1 < n; i++) th.emplace_back(one, i);
    one(n - 1);
    for (auto& t : th) t.join();
    for (int i = 0; i < n; i++) if (status[i] < 0) return status[i];
    return 0;
}
