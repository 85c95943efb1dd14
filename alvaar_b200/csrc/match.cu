// match.cu -- projection-gated matching of the local map to a keyframe's keypoints on the GPU.
//
// What is computed (identical (keypoint -> map point) maps; the CPU restatement is oracle/match_oracle.c, pinned to the
// reference's own Mapper running on its own Frame / MapPoint / MapManager objects):
//   Mapper::matchToMap                     src/slam/src/mapper.cpp:354-587   (caller matchingToLocalMap :293-352)
//   MapPoint::computeMinDescDist           src/slam/src/map_point.cpp:204-222  (cv::norm(NORM_HAMMING), all pairs)
//   Frame::getSurroundingKeypoints         src/slam/src/frame.cpp:313-341
//   CameraCalibration::projectCamToImageDist  src/slam/src/camera_calibration.cpp:34-55  (with distortion: camera_model.h,
//                                             radial-tangential, its full 14-coefficient form, or equidistant fisheye)
//
// How: the reference walks hash maps (map point -> shared_ptr -> per-keyframe descriptor map -> cv::Mat) once per candidate.
// Here the map lives in flat SoA arenas in HBM (world points, CSR observation lists, CSR descriptor lists) and one warp
// handles one local map point: the gates are scalar, the per-candidate work is warp-parallel -- keyframe-set disjointness as
// a 64-bit mask intersection, co-projection errors one keyframe per lane (summed in the reference's order: it accumulates in
// float), the all-pairs 256-bit Hamming minimum with __popc and a shuffle reduction.  The "best / second best / ratio" logic
// per map point and the "smallest distance, last one wins" rule per keypoint are order-sensitive; the first runs in
// candidate order inside the warp, the second is a 64-bit atomicMin on (distance, reversed processing index).
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include "map_geom.cuh"
#include <math.h>

namespace {

struct MatchParams {
    int w, h, cell, ncw, nch;
    double fx, fy, cx, cy;
    const double* Twc_cur;
    int n_kp;
    const int32_t* kp_mp;
    const float* kp_px;
    int nkp3d;
    int n_kf;
    const double* kf_Twc;
    int n_mp;
    const double* mp_wpt;
    const uint8_t* mp_is3d;
    const int32_t* obs_start;
    const int32_t* obs_kf;
    const float* obs_px;
    const int32_t* desc_start;
    const uint8_t* desc;
    int n_local;
    const int32_t* local_mp;
    float max_px_dist, min_dist, view_th;
    // scratch
    uint8_t* mp_observed;
    int32_t* kp_cell;
    int32_t* cell_start;
    int32_t* cell_kp;
    unsigned long long* kbest;
    int32_t* kp_match;
    float* kp_dist;
    int32_t* n_match;
    double dist[4];   // k1 k2 p1 p2 (LENS_RADTAN) or k1 k2 k3 k4 (LENS_FISHEYE)
};
// LENS_FULL's parameters: the same, and the 14 coefficients with their tilt matrices (the other lenses keep MatchParams)
struct MatchParamsFull : MatchParams { alva_cam::LensFull L; };
template <int LENS> struct MatchArgs { using type = MatchParams; };
template <> struct MatchArgs<alva_geom::LENS_FULL> { using type = MatchParamsFull; };

using alva_geom::world_to_cam;
using alva_geom::LENS_NONE;
using alva_geom::LENS_RADTAN;
using alva_geom::LENS_FISHEYE;
using alva_geom::LENS_FULL;
template <int LENS>
__device__ __forceinline__ void project_cam(const typename MatchArgs<LENS>::type& P, const double* c, float* px) {
    const double K4[4] = {P.fx, P.fy, P.cx, P.cy};
    if constexpr (LENS == LENS_FULL) alva_geom::project_cam<LENS>(K4, nullptr, c, px, &P.L);
    else alva_geom::project_cam<LENS>(K4, P.dist, c, px);
}

// one CTA: observed flags, the frame's grid (cell -> keypoints in insertion order), per-keypoint result keys
__global__ void __launch_bounds__(1024) match_prepare_kernel(const MatchParams P) {
    const int tid = threadIdx.x, nt = blockDim.x, ncells = P.ncw * P.nch;
    for (int i = tid; i < P.n_mp; i += nt) P.mp_observed[i] = 0;
    for (int i = tid; i < P.n_kp; i += nt) P.kbest[i] = 0xffffffffffffffffull;
    if (tid == 0) *P.n_match = 0;
    __syncthreads();
    for (int i = tid; i < P.n_kp; i += nt) {
        if (P.kp_mp[i] >= 0 && P.kp_mp[i] < P.n_mp) P.mp_observed[P.kp_mp[i]] = 1;
        const int r = (int)floorf(P.kp_px[2 * i + 1] / (float)P.cell), c = (int)floorf(P.kp_px[2 * i] / (float)P.cell);
        const int idx = r * P.ncw + c;
        P.kp_cell[i] = (r >= 0 && c >= 0 && c < P.ncw && idx < ncells) ? idx : -1;
    }
    __syncthreads();
    // stable counting sort: thread per cell scans the keypoints in insertion order (n_kp x ncells is tiny)
    __shared__ int total;
    if (tid == 0) total = 0;
    for (int c0 = 0; c0 < ncells; c0 += nt) {
        const int c = c0 + tid;
        int cnt = 0;
        if (c < ncells)
            for (int i = 0; i < P.n_kp; i++) cnt += (P.kp_cell[i] == c);
        // exclusive scan of cnt over this chunk of cells (serial by thread 0 over nt values kept in cell_start)
        if (c < ncells) P.cell_start[c + 1] = cnt;
        __syncthreads();
        if (tid == 0) {
            int run = total;
            const int hi = min(ncells, c0 + nt);
            for (int k = c0; k < hi; k++) { const int v = P.cell_start[k + 1]; P.cell_start[k] = run; run += v; }
            P.cell_start[hi] = run;
            total = run;
        }
        __syncthreads();
        if (c < ncells) {
            int pos = P.cell_start[c];
            for (int i = 0; i < P.n_kp; i++)
                if (P.kp_cell[i] == c) P.cell_kp[pos++] = i;
        }
        __syncthreads();
    }
}

template <int LENS>
__global__ void __launch_bounds__(128) match_local_kernel(const typename MatchArgs<LENS>::type P) {
    const int lane = threadIdx.x & 31;
    const int li = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
    if (li >= P.n_local) return;
    const int m = P.local_mp[li];
    if (m < 0 || m >= P.n_mp) return;
    if (P.mp_observed[m]) return;                                               // frame.isObservingKeypoint (mapper.cpp:404)
    const int d0 = P.desc_start[m], nd = P.desc_start[m + 1] - d0;
    if (!P.mp_is3d[m] || nd == 0) return;                                       // :415
    const double wpt[3] = {P.mp_wpt[3 * m], P.mp_wpt[3 * m + 1], P.mp_wpt[3 * m + 2]};
    double campt[3];
    world_to_cam(P.Twc_cur, wpt, campt);
    if (campt[2] < 0.1) return;                                                 // :425
    const float view_angle = (float)(campt[2] / sqrt(campt[0] * campt[0] + campt[1] * campt[1] + campt[2] * campt[2]));
    if (fabs((double)view_angle) < (double)P.view_th) return;                   // :432
    float proj[2];
    project_cam<LENS>(P, campt, proj);
    if (!(proj[0] >= 0 && proj[1] >= 0 && (double)proj[0] < (double)P.w && (double)proj[1] < (double)P.h)) return;
    // keyframes observing this map point, as a bit mask over keyframe indices (n_kf <= 64)
    const int o0 = P.obs_start[m], no = P.obs_start[m + 1] - o0;
    unsigned long long mymask = 0;
    for (int a = lane; a < no; a += 32) mymask |= 1ull << P.obs_kf[o0 + a];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mymask |= __shfl_xor_sync(0xffffffffu, mymask, off);

    const int ncells = P.ncw * P.nch;
    int bestKp = -1, secKp = -1;
    float bestDist = P.min_dist, secDist = P.min_dist;
    const int rkp = (int)floorf(proj[1] / (float)P.cell), ckp = (int)floorf(proj[0] / (float)P.cell);
    for (int r = rkp - 1; r < rkp + 1; r++)
        for (int c = ckp - 1; c < ckp + 1; c++) {
            const int idx = r * P.ncw + c;
            if (r < 0 || c < 0 || idx >= ncells) continue;
            for (int s = P.cell_start[idx]; s < P.cell_start[idx + 1]; s++) {
                const int k = P.cell_kp[s];
                const int km = P.kp_mp[k];
                if (km < 0 || km >= P.n_mp) continue;
                const float ddx = proj[0] - P.kp_px[2 * k], ddy = proj[1] - P.kp_px[2 * k + 1];
                const float pxDist = (float)sqrt((double)ddx * (double)ddx + (double)ddy * (double)ddy);
                if (pxDist > P.max_px_dist) continue;                           // :454
                const int kd0 = P.desc_start[km], knd = P.desc_start[km + 1] - kd0;
                if (knd == 0) continue;                                         // :470
                const int ko0 = P.obs_start[km], kno = P.obs_start[km + 1] - ko0;
                // candidate only if the two map points are never observed in the same keyframe (:476-491)
                unsigned long long kmask = 0;
                for (int a = lane; a < kno; a += 32) kmask |= 1ull << P.obs_kf[ko0 + a];
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) kmask |= __shfl_xor_sync(0xffffffffu, kmask, off);
                if (kmask & mymask) continue;
                // mean distance between the keypoint's pixel in each of its keyframes and the map point projected there
                // (:493-521); the reference accumulates in float, in ascending keyframe order
                float co = 0.f;
                for (int a0 = 0; a0 < kno; a0 += 32) {
                    double dist = 0.0;
                    if (a0 + lane < kno) {
                        double cc[3];
                        float pp[2];
                        world_to_cam(P.kf_Twc + 7 * P.obs_kf[ko0 + a0 + lane], wpt, cc);
                        project_cam<LENS>(P, cc, pp);
                        const float ex = P.obs_px[2 * (ko0 + a0 + lane)] - pp[0], ey = P.obs_px[2 * (ko0 + a0 + lane) + 1] - pp[1];
                        dist = sqrt((double)ex * (double)ex + (double)ey * (double)ey);
                    }
                    const int cnt = min(32, kno - a0);
                    for (int j = 0; j < cnt; j++) co = (float)((double)co + __shfl_sync(0xffffffffu, dist, j));
                }
                if (co / (float)kno > P.max_px_dist) continue;
                // MapPoint::computeMinDescDist: minimum Hamming distance over all descriptor pairs
                int dmin = 1000;
                const int npairs = nd * knd;
                for (int pr = lane; pr < npairs; pr += 32) {
                    const int a = pr / knd, b = pr - a * knd;
                    const uint4* A = reinterpret_cast<const uint4*>(P.desc + 32 * (size_t)(d0 + a));
                    const uint4* B = reinterpret_cast<const uint4*>(P.desc + 32 * (size_t)(kd0 + b));
                    const uint4 a0v = __ldg(A), a1v = __ldg(A + 1), b0v = __ldg(B), b1v = __ldg(B + 1);
                    const int hd = __popc(a0v.x ^ b0v.x) + __popc(a0v.y ^ b0v.y) + __popc(a0v.z ^ b0v.z) + __popc(a0v.w ^ b0v.w) +
                                   __popc(a1v.x ^ b1v.x) + __popc(a1v.y ^ b1v.y) + __popc(a1v.z ^ b1v.z) + __popc(a1v.w ^ b1v.w);
                    dmin = min(dmin, hd);
                }
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) dmin = min(dmin, __shfl_xor_sync(0xffffffffu, dmin, off));
                const float dist = (float)dmin;
                if (dist <= bestDist) { secDist = bestDist; secKp = bestKp; bestDist = dist; bestKp = k; }   // :525-537
                else if (dist <= secDist) { secDist = dist; secKp = k; }
            }
        }
    if (bestKp != -1 && secKp != -1 && 0.9 * (double)secDist < (double)bestDist) bestKp = -1;                // :540-546
    if (bestKp < 0) return;
    // per keypoint: smallest distance, the LAST such map point in processing order wins (`<=`, :565-585)
    if (lane == 0) {
        const unsigned long long key = ((unsigned long long)(unsigned)(int)bestDist << 32) | (unsigned)(0xffffffffu - (unsigned)li);
        atomicMin(P.kbest + bestKp, key);
    }
}

__global__ void match_finalize_kernel(const MatchParams P) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P.n_kp) return;
    const unsigned long long key = P.kbest[k];
    if (key == 0xffffffffffffffffull) { P.kp_match[k] = -1; if (P.kp_dist) P.kp_dist[k] = -1.f; return; }
    const unsigned li = 0xffffffffu - (unsigned)(key & 0xffffffffu);
    P.kp_match[k] = P.local_mp[li];
    if (P.kp_dist) P.kp_dist[k] = (float)(unsigned)(key >> 32);
    atomicAdd(P.n_match, 1);
}

// lens: LENS_NONE (coef4 unused), LENS_RADTAN or LENS_FISHEYE with its four coefficients, or LENS_FULL with F (checked by the
// caller)
int match_to_map_launch(alva_ctx* ctx, int w, int h, int cell, double fx, double fy, double cx, double cy, const double* Twc_cur,
                        int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf, const double* kf_Twc, int n_mp,
                        const double* mp_wpt, const uint8_t* mp_is3d, const int32_t* obs_start, const int32_t* obs_kf,
                        const float* obs_px, const int32_t* desc_start, const uint8_t* desc, int n_local, const int32_t* local_mp,
                        float max_proj_err, float dist_ratio, int32_t* kp_match, float* kp_dist, int32_t* n_match, int lens,
                        const double* coef4, const alva_cam::LensFull* F = nullptr) {
    if (!ctx || !Twc_cur || !kp_mp || !kp_px || !kf_Twc || !mp_wpt || !mp_is3d || !obs_start || !obs_kf || !obs_px || !desc_start ||
        !desc || !local_mp || !kp_match || !n_match || n_kp < 1 || n_mp < 1 || n_local < 1 || cell < 1) {
        alva_set_error("alva_k_match_to_map: bad argument");
        return ALVA_E_INVALID;
    }
    if (n_kf > 64) { alva_set_error("alva_k_match_to_map: at most 64 keyframes (the reference's window is 30), got %d", n_kf); return ALVA_E_INVALID; }
    if (((uintptr_t)desc & 15) != 0) { alva_set_error("alva_k_match_to_map: desc must be 16-byte aligned"); return ALVA_E_INVALID; }
    MatchParamsFull PF{};
    MatchParams& P = PF;
    if (lens == LENS_FULL) PF.L = *F;
    else if (lens != LENS_NONE) for (int i = 0; i < 4; i++) P.dist[i] = coef4[i];
    P.w = w; P.h = h; P.cell = cell;
    P.ncw = (int)ceilf((float)w / (float)cell); P.nch = (int)ceilf((float)h / (float)cell);   // frame.cpp:14-15
    P.fx = fx; P.fy = fy; P.cx = cx; P.cy = cy;
    P.Twc_cur = Twc_cur; P.n_kp = n_kp; P.kp_mp = kp_mp; P.kp_px = kp_px; P.nkp3d = nkp3d; P.n_kf = n_kf; P.kf_Twc = kf_Twc;
    P.n_mp = n_mp; P.mp_wpt = mp_wpt; P.mp_is3d = mp_is3d; P.obs_start = obs_start; P.obs_kf = obs_kf; P.obs_px = obs_px;
    P.desc_start = desc_start; P.desc = desc; P.n_local = n_local; P.local_mp = local_mp;
    // mapper.cpp:365-385, 436: thresholds in the reference's float arithmetic
    const float fovV = (float)(0.5 * h / fy), fovH = (float)(0.5 * w / fx);
    P.view_th = cosf(fovH > fovV ? atanf(fovH) : atanf(fovV));
    P.max_px_dist = max_proj_err;
    if (nkp3d < 30) P.max_px_dist = (float)(P.max_px_dist * 2.);
    P.min_dist = (float)(32 * dist_ratio * 8.);
    const int ncells = P.ncw * P.nch;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t b0 = al((size_t)n_mp), b1 = al((size_t)n_kp * 4), b2 = al((size_t)(ncells + 2) * 4), b3 = al((size_t)n_kp * 4), b4 = al((size_t)n_kp * 8);
    uint8_t* ws = (uint8_t*)alva_scratch(ctx, b0 + b1 + b2 + b3 + b4 + 256);
    if (!ws) return ALVA_E_CUDA;
    P.mp_observed = ws; P.kp_cell = (int32_t*)(ws + b0); P.cell_start = (int32_t*)(ws + b0 + b1); P.cell_kp = (int32_t*)(ws + b0 + b1 + b2);
    P.kbest = (unsigned long long*)(ws + b0 + b1 + b2 + b3);
    P.kp_match = kp_match; P.kp_dist = kp_dist; P.n_match = n_match;
    match_prepare_kernel<<<1, 1024, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    if (lens == LENS_FULL) match_local_kernel<LENS_FULL><<<(n_local * 32 + 127) / 128, 128, 0, ctx->stream>>>(PF);
    else if (lens == LENS_RADTAN) match_local_kernel<LENS_RADTAN><<<(n_local * 32 + 127) / 128, 128, 0, ctx->stream>>>(P);
    else if (lens == LENS_FISHEYE) match_local_kernel<LENS_FISHEYE><<<(n_local * 32 + 127) / 128, 128, 0, ctx->stream>>>(P);
    else match_local_kernel<LENS_NONE><<<(n_local * 32 + 127) / 128, 128, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    match_finalize_kernel<<<(n_kp + 255) / 256, 256, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

}  // namespace

extern "C" int alva_k_match_to_map_dist(alva_ctx* ctx, int w, int h, int cell, double fx, double fy, double cx, double cy,
                                        const double* Twc_cur, int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf,
                                        const double* kf_Twc, int n_mp, const double* mp_wpt, const uint8_t* mp_is3d,
                                        const int32_t* obs_start, const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start,
                                        const uint8_t* desc, int n_local, const int32_t* local_mp, float max_proj_err, float dist_ratio,
                                        int32_t* kp_match, float* kp_dist, int32_t* n_match, const double* dist4) { AlvaDeviceGuard guard__(ctx);
    bool dist = false;
    if (dist4)
        for (int i = 0; i < 4; i++) {
            if (!isfinite(dist4[i])) { alva_set_error("alva_k_match_to_map_dist: non-finite distortion coefficient"); return ALVA_E_INVALID; }
            dist = dist || dist4[i] != 0.0;
        }
    return match_to_map_launch(ctx, w, h, cell, fx, fy, cx, cy, Twc_cur, n_kp, kp_mp, kp_px, nkp3d, n_kf, kf_Twc, n_mp, mp_wpt, mp_is3d,
                               obs_start, obs_kf, obs_px, desc_start, desc, n_local, local_mp, max_proj_err, dist_ratio, kp_match, kp_dist,
                               n_match, dist ? LENS_RADTAN : LENS_NONE, dist4);
}

extern "C" int alva_k_match_to_map_fisheye(alva_ctx* ctx, int w, int h, int cell, double fx, double fy, double cx, double cy,
                                           const double* Twc_cur, int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf,
                                           const double* kf_Twc, int n_mp, const double* mp_wpt, const uint8_t* mp_is3d,
                                           const int32_t* obs_start, const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start,
                                           const uint8_t* desc, int n_local, const int32_t* local_mp, float max_proj_err, float dist_ratio,
                                           int32_t* kp_match, float* kp_dist, int32_t* n_match, const double* fisheye4) { AlvaDeviceGuard guard__(ctx);
    if (!fisheye4) { alva_set_error("alva_k_match_to_map_fisheye: fisheye4 is required (zeros are a valid lens)"); return ALVA_E_INVALID; }
    for (int i = 0; i < 4; i++)
        if (!isfinite(fisheye4[i])) { alva_set_error("alva_k_match_to_map_fisheye: non-finite coefficient"); return ALVA_E_INVALID; }
    return match_to_map_launch(ctx, w, h, cell, fx, fy, cx, cy, Twc_cur, n_kp, kp_mp, kp_px, nkp3d, n_kf, kf_Twc, n_mp, mp_wpt, mp_is3d,
                               obs_start, obs_kf, obs_px, desc_start, desc, n_local, local_mp, max_proj_err, dist_ratio, kp_match, kp_dist,
                               n_match, LENS_FISHEYE, fisheye4);
}

extern "C" int alva_k_match_to_map_full(alva_ctx* ctx, int w, int h, int cell, double fx, double fy, double cx, double cy,
                                        const double* Twc_cur, int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf,
                                        const double* kf_Twc, int n_mp, const double* mp_wpt, const uint8_t* mp_is3d,
                                        const int32_t* obs_start, const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start,
                                        const uint8_t* desc, int n_local, const int32_t* local_mp, float max_proj_err, float dist_ratio,
                                        int32_t* kp_match, float* kp_dist, int32_t* n_match, const double* coeffs, int ncoeffs) { AlvaDeviceGuard guard__(ctx);
    alva_cam::LensFull L;
    if (!alva_cam::make_lens_full(coeffs, ncoeffs, L)) {
        alva_set_error("alva_k_match_to_map_full: coeffs must hold 4, 5, 8, 12 or 14 finite values with |tau_x|, |tau_y| < pi/2");
        return ALVA_E_INVALID;
    }
    return match_to_map_launch(ctx, w, h, cell, fx, fy, cx, cy, Twc_cur, n_kp, kp_mp, kp_px, nkp3d, n_kf, kf_Twc, n_mp, mp_wpt, mp_is3d,
                               obs_start, obs_kf, obs_px, desc_start, desc, n_local, local_mp, max_proj_err, dist_ratio, kp_match, kp_dist,
                               n_match, LENS_FULL, nullptr, &L);
}

extern "C" int alva_k_match_to_map(alva_ctx* ctx, int w, int h, int cell, double fx, double fy, double cx, double cy,
                                   const double* Twc_cur, int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf,
                                   const double* kf_Twc, int n_mp, const double* mp_wpt, const uint8_t* mp_is3d,
                                   const int32_t* obs_start, const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start,
                                   const uint8_t* desc, int n_local, const int32_t* local_mp, float max_proj_err, float dist_ratio,
                                   int32_t* kp_match, float* kp_dist, int32_t* n_match) {
    return alva_k_match_to_map_dist(ctx, w, h, cell, fx, fy, cx, cy, Twc_cur, n_kp, kp_mp, kp_px, nkp3d, n_kf, kf_Twc, n_mp, mp_wpt, mp_is3d,
                                    obs_start, obs_kf, obs_px, desc_start, desc, n_local, local_mp, max_proj_err, dist_ratio, kp_match,
                                    kp_dist, n_match, nullptr);
}
