// klt.cu -- pyramidal Lucas-Kanade tracking of keypoints between consecutive frames, forward-backward checked, for sm_90a.
//
// What is computed (bit-exact with the reference -- positions as float bit patterns, status, min-eigenvalue; the CPU
// restatement is oracle/klt_oracle.c):
//   cv::calcOpticalFlowPyrLK on prebuilt pyramids, flags USE_INITIAL_FLOW | LK_GET_MIN_EIGENVALS, 9x9 window
//        reference: opencv video/src/lkpyramid.cpp:1238-1398, LKTrackerInvoker::operator() :183-722
//   FeatureTracker::fbKltTracking          src/slam/src/feature_tracker.cpp:5-111  (caller visual_frontend.cpp:103-243)
//
// How: every keypoint is independent through all pyramid levels AND through the backward pass, so ONE launch does
// forward LK on all levels, the reference's gates, and the backward LK -- one warp per keypoint, nothing leaves the SM
// between the steps (the reference makes 2 x (levels + 1) passes over its point vectors).
//   * lanes 0..26 own 3 adjacent window pixels each (81 = 9 x 9): bilinear samples in Q14 fixed point, integer exact;
//   * the reference accumulates its (integer-valued) products in float32, and the sums exceed 2^24, so the ORDER is part
//     of the result: it is the order of OpenCV's SSE universal-intrinsic path -- four lanes striding the first 8 window
//     columns plus a scalar accumulator for column 8, lanes reduced as (l0 + l2) + (l1 + l3).  Here 15 (covariance) /
//     10 (mismatch vector) lanes each replay ONE of those accumulator chains from the per-warp shared window, and warp
//     shuffles combine them in the reference's order.  Everything else is parallel;
//   * float expressions are compiled with -fmad=false (Makefile): the reference is SSE code without FMA contraction.
// The 9-px REFLECT_101 image border / constant-0 derivative border that buildOpticalFlowPyramid stores around each level
// (lkpyramid.cpp:726-822) are produced by index arithmetic on the tightly packed levels.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include <float.h>

namespace {

constexpr int WIN = 9;
constexpr int KLT_WARPS = 4;

struct KltParams {
    const uint8_t* prev_img[4];
    const int16_t* prev_der[4];
    const uint8_t* cur_img[4];
    const int16_t* cur_der[4];
    int w[4], h[4];
    int nframes, npts, max_level, max_count, use_initial;
    double eps2;
    float min_eig_thr, error_value, max_fb_dist;
    const float* pts;            // [nframes][npts][2]
    float* next;                 // [nframes][npts][2] in/out
    const int32_t* npts_per_frame;
    uint8_t* status;             // LK: status; FB: good
    float* err;                  // LK only
};

struct __align__(16) WarpWin {
    short dx[84], dy[84], diff[84];
};

__device__ __forceinline__ int refl(int p, int n) { return p < 0 ? -p : (p >= n ? 2 * n - 2 - p : p); }   // n >= 10, |overhang| <= 9

// one pyramid level of one point (LKTrackerInvoker::operator() body); all lanes hold the same scalars
__device__ __forceinline__ void lk_level(const uint8_t* __restrict__ I, const int16_t* __restrict__ dI,
                                         const uint8_t* __restrict__ J, int w, int h, int level, int max_level,
                                         bool use_initial, float px, float py, float& nextx, float& nexty, int& status,
                                         float& err, WarpWin& S, int lane, int max_count, double eps2, float min_eig_thr) {
    const float half = (float)(WIN - 1) * 0.5f;
    const float scale = (float)(1. / (double)(1 << level));
    float prevx = px * scale, prevy = py * scale;
    float nx, ny;
    if (level == max_level) {
        if (use_initial) { nx = nextx * scale; ny = nexty * scale; }
        else { nx = prevx; ny = prevy; }
    } else { nx = nextx * 2.f; ny = nexty * 2.f; }
    nextx = nx; nexty = ny;
    prevx -= half; prevy -= half;
    const int ipx = (int)floorf(prevx), ipy = (int)floorf(prevy);
    if (ipx < -WIN || ipx >= w || ipy < -WIN || ipy >= h) {
        if (level == 0) { status = 0; err = 0.f; }
        return;
    }
    float a = prevx - (float)ipx, b = prevy - (float)ipy;
    int iw00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
    int iw01 = __float2int_rn(a * (1.f - b) * 16384.f);
    int iw10 = __float2int_rn((1.f - a) * b * 16384.f);
    int iw11 = 16384 - iw00 - iw01 - iw10;

    const bool pix = lane < 27;
    const int wy = lane / 3, wx = 3 * (lane - 3 * wy);       // this lane's window row and first column
    int Iw[3] = {0, 0, 0};
    __syncwarp();
    if (pix) {
        const int X = ipx + wx, Y = ipy + wy;
        int i0[4], i1[4], dx0[4], dx1[4], dy0[4], dy1[4];
        const uint32_t* D = reinterpret_cast<const uint32_t*>(dI);
        if (ipx >= 0 && ipy >= 0 && ipx + WIN < w && ipy + WIN < h) {   // whole footprint inside the image (warp-uniform)
            const size_t o = (size_t)Y * w + X;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                i0[k] = __ldg(I + o + k);
                i1[k] = __ldg(I + o + w + k);
                const uint32_t d0 = __ldg(D + o + k), d1 = __ldg(D + o + w + k);
                dx0[k] = (int)(short)(d0 & 0xffffu); dy0[k] = (int)d0 >> 16;
                dx1[k] = (int)(short)(d1 & 0xffffu); dy1[k] = (int)d1 >> 16;
            }
        } else {
            const int y0 = refl(Y, h), y1 = refl(Y + 1, h);
            const bool yin0 = (Y >= 0 && Y < h), yin1 = (Y + 1 >= 0 && Y + 1 < h);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int xr = refl(X + k, w);
                const bool xin = (X + k >= 0 && X + k < w);
                i0[k] = __ldg(I + (size_t)y0 * w + xr);
                i1[k] = __ldg(I + (size_t)y1 * w + xr);
                const uint32_t d0 = (xin && yin0) ? __ldg(D + (size_t)y0 * w + xr) : 0u;
                const uint32_t d1 = (xin && yin1) ? __ldg(D + (size_t)y1 * w + xr) : 0u;
                dx0[k] = (int)(short)(d0 & 0xffffu); dy0[k] = (int)d0 >> 16;
                dx1[k] = (int)(short)(d1 & 0xffffu); dy1[k] = (int)d1 >> 16;
            }
        }
#pragma unroll
        for (int k = 0; k < 3; k++) {
            Iw[k] = (i0[k] * iw00 + i0[k + 1] * iw01 + i1[k] * iw10 + i1[k + 1] * iw11 + (1 << 8)) >> 9;
            const int ix = (dx0[k] * iw00 + dx0[k + 1] * iw01 + dx1[k] * iw10 + dx1[k + 1] * iw11 + (1 << 13)) >> 14;
            const int iy = (dy0[k] * iw00 + dy0[k + 1] * iw01 + dy1[k] * iw10 + dy1[k + 1] * iw11 + (1 << 13)) >> 14;
            S.dx[wy * WIN + wx + k] = (short)ix;
            S.dy[wy * WIN + wx + k] = (short)iy;
        }
    }
    __syncwarp();

    // covariance matrix: chain lanes.  group g = lane >> 3 (0: A11, 1: A12, 2: A22), chain c = lane & 7 (0..3: SIMD lanes,
    // 4: the scalar accumulator of column 8)
    const int grp = lane >> 3, ch = lane & 7;
    float q = 0.f;
    if (grp < 3 && ch < 5) {
#pragma unroll
        for (int y = 0; y < WIN; y++) {
            if (ch < 4) {
#pragma unroll
                for (int hh = 0; hh < 2; hh++) {
                    const float fx = (float)S.dx[y * WIN + ch + 4 * hh], fy = (float)S.dy[y * WIN + ch + 4 * hh];
                    const float p = grp == 0 ? fx * fx : (grp == 1 ? fx * fy : fy * fy);
                    q = p + q;
                }
            } else {
                const int ix = S.dx[y * WIN + 8], iy = S.dy[y * WIN + 8];
                q += (float)(grp == 0 ? ix * ix : (grp == 1 ? ix * iy : iy * iy));
            }
        }
    }
    float A[3];
#pragma unroll
    for (int g = 0; g < 3; g++) {
        const float q0 = __shfl_sync(0xffffffffu, q, 8 * g), q1 = __shfl_sync(0xffffffffu, q, 8 * g + 1);
        const float q2 = __shfl_sync(0xffffffffu, q, 8 * g + 2), q3 = __shfl_sync(0xffffffffu, q, 8 * g + 3);
        const float s = __shfl_sync(0xffffffffu, q, 8 * g + 4);
        A[g] = (s + ((q0 + q2) + (q1 + q3))) * (1.f / (1 << 20));
    }
    const float a11 = A[0], a12 = A[1], a22 = A[2];
    float D = a11 * a22 - a12 * a12;
    const float min_eig = (a22 + a11 - __fsqrt_rn((a11 - a22) * (a11 - a22) + 4.f * a12 * a12)) / (float)(2 * WIN * WIN);
    err = min_eig;
    if (min_eig < min_eig_thr || D < FLT_EPSILON) {
        if (level == 0) status = 0;
        return;
    }
    D = 1.f / D;

    // mismatch-vector chains: lanes 0..4 -> b1 (dx), lanes 8..12 -> b2 (dy); chain c < 4 pairs columns (c, c + 4), chain 4 = column 8
    int Da[WIN], Db[WIN];
    const bool chain = (grp < 2 && ch < 5);
    if (chain) {
        const short* src = grp == 0 ? S.dx : S.dy;
#pragma unroll
        for (int y = 0; y < WIN; y++) {
            Da[y] = src[y * WIN + (ch < 4 ? ch : 8)];
            Db[y] = ch < 4 ? src[y * WIN + ch + 4] : 0;
        }
    }
    const int ca = ch < 4 ? ch : 8, cb = ch < 4 ? ch + 4 : 8;

    nx -= half; ny -= half;
    float pdx = 0.f, pdy = 0.f;
    for (int j = 0; j < max_count; j++) {
        const int inx = (int)floorf(nx), iny = (int)floorf(ny);
        if (inx < -WIN || inx >= w || iny < -WIN || iny >= h) {
            if (level == 0) status = 0;
            break;
        }
        a = nx - (float)inx; b = ny - (float)iny;
        iw00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
        iw01 = __float2int_rn(a * (1.f - b) * 16384.f);
        iw10 = __float2int_rn((1.f - a) * b * 16384.f);
        iw11 = 16384 - iw00 - iw01 - iw10;
        __syncwarp();
        if (pix) {
            const int X = inx + wx, Y = iny + wy;
            int j0[4], j1[4];
            if (inx >= 0 && iny >= 0 && inx + WIN < w && iny + WIN < h) {   // whole 10x10 footprint inside the image (warp-uniform)
                const uint8_t* r0 = J + (size_t)Y * w + X;
#pragma unroll
                for (int k = 0; k < 4; k++) { j0[k] = __ldg(r0 + k); j1[k] = __ldg(r0 + w + k); }
            } else {
                const uint8_t* r0 = J + (size_t)refl(Y, h) * w;
                const uint8_t* r1 = J + (size_t)refl(Y + 1, h) * w;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int xr = refl(X + k, w);
                    j0[k] = __ldg(r0 + xr); j1[k] = __ldg(r1 + xr);
                }
            }
#pragma unroll
            for (int k = 0; k < 3; k++)
                S.diff[wy * WIN + wx + k] =
                    (short)(((j0[k] * iw00 + j0[k + 1] * iw01 + j1[k] * iw10 + j1[k + 1] * iw11 + (1 << 8)) >> 9) - Iw[k]);
        }
        __syncwarp();
        float qb = 0.f;
        if (chain) {
#pragma unroll
            for (int y = 0; y < WIN; y++) {
                const int d0 = S.diff[y * WIN + ca], d1 = S.diff[y * WIN + cb];
                qb += (float)(d0 * Da[y] + d1 * Db[y]);
            }
        }
        // qb0 = (bx c0, by c0, bx c1, by c1), qb1 = (bx c2, by c2, bx c3, by c3); s = qb0 + qb1; ib += (s0 + 0) + (s2 + 0)
        float bb[2];
#pragma unroll
        for (int g = 0; g < 2; g++) {
            const float c0 = __shfl_sync(0xffffffffu, qb, 8 * g), c1 = __shfl_sync(0xffffffffu, qb, 8 * g + 1);
            const float c2 = __shfl_sync(0xffffffffu, qb, 8 * g + 2), c3 = __shfl_sync(0xffffffffu, qb, 8 * g + 3);
            const float sc = __shfl_sync(0xffffffffu, qb, 8 * g + 4);
            bb[g] = (sc + ((c0 + c2) + (c1 + c3))) * (1.f / (1 << 20));
        }
        const float b1 = bb[0], b2 = bb[1];
        const float dx = (a12 * b2 - a22 * b1) * D;
        const float dy = (a12 * b1 - a11 * b2) * D;
        nx += dx; ny += dy;
        nextx = nx + half; nexty = ny + half;
        if ((double)dx * (double)dx + (double)dy * (double)dy <= eps2) break;
        if (j > 0 && fabs((double)(dx + pdx)) < 0.01 && fabs((double)(dy + pdy)) < 0.01) {
            nextx -= dx * 0.5f; nexty -= dy * 0.5f;
            break;
        }
        pdx = dx; pdy = dy;
    }
}

template <bool FB>
__global__ void __launch_bounds__(KLT_WARPS * 32, 6) klt_kernel(const KltParams P) {
    __shared__ WarpWin win[KLT_WARPS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long g = (long long)blockIdx.x * KLT_WARPS + wid;
    if (g >= (long long)P.nframes * P.npts) return;
    const int f = (int)(g / P.npts), i = (int)(g - (long long)f * P.npts);
    const int n = P.npts_per_frame ? P.npts_per_frame[f] : P.npts;
    const size_t pi = (size_t)f * P.npts + i;
    if (i >= n) {
        if (lane == 0) { P.status[pi] = 0; if (!FB && P.err) P.err[pi] = 0.f; }
        return;
    }
    WarpWin& S = win[wid];
    const float px = P.pts[2 * pi], py = P.pts[2 * pi + 1];
    float nextx = P.next[2 * pi], nexty = P.next[2 * pi + 1];
    int status = 1;
    float err = 0.f;
    for (int level = P.max_level; level >= 0; level--) {
        const size_t off = (size_t)f * P.w[level] * P.h[level];
        lk_level(P.prev_img[level] + off, P.prev_der[level] + 2 * off, P.cur_img[level] + off, P.w[level], P.h[level], level,
                 P.max_level, P.use_initial != 0, px, py, nextx, nexty, status, err, S, lane, P.max_count, P.eps2,
                 P.min_eig_thr);
    }
    if (!FB) {
        if (lane == 0) {
            P.next[2 * pi] = nextx; P.next[2 * pi + 1] = nexty;
            P.status[pi] = (uint8_t)status;
            if (P.err) P.err[pi] = err;
        }
        return;
    }
    // FeatureTracker::fbKltTracking gates (feature_tracker.cpp:48-72), then backward LK on level 0 (:83-87) and the
    // forward-backward distance gate (:103)
    bool good = status && !(err > P.error_value) && (1.0f <= nextx && nextx < (float)P.w[0] - 1.0f && 1.0f <= nexty &&
                                                     nexty < (float)P.h[0] - 1.0f);
    if (good) {
        float backx = px, backy = py;
        int st2 = 1;
        float e2 = 0.f;
        const size_t off = (size_t)f * P.w[0] * P.h[0];
        lk_level(P.cur_img[0] + off, P.cur_der[0] + 2 * off, P.prev_img[0] + off, P.w[0], P.h[0], 0, 0, true, nextx, nexty,
                 backx, backy, st2, e2, S, lane, P.max_count, P.eps2, P.min_eig_thr);
        if (!st2) good = false;
        else {
            const float ddx = px - backx, ddy = py - backy;
            if (sqrt((double)ddx * (double)ddx + (double)ddy * (double)ddy) > (double)P.max_fb_dist) good = false;
        }
    }
    if (lane == 0) {
        P.next[2 * pi] = nextx; P.next[2 * pi + 1] = nexty;
        P.status[pi] = good ? 1 : 0;
    }
}

int fill_params(KltParams& P, const uint8_t* const* prev_img, const int16_t* const* prev_der, const uint8_t* const* cur_img,
                const int16_t* const* cur_der, int w, int h, int nframes, int pyr_levels, int levels, int win, int max_count,
                double epsilon, const char* who) {
    if (win != WIN) { alva_set_error("%s: only the reference's 9x9 window is built (got %d)", who, win); return ALVA_E_INVALID; }
    if (pyr_levels < 0 || pyr_levels > 3 || levels < 0 || nframes < 1) { alva_set_error("%s: bad level / frame count", who); return ALVA_E_INVALID; }
    if (levels > pyr_levels) levels = pyr_levels;   // feature_tracker.cpp:18-21, lkpyramid.cpp:1315,1338
    int ww = w, hh = h;
    for (int k = 0; k <= levels; k++) {
        if (ww <= WIN || hh <= WIN) { alva_set_error("%s: level %d is %dx%d, not larger than the window", who, k, ww, hh); return ALVA_E_INVALID; }
        if (!prev_img[k] || !prev_der[k] || !cur_img[k] || (cur_der && !cur_der[k])) { alva_set_error("%s: null level %d", who, k); return ALVA_E_INVALID; }
        P.prev_img[k] = prev_img[k]; P.prev_der[k] = prev_der[k]; P.cur_img[k] = cur_img[k];
        P.cur_der[k] = cur_der ? cur_der[k] : nullptr;
        P.w[k] = ww; P.h[k] = hh;
        ww = (ww + 1) / 2; hh = (hh + 1) / 2;
    }
    P.nframes = nframes; P.max_level = levels;
    P.max_count = max_count < 0 ? 0 : (max_count > 100 ? 100 : max_count);       // lkpyramid.cpp:1351-1354
    const double e = epsilon < 0 ? 0 : (epsilon > 10 ? 10 : epsilon);            // :1355-1359
    P.eps2 = e * e;
    P.min_eig_thr = 1e-4f;
    return 0;
}

}  // namespace

extern "C" int alva_k_klt_lk(alva_ctx* ctx, const uint8_t* const* prev_img, const int16_t* const* prev_der,
                             const uint8_t* const* cur_img, int w, int h, int nframes, int pyr_levels, int levels, int win,
                             int max_count, double epsilon, int use_initial, const float* pts, float* next,
                             const int32_t* npts_per_frame, int npts, uint8_t* status, float* err) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !prev_img || !prev_der || !cur_img || !pts || !next || !status || npts < 1) { alva_set_error("alva_k_klt_lk: bad argument"); return ALVA_E_INVALID; }
    KltParams P{};
    if (int e = fill_params(P, prev_img, prev_der, cur_img, nullptr, w, h, nframes, pyr_levels, levels, win, max_count, epsilon, "alva_k_klt_lk")) return e;
    P.npts = npts; P.use_initial = use_initial; P.pts = pts; P.next = next; P.npts_per_frame = npts_per_frame;
    P.status = status; P.err = err;
    const long long warps = (long long)nframes * npts;
    klt_kernel<false><<<(unsigned)((warps + KLT_WARPS - 1) / KLT_WARPS), KLT_WARPS * 32, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_klt_fb(alva_ctx* ctx, const uint8_t* const* prev_img, const int16_t* const* prev_der,
                             const uint8_t* const* cur_img, const int16_t* const* cur_der, int w, int h, int nframes,
                             int pyr_levels, int levels, int win, float error_value, float max_fb_dist, const float* pts,
                             float* priors, const int32_t* npts_per_frame, int npts, uint8_t* good) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !prev_img || !prev_der || !cur_img || !cur_der || !pts || !priors || !good || npts < 1) { alva_set_error("alva_k_klt_fb: bad argument"); return ALVA_E_INVALID; }
    KltParams P{};
    // FeatureTracker(30, 0.01): kltConvCriteria_ (src/slam/src/system.cpp:31 -> feature_tracker.hpp:14)
    if (int e = fill_params(P, prev_img, prev_der, cur_img, cur_der, w, h, nframes, pyr_levels, levels, win, 30, 0.01f, "alva_k_klt_fb")) return e;
    P.npts = npts; P.use_initial = 1; P.pts = pts; P.next = priors; P.npts_per_frame = npts_per_frame;
    P.status = good; P.err = nullptr; P.error_value = error_value; P.max_fb_dist = max_fb_dist;
    const long long warps = (long long)nframes * npts;
    klt_kernel<true><<<(unsigned)((warps + KLT_WARPS - 1) / KLT_WARPS), KLT_WARPS * 32, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}
