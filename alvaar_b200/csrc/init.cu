// init.cu -- map initialisation on the GPU: the reference's 5-point essential-matrix RANSAC + non-linear refinement
// (MultiViewGeometry::compute5ptEssentialMatrix, src/slam/src/multi_view_geometry.cpp:225-318; caller
// VisualFrontend::checkReadyForInit, visual_frontend.cpp:419-552) and the mid-point triangulation the mapper builds the
// first map points with (MultiViewGeometry::triangulate, multi_view_geometry.cpp:12-22; caller Mapper::triangulateTemporal,
// mapper.cpp:157-291).
//
// The reference runs RANSAC serially: draw 8 indices, solve Nister's five-point problem (<= 10 essential matrices x 4
// decompositions, disambiguated on the 8 sample points), count the inliers of the winner over all N correspondences, update
// the adaptive iteration bound k.  The draws do not depend on the outcome of earlier iterations (one persistent partial
// Fisher-Yates shuffle fed by mt19937), so here a CTA solves CHUNK hypotheses at once (one thread each), counts their inliers
// warp-parallel, and one thread replays the reference's sequential bookkeeping (alva_init::RansacState) over them in draw
// order -- same selected model, same iteration count, same inlier set.  The refinement minimises the reference's cost
// (sum over inliers of (e1 + e2)^2, 6 parameters [t, cayley]) by Levenberg-Marquardt with the residuals, Jacobian rows and
// normal-equation sums spread over the CTA (fixed-order reductions: bit-reproducible).
// This runs once per map initialisation; it is latency-bound FP64 scalar work (a few thousand flops per hypothesis and
// point) and nowhere near any roofline -- the point is that no per-frame or per-keyframe step ever leaves the device.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include "init_core.h"
#include "lmdif_core.h"
#include <limits>
#include <random>
#include <vector>

namespace {

using namespace alva_init;

constexpr int INIT_THREADS = 128;
constexpr int CHUNK = 32;   // hypotheses solved per round (one per thread of the first warp; the solver's local arrays make it
                            // local-memory bound, so more hypotheses per round mean more local-memory traffic per thread)

struct EssentialParams {
    const double* bv1; const double* bv2; const int32_t* counts; int cap;
    int max_iter; int optimize; double threshold;
    const int32_t* rnd; int table_len;
    double* Rt; uint8_t* outlier; double* info;
    double* work; int32_t* inl;   // optimize == 2: [nprob][8 * cap] doubles + [nprob][cap] inlier indices for the MINPACK-style refinement
};

__device__ __forceinline__ double block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0;
    for (int w = 0; w < INIT_THREADS / 32; w++) s += red[w];
    return s;
}

__global__ void __launch_bounds__(INIT_THREADS) essential_kernel(const EssentialParams P) {
    extern __shared__ int sh_idx[];   // the sampler's persistent shuffle
    __shared__ double models[CHUNK][12];
    __shared__ int sidx[CHUNK][8];
    __shared__ int valid[CHUNK], cnt[CHUNK];
    __shared__ double bestm[12], xs[6], xn[6], Hs[36], gs[6], red[INIT_THREADS / 32];
    __shared__ RansacState rs;
    __shared__ int done, flag;
    const int prob = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = P.counts ? min(P.counts[prob], P.cap) : P.cap;
    const double* bv1 = P.bv1 + (size_t)prob * P.cap * 3;
    const double* bv2 = P.bv2 + (size_t)prob * P.cap * 3;
    uint8_t* outlier = P.outlier + (size_t)prob * P.cap;
    double* info = P.info ? P.info + 4 * prob : nullptr;
    for (int i = tid; i < P.cap; i += INIT_THREADS) outlier[i] = i < n ? 0 : 1;
    if (n < 8) {   // compute5ptEssentialMatrix: fewer than 8 correspondences -> false
        if (tid == 0 && info) { info[0] = 0; info[1] = 0; info[2] = 0; info[3] = 0; }
        return;
    }
    for (int i = tid; i < n; i += INIT_THREADS) sh_idx[i] = i;
    if (tid == 0) { rs.init(P.max_iter); done = 0; }
    __syncthreads();
    int base_draw = 0;
    while (true) {
        if (tid == 0) {   // CHUNK draws of 8 indices, continuing the shuffle (SampleConsensusProblem::drawIndexSample)
            for (int h = 0; h < CHUNK; h++) {
                const int d = base_draw + h;
                for (int i = 0; i < 8; i++) {
                    const int32_t r = 8 * d + i < P.table_len ? P.rnd[8 * d + i] : 0;
                    const int j = i + (int)((uint32_t)r % (uint32_t)(n - i));
                    const int t = sh_idx[i]; sh_idx[i] = sh_idx[j]; sh_idx[j] = t;
                }
                for (int i = 0; i < 8; i++) sidx[h][i] = sh_idx[i];
            }
        }
        __syncthreads();
        if (tid < CHUNK) {
            double m[12];
            const bool ok = relpose_sample_model(bv1, bv2, sidx[tid], m);
            valid[tid] = ok ? 1 : 0;
            for (int i = 0; i < 12; i++) models[tid][i] = m[i];
        }
        __syncthreads();
        for (int h = warp; h < CHUNK; h += INIT_THREADS / 32) {   // countWithinDistance, one warp per hypothesis
            int c = 0;
            if (valid[h])
                for (int i = lane; i < n; i += 32) c += relpose_dist(models[h], models[h] + 9, bv1 + 3 * i, bv2 + 3 * i) < P.threshold;
            c = __reduce_add_sync(0xffffffffu, c);
            if (lane == 0) cnt[h] = c;
        }
        __syncthreads();
        if (tid == 0) {
            for (int h = 0; h < CHUNK; h++) {
                if (!rs.running()) { done = 1; break; }
                bool stop;
                if (rs.consume(valid[h] != 0, cnt[h], n, stop))
                    for (int i = 0; i < 12; i++) bestm[i] = models[h][i];
                if (stop) { done = 1; break; }
            }
            if (!rs.running()) done = 1;
            if (8 * (base_draw + 2 * CHUNK) > P.table_len) done = 1;   // table exhausted (cannot happen: sized for max_skip)
        }
        __syncthreads();
        if (done) break;
        base_draw += CHUNK;
    }
    if (!rs.have) {
        if (tid == 0 && info) { info[0] = 0; info[1] = 0; info[2] = rs.iterations; info[3] = rs.draws; }
        for (int i = tid; i < n; i += INIT_THREADS) outlier[i] = 1;
        return;
    }
    // selectWithinDistance with the best model
    int mine = 0;
    for (int i = tid; i < n; i += INIT_THREADS) {
        const bool in = relpose_dist(bestm, bestm + 9, bv1 + 3 * i, bv2 + 3 * i) < P.threshold;
        outlier[i] = in ? 0 : 1;
        mine += in;
    }
    const int m = (int)(block_sum((double)mine, red) + 0.5);
    if (tid == 0 && info) { info[0] = m >= 10 ? 1 : 0; info[1] = m; info[2] = rs.iterations; info[3] = rs.draws; }
    if (m < 10) return;   // multi_view_geometry.cpp:283-286: fewer than 10 inliers -> false
    if (P.optimize == 2) {
        // the reference's own minimiser restated (lmdif_core.h): MINPACK Levenberg-Marquardt on a forward-difference Jacobian,
        // ftol = xtol = 10 eps, maxfev 1000 (relative_pose/methods.cpp:1152-1177).  One thread: the stage runs once per session.
        __syncthreads();
        if (tid == 0) {
            int32_t* inl = P.inl + (size_t)prob * P.cap;
            int mm = 0;
            for (int i = 0; i < n; i++) if (!outlier[i]) inl[mm++] = i;
            double x[6];
            for (int i = 0; i < 3; i++) x[i] = bestm[9 + i];
            rot2cayley(bestm, x + 3);
            double* w = P.work + (size_t)prob * P.cap * 8;
            auto fun = [&](const double* xx, double* f) {
                double R[9];
                cayley2rot(xx + 3, R);
                for (int i = 0; i < mm; i++) f[i] = relpose_dist(R, xx, bv1 + 3 * inl[i], bv2 + 3 * inl[i]);
            };
            alva_lm::lmdif(fun, mm, x, w, w + mm, w + 7 * (size_t)mm, 10 * DBL_EPSILON, 10 * DBL_EPSILON, 1000);
            for (int i = 0; i < 3; i++) bestm[9 + i] = x[i];
            cayley2rot(x + 3, bestm);
        }
        __syncthreads();
    } else if (P.optimize) {
        if (tid == 0) { for (int i = 0; i < 3; i++) xs[i] = bestm[9 + i]; rot2cayley(bestm, xs + 3); }
        __syncthreads();
        double local = 0;
        for (int i = tid; i < n; i += INIT_THREADS)
            if (!outlier[i]) { const double f = nl_point(xs, bv1 + 3 * i, bv2 + 3 * i, nullptr); local += f * f; }
        double cost = block_sum(local, red), lambda = 1e-3;
        for (int it = 0; it < 200; it++) {
            double acc[27];
            for (int k = 0; k < 27; k++) acc[k] = 0;
            for (int i = tid; i < n; i += INIT_THREADS) {
                if (outlier[i]) continue;
                double J[6];
                const double f = nl_point(xs, bv1 + 3 * i, bv2 + 3 * i, J);
                int k = 0;
                for (int a = 0; a < 6; a++)
                    for (int b = 0; b <= a; b++) acc[k++] += J[a] * J[b];
                for (int a = 0; a < 6; a++) acc[21 + a] -= J[a] * f;
            }
            for (int k = 0; k < 27; k++) {
                const double s = block_sum(acc[k], red);
                if (tid == 0) {
                    if (k < 21) { int a = 0, r = k; while (r > a) { r -= a + 1; a++; } Hs[6 * a + r] = s; Hs[6 * r + a] = s; }
                    else gs[k - 21] = s;
                }
            }
            __syncthreads();
            bool improved = false;
            double step_rel = 0;
            for (int tries = 0; tries < 40 && !improved; tries++) {
                if (tid == 0) {
                    double dx[6];
                    flag = solve6_damped(Hs, gs, lambda, dx) ? 1 : 0;
                    if (flag) {
                        double nx = 0, nd = 0;
                        for (int a = 0; a < 6; a++) { xn[a] = xs[a] + dx[a]; nx += xs[a] * xs[a]; nd += dx[a] * dx[a]; }
                        models[0][0] = sqrt(nd) / fmax(sqrt(nx), 1e-300);   // scratch: relative step length
                    }
                }
                __syncthreads();
                if (!flag) { lambda *= 10; __syncthreads(); continue; }
                const double srel = models[0][0];
                double l2 = 0;
                for (int i = tid; i < n; i += INIT_THREADS)
                    if (!outlier[i]) { const double f = nl_point(xn, bv1 + 3 * i, bv2 + 3 * i, nullptr); l2 += f * f; }
                const double c2 = block_sum(l2, red);
                if (c2 < cost) {
                    const double rel = (cost - c2) / cost;
                    step_rel = rel < 1e-15 ? 0.0 : srel;
                    cost = c2; lambda = fmax(lambda * 0.1, 1e-12); improved = true;
                    __syncthreads();
                    if (tid < 6) xs[tid] = xn[tid];
                } else lambda *= 10;
                __syncthreads();
            }
            if (!improved || step_rel < 1e-13) break;
        }
        if (tid == 0) { for (int i = 0; i < 3; i++) bestm[9 + i] = xs[i]; cayley2rot(xs + 3, bestm); }
        __syncthreads();
    }
    if (tid < 12) {
        const int r = tid / 4, c = tid % 4;
        P.Rt[12 * prob + tid] = c < 3 ? bestm[3 * r + c] : bestm[9 + r];
    }
}

__global__ void triangulate_kernel(const double* __restrict__ Tlr, const double* __restrict__ bvl, const double* __restrict__ bvr, int n,
                                   double* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x = Tlr[3], y = Tlr[4], z = Tlr[5], w = Tlr[6];   // Eigen::Quaterniond::toRotationMatrix
    const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
    const double t[3] = {Tlr[0], Tlr[1], Tlr[2]};
    double p[3];
    triangulate2(R, t, bvl + 3 * i, bvr + 3 * i, p);
    out[3 * i] = p[0]; out[3 * i + 1] = p[1]; out[3 * i + 2] = p[2];
}

}  // namespace

// SampleConsensusProblem::rnd(): the reference's own objects evaluated by this host's libstdc++ (as pose.cu does)
static void make_rnd_table_init(uint32_t seed, int n, std::vector<int32_t>& out) {
    std::mt19937 alg(seed);
    std::uniform_int_distribution<> dist(0, std::numeric_limits<int>::max());
    out.resize(n);
    for (int i = 0; i < n; i++) out[i] = dist(alg);
}

extern "C" int alva_k_essential_5pt(alva_ctx* ctx, int nprob, int cap, const double* bv1, const double* bv2, const int32_t* counts,
                                    int max_iter, float err_px, int optimize, float fx, float fy, uint32_t seed, double* Rt_out,
                                    uint8_t* outlier, double* info) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !bv1 || !bv2 || !Rt_out || !outlier || nprob < 1 || cap < 1 || max_iter < 1 || max_iter > 1024) {
        alva_set_error("alva_k_essential_5pt: bad argument");
        return ALVA_E_INVALID;
    }
    if (cap > 8192) { alva_set_error("alva_k_essential_5pt: at most 8192 correspondences per problem (got %d)", cap); return ALVA_E_INVALID; }
    float focal = fx + fy;   // threshold in the reference's float arithmetic (multi_view_geometry.cpp:274-278)
    focal = (float)(focal / 2.);
    EssentialParams P{};
    P.threshold = 2.0 * (1.0 - cosf(atanf(err_px / focal)));
    P.bv1 = bv1; P.bv2 = bv2; P.counts = counts; P.cap = cap; P.max_iter = max_iter; P.optimize = optimize;
    P.table_len = 8 * (11 * max_iter + 3 * CHUNK);
    const size_t tab_b = 0;   // (the sampler table lives on the context)
    const size_t work_b = optimize == 2 ? (size_t)nprob * cap * 8 * sizeof(double) : 0;
    const size_t inl_b = optimize == 2 ? (((size_t)nprob * cap * 4 + 255) & ~(size_t)255) : 0;
    uint8_t* scr = (uint8_t*)alva_scratch(ctx, tab_b + work_b + inl_b + 256);
    if (!scr) return ALVA_E_CUDA;
    P.work = (double*)(scr + tab_b); P.inl = (int32_t*)(scr + tab_b + work_b);
    P.Rt = Rt_out; P.outlier = outlier; P.info = info;
    // the sampler table depends only on (seed, length): kept on the device across calls -- a per-call upload from pageable memory
    // made every call wait for the stream to drain (the loop-closure detector calls this every step)
    if (!ctx->init_tab || ctx->init_tab_len != P.table_len || ctx->init_tab_seed != seed) {
        std::vector<int32_t> host_tab;
        make_rnd_table_init(seed, P.table_len, host_tab);
        ctx->ws_epoch++;
        if (ctx->init_tab) { ALVA_CUDA(cudaStreamSynchronize(ctx->stream)); ALVA_CUDA(cudaFree(ctx->init_tab)); ctx->init_tab = nullptr; }
        ALVA_CUDA(cudaMalloc(&ctx->init_tab, (size_t)P.table_len * 4));
        ALVA_CUDA(cudaMemcpy(ctx->init_tab, host_tab.data(), (size_t)P.table_len * 4, cudaMemcpyHostToDevice));
        ctx->init_tab_len = P.table_len; ctx->init_tab_seed = seed;
    }
    P.rnd = (const int32_t*)ctx->init_tab;
    essential_kernel<<<nprob, INIT_THREADS, (size_t)cap * sizeof(int), ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_triangulate(alva_ctx* ctx, const double* Tlr, const double* bvl, const double* bvr, int n, double* out) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !Tlr || !bvl || !bvr || !out || n < 0) { alva_set_error("alva_k_triangulate: bad argument"); return ALVA_E_INVALID; }
    if (n == 0) return 0;
    triangulate_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(Tlr, bvl, bvr, n, out);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}
