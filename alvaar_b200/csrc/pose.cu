// pose.cu -- per-frame camera pose on the GPU: P3P (Kneip) inside a Least-Median-of-Squares loop, then the motion-only
// Levenberg-Marquardt refinement (PnP), batched over independent problems (one per frame / camera stream).
//
// What is computed (fp64; parity: pose within 1e-4 relative, inlier / outlier sets equal -- tests/test_gpu_pose.py; the CPU
// restatement is oracle/pose_oracle.c):
//   MultiViewGeometry::p3pRansac (optimize = false)   src/slam/src/multi_view_geometry.cpp:24-127
//        opengv::sac::Lmeds::computeModel             opengv/include/opengv/sac/implementation/Lmeds.hpp:40-190
//        sampling                                     opengv/include/opengv/sac/implementation/SampleConsensusProblem.hpp:62-120
//        AbsolutePoseSacProblem (KNEIP)               opengv/src/sac_problems/absolute_pose/AbsolutePoseSacProblem.cpp:40-210
//        p3p_kneip_main, o4_roots                     opengv/src/absolute_pose/modules/main.cpp:50-220, src/math/roots.cpp:88-136
//   MultiViewGeometry::ceresPnP                       src/slam/src/multi_view_geometry.cpp:129-223
//        DirectSE3::ReprojectionErrorSE3::Evaluate    src/slam/src/ceres_parametrization.cpp:96-155
//        Ceres trust-region LM (DENSE_QR)             same loop as ba.cu restates for the local BA
//   caller VisualFrontend::computePose                src/slam/src/visual_frontend.cpp:245-417
//
// How: the reference runs 100 hypotheses x (P3P + N distances + std::sort) serially.  Here
//   * the sampler's partial Fisher-Yates shuffle is the only serial piece (one thread, ~500 swaps in shared memory; its
//     random numbers are a host-made table: std::mt19937 through libstdc++'s uniform_int_distribution is x >> 1);
//   * all hypotheses of a problem are solved at once (thread per draw), kept in the reference's order;
//   * one CTA per (hypothesis, problem) computes the N squared distances and takes the median by a bitonic sort in
//     shared memory; a last kernel picks the first strict minimum, classifies inliers and checks orthogonality;
//   * P3P-RANSAC (alva_k_p3p_ransac, System's relocalisation) runs the same hypotheses kernel, counts each hypothesis'
//     inliers instead of sorting, and the last kernel picks the first strict maximum;
//   * the PnP refinement is one CTA per problem with every LM decision on the device (fixed-order reductions: the result
//     is bit-reproducible run to run).
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include <float.h>
#include <random>
#include <vector>

namespace {

// ------------------------------------------------------------------ complex helpers (double)
struct cd { double x, y; };
__device__ __forceinline__ cd cmk(double x, double y) { cd r; r.x = x; r.y = y; return r; }
__device__ __forceinline__ cd cadd(cd a, cd b) { return cmk(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ cd csub(cd a, cd b) { return cmk(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ cd cscale(cd a, double s) { return cmk(a.x * s, a.y * s); }
__device__ __forceinline__ cd cdivc(cd a, cd b) {
    const double d = b.x * b.x + b.y * b.y;
    return cmk((a.x * b.x + a.y * b.y) / d, (a.y * b.x - a.x * b.y) / d);
}
__device__ cd csqrtd(cd z) {
    if (z.x == 0.0 && z.y == 0.0) return cmk(0.0, z.y);
    const double t = sqrt((fabs(z.x) + hypot(z.x, z.y)) * 0.5);
    if (z.x >= 0.0) return cmk(t, z.y / (2.0 * t));
    return cmk(fabs(z.y) / (2.0 * t), copysign(t, z.y));
}
// std::pow(std::complex<double>, double) as libstdc++ evaluates it: real pow for positive reals, else polar(exp(y log|z|), y arg z)
__device__ cd cpow_real(cd z, double y) {
    if (z.y == 0.0 && z.x > 0.0) return cmk(pow(z.x, y), 0.0);
    const double lr = log(hypot(z.x, z.y)), th = atan2(z.y, z.x);
    const double rho = exp(y * lr);
    double s, c;
    sincos(y * th, &s, &c);
    return cmk(rho * c, rho * s);
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* o) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double norm3(const double* a) { return sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }

// opengv::math::o4_roots: Ferrari in complex arithmetic, real parts of all four roots
__device__ void o4_roots(const double* p, double* roots) {
    const double A = p[0], B = p[1], C = p[2], D = p[3], E = p[4];
    const double A2 = A * A, B2 = B * B, A3 = A2 * A, B3 = B2 * B, A4 = A3 * A, B4 = B3 * B;
    const double alpha = -3 * B2 / (8 * A2) + C / A;
    const double beta = B3 / (8 * A3) - B * C / (2 * A2) + D / A;
    const double gamma = -3 * B4 / (256 * A4) + B2 * C / (16 * A3) - B * D / (4 * A2) + E / A;
    const double alpha2 = alpha * alpha, alpha3 = alpha2 * alpha;
    const cd P = cmk(-alpha2 / 12 - gamma, 0.0);
    const cd Q = cmk(-alpha3 / 108 + alpha * gamma / 3 - beta * beta / 8, 0.0);
    const cd R = cadd(cscale(Q, -0.5), csqrtd(cadd(cscale(cpow_real(Q, 2.0), 0.25), cscale(cpow_real(P, 3.0), 1.0 / 27.0))));
    const cd U = cpow_real(R, 1.0 / 3.0);
    cd y;
    if (U.x == 0.0) y = csub(cmk(-5.0 * alpha / 6.0, 0.0), cpow_real(Q, 1.0 / 3.0));
    else y = cadd(csub(cmk(-5.0 * alpha / 6.0, 0.0), cdivc(P, cscale(U, 3.0))), U);
    const cd w = csqrtd(cmk(alpha + 2.0 * y.x, 2.0 * y.y));
    const cd bw = cdivc(cmk(2.0 * beta, 0.0), w);
    const cd base = cmk(3.0 * alpha + 2.0 * y.x, 2.0 * y.y);
    const cd a1 = cadd(base, bw), a2 = csub(base, bw);
    const cd s1 = csqrtd(cmk(-a1.x, -a1.y)), s2 = csqrtd(cmk(-a2.x, -a2.y));
    const double sh = -B / (4.0 * A);
    roots[0] = sh + 0.5 * (w.x + s1.x);
    roots[1] = sh + 0.5 * (w.x - s1.x);
    roots[2] = sh + 0.5 * (-w.x + s2.x);
    roots[3] = sh + 0.5 * (-w.x - s2.x);
}

// 1 - f . normalise(R^T (X - t)), T = [R | t] 3x4 row-major
__device__ __forceinline__ double bearing_dist(const double* T, const double* X, const double* f) {
    double q[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const double tr = -(T[i] * T[3] + T[4 + i] * T[7] + T[8 + i] * T[11]);
        q[i] = T[i] * X[0] + T[4 + i] * X[1] + T[8 + i] * X[2] + tr;
    }
    const double n = norm3(q);
    return 1.0 - (q[0] / n * f[0] + q[1] / n * f[1] + q[2] / n * f[2]);
}

// AbsolutePoseSacProblem::computeModelCoefficients (KNEIP): P3P on sample points 0..2, the 4th picks among the 4 roots
__device__ bool p3p_sample_model(const double* __restrict__ bvs, const double* __restrict__ wpts, const int* idx, double* Tout) {
    double f[9], p[9];
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int i = 0; i < 3; i++) { f[3 * k + i] = bvs[3 * idx[k] + i]; p[3 * k + i] = wpts[3 * idx[k] + i]; }
    const double *P1 = p, *P2 = p + 3, *P3 = p + 6;
    double t1[3], t2[3], c[3];
    for (int i = 0; i < 3; i++) { t1[i] = P2[i] - P1[i]; t2[i] = P3[i] - P1[i]; }
    cross3(t1, t2, c);
    if (norm3(c) == 0.0) return false;
    const double *f1 = f, *f2 = f + 3, *f3 = f + 6;
    double T[9], f3t[3];
    for (int pass = 0; pass < 2; pass++) {
        double e3[3], e2[3];
        cross3(f1, f2, e3);
        const double n = norm3(e3);
        for (int i = 0; i < 3; i++) e3[i] /= n;
        cross3(e3, f1, e2);
        for (int i = 0; i < 3; i++) { T[i] = f1[i]; T[3 + i] = e2[i]; T[6 + i] = e3[i]; }
        for (int i = 0; i < 3; i++) f3t[i] = T[3 * i] * f3[0] + T[3 * i + 1] * f3[1] + T[3 * i + 2] * f3[2];
        if (pass == 0 && f3t[2] > 0) { f1 = f + 3; f2 = f; P1 = p + 3; P2 = p; }
        else break;
    }
    double n1[3], n2[3], n3[3], d[3], N[9];
    for (int i = 0; i < 3; i++) n1[i] = P2[i] - P1[i];
    { const double n = norm3(n1); for (int i = 0; i < 3; i++) n1[i] /= n; }
    for (int i = 0; i < 3; i++) d[i] = P3[i] - P1[i];
    cross3(n1, d, n3);
    { const double n = norm3(n3); for (int i = 0; i < 3; i++) n3[i] /= n; }
    cross3(n3, n1, n2);
    for (int i = 0; i < 3; i++) { N[i] = n1[i]; N[3 + i] = n2[i]; N[6 + i] = n3[i]; }
    double P3n[3];
    for (int i = 0; i < 3; i++) P3n[i] = N[3 * i] * d[0] + N[3 * i + 1] * d[1] + N[3 * i + 2] * d[2];
    const double d_12 = norm3(t1);
    const double f_1 = f3t[0] / f3t[2], f_2 = f3t[1] / f3t[2], p_1 = P3n[0], p_2 = P3n[1];
    const double cos_beta = f1[0] * f2[0] + f1[1] * f2[1] + f1[2] * f2[2];
    double b = 1 / (1 - cos_beta * cos_beta) - 1;
    b = cos_beta < 0 ? -sqrt(b) : sqrt(b);
    const double f_1_pw2 = f_1 * f_1, f_2_pw2 = f_2 * f_2, p_1_pw2 = p_1 * p_1, p_1_pw3 = p_1_pw2 * p_1, p_1_pw4 = p_1_pw3 * p_1;
    const double p_2_pw2 = p_2 * p_2, p_2_pw3 = p_2_pw2 * p_2, p_2_pw4 = p_2_pw3 * p_2, d_12_pw2 = d_12 * d_12, b_pw2 = b * b;
    double fac[5];
    fac[0] = -f_2_pw2 * p_2_pw4 - p_2_pw4 * f_1_pw2 - p_2_pw4;
    fac[1] = 2 * p_2_pw3 * d_12 * b + 2 * f_2_pw2 * p_2_pw3 * d_12 * b - 2 * f_2 * p_2_pw3 * f_1 * d_12;
    fac[2] = -f_2_pw2 * p_2_pw2 * p_1_pw2 - f_2_pw2 * p_2_pw2 * d_12_pw2 * b_pw2 - f_2_pw2 * p_2_pw2 * d_12_pw2 + f_2_pw2 * p_2_pw4 +
             p_2_pw4 * f_1_pw2 + 2 * p_1 * p_2_pw2 * d_12 + 2 * f_1 * f_2 * p_1 * p_2_pw2 * d_12 * b - p_2_pw2 * p_1_pw2 * f_1_pw2 +
             2 * p_1 * p_2_pw2 * f_2_pw2 * d_12 - p_2_pw2 * d_12_pw2 * b_pw2 - 2 * p_1_pw2 * p_2_pw2;
    fac[3] = 2 * p_1_pw2 * p_2 * d_12 * b + 2 * f_2 * p_2_pw3 * f_1 * d_12 - 2 * f_2_pw2 * p_2_pw3 * d_12 * b - 2 * p_1 * p_2 * d_12_pw2 * b;
    fac[4] = -2 * f_2 * p_2_pw2 * f_1 * p_1 * d_12 * b + f_2_pw2 * p_2_pw2 * d_12_pw2 + 2 * p_1_pw3 * d_12 - p_1_pw2 * d_12_pw2 +
             f_2_pw2 * p_2_pw2 * p_1_pw2 - p_1_pw4 - 2 * f_2_pw2 * p_2_pw2 * p_1 * d_12 + p_2_pw2 * f_1_pw2 * p_1_pw2 +
             f_2_pw2 * p_2_pw2 * d_12_pw2 * b_pw2;
    double roots[4];
    o4_roots(fac, roots);
    double best = 1000000.0;
    bool have = false;
    const double* X4 = wpts + 3 * idx[3];
    const double* f4 = bvs + 3 * idx[3];
    for (int k = 0; k < 4; k++) {
        const double r = roots[k];
        const double cot_alpha = (-f_1 * p_1 / f_2 - r * p_2 + d_12 * b) / (-f_1 * r * p_2 / f_2 + p_1 - d_12);
        const double cos_theta = r, sin_theta = sqrt(1 - r * r);
        const double sin_alpha = sqrt(1 / (cot_alpha * cot_alpha + 1));
        double cos_alpha = sqrt(1 - sin_alpha * sin_alpha);
        if (cot_alpha < 0) cos_alpha = -cos_alpha;
        const double k0 = sin_alpha * b + cos_alpha;
        const double Cc[3] = {d_12 * cos_alpha * k0, cos_theta * d_12 * sin_alpha * k0, sin_theta * d_12 * sin_alpha * k0};
        const double Rm[9] = {-cos_alpha, -sin_alpha * cos_theta, -sin_alpha * sin_theta,
                              sin_alpha,  -cos_alpha * cos_theta, -cos_alpha * sin_theta,
                              0.0,        -sin_theta,             cos_theta};
        double S[12], NR[9];
        for (int i = 0; i < 3; i++) S[4 * i + 3] = P1[i] + (N[i] * Cc[0] + N[3 + i] * Cc[1] + N[6 + i] * Cc[2]);
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) NR[3 * i + j] = N[i] * Rm[3 * j] + N[3 + i] * Rm[3 * j + 1] + N[6 + i] * Rm[3 * j + 2];
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) S[4 * i + j] = NR[3 * i] * T[j] + NR[3 * i + 1] * T[3 + j] + NR[3 * i + 2] * T[6 + j];
        const double sc = bearing_dist(S, X4, f4);
        if (sc < best) {
            best = sc; have = true;
            for (int i = 0; i < 12; i++) Tout[i] = S[i];
        }
    }
    return have;
}

// ------------------------------------------------------------------ kernel A: draws -> hypotheses (one CTA per problem)
constexpr int HYP_THREADS = 128;
struct LmedsParams {
    const double* bvs; const double* wpts; const int32_t* counts;
    int cap, max_iter, max_skip, table_len;
    const int32_t* rnd;      // SampleConsensusProblem::rnd() sequence for the seed
    double* hyp;             // [nprob][max_iter][12]
    int32_t* nhyp;           // [nprob][2]: valid hypotheses, draws consumed
    double* pen;             // [nprob][max_iter]
    double threshold;
    double* Twc; uint8_t* outlier; double* info;
};

__global__ void __launch_bounds__(HYP_THREADS) p3p_hypotheses_kernel(const LmedsParams P) {
    extern __shared__ int sh[];                 // shuffled_indices_ [n]
    __shared__ int sidx[HYP_THREADS][4];
    __shared__ int wcount[HYP_THREADS / 32];
    __shared__ int s_nvalid, s_skipped, s_draws, s_go;
    const int prob = blockIdx.x, tid = threadIdx.x;
    const int n = P.counts ? min(P.counts[prob], P.cap) : P.cap;
    const double* bvs = P.bvs + (size_t)prob * P.cap * 3;
    const double* wpts = P.wpts + (size_t)prob * P.cap * 3;
    if (n < 4) { if (tid == 0) { P.nhyp[2 * prob] = 0; P.nhyp[2 * prob + 1] = 0; } return; }
    for (int i = tid; i < n; i += HYP_THREADS) sh[i] = i;
    if (tid == 0) { s_nvalid = 0; s_skipped = 0; s_draws = 0; s_go = 1; }
    __syncthreads();
    while (s_go) {
        const int d0 = s_draws;
        if (tid == 0) {
            for (int k = 0; k < HYP_THREADS; k++) {
                const int base = 4 * (d0 + k);
                if (base + 3 >= P.table_len) { sidx[k][0] = -1; continue; }
                for (int i = 0; i < 4; i++) {
                    const int j = i + (int)((uint32_t)P.rnd[base + i] % (uint32_t)(n - i));
                    const int t = sh[i]; sh[i] = sh[j]; sh[j] = t;
                }
                for (int i = 0; i < 4; i++) sidx[k][i] = sh[i];
            }
        }
        __syncthreads();
        double T[12];
        int idx[4] = {sidx[tid][0], sidx[tid][1], sidx[tid][2], sidx[tid][3]};
        const bool drawn = idx[0] >= 0;
        const bool valid = drawn && p3p_sample_model(bvs, wpts, idx, T);
        // ordered accounting: draw k counts only while iterations < max_iter and skipped < max_skip (Lmeds.hpp:78)
        const unsigned bal = __ballot_sync(0xffffffffu, valid);
        const int lane = tid & 31, wid = tid >> 5;
        if (lane == 0) wcount[wid] = __popc(bal);
        __syncthreads();
        int vb = __popc(bal & ((1u << lane) - 1u));
        for (int w = 0; w < wid; w++) vb += wcount[w];
        const int sb = tid - vb;
        const int nv0 = s_nvalid, sk0 = s_skipped;
        const bool processed = drawn && (nv0 + vb < P.max_iter) && (sk0 + sb < P.max_skip);
        if (processed && valid) {
            double* out = P.hyp + ((size_t)prob * P.max_iter + nv0 + vb) * 12;
            for (int i = 0; i < 12; i++) out[i] = T[i];
        }
        const int pv = __syncthreads_count(processed && valid);
        const int pi = __syncthreads_count(processed && !valid);
        const int und = __syncthreads_count(!drawn);
        if (tid == 0) {
            s_nvalid = nv0 + pv; s_skipped = sk0 + pi; s_draws = d0 + pv + pi;
            s_go = (s_nvalid < P.max_iter && s_skipped < P.max_skip && und == 0) ? 1 : 0;
            // the shuffle state must continue right after the last processed draw: a chunk is only partially consumed when
            // the loop ends, so over-generation is harmless
        }
        __syncthreads();
    }
    if (tid == 0) { P.nhyp[2 * prob] = s_nvalid; P.nhyp[2 * prob + 1] = s_draws; }
}

// ------------------------------------------------------------------ kernel B: median of squared distances per hypothesis
constexpr int MED_THREADS = 256;
__global__ void __launch_bounds__(MED_THREADS) p3p_median_kernel(const LmedsParams P, int npow2) {
    extern __shared__ unsigned long long keys[];
    const int prob = blockIdx.y, hy = blockIdx.x, tid = threadIdx.x;
    if (hy >= P.nhyp[2 * prob]) return;
    const int n = P.counts ? min(P.counts[prob], P.cap) : P.cap;
    const double* bvs = P.bvs + (size_t)prob * P.cap * 3;
    const double* wpts = P.wpts + (size_t)prob * P.cap * 3;
    double T[12];
    const double* Tg = P.hyp + ((size_t)prob * P.max_iter + hy) * 12;
#pragma unroll
    for (int i = 0; i < 12; i++) T[i] = Tg[i];
    // only the smallest power of two >= n takes part in the sort
    int m = 1;
    while (m < n) m <<= 1;
    for (int i = tid; i < m; i += MED_THREADS) {
        unsigned long long k = 0xffffffffffffffffull;
        if (i < n) {
            double d = bearing_dist(T, wpts + 3 * i, bvs + 3 * i);
            if (d < 0) d = 0;
            d = d * d;
            k = (d == d) ? (unsigned long long)__double_as_longlong(d) : 0xfff8000000000000ull;   // non-negative: bits are monotonic
        }
        keys[i] = k;
    }
    __syncthreads();
    for (int k = 2; k <= m; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < m; i += MED_THREADS) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long a = keys[i], b = keys[l];
                    const bool up = (i & k) == 0;
                    if ((a > b) == up) { keys[i] = b; keys[l] = a; }
                }
            }
            __syncthreads();
        }
    if (tid == 0) {
        const int mid = n / 2;
        const double hi = __longlong_as_double((long long)keys[mid]);
        const double pen = (n % 2 == 0) ? (__longlong_as_double((long long)keys[mid - 1]) + hi) / 2 : hi;
        P.pen[(size_t)prob * P.max_iter + hy] = pen;
    }
}

// ------------------------------------------------------------------ kernel B': inlier count per hypothesis (RANSAC)
// one CTA per (hypothesis, problem): pen[k] = #points with bearing distance <= threshold under hypothesis k
__global__ void __launch_bounds__(MED_THREADS) p3p_inlier_count_kernel(const LmedsParams P) {
    __shared__ int cnt[MED_THREADS];
    const int prob = blockIdx.y, hy = blockIdx.x, tid = threadIdx.x;
    if (hy >= P.nhyp[2 * prob]) return;
    const int n = P.counts ? min(P.counts[prob], P.cap) : P.cap;
    const double* bvs = P.bvs + (size_t)prob * P.cap * 3;
    const double* wpts = P.wpts + (size_t)prob * P.cap * 3;
    double T[12];
    const double* Tg = P.hyp + ((size_t)prob * P.max_iter + hy) * 12;
#pragma unroll
    for (int i = 0; i < 12; i++) T[i] = Tg[i];
    int mine = 0;
    for (int i = tid; i < n; i += MED_THREADS) mine += bearing_dist(T, wpts + 3 * i, bvs + 3 * i) <= P.threshold;
    cnt[tid] = mine;
    __syncthreads();
    for (int s = MED_THREADS / 2; s > 0; s >>= 1) { if (tid < s) cnt[tid] += cnt[tid + s]; __syncthreads(); }
    if (tid == 0) P.pen[(size_t)prob * P.max_iter + hy] = (double)cnt[0];
}

// ------------------------------------------------------------------ kernel C: best model, inliers, checks
// LMedS (RANSAC = false): the first strict minimum of the median; RANSAC: the first strict maximum of the inlier count (a
// hypothesis without inliers is never selected).  info[2] = the best median (LMedS) / the selected hypothesis' index (RANSAC).
template <bool RANSAC>
__global__ void __launch_bounds__(256) p3p_select_kernel(const LmedsParams P) {
    __shared__ int s_best;
    __shared__ double s_pen;
    const int prob = blockIdx.x, tid = threadIdx.x;
    const int n = P.counts ? min(P.counts[prob], P.cap) : P.cap;
    const int nh = P.nhyp[2 * prob];
    uint8_t* outl = P.outlier + (size_t)prob * P.cap;
    double* info = P.info ? P.info + 4 * prob : nullptr;
    if (tid == 0) {
        double best = RANSAC ? 0.0 : DBL_MAX;
        int bi = -1;
        for (int k = 0; k < nh; k++) {
            const double v = P.pen[(size_t)prob * P.max_iter + k];
            if (RANSAC ? v > best : v < best) { best = v; bi = k; }
        }
        s_best = bi; s_pen = RANSAC ? (double)bi : best;
    }
    __syncthreads();
    const int bi = s_best;
    if (bi < 0) {
        for (int i = tid; i < P.cap; i += blockDim.x) outl[i] = 1;
        if (tid == 0 && info) { info[0] = 0; info[1] = 0; info[2] = DBL_MAX; info[3] = P.nhyp[2 * prob + 1]; }
        return;
    }
    double T[12];
    const double* Tg = P.hyp + ((size_t)prob * P.max_iter + bi) * 12;
#pragma unroll
    for (int i = 0; i < 12; i++) T[i] = Tg[i];
    const double* bvs = P.bvs + (size_t)prob * P.cap * 3;
    const double* wpts = P.wpts + (size_t)prob * P.cap * 3;
    int mine = 0;
    for (int i = tid; i < P.cap; i += blockDim.x) {
        bool out = true;
        if (i < n) out = !(bearing_dist(T, wpts + 3 * i, bvs + 3 * i) <= P.threshold);
        outl[i] = out ? 1 : 0;
        mine += (i < n && !out);
    }
    // deterministic count
    __shared__ int cnt[256];
    cnt[tid] = mine;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) { if (tid < s) cnt[tid] += cnt[tid + s]; __syncthreads(); }
    if (tid == 0) {
        double e = 0;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                const double v = T[4 * i] * T[4 * j] + T[4 * i + 1] * T[4 * j + 1] + T[4 * i + 2] * T[4 * j + 2] - (i == j ? 1.0 : 0.0);
                e += v * v;
            }
        const int ninl = cnt[0];
        const bool ok = ninl >= 5 && sqrt(e) < 1e-10;   // multi_view_geometry.cpp:83-92, Sophus::isOrthogonal
        for (int i = 0; i < 12; i++) P.Twc[12 * prob + i] = T[i];
        if (info) { info[0] = ok ? 1 : 0; info[1] = ninl; info[2] = s_pen; info[3] = P.nhyp[2 * prob + 1]; }
    }
}

// ================================================================== PnP (one CTA per problem)
constexpr int PNP_THREADS = 128;

__device__ __forceinline__ void q_to_R(const double* q, double* R) {
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}

// SE3Parameterization::Plus: exp(delta) * T, delta = [upsilon, omega]  (ceres_parametrization.hpp:224-240, Sophus se3.hpp / so3.hpp)
__device__ void se3_plus(const double* x, const double* delta, double* out) {
    const double* ups = delta;
    const double* om = delta + 3;
    const double theta_sq = om[0] * om[0] + om[1] * om[1] + om[2] * om[2];
    double theta, imag, real;
    const double eps = 1e-10;
    if (theta_sq < eps * eps) {
        theta = 0;
        const double t4 = theta_sq * theta_sq;
        imag = 0.5 - (1.0 / 48.0) * theta_sq + (1.0 / 3840.0) * t4;
        real = 1.0 - (1.0 / 8.0) * theta_sq + (1.0 / 384.0) * t4;
    } else {
        theta = sqrt(theta_sq);
        const double half = 0.5 * theta;
        imag = sin(half) / theta;
        real = cos(half);
    }
    const double dq[4] = {imag * om[0], imag * om[1], imag * om[2], real};
    double Rd[9];
    q_to_R(dq, Rd);   // dq is unit up to rounding; the oracle uses it un-normalised, the difference is ~1e-16
    const double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0};
    double O2[9], V[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) O2[3 * i + j] = O[3 * i] * O[j] + O[3 * i + 1] * O[3 + j] + O[3 * i + 2] * O[6 + j];
    if (theta < eps) { for (int i = 0; i < 9; i++) V[i] = Rd[i]; }
    else {
        const double a = (1 - cos(theta)) / theta_sq, b = (theta - sin(theta)) / (theta_sq * theta);
        for (int i = 0; i < 9; i++) V[i] = ((i % 4 == 0) ? 1.0 : 0.0) + a * O[i] + b * O2[i];
    }
    double qn[4];
    { const double n = sqrt(x[3] * x[3] + x[4] * x[4] + x[5] * x[5] + x[6] * x[6]); for (int i = 0; i < 4; i++) qn[i] = x[3 + i] / n; }
    for (int i = 0; i < 3; i++)
        out[i] = (V[3 * i] * ups[0] + V[3 * i + 1] * ups[1] + V[3 * i + 2] * ups[2]) + (Rd[3 * i] * x[0] + Rd[3 * i + 1] * x[1] + Rd[3 * i + 2] * x[2]);
    const double ax = dq[0], ay = dq[1], az = dq[2], aw = dq[3], bx = qn[0], by = qn[1], bz = qn[2], bw = qn[3];
    double qo[4] = {aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                    aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz};
    const double nn = sqrt(qo[0] * qo[0] + qo[1] * qo[1] + qo[2] * qo[2] + qo[3] * qo[3]);
    for (int i = 0; i < 4; i++) out[3 + i] = qo[i] / nn;
}

// ReprojectionErrorSE3::Evaluate with R = R_wc precomputed: res, (optional) 2x6 local Jacobian; returns depth-positive
__device__ __forceinline__ bool pnp_eval(const double* K, const double* R, const double* t, const double* X, const double* uv,
                                         double* res, double* J) {
    const double d[3] = {X[0] - t[0], X[1] - t[1], X[2] - t[2]};
    double c[3];
#pragma unroll
    for (int i = 0; i < 3; i++) c[i] = R[i] * d[0] + R[3 + i] * d[1] + R[6 + i] * d[2];
    const double iz = 1. / c[2];
    res[0] = K[0] * c[0] * iz + K[2] - uv[0];
    res[1] = K[1] * c[1] * iz + K[3] - uv[1];
    if (J) {
        const double iz2 = iz * iz;
        const double Jc[6] = {iz * K[0], 0, -c[0] * iz2 * K[0], 0, iz * K[1], -c[1] * iz2 * K[1]};
        double JR[6];
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
            for (int k = 0; k < 3; k++) JR[3 * r + k] = Jc[3 * r] * R[3 * k] + Jc[3 * r + 1] * R[3 * k + 1] + Jc[3 * r + 2] * R[3 * k + 2];
        const double Sk[9] = {0, -X[2], X[1], X[2], 0, -X[0], -X[1], X[0], 0};
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
            for (int k = 0; k < 3; k++) {
                J[6 * r + k] = -JR[3 * r + k];
                J[6 * r + 3 + k] = JR[3 * r] * Sk[k] + JR[3 * r + 1] * Sk[3 + k] + JR[3 * r + 2] * Sk[6 + k];
            }
    }
    return c[2] > 0;
}
__device__ __forceinline__ void huber_rho(double s, double delta, double& rho0, double& rho1) {
    if (delta > 0 && s > delta * delta) {
        const double r = sqrt(s);
        rho0 = 2 * delta * r - delta * delta;
        const double v = delta / r;
        rho1 = v > DBL_MIN ? v : DBL_MIN;
    } else { rho0 = s; rho1 = 1.0; }
}

struct PnpShared {
    double red[PNP_THREADS / 32][28];
    double H[21], g[6], cost;          // block-reduced linearisation (H upper triangle, row-major)
    double pose[7], cand[7], last[7], R[9];
    double nf[6], sc[6], diag[6];
    double radius, decrease_factor, x_cost, xn, gmax, model_change, cand_cost;
    double se_min, se_cur, se_ref, se_cand, se_acc_ref, se_acc_cand;
    int reuse_diagonal, invalid_steps, n_success, n_iter, term, iteration, last_success, action;
};

// fixed-order block reduction of NV per-thread doubles into dst (all threads call; result valid after the trailing sync)
template <int NV>
__device__ void block_reduce(double* v, PnpShared& S, double* dst) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; k++) {
        double x = v[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) x += __shfl_down_sync(0xffffffffu, x, off);
        if (lane == 0) S.red[wid][k] = x;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        double x = 0;
        for (int w = 0; w < PNP_THREADS / 32; w++) x += S.red[w][threadIdx.x];
        dst[threadIdx.x] = x;
    }
    __syncthreads();
}

struct PnpProblem { const double* K; const double* uv; const double* X; const uint8_t* removed; int n; double huber; };

__device__ void pnp_linearize(const PnpProblem& Q, const double* pose, PnpShared& S) {
    if (threadIdx.x == 0) q_to_R(pose + 3, S.R);
    __syncthreads();
    double R[9], t[3] = {pose[0], pose[1], pose[2]};
#pragma unroll
    for (int i = 0; i < 9; i++) R[i] = S.R[i];
    double acc[28];
#pragma unroll
    for (int k = 0; k < 28; k++) acc[k] = 0;
    for (int i = threadIdx.x; i < Q.n; i += PNP_THREADS) {
        if (Q.removed && Q.removed[i]) continue;
        double r[2], J[12];
        pnp_eval(Q.K, R, t, Q.X + 3 * i, Q.uv + 2 * i, r, J);
        double r0, r1;
        huber_rho(r[0] * r[0] + r[1] * r[1], Q.huber, r0, r1);
        const double sc = sqrt(r1);
        r[0] *= sc; r[1] *= sc;
#pragma unroll
        for (int k = 0; k < 12; k++) J[k] *= sc;
        int o = 0;
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = a; b < 6; b++) acc[o++] += J[a] * J[b] + J[6 + a] * J[6 + b];
#pragma unroll
        for (int a = 0; a < 6; a++) acc[21 + a] += J[a] * r[0] + J[6 + a] * r[1];
        acc[27] += 0.5 * r0;
    }
    block_reduce<28>(acc, S, S.H);   // H[21], g[6], cost are contiguous in PnpShared
}
__device__ void pnp_cost(const PnpProblem& Q, const double* pose, PnpShared& S, double* dst) {
    if (threadIdx.x == 0) q_to_R(pose + 3, S.R);
    __syncthreads();
    double R[9], t[3] = {pose[0], pose[1], pose[2]};
#pragma unroll
    for (int i = 0; i < 9; i++) R[i] = S.R[i];
    double acc[1] = {0};
    for (int i = threadIdx.x; i < Q.n; i += PNP_THREADS) {
        if (Q.removed && Q.removed[i]) continue;
        double r[2], r0, r1;
        pnp_eval(Q.K, R, t, Q.X + 3 * i, Q.uv + 2 * i, r, nullptr);
        huber_rho(r[0] * r[0] + r[1] * r[1], Q.huber, r0, r1);
        acc[0] += 0.5 * r0;
    }
    block_reduce<1>(acc, S, dst);
}
__device__ __forceinline__ double Hget(const double* H, int a, int b) {   // upper triangle, row-major packed
    if (a > b) { const int t = a; a = b; b = t; }
    return H[a * 6 - a * (a - 1) / 2 + (b - a)];
}
__device__ bool chol6(const double* Sm, const double* b, double* x) {
    double L[36];
    for (int i = 0; i < 36; i++) L[i] = Sm[i];
    for (int j = 0; j < 6; j++) {
        double d = L[6 * j + j];
        for (int k = 0; k < j; k++) d -= L[6 * j + k] * L[6 * j + k];
        if (!(d > 0)) return false;
        d = sqrt(d);
        L[6 * j + j] = d;
        for (int i = j + 1; i < 6; i++) {
            double s = L[6 * i + j];
            for (int k = 0; k < j; k++) s -= L[6 * i + k] * L[6 * j + k];
            L[6 * i + j] = s / d;
        }
    }
    for (int i = 0; i < 6; i++) { double s = b[i]; for (int k = 0; k < i; k++) s -= L[6 * i + k] * x[k]; x[i] = s / L[6 * i + i]; }
    for (int i = 5; i >= 0; i--) { double s = x[i]; for (int k = i + 1; k < 6; k++) s -= L[6 * k + i] * x[k]; x[i] = s / L[6 * i + i]; }
    return true;
}
__device__ __forceinline__ double v7norm(const double* p) { double s = 0; for (int i = 0; i < 7; i++) s += p[i] * p[i]; return sqrt(s); }
__device__ __forceinline__ double v7diff(const double* a, const double* b, bool inf) {
    double s = 0;
    for (int i = 0; i < 7; i++) { const double e = fabs(a[i] - b[i]); if (inf) { if (e > s) s = e; } else s += e * e; }
    return inf ? s : sqrt(s);
}

// one ceres::Solve (trust-region LM, one 6-dof block) executed by the whole CTA; S.pose in/out, S.last = last evaluated point
__device__ void pnp_solve(const PnpProblem& Q, PnpShared& S, int max_iter, double* summary) {
    const int tid = threadIdx.x;
    pnp_linearize(Q, S.pose, S);
    if (tid == 0) {
        S.radius = 1e4; S.decrease_factor = 2.0; S.reuse_diagonal = 0; S.invalid_steps = 0;
        S.x_cost = S.cost;
        for (int i = 0; i < 7; i++) S.last[i] = S.pose[i];
        for (int i = 0; i < 6; i++) { S.nf[i] = Hget(S.H, i, i); S.sc[i] = 1.0 / (1.0 + sqrt(S.nf[i])); }
        S.xn = v7norm(S.pose);
        S.se_min = S.se_cur = S.se_ref = S.se_cand = S.x_cost; S.se_acc_ref = S.se_acc_cand = 0;
        S.n_success = 0; S.n_iter = 0; S.term = 1; S.iteration = 0; S.last_success = 1;
        summary[0] = S.x_cost;
        double gneg[6], c[7];
        for (int i = 0; i < 6; i++) gneg[i] = -S.g[i];
        se3_plus(S.pose, gneg, c);
        S.gmax = v7diff(S.pose, c, true);
    }
    __syncthreads();
    for (;;) {
        if (tid == 0) {
            int action = 1;   // 0 stop, 1 evaluate candidate, 2 retry (invalid step)
            if (S.last_success) S.n_success++;
            S.n_iter++;
            if (S.iteration >= max_iter) { S.term = 1; action = 0; }
            else if (S.last_success && S.gmax <= 1e-10) { S.term = 0; action = 0; }
            else if (S.radius <= 1e-32) { S.term = 0; action = 0; }
            if (action) {
                S.iteration++;
                S.last_success = 0;
                if (!S.reuse_diagonal)
                    for (int i = 0; i < 6; i++) S.diag[i] = fmin(fmax(S.nf[i] * S.sc[i] * S.sc[i], 1e-6), 1e32);
                S.reuse_diagonal = 1;
                double Sm[36], rhs[6], y[6];
                for (int a = 0; a < 6; a++) {
                    rhs[a] = S.g[a] * S.sc[a];
                    for (int b = 0; b < 6; b++) Sm[6 * a + b] = Hget(S.H, a, b) * S.sc[a] * S.sc[b];
                    Sm[7 * a] += S.diag[a] / S.radius;
                }
                const bool ok = chol6(Sm, rhs, y);
                double mc = -1;
                if (ok) {
                    double lin = 0, quad = 0;
                    for (int a = 0; a < 6; a++) {
                        lin += -y[a] * rhs[a];
                        for (int b = 0; b < 6; b++) quad += y[a] * (Hget(S.H, a, b) * S.sc[a] * S.sc[b]) * y[b];
                    }
                    mc = -(lin + 0.5 * quad);
                }
                if (!ok || !(mc > 0.0)) {
                    if (++S.invalid_steps >= 5) { S.term = 2; action = 0; }
                    else { S.radius *= 0.5; S.reuse_diagonal = 1; action = 2; }
                } else {
                    S.invalid_steps = 0;
                    S.model_change = mc;
                    double df[6];
                    for (int i = 0; i < 6; i++) df[i] = -y[i] * S.sc[i];
                    se3_plus(S.pose, df, S.cand);
                }
            }
            S.action = action;
        }
        __syncthreads();
        const int action = S.action;
        if (action == 0) break;
        if (action == 2) continue;
        pnp_cost(Q, S.cand, S, &S.cand_cost);
        if (tid == 0) {
            int act = 2;   // 0 stop, 1 accepted (re-linearise), 2 rejected
            for (int i = 0; i < 7; i++) S.last[i] = S.cand[i];
            const double step_norm = v7diff(S.pose, S.cand, false);
            if (step_norm <= 1e-8 * (S.xn + 1e-8)) { S.term = 0; act = 0; }
            else if (fabs(S.x_cost - S.cand_cost) <= 1e-3 * S.x_cost) { S.term = 0; act = 0; }
            else {
                const double rel = (S.se_cur - S.cand_cost) / S.model_change;
                const double hist = (S.se_ref - S.cand_cost) / (S.se_acc_ref + S.model_change);
                const double quality = rel > hist ? rel : hist;
                if (quality > 1e-3) {
                    for (int i = 0; i < 7; i++) S.pose[i] = S.cand[i];
                    S.xn = v7norm(S.pose);
                    S.radius = S.radius / fmax(1.0 / 3.0, 1.0 - pow(2.0 * quality - 1.0, 3));
                    S.radius = fmin(1e16, S.radius);
                    S.decrease_factor = 2.0;
                    S.reuse_diagonal = 0;
                    S.se_cur = S.cand_cost; S.se_acc_cand += S.model_change; S.se_acc_ref += S.model_change;
                    bool nonmono = false;
                    if (S.se_cur < S.se_min) { S.se_min = S.se_cur; S.se_cand = S.se_cur; S.se_acc_cand = 0; }
                    else { nonmono = true; if (S.se_cur > S.se_cand) { S.se_cand = S.se_cur; S.se_acc_cand = 0; } }
                    if (!nonmono) { S.se_ref = S.se_cand; S.se_acc_ref = S.se_acc_cand; }
                    S.last_success = 1;
                    act = 1;
                } else {
                    S.radius = S.radius / S.decrease_factor;
                    S.decrease_factor *= 2.0;
                    S.reuse_diagonal = 1;
                }
            }
            S.action = act;
        }
        __syncthreads();
        const int act = S.action;
        if (act == 0) break;
        if (act == 1) {
            pnp_linearize(Q, S.pose, S);
            if (tid == 0) {
                S.x_cost = S.cost;
                for (int i = 0; i < 6; i++) S.nf[i] = Hget(S.H, i, i);
                double gneg[6], c[7];
                for (int i = 0; i < 6; i++) gneg[i] = -S.g[i];
                se3_plus(S.pose, gneg, c);
                S.gmax = v7diff(S.pose, c, true);
            }
            __syncthreads();
        }
    }
    if (tid == 0) { summary[1] = S.x_cost; summary[2] = S.n_success; summary[3] = S.n_iter; summary[4] = S.term; }
    __syncthreads();
}

struct PnpParams {
    const double* K; const double* uv; const double* X; const int32_t* counts;
    int cap, max_iter, use_robust, apply_l2;
    double huber, chi2;
    double* poses; uint8_t* outlier; double* summary;
};

__global__ void __launch_bounds__(PNP_THREADS) pnp_kernel(const PnpParams P) {
    __shared__ PnpShared S;
    __shared__ int s_nbad;
    const int prob = blockIdx.x, tid = threadIdx.x;
    const int n = P.counts ? min(P.counts[prob], P.cap) : P.cap;
    uint8_t* outl = P.outlier + (size_t)prob * P.cap;
    double* summ = P.summary + 12 * prob;
    PnpProblem Q{P.K + 4 * prob, P.uv + (size_t)prob * P.cap * 2, P.X + (size_t)prob * P.cap * 3, nullptr, n,
                 P.use_robust ? P.huber : 0.0};
    if (tid < 12) summ[tid] = 0;
    if (tid < 7) S.pose[tid] = P.poses[7 * prob + tid];
    __syncthreads();
    if (n < 1) { for (int i = tid; i < P.cap; i += PNP_THREADS) outl[i] = 0; return; }
    pnp_solve(Q, S, P.max_iter, summ);
    // flag at the LAST evaluated point (the functors keep chi2err_ / isDepthPositive_ of their last Evaluate call)
    if (tid == 0) q_to_R(S.last + 3, S.R);
    __syncthreads();
    int mine = 0;
    for (int i = tid; i < P.cap; i += PNP_THREADS) {
        uint8_t o = 0;
        if (i < n) {
            double r[2];
            const bool dp = pnp_eval(Q.K, S.R, S.last, Q.X + 3 * i, Q.uv + 2 * i, r, nullptr);
            o = (r[0] * r[0] + r[1] * r[1] > P.chi2 || !dp) ? 1 : 0;
        }
        outl[i] = o;
        mine += o;
    }
    {
        __shared__ int cnt[PNP_THREADS];
        cnt[tid] = mine;
        __syncthreads();
        for (int s = PNP_THREADS / 2; s > 0; s >>= 1) { if (tid < s) cnt[tid] += cnt[tid + s]; __syncthreads(); }
        if (tid == 0) s_nbad = cnt[0];
        __syncthreads();
    }
    const int bad = s_nbad;
    int usable = (int)(summ[4] != 2.0);
    if (bad == n) {   // multi_view_geometry.cpp:205-208: return false before the pose is read back
        if (tid == 0) { summ[10] = 0; summ[11] = bad; }
        return;
    }
    if (P.apply_l2 && bad > 0) {
        __threadfence_block();
        Q.removed = outl;
        Q.huber = 0.0;
        pnp_solve(Q, S, P.max_iter, summ + 5);
        usable = (int)(summ[9] != 2.0);
    }
    if (tid < 7) P.poses[7 * prob + tid] = S.pose[tid];
    if (tid == 0) { summ[10] = usable; summ[11] = bad; }
}


// ---- P3P -> PnP hand-over on the device (System's per-frame pose without a host round trip in between) ----------------------
// What VisualFrontend::computePose does on the host between the two solvers (visual_frontend.cpp:300-357): the P3P pose becomes
// the PnP start (rotation matrix -> Eigen quaternion), the P3P outliers leave the correspondence list (order kept).
__global__ void __launch_bounds__(256) pnp_from_p3p_kernel(int cap, const int32_t* __restrict__ counts, int n_fixed,
                                                           const double* __restrict__ T12, const uint8_t* __restrict__ outl,
                                                           const double* __restrict__ uv, const double* __restrict__ X,
                                                           double* __restrict__ uv2, double* __restrict__ X2, int32_t* __restrict__ n2,
                                                           double* __restrict__ pose7) {
    __shared__ int woff[8];
    __shared__ int base_s;
    const int prob = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = counts ? min(counts[prob], cap) : n_fixed;
    const uint8_t* o = outl + (size_t)prob * cap;
    const double *u = uv + (size_t)prob * cap * 2, *x = X + (size_t)prob * cap * 3;
    double *u2 = uv2 + (size_t)prob * cap * 2, *x2 = X2 + (size_t)prob * cap * 3;
    if (tid == 0) {
        base_s = 0;
        // Se3::setR (system_core.h) = Eigen's matrix -> quaternion, then normalised; no contraction (the host compiles it with
        // -ffp-contract=off)
        const double* T = T12 + 12 * prob;
        const double M[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
        double q[4];
        double tr = __dadd_rn(__dadd_rn(M[0], M[4]), M[8]);
        if (tr > 0) {
            tr = sqrt(__dadd_rn(tr, 1.0));
            q[3] = __dmul_rn(0.5, tr); tr = 0.5 / tr;
            q[0] = __dmul_rn(__dsub_rn(M[7], M[5]), tr); q[1] = __dmul_rn(__dsub_rn(M[2], M[6]), tr); q[2] = __dmul_rn(__dsub_rn(M[3], M[1]), tr);
        } else {
            int i = 0;
            if (M[4] > M[0]) i = 1;
            if (M[8] > M[4 * i]) i = 2;
            const int j = (i + 1) % 3, k = (j + 1) % 3;
            tr = sqrt(__dadd_rn(__dsub_rn(__dsub_rn(M[4 * i], M[4 * j]), M[4 * k]), 1.0));
            q[i] = __dmul_rn(0.5, tr); tr = 0.5 / tr;
            q[3] = __dmul_rn(__dsub_rn(M[3 * k + j], M[3 * j + k]), tr);
            q[j] = __dmul_rn(__dadd_rn(M[3 * j + i], M[3 * i + j]), tr);
            q[k] = __dmul_rn(__dadd_rn(M[3 * k + i], M[3 * i + k]), tr);
        }
        const double nn = sqrt(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])), __dmul_rn(q[3], q[3])));
        double* p = pose7 + 7 * prob;
        p[0] = T[3]; p[1] = T[7]; p[2] = T[11];
        for (int c = 0; c < 4; c++) p[3 + c] = q[c] / nn;
    }
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += 256) {
        const int i = i0 + tid;
        const bool keep = i < n && o[i] == 0;
        const uint32_t m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) woff[warp] = __popc(m);
        __syncthreads();
        int off = base_s;
        for (int w = 0; w < warp; w++) off += woff[w];
        if (keep) {
            const int d = off + __popc(m & ((1u << lane) - 1u));
            u2[2 * d] = u[2 * i]; u2[2 * d + 1] = u[2 * i + 1];
            x2[3 * d] = x[3 * i]; x2[3 * d + 1] = x[3 * i + 1]; x2[3 * d + 2] = x[3 * i + 2];
        }
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < 8; w++) t += woff[w]; base_s += t; }
        __syncthreads();
    }
    if (tid == 0) n2[prob] = base_s;
}

}  // namespace

// SampleConsensusProblem::rnd() for a given seed: std::uniform_int_distribution<int>(0, INT_MAX) over std::mt19937 -- the very
// objects the reference uses (SampleConsensusProblem.hpp:41-48), evaluated by this host's libstdc++
static void make_rnd_table(uint32_t seed, int n, std::vector<int32_t>& out) {
    std::mt19937 alg(seed);
    std::uniform_int_distribution<> dist(0, std::numeric_limits<int>::max());
    out.resize(n);
    for (int i = 0; i < n; i++) out[i] = dist(alg);
}

// the sampler table depends only on (seed, length) and a longer table starts with the shorter one: kept on the device across
// calls (System draws it every frame) and regrown only when a caller needs more of it or another seed
static int p3p_rnd_table(alva_ctx* ctx, uint32_t seed, int len) {
    if (ctx->p3p_tab && ctx->p3p_tab_len >= len && ctx->p3p_tab_seed == seed) return 0;
    std::vector<int32_t> host_tab;
    make_rnd_table(seed, len, host_tab);
    ctx->ws_epoch++;
    if (ctx->p3p_tab) { ALVA_CUDA(cudaStreamSynchronize(ctx->stream)); ALVA_CUDA(cudaFree(ctx->p3p_tab)); ctx->p3p_tab = nullptr; }
    ALVA_CUDA(cudaMalloc(&ctx->p3p_tab, (size_t)len * 4));
    ALVA_CUDA(cudaMemcpy(ctx->p3p_tab, host_tab.data(), (size_t)len * 4, cudaMemcpyHostToDevice));
    ctx->p3p_tab_len = len; ctx->p3p_tab_seed = seed;
    return 0;
}

extern "C" int alva_k_p3p_lmeds(alva_ctx* ctx, int nprob, int cap, const double* bvs, const double* wpts, const int32_t* counts,
                                int max_iter, float err_px, float fx, float fy, uint32_t seed, double* Twc_out,
                                uint8_t* outlier, double* info) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !bvs || !wpts || !Twc_out || !outlier || nprob < 1 || cap < 1 || max_iter < 1 || max_iter > 1024) {
        alva_set_error("alva_k_p3p_lmeds: bad argument");
        return ALVA_E_INVALID;
    }
    if (cap > 4096) { alva_set_error("alva_k_p3p_lmeds: at most 4096 points per problem (got %d)", cap); return ALVA_E_INVALID; }
    // threshold in the reference's float arithmetic (multi_view_geometry.cpp:70-75)
    float focal = fx + fy;
    focal = (float)(focal / 2.);
    LmedsParams P{};
    P.threshold = 1.0 - cosf(atanf(err_px / focal));
    P.bvs = bvs; P.wpts = wpts; P.counts = counts; P.cap = cap; P.max_iter = max_iter; P.max_skip = max_iter * 10;
    P.table_len = 4 * (max_iter + P.max_skip + HYP_THREADS);
    const size_t hyp_b = (size_t)nprob * max_iter * 12 * sizeof(double), pen_b = (size_t)nprob * max_iter * sizeof(double);
    const size_t tab_b = ((size_t)P.table_len * 4 + 255) & ~(size_t)255, nh_b = ((size_t)nprob * 8 + 255) & ~(size_t)255;
    uint8_t* ws = (uint8_t*)alva_scratch(ctx, hyp_b + pen_b + tab_b + nh_b + 1024);
    if (!ws) return ALVA_E_CUDA;
    P.hyp = (double*)ws; P.pen = (double*)(ws + hyp_b);
    int32_t* tab = (int32_t*)(ws + hyp_b + pen_b);
    P.rnd = tab; P.nhyp = (int32_t*)(ws + hyp_b + pen_b + tab_b);
    P.Twc = Twc_out; P.outlier = outlier; P.info = info;
    (void)tab;
    if (int e = p3p_rnd_table(ctx, seed, P.table_len)) return e;
    P.rnd = (const int32_t*)ctx->p3p_tab;
    p3p_hypotheses_kernel<<<nprob, HYP_THREADS, (size_t)cap * sizeof(int), ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    int m = 1;
    while (m < cap) m <<= 1;
    p3p_median_kernel<<<dim3(max_iter, nprob), MED_THREADS, (size_t)m * 8, ctx->stream>>>(P, m);
    ALVA_LAUNCH_CHECK(ctx);
    p3p_select_kernel<false><<<nprob, 256, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// P3P-RANSAC: the sampler and hypotheses of alva_k_p3p_lmeds (the same kernel: the same seed gives the same hypotheses),
// each scored by its inlier count at the same threshold; the first strict maximum is the model
extern "C" int alva_k_p3p_ransac(alva_ctx* ctx, int nprob, int cap, const double* bvs, const double* wpts, const int32_t* counts,
                                 int max_iter, float err_px, float fx, float fy, uint32_t seed, double* Twc_out,
                                 uint8_t* outlier, double* info) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !bvs || !wpts || !Twc_out || !outlier || nprob < 1 || cap < 1 || max_iter < 1 || max_iter > 1024) {
        alva_set_error("alva_k_p3p_ransac: bad argument");
        return ALVA_E_INVALID;
    }
    if (cap > 8192) { alva_set_error("alva_k_p3p_ransac: at most 8192 points per problem (got %d)", cap); return ALVA_E_INVALID; }
    float focal = fx + fy;
    focal = (float)(focal / 2.);
    LmedsParams P{};
    P.threshold = 1.0 - cosf(atanf(err_px / focal));
    P.bvs = bvs; P.wpts = wpts; P.counts = counts; P.cap = cap; P.max_iter = max_iter; P.max_skip = max_iter * 10;
    P.table_len = 4 * (max_iter + P.max_skip + HYP_THREADS);
    const size_t hyp_b = (size_t)nprob * max_iter * 12 * sizeof(double), pen_b = (size_t)nprob * max_iter * sizeof(double);
    const size_t nh_b = ((size_t)nprob * 8 + 255) & ~(size_t)255;
    uint8_t* ws = (uint8_t*)alva_scratch(ctx, hyp_b + pen_b + nh_b + 1024);
    if (!ws) return ALVA_E_CUDA;
    P.hyp = (double*)ws; P.pen = (double*)(ws + hyp_b); P.nhyp = (int32_t*)(ws + hyp_b + pen_b);
    P.Twc = Twc_out; P.outlier = outlier; P.info = info;
    if (int e = p3p_rnd_table(ctx, seed, P.table_len)) return e;
    P.rnd = (const int32_t*)ctx->p3p_tab;
    p3p_hypotheses_kernel<<<nprob, HYP_THREADS, (size_t)cap * sizeof(int), ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    p3p_inlier_count_kernel<<<dim3(max_iter, nprob), MED_THREADS, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    p3p_select_kernel<true><<<nprob, 256, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_pnp(alva_ctx* ctx, int nprob, int cap, const double* K, const double* uv, const double* X,
                          const int32_t* counts, double* poses, double huber_delta, double chi2_thr, int max_iter,
                          int use_robust, int apply_l2, uint8_t* outlier, double* summary) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !K || !uv || !X || !poses || !outlier || !summary || nprob < 1 || cap < 1 || max_iter < 0) {
        alva_set_error("alva_k_pnp: bad argument");
        return ALVA_E_INVALID;
    }
    PnpParams P{K, uv, X, counts, cap, max_iter, use_robust, apply_l2, huber_delta, chi2_thr, poses, outlier, summary};
    pnp_kernel<<<nprob, PNP_THREADS, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// internal (system.cu): P3P-LMedS -> hand-over -> PnP for ONE problem, everything on the stream, no host synchronisation.
// bvs / X / uv: the n correspondences (device); K4: calibration (device, 4 doubles); T12 + info: P3P's result ([12] + [4]);
// o1 [cap]: P3P outliers; uv2 / X2 [cap]: scratch for the surviving correspondences; n2: their count; pose7: PnP start -> result;
// o2 [cap]: PnP outliers over the survivors; summ [12]: PnP summary.
int alva_pose_chain_launch(alva_ctx* ctx, int n, int cap, const double* bvs, const double* X, const double* uv, const double* K4,
                           float fx, float fy, uint32_t seed, double* T12, double* info, uint8_t* o1, double* uv2, double* X2,
                           int32_t* n2, double* pose7, uint8_t* o2, double* summ, double huber, double chi2) {
    if (int e = alva_k_p3p_lmeds(ctx, 1, n, bvs, X, nullptr, 100, 3.0f, fx, fy, seed, T12, o1, info)) return e;
    pnp_from_p3p_kernel<<<1, 256, 0, ctx->stream>>>(cap, nullptr, n, T12, o1, uv, X, uv2, X2, n2, pose7);
    ALVA_LAUNCH_CHECK(ctx);
    return alva_k_pnp(ctx, 1, cap, K4, uv2, X2, n2, pose7, huber, chi2, 5, 1, 1, o2, summ);
}

// internal (system.cu): the pose of a relocalised frame -- P3P-RANSAC (max_iter hypotheses) on the counts[0] correspondences
// alva_reloc_compact_launch wrote, the same hand-over as alva_pose_chain_launch, PnP on the RANSAC inliers; no host
// synchronisation.  Buffers as alva_pose_chain_launch, every point list [cap].
int alva_reloc_pose_launch(alva_ctx* ctx, int cap, const int32_t* counts, const double* bvs, const double* X, const double* uv,
                           const double* K4, float fx, float fy, uint32_t seed, int max_iter, double* T12, double* info, uint8_t* o1,
                           double* uv2, double* X2, int32_t* n2, double* pose7, uint8_t* o2, double* summ, double huber, double chi2) {
    if (int e = alva_k_p3p_ransac(ctx, 1, cap, bvs, X, counts, max_iter, 3.0f, fx, fy, seed, T12, o1, info)) return e;
    pnp_from_p3p_kernel<<<1, 256, 0, ctx->stream>>>(cap, counts, 0, T12, o1, uv, X, uv2, X2, n2, pose7);
    ALVA_LAUNCH_CHECK(ctx);
    return alva_k_pnp(ctx, 1, cap, K4, uv2, X2, n2, pose7, huber, chi2, 5, 1, 1, o2, summ);
}
