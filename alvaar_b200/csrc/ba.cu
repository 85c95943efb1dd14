// ba.cu -- local bundle adjustment (anchored inverse depth, SE(3) poses) on sm_90a: residual/Jacobian build,
// Huber re-weighting, Schur-complement reduction to the reduced camera system, dense Cholesky, back-substitution and
// Ceres' Levenberg-Marquardt trust-region control flow -- all on the device, batched over independent problems.
//
// Reference behaviour (CPU restatement: oracle/ba_oracle.c; pinned against ceres::Solve itself):
//   cost functor      DirectSE3::ReprojectionErrorKSE3AnchInvDepth::Evaluate   src/slam/src/ceres_parametrization.cpp:157-269
//   plus-op           SE3Parameterization::Plus                                src/slam/src/ceres_parametrization.hpp:224-240
//   problem / options Optimizer::localBA                                       src/slam/src/optimizer.cpp:20-262
//   robust loss       HuberLoss + Corrector                                    ceres-solver/internal/ceres/loss_function.cc:48-62, corrector.cc:36-134
//   Schur reduction   SchurEliminator::Eliminate / BackSubstitute              ceres-solver/internal/ceres/schur_eliminator_impl.h:176-375
//   LM shell          LevenbergMarquardtStrategy, TrustRegionMinimizer         levenberg_marquardt_strategy.cc:66-160, trust_region_minimizer.cc
//
// FP64 throughout (the north-star tolerance is 1e-4 relative; we land at ~1e-9).  The e-blocks are 1-dimensional
// (inverse depth), so (E'E)^-1 is a scalar reciprocal per landmark; the reduced system is <= 21 free poses x 6 = 126 wide
// (a problem with more is refused, termination 2) and lives in ONE CTA's shared memory for the (blocked) Cholesky / triangular solves; the Schur complement itself is
// assembled block-wise by a gather kernel (one warp per 6x6 pose-pair block, no atomics, bit-reproducible).  The trust-region decisions
// (accept / reject, radius update, function / parameter / gradient tolerance) run in single-CTA "control" kernels
// that read and write a device-resident state block, so an entire solve is a fixed launch sequence with no host
// synchronisation (graph-capturable).
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include <math.h>
#include <float.h>
#include <string.h>

namespace {

constexpr int NMAX = 128;   // max reduced-system width (>= 6 * free poses), padded
constexpr int LIN_THREADS = 128;
constexpr int NBMAX = NMAX / 6;                 // 21 free poses at most
constexpr int MAXKEYS = NBMAX * (NBMAX + 1) / 2;   // upper-triangular 6x6 blocks of the reduced system (grid of the gather kernel)
constexpr int BS_THREADS = 128;                // back-substitution CTA

struct BaState {
    double radius, decrease_factor, x_cost, cand_cost, xnorm, gmax, model_change;
    double se_min, se_cur, se_ref, se_cand, se_acc_ref, se_acc_cand;
    double initial_cost, push_cost;
    int reuse_diagonal, invalid_steps, iteration, last_success, n_success, n_iter, term, done;
    int relin, step_ok, ncols, chol_ok;
    int use_gather, nb, nbad, has_last;   // nbad / has_last: alva_k_ba_local (outliers removed, last evaluated point is cand)
    int skipped, pad0;
};

// per-problem views into the workspace
struct BaProblem {
    // inputs
    const double* calib;       // [4]
    double* poses;             // [nkf*7] in/out
    const uint8_t* pose_const; // [nkf]
    double* invd;              // [nlm]   in/out
    const int32_t* anch_kf;    // [nlm]
    const double* anch_uv;     // [nlm*2]
    const int32_t* obs_kf;     // [nobs]
    const int32_t* obs_lm;     // [nobs]  (-1 = unused slot)
    const double* obs_uv;      // [nobs*2]
    // workspace
    double *res, *Ja, *Jd;                  // per obs: 2, 12, 2 (the observer's Jacobian is -Ja exactly: see ba_evaluate)
    double *wp;                             // per obs: 6  (F_p^T e)
    double *nf, *gf, *scf, *diagf, *Df;     // [NMAX]
    double *ne, *ge, *sce, *diage, *De;     // [nlm]
    double *ete, *etb, *wa, *ye;            // [nlm], [nlm], [nlm*6], [nlm]
    double *S, *rhs, *yf;                   // [NMAX*NMAX], [NMAX], [NMAX]
    double *cand_poses, *cand_invd;         // [nkf*7], [nlm]
    double *cost_part;                      // [nblk]
    int32_t *pose_col;                      // [nkf]
    int32_t *lm_start, *lm_obs;             // CSR landmark -> observations: [nlm+1], [nobs]
    double* Wt;                             // dense Schur path: [nlm_pad][NMAX]
    double* mc_part;                        // model-cost partials, one per back-substitution CTA
    double* ga_part;                        // gather Schur: [NBMAX][GA_SPLIT][42] partial sums of the diagonal blocks
    int32_t* ga_ticket;                     // gather Schur: [NBMAX] arrival counters of a diagonal block's parts (wrap to 0)
    int32_t *obs_col, *anch_col;            // reduced-system column of each observation's / landmark anchor's pose (-1: fixed)
    int32_t *pstart;                        // gather Schur: [NBMAX + 1] ranges of plist per free pose
    uint32_t *plist;                        // gather Schur: (landmark << 8) | slot, every (landmark, slot) seeing that pose, by landmark
    int32_t *blk_start;                     // gather Schur: [NBMAX*NBMAX + 1] entry COUNTS per 6x6 block (bi <= bj), row-major, at [blk + 1]
    int32_t *blk_off;                       // gather Schur: [NBMAX*NBMAX] first entry of each block
    uint64_t *pairs;                        // gather Schur: per block, in plist order: landmark << 48 | slot_u << 40 | slot_v << 32 |
                                            //   observation index of slot_u << 16 | of slot_v (0xffff for the anchor slot)
    // alva_k_ba_local only (null otherwise): obs_lm above then points at obs_lm_w, the working copy removals are made in
    const int32_t* obs_lm_in;               // caller's obs_lm
    int32_t* obs_lm_w;                      // [nobs]
    int32_t* flags;                         // [nobs] out: 0 kept, 1 removed after solve 1, 2 flagged after solve 2
    double *last_poses, *last_invd;         // point of the cost functors' last evaluation (see ba_post_kernel)
    BaState* st;
};

struct BaDims { int nkf, nlm, nobs, nblk; double huber; int max_iter; int nlm_pad; int ecap; int nbs; int pass; };

// ------------------------------------------------------------------------------------------ SE(3) helpers
__device__ __forceinline__ void quat_to_R(const double* q, double* R) {   // q = (x,y,z,w), normalised here
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

// SE3Parameterization::Plus: out = exp([ups, om]) * (t, q)   (Sophus se3.hpp:763-784, so3.hpp:585-621)
__device__ void se3_plus(const double* x, const double* delta, double* out) {
    const double* ups = delta;
    const double* om = delta + 3;
    const double theta_sq = om[0] * om[0] + om[1] * om[1] + om[2] * om[2];
    const double eps = 1e-10;
    double theta, imag, real;
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
    quat_to_R(dq, Rd);
    const double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0};
    double V[9];
    if (theta < eps) {
        for (int i = 0; i < 9; i++) V[i] = Rd[i];
    } else {
        const double a = (1 - cos(theta)) / theta_sq, b = (theta - sin(theta)) / (theta_sq * theta);
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                double o2 = 0;
                for (int k = 0; k < 3; k++) o2 += O[3 * i + k] * O[3 * k + j];
                V[3 * i + j] = (i == j ? 1.0 : 0.0) + a * O[3 * i + j] + b * o2;
            }
    }
    for (int i = 0; i < 3; i++)
        out[i] = V[3 * i] * ups[0] + V[3 * i + 1] * ups[1] + V[3 * i + 2] * ups[2] + Rd[3 * i] * x[0] + Rd[3 * i + 1] * x[1] +
                 Rd[3 * i + 2] * x[2];
    const double qn = sqrt(x[3] * x[3] + x[4] * x[4] + x[5] * x[5] + x[6] * x[6]);
    const double bx = x[3] / qn, by = x[4] / qn, bz = x[5] / qn, bw = x[6] / qn;
    const double ax = dq[0], ay = dq[1], az = dq[2], aw = dq[3];
    double q[4] = {aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                   aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz};
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int i = 0; i < 4; i++) out[3 + i] = q[i] / n;
}

// ReprojectionErrorKSE3AnchInvDepth::Evaluate; Ja/Jp are the LOCAL 2x6 Jacobians (J_global * [I6; 0]).  Jp is Ja negated, entry
// for entry and bit for bit (negation is exact, also after the Huber scaling), so the solver's workspace keeps Ja alone and reads
// -Ja for the observer: 16 instead of 28 doubles per observation to write and read back every iteration.
__device__ __forceinline__ bool ba_evaluate(const double* calib, const double* anch, const double* pose, double invd, double u,
                                            double v, double ua, double va, double* res, double* Ja, double* Jp, double* Jd) {
    const double fx = calib[0], fy = calib[1], cx = calib[2], cy = calib[3];
    double Rwa[9], Rwc[9];
    quat_to_R(anch + 3, Rwa);
    quat_to_R(pose + 3, Rwc);
    const double zanch = 1.0 / invd;
    const double ap[3] = {zanch * (ua - cx) / fx, zanch * (va - cy) / fy, zanch};
    double Ra[3], wpt[3];
    for (int i = 0; i < 3; i++) {
        Ra[i] = Rwa[3 * i] * ap[0] + Rwa[3 * i + 1] * ap[1] + Rwa[3 * i + 2] * ap[2];
        wpt[i] = Ra[i] + anch[i];
    }
    const double d[3] = {wpt[0] - pose[0], wpt[1] - pose[1], wpt[2] - pose[2]};
    double cp[3];
    for (int i = 0; i < 3; i++) cp[i] = Rwc[i] * d[0] + Rwc[3 + i] * d[1] + Rwc[6 + i] * d[2];
    const double iz = 1.0 / cp[2];
    res[0] = fx * cp[0] * iz + cx - u;
    res[1] = fy * cp[1] * iz + cy - v;
    if (Ja) {
        const double iz2 = iz * iz;
        const double Jc[6] = {iz * fx, 0, -cp[0] * iz2 * fx, 0, iz * fy, -cp[1] * iz2 * fy};
        double JR[6];
        for (int r = 0; r < 2; r++)
            for (int c = 0; c < 3; c++)
                JR[3 * r + c] = Jc[3 * r] * Rwc[3 * c] + Jc[3 * r + 1] * Rwc[3 * c + 1] + Jc[3 * r + 2] * Rwc[3 * c + 2];
        const double Sk[9] = {0, -wpt[2], wpt[1], wpt[2], 0, -wpt[0], -wpt[1], wpt[0], 0};
        for (int r = 0; r < 2; r++)
            for (int c = 0; c < 3; c++) {
                const double js = JR[3 * r] * Sk[c] + JR[3 * r + 1] * Sk[3 + c] + JR[3 * r + 2] * Sk[6 + c];
                Ja[6 * r + c] = JR[3 * r + c];
                Ja[6 * r + 3 + c] = -js;
                Jp[6 * r + c] = -JR[3 * r + c];
                Jp[6 * r + 3 + c] = js;
            }
        for (int r = 0; r < 2; r++) Jd[r] = -zanch * (JR[3 * r] * Ra[0] + JR[3 * r + 1] * Ra[1] + JR[3 * r + 2] * Ra[2]);
    }
    return cp[2] > 0;
}

__device__ __forceinline__ void huber(double s, double delta, double& rho0, double& rho1) {
    if (delta > 0 && s > delta * delta) {
        const double r = sqrt(s);
        rho0 = 2 * delta * r - delta * delta;
        rho1 = fmax(DBL_MIN, delta / r);
    } else { rho0 = s; rho1 = 1.0; }
}

// 16-byte loads / stores of the workspace's per-observation records (res, Jd: 2 doubles; Ja: 12; wp: 6) and per-landmark F'e (wa: 6).
// Every workspace array starts 16-byte aligned (ba_prepare) and every record is an even number of doubles, so a record moves in
// N / 2 vector accesses instead of N scalar ones: half the memory instructions and L2 requests, the same values.  The BA kernels
// that read these records per observation or per Schur entry issue little else.
template <int N>
__device__ __forceinline__ void ld2(const double* p, double* v) {
#pragma unroll
    for (int i = 0; i < N / 2; i++) { const double2 t = reinterpret_cast<const double2*>(p)[i]; v[2 * i] = t.x; v[2 * i + 1] = t.y; }
}
template <int N>
__device__ __forceinline__ void st2(double* p, const double* v) {
#pragma unroll
    for (int i = 0; i < N / 2; i++) reinterpret_cast<double2*>(p)[i] = make_double2(v[2 * i], v[2 * i + 1]);
}

// deterministic block reduction (fixed tree), result valid in thread 0
template <int NT>
__device__ __forceinline__ double block_sum(double v, double* sm) {
    sm[threadIdx.x] = v;
    __syncthreads();
    for (int s = NT / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
        __syncthreads();
    }
    return sm[0];
}

// the same for any block size that is a multiple of 32 (<= 1024): butterfly inside each warp, then the warps in order.  Every
// thread of the block must call; the result is returned to all.  sm: >= 33 doubles.
__device__ __forceinline__ double block_sum_dyn(double v, double* sm) {
#pragma unroll
    for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    __syncthreads();   // earlier readers of sm are done
    if (lane == 0) sm[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < nw; w++) t += sm[w]; sm[32] = t; }
    __syncthreads();
    return sm[32];
}
__device__ __forceinline__ double block_max_dyn(double v, double* sm) {
#pragma unroll
    for (int off = 16; off; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (lane == 0) sm[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) { double t = sm[0]; for (int w = 1; w < nw; w++) t = fmax(t, sm[w]); sm[32] = t; }
    __syncthreads();
    return sm[32];
}

// ------------------------------------------------------------------------------------------ setup (1 CTA / problem)
// Structure of the problem, computed once per solve: free-pose columns, landmark -> observation CSR, and per free pose
// the list of (landmark, slot) pairs that see it (slot 0 = anchor keyframe, 1 + k = the landmark's k-th observation).
// The pose lists are an order-preserving multisplit (warp match + prefix), so every list -- and every floating-point
// sum taken over one later -- has a fixed order: the whole solve is bit-reproducible.
constexpr int SETUP_THREADS = 1024;
__global__ void __launch_bounds__(SETUP_THREADS) ba_setup_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.x];
    if (threadIdx.x < NBMAX) P.ga_ticket[threadIdx.x] = 0;   // arrival counters of the gather kernel's diagonal parts
    __shared__ int ref[256];
    __shared__ int scan_s[SETUP_THREADS + 1];
    __shared__ int wcount[32][NBMAX + 1];
    __shared__ int run[NBMAX + 1], pl_base[NBMAX + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NT = SETUP_THREADS;
    if (D.pass == 1 && (P.st->nbad == 0 || !(D.huber > 0))) {
        // second solve of localBA runs only if the first one lost residuals (optimizer.cpp:305): otherwise every kernel
        // of this pass is a no-op for this problem
        if (tid == 0) { P.st->done = 1; P.st->skipped = 1; P.st->use_gather = 0; P.st->has_last = 0; }
        return;
    }
    for (int k = tid; k < 256; k += NT) ref[k] = 0;
    for (int l = tid; l <= D.nlm; l += NT) P.lm_start[l] = 0;
    __syncthreads();
    // counts per landmark (exact integer atomics) and referenced poses
    for (int o = tid; o < D.nobs; o += NT) {
        const int l = P.obs_lm[o];
        if (l < 0) continue;
        atomicAdd(&P.lm_start[l + 1], 1);
        ref[P.anch_kf[l]] = 1;
        ref[P.obs_kf[o]] = 1;
    }
    __syncthreads();
    if (tid == 0) {
        int c = 0;
        for (int k = 0; k < D.nkf; k++) {
            if (!P.pose_const[k] && ref[k]) { P.pose_col[k] = c; c += 6; }
            else P.pose_col[k] = -1;
        }
        BaState& s = *P.st;
        s.ncols = c;
        s.radius = 1e4; s.decrease_factor = 2.0; s.reuse_diagonal = 0; s.invalid_steps = 0; s.iteration = 0;
        s.last_success = 1; s.n_success = 0; s.n_iter = 0; s.term = 1; s.done = 0; s.relin = 1; s.step_ok = 0;
        s.se_acc_ref = 0; s.se_acc_cand = 0; s.gmax = 1.0; s.model_change = 0; s.cand_cost = 0;
        s.chol_ok = 1; s.use_gather = 0; s.nb = c / 6; s.has_last = 0; s.skipped = 0;
        if (c > 6 * NBMAX) {
            // more free poses than the reduced-system buffers hold (NBMAX): refuse the problem -- every later kernel returns at
            // once for a finished problem and the parameters stay untouched -- instead of writing past S / rhs.  term 2 = failure.
            // ba_pre_body never runs, so the costs are set here: the summary reads 0, 0 rather than what the workspace last held.
            for (int k = 0; k < D.nkf; k++) P.pose_col[k] = -1;
            s.ncols = 0; s.nb = 0; s.done = 1; s.term = 2;
            s.initial_cost = 0; s.x_cost = 0;
        }
    }
    // exclusive scan of counts -> lm_start
    {
        const int chunk = (D.nlm + NT) / NT;
        const int b = tid * chunk + 1, e = min(b + chunk, D.nlm + 1);
        int sum = 0;
        for (int i = b; i < e; i++) sum += P.lm_start[i];
        scan_s[tid + 1] = sum;
        if (tid == 0) scan_s[0] = 0;
        __syncthreads();
        if (warp == 0) {   // inclusive scan of the NT partials, 32 per lane
            int v[NT / 32], t = 0;
            for (int i = 0; i < NT / 32; i++) { t += scan_s[1 + lane * (NT / 32) + i]; v[i] = t; }
            int incl = t;
            for (int off = 1; off < 32; off <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += u; }
            const int excl = incl - t;
            for (int i = 0; i < NT / 32; i++) scan_s[1 + lane * (NT / 32) + i] = excl + v[i];
        }
        __syncthreads();
        int r = scan_s[tid];
        for (int i = b; i < e; i++) { r += P.lm_start[i]; P.lm_start[i] = r; }
        __syncthreads();
    }
    // landmark -> observation lists.  Common case: obs_lm is non-decreasing (the reference emits observations grouped by
    // landmark), then the list is a contiguous index range found by binary search; otherwise a linear scan.
    for (int l = tid; l < D.nlm; l += NT) {
        const int b = P.lm_start[l], e = P.lm_start[l + 1];
        if (e == b) continue;
        int lo = 0, hi = D.nobs;
        while (lo < hi) { const int mid = (lo + hi) >> 1; const int v = P.obs_lm[mid]; if (v >= 0 && v < l) lo = mid + 1; else hi = mid; }
        bool grouped = (lo + (e - b) <= D.nobs);
        for (int i = 0; grouped && i < e - b; i++) grouped = (P.obs_lm[lo + i] == l);
        if (grouped) { for (int i = 0; i < e - b; i++) P.lm_obs[b + i] = lo + i; }
        else { int c = b; for (int o = 0; o < D.nobs && c < e; o++) if (P.obs_lm[o] == l) P.lm_obs[c++] = o; }
    }
    for (int l = tid; l < D.nlm; l += NT) P.anch_col[l] = P.pose_col[P.anch_kf[l]];
    for (int o = tid; o < D.nobs; o += NT) P.obs_col[o] = P.obs_lm[o] >= 0 ? P.pose_col[P.obs_kf[o]] : -1;
    for (int i = tid; i <= NBMAX; i += NT) { run[i] = 0; pl_base[i] = 0; }
    __syncthreads();
    // ---- per-pose (landmark, slot) lists: items = [anchor of every used landmark] ++ [CSR positions in order]
    const int nobs_used = P.lm_start[D.nlm];
    const int nitems = D.nlm + nobs_used;
    auto item = [&](int t, int& key, uint32_t& val) {
        key = -1; val = 0;
        if (t < D.nlm) {
            if (P.lm_start[t + 1] > P.lm_start[t] && P.anch_col[t] >= 0) { key = P.anch_col[t] / 6; val = (uint32_t)t << 8; }
        } else if (t < nitems) {
            const int i = t - D.nlm, o = P.lm_obs[i], l = P.obs_lm[o];
            if (P.obs_col[o] >= 0) { key = P.obs_col[o] / 6; val = ((uint32_t)l << 8) | (uint32_t)(i - P.lm_start[l] + 1); }
        }
    };
    int maxobs = 0;
    for (int l = tid; l < D.nlm; l += NT) maxobs = max(maxobs, P.lm_start[l + 1] - P.lm_start[l]);
    for (int t = tid; t < nitems; t += NT) {   // pass 0: totals per pose
        int key; uint32_t val;
        item(t, key, val);
        if (key >= 0) atomicAdd(&pl_base[key + 1], 1);
    }
    __syncthreads();
    if (tid == 0) {
        P.pstart[0] = 0;
        for (int k = 0; k < NBMAX; k++) { P.pstart[k + 1] = pl_base[k + 1]; pl_base[k + 1] += pl_base[k]; }   // pstart[k+1] = count
    }
    __syncthreads();
    for (int t0 = 0; t0 < nitems; t0 += NT) {   // pass 1: ordered fill
        for (int i = tid; i < 32 * (NBMAX + 1); i += NT) (&wcount[0][0])[i] = 0;
        __syncthreads();
        int key; uint32_t val;
        item(t0 + tid, key, val);
        const uint32_t m = __match_any_sync(0xffffffffu, key);
        const int rank = __popc(m & ((1u << lane) - 1));
        if (key >= 0 && rank == 0) wcount[warp][key] = __popc(m);
        __syncthreads();
        if (tid < NBMAX) {   // exclusive prefix over the warps, per key
            int acc = 0;
            for (int wv = 0; wv < 32; wv++) { const int c = wcount[wv][tid]; wcount[wv][tid] = acc; acc += c; }
            scan_s[tid] = acc;   // chunk total of this key
        }
        __syncthreads();
        if (key >= 0) P.plist[pl_base[key] + run[key] + wcount[warp][key] + rank] = val;
        __syncthreads();
        if (tid < NBMAX) run[tid] += scan_s[tid];
        __syncthreads();
    }
    // the gather path packs (landmark, slot_u, slot_v) into 32 bits
    maxobs = max(maxobs, __shfl_xor_sync(0xffffffffu, maxobs, 16)); maxobs = max(maxobs, __shfl_xor_sync(0xffffffffu, maxobs, 8));
    maxobs = max(maxobs, __shfl_xor_sync(0xffffffffu, maxobs, 4)); maxobs = max(maxobs, __shfl_xor_sync(0xffffffffu, maxobs, 2));
    maxobs = max(maxobs, __shfl_xor_sync(0xffffffffu, maxobs, 1));
    if (lane == 0) scan_s[warp] = maxobs;
    __syncthreads();
    if (tid == 0) {
        int mo = 0;
        for (int i = 0; i < NT / 32; i++) mo = max(mo, scan_s[i]);
        P.st->use_gather = (mo < 255 && D.nlm < 65536 && D.nobs < 65535) ? 1 : 0;
    }
}

// ------------------------------------------------------------------------------------------ linearise (thread / obs)
// FULL: residuals + Jacobians at the current point (column norms and gradient follow in ba_stats_kernel, without atomics);
// otherwise cost only at the candidate point.  Per-block cost partials (deterministic order in the control kernels).
// one observation: cost (FULL: + corrected residual and Jacobians stored) at `poses` / `invd_l`
template <bool FULL>
__device__ __forceinline__ double lin_obs(const BaProblem& P, const BaDims& D, int o, int l, const double* poses, double invd_l) {
    const int ka = P.anch_kf[l], kp = P.obs_kf[o];
    double r[2], Ja[12], Jp[12], Jd[2];
    ba_evaluate(P.calib, poses + 7 * ka, poses + 7 * kp, invd_l, P.obs_uv[2 * o], P.obs_uv[2 * o + 1], P.anch_uv[2 * l],
                P.anch_uv[2 * l + 1], r, FULL ? Ja : nullptr, Jp, Jd);
    double rho0, rho1;
    huber(r[0] * r[0] + r[1] * r[1], D.huber, rho0, rho1);
    if (FULL) {
        const double sc = sqrt(rho1);
        r[0] *= sc; r[1] *= sc;
        st2<2>(P.res + 2 * o, r);
        Jd[0] *= sc; Jd[1] *= sc;
        st2<2>(P.Jd + 2 * o, Jd);
#pragma unroll
        for (int i = 0; i < 12; i++) Ja[i] *= sc;
        st2<12>(P.Ja + 12 * o, Ja);   // Jp = -Ja: not stored
    }
    return 0.5 * rho0;
}

template <bool FULL>
__global__ void __launch_bounds__(LIN_THREADS, 7) ba_linearize_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.y];
    __shared__ double red[LIN_THREADS];
    const BaState& st = *P.st;
    const bool active = FULL ? (st.relin && !st.done) : !st.done;
    if (!active) return;   // uniform per CTA
    const int o = blockIdx.x * LIN_THREADS + threadIdx.x;
    double cost = 0;
    const int l = o < D.nobs ? P.obs_lm[o] : -1;
    if (l >= 0) cost = lin_obs<FULL>(P, D, o, l, FULL ? P.poses : P.cand_poses, (FULL ? P.invd : P.cand_invd)[l]);
    const double tot = block_sum<LIN_THREADS>(cost, red);
    if (threadIdx.x == 0) P.cost_part[blockIdx.x] = tot;
}

// squared column norm and gradient entry of one landmark's inverse-depth column
__device__ __forceinline__ void stats_landmark(const BaProblem& P, int l) {
    double ne = 0, ge = 0;
    for (int i = P.lm_start[l]; i < P.lm_start[l + 1]; i++) {
        const int o = P.lm_obs[i];
        double d[2], q[2];
        ld2<2>(P.Jd + 2 * o, d);
        ld2<2>(P.res + 2 * o, q);
        ne += d[0] * d[0] + d[1] * d[1];
        ge += d[0] * q[0] + d[1] * q[1];
    }
    P.ne[l] = ne;
    P.ge[l] = ge;
}
// thread gt of the BS_THREADS that share free pose b: its share (stride BS_THREADS over the pose's (landmark, slot) list) of the
// six squared column norms v[0..5] and gradient entries v[6..11]
__device__ __forceinline__ void stats_pose_partial(const BaProblem& P, int b, int gt, double* v) {
    int eb = 0;
    for (int i = 0; i < b; i++) eb += P.pstart[i + 1];
    const int ee = eb + P.pstart[b + 1];
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = 0;
    for (int idx = eb + gt; idx < ee; idx += BS_THREADS) {
        const uint32_t en = P.plist[idx];
        const int l = en >> 8, su = en & 0xff;
        const int ob = P.lm_start[l];
        if (su) {
            const int o = P.lm_obs[ob + su - 1];
            double q[2], J[12];
            ld2<2>(P.res + 2 * o, q);
            ld2<12>(P.Ja + 12 * o, J);
            const double r0 = q[0], r1 = q[1];
#pragma unroll
            for (int c = 0; c < 6; c++) {
                const double j0 = -J[c], j1 = -J[6 + c];
                v[c] += j0 * j0 + j1 * j1;
                v[6 + c] += j0 * r0 + j1 * r1;
            }
        } else {
            for (int i = ob; i < P.lm_start[l + 1]; i++) {
                const int o = P.lm_obs[i];
                double q[2], J[12];
                ld2<2>(P.res + 2 * o, q);
                ld2<12>(P.Ja + 12 * o, J);
                const double r0 = q[0], r1 = q[1];
#pragma unroll
                for (int c = 0; c < 6; c++) {
                    const double j0 = J[c], j1 = J[6 + c];
                    v[c] += j0 * j0 + j1 * j1;
                    v[6 + c] += j0 * r0 + j1 * r1;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ column norms and gradient
// Squared column norms of the (unscaled) Jacobian and the gradient J'r, in fixed summation order:
//   blocks [0, nbs)          : thread per landmark -> inverse-depth column (ne, ge)
//   blocks [nbs, nbs+NBMAX)  : 4 warps per free pose over its (landmark, slot) list -> 6 pose columns (nf, gf)
__global__ void __launch_bounds__(BS_THREADS) ba_stats_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.y];
    const BaState& st = *P.st;
    if (st.done || !st.relin) return;
    __shared__ double part[4][12];
    if ((int)blockIdx.x < D.nbs) {
        const int l = blockIdx.x * BS_THREADS + threadIdx.x;
        if (l >= D.nlm) return;
        stats_landmark(P, l);
        return;
    }
    const int b = blockIdx.x - D.nbs;
    if (b >= st.ncols / 6) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double v[12];
    stats_pose_partial(P, b, threadIdx.x, v);
#pragma unroll
    for (int i = 0; i < 12; i++) {
#pragma unroll
        for (int off = 16; off; off >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], off);
        if (lane == 0) part[warp][i] = v[i];
    }
    __syncthreads();
    if (threadIdx.x < 12) {
        const double t = part[0][threadIdx.x] + part[1][threadIdx.x] + part[2][threadIdx.x] + part[3][threadIdx.x];
        if (threadIdx.x < 6) P.nf[6 * b + threadIdx.x] = t;
        else P.gf[6 * b + threadIdx.x - 6] = t;
    }
}

// ------------------------------------------------------------------------------------------ gather-form Schur: block lists
// For block row bi: every (landmark, slot_u) of pose bi's list is paired with the landmark's slots holding pose bj >= bi
// (bj == bi: slot_v >= slot_u, each unordered pair once).  MODE 0 counts the entries of each block, MODE 1 fills them in
// list order (ballot-ordered appends).  One warp per block row.
template <int MODE>
__global__ void __launch_bounds__(32) ba_pairs_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.y];
    BaState& st = *P.st;
    const int nb = st.ncols / 6, bi = blockIdx.x, lane = threadIdx.x;
    if (!st.use_gather) return;
    __shared__ int cnt[NBMAX];    // running entry count of block (bi, bj)
    __shared__ int boff[NBMAX];   // MODE 1: start of block (bi, bj)
    if (bi >= nb) {
        if (MODE == 0) for (int bj = lane; bj < NBMAX; bj += 32) P.blk_start[bi * NBMAX + bj + 1] = 0;
        return;
    }
    int base_row = 0;   // MODE 1: entries of all preceding block rows
    if (MODE == 1) {
        int sum = 0;
        for (int i = lane; i < bi * NBMAX; i += 32) sum += P.blk_start[i + 1];
#pragma unroll
        for (int off = 16; off; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
        base_row = sum;
    }
    if (lane < NBMAX) cnt[lane] = 0;
    if (lane == 0) {
        int run = base_row;
        for (int bj = 0; bj < NBMAX; bj++) {
            boff[bj] = run;
            if (MODE == 1) { P.blk_off[bi * NBMAX + bj] = run; run += P.blk_start[bi * NBMAX + bj + 1]; }
        }
    }
    __syncwarp();
    int eb = 0;
    for (int i = 0; i < bi; i++) eb += P.pstart[i + 1];
    const int ee = eb + P.pstart[bi + 1];
    for (int c0 = eb; c0 < ee; c0 += 32) {
        const int idx = c0 + lane;
        const bool live = idx < ee;
        const uint32_t en = live ? P.plist[idx] : 0u;
        const int l = en >> 8, su = en & 0xff;
        const int ob = live ? P.lm_start[l] : 0, ns = live ? P.lm_start[l + 1] - ob : -1;
        // the reduced-system columns of the first four slots, fetched together (independent loads) before the serial rounds
        int cv0 = -1, cv1 = -1, cv2 = -1, cv3 = -1, o1 = -1, o2 = -1, o3 = -1, ou = 0xffff;
        if (live) {
            cv0 = P.anch_col[l];
            o1 = ns >= 1 ? P.lm_obs[ob] : -1; o2 = ns >= 2 ? P.lm_obs[ob + 1] : -1; o3 = ns >= 3 ? P.lm_obs[ob + 2] : -1;
            if (o1 >= 0) cv1 = P.obs_col[o1];
            if (o2 >= 0) cv2 = P.obs_col[o2];
            if (o3 >= 0) cv3 = P.obs_col[o3];
            if (MODE == 1 && su) ou = su == 1 ? o1 : su == 2 ? o2 : su == 3 ? o3 : P.lm_obs[ob + su - 1];
        }
        for (int sv = 0; sv <= 255; sv++) {                 // slot-major rounds (ns is small: 3 in the reference's problems)
            if (!__any_sync(0xffffffffu, live && sv <= ns)) break;
            int bjv = -1, bjv_ov = 0xffff;
            if (live && sv <= ns) {
                const int ov = sv == 0 ? 0xffff : sv == 1 ? o1 : sv == 2 ? o2 : sv == 3 ? o3 : P.lm_obs[ob + sv - 1];
                bjv_ov = ov;
                const int cv = sv == 0 ? cv0 : sv == 1 ? cv1 : sv == 2 ? cv2 : sv == 3 ? cv3 : P.obs_col[ov];
                if (cv >= 0) { const int bj = cv / 6; if (bj > bi || (bj == bi && sv >= su)) bjv = bj; }
                // a landmark seen twice from one keyframe (two slots on the same pose) needs the transposed contribution
                // as well; localBA never builds that, so such problems simply take the atomic Schur path instead
                if (MODE == 0 && cv >= 0 && cv / 6 == bi && sv > su) st.use_gather = 0;
            }
            // lanes that hit the same block append in lane order: one match instead of one ballot per block
            const uint32_t m = __match_any_sync(0xffffffffu, bjv);
            if (bjv >= 0) {
                const int rank = __popc(m & ((1u << lane) - 1));
                const int old = cnt[bjv];
                if (MODE == 1) {
                    const int pos = boff[bjv] + old + rank;
                    if (pos < D.ecap)
                        P.pairs[pos] = ((uint64_t)l << 48) | ((uint64_t)su << 40) | ((uint64_t)sv << 32) | ((uint64_t)(ou & 0xffff) << 16) |
                                       (uint64_t)(bjv_ov & 0xffff);
                }
                __syncwarp(m);
                if (rank == 0) cnt[bjv] = old + __popc(m);
            }
            __syncwarp();
        }
    }
    if (MODE == 0) {
        if (lane < NBMAX) P.blk_start[bi * NBMAX + lane + 1] = cnt[lane];
    } else if (bi == nb - 1 && lane == 0) {
        int total = base_row;
        for (int bj = 0; bj < NBMAX; bj++) total += cnt[bj];
        if (total > D.ecap) st.use_gather = 0;   // structure too large for the entry buffer: the atomic path takes over
    }
}

// ------------------------------------------------------------------------------------------ control: before the step
// TrustRegionMinimizer::{IterationZero, FinalizeIterationAndCheckIfMinimizerCanContinue} + LM ComputeStep's diagonal.
constexpr int CT_THREADS = 1024;   // control kernels: one CTA per problem; their loops over landmarks are chains of L2 round trips, so be wide
// (one CTA of any size that is a multiple of 32; every thread calls)
__device__ void ba_pre_body(const BaProblem& P, const BaDims& D) {
    BaState& st = *P.st;
    __shared__ double red[34];
    __shared__ int go;
    const int tid = threadIdx.x, NT = blockDim.x;
    const int n = st.ncols;
    if (st.done) return;
    if (st.relin) {
        // cost at the (new) current point, in a fixed summation order
        double c = 0;
        for (int i = tid; i < D.nblk; i += NT) c += P.cost_part[i];
        const double x_cost = block_sum_dyn(c, red);
        // |x|
        double xn = 0;
        for (int k = tid; k < D.nkf; k += NT)
            if (P.pose_col[k] >= 0) for (int i = 0; i < 7; i++) xn += P.poses[7 * k + i] * P.poses[7 * k + i];
        for (int l = tid; l < D.nlm; l += NT)
            if (P.lm_start[l + 1] > P.lm_start[l]) xn += P.invd[l] * P.invd[l];
        xn = block_sum_dyn(xn, red);
        // gradient max-norm |x - Plus(x, -g)|_inf
        double gm = 0;
        for (int k = tid; k < D.nkf; k += NT) {
            const int c0 = P.pose_col[k];
            if (c0 < 0) continue;
            double dlt[6], out[7];
            for (int i = 0; i < 6; i++) dlt[i] = -P.gf[c0 + i];
            se3_plus(P.poses + 7 * k, dlt, out);
            for (int i = 0; i < 7; i++) gm = fmax(gm, fabs(P.poses[7 * k + i] - out[i]));
        }
        for (int l = tid; l < D.nlm; l += NT)
            if (P.lm_start[l + 1] > P.lm_start[l]) gm = fmax(gm, fabs(P.ge[l]));
        gm = block_max_dyn(gm, red);
        if (st.iteration == 0) {   // Jacobi scaling is fixed at iteration 0 (trust_region_minimizer.cc:266-275)
            for (int i = tid; i < n; i += NT) P.scf[i] = 1.0 / (1.0 + sqrt(P.nf[i]));
            for (int l = tid; l < D.nlm; l += NT) P.sce[l] = 1.0 / (1.0 + sqrt(P.ne[l]));
        }
        __syncthreads();
        if (tid == 0) {
            st.x_cost = x_cost; st.xnorm = sqrt(xn); st.gmax = gm; st.push_cost = x_cost;
            if (st.iteration == 0) {
                st.initial_cost = x_cost;
                st.se_min = st.se_cur = st.se_ref = st.se_cand = x_cost;
            }
            st.relin = 0;
        }
    }
    __syncthreads();
    if (tid == 0) {
        // FinalizeIterationAndCheckIfMinimizerCanContinue
        if (st.last_success) st.n_success++;
        st.n_iter++;
        int cont = 1;
        if (st.iteration >= D.max_iter) { st.term = 1; cont = 0; }
        else if (st.last_success && st.gmax <= 1e-10) { st.term = 0; cont = 0; }
        else if (st.radius <= 1e-32) { st.term = 0; cont = 0; }
        if (!cont) st.done = 1;
        else { st.iteration++; st.last_success = 0; }
        go = cont;
    }
    __syncthreads();
    if (!go) return;
    // LM diagonal (levenberg_marquardt_strategy.cc:76-88)
    const bool reuse = st.reuse_diagonal;
    const double radius = st.radius;
    __syncthreads();   // everyone has read the state before thread 0 updates it below
    for (int i = tid; i < n; i += NT) {
        if (!reuse) P.diagf[i] = fmin(fmax(P.nf[i] * P.scf[i] * P.scf[i], 1e-6), 1e32);
        P.Df[i] = sqrt(P.diagf[i] / radius);
    }
    for (int l = tid; l < D.nlm; l += NT) {
        if (!reuse) P.diage[l] = fmin(fmax(P.ne[l] * P.sce[l] * P.sce[l], 1e-6), 1e32);
        P.De[l] = sqrt(P.diage[l] / radius);
    }
    for (int i = tid; i < NMAX * NMAX; i += NT) P.S[i] = 0;
    for (int i = tid; i < NMAX; i += NT) P.rhs[i] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += NT) P.S[i * NMAX + i] = P.Df[i] * P.Df[i];
    if (tid == 0) st.reuse_diagonal = 1;
}

__global__ void __launch_bounds__(CT_THREADS) ba_pre_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.x];
    ba_pre_body(P, D);
}

// ------------------------------------------------------------------------------------------ Schur (thread / landmark)
// S += F'F - (E'F)'(E'E + D^2)^-1 (E'F),  rhs += F'b - (E'F)'(E'E + D^2)^-1 E'b  for this landmark's rows
// DENSE = true: the -(E'F)'(E'E)^-1(E'F) term is NOT accumulated here; instead the landmark's row of
// Wt = diag(E'E + D^2)^-1/2 (E'F)  (nlm x 128, zero outside the landmark's pose blocks) is written for the FP64
// tensor-core SYRK below (S -= Wt' Wt), which is where that term is a genuine dense contraction.
template <bool DENSE>
__device__ void schur_landmark(const BaProblem& P, const BaDims& D, int l) {
    if (DENSE) {   // rows are rewritten every iteration; padding rows and unused landmarks stay zero
        double* row = P.Wt + (size_t)l * NMAX;
        for (int i = 0; i < NMAX; i++) row[i] = 0.0;
    }
    if (l >= D.nlm) return;
    const int b = P.lm_start[l], e = P.lm_start[l + 1];
    if (e == b) return;
    const int ca = P.pose_col[P.anch_kf[l]];
    const double sce = P.sce[l];
    double ete = P.De[l] * P.De[l], etb = 0, wa[6] = {0, 0, 0, 0, 0, 0};
    double sca[6];
    for (int c = 0; c < 6; c++) sca[c] = ca >= 0 ? P.scf[ca + c] : 0.0;
    double Saa[36];
    for (int i = 0; i < 36; i++) Saa[i] = 0;
    double rha[6] = {0, 0, 0, 0, 0, 0};
    for (int i = b; i < e; i++) {
        const int o = P.lm_obs[i];
        const int cp = P.pose_col[P.obs_kf[o]];
        const double e0 = P.Jd[2 * o] * sce, e1 = P.Jd[2 * o + 1] * sce;
        const double r0 = P.res[2 * o], r1 = P.res[2 * o + 1];
        ete += e0 * e0 + e1 * e1;
        etb += e0 * r0 + e1 * r1;
        double Fa[12], Fp[12];
        for (int c = 0; c < 6; c++) {
            Fa[c] = P.Ja[12 * o + c] * sca[c]; Fa[6 + c] = P.Ja[12 * o + 6 + c] * sca[c];
            const double s = cp >= 0 ? P.scf[cp + c] : 0.0;
            Fp[c] = -P.Ja[12 * o + c] * s; Fp[6 + c] = -P.Ja[12 * o + 6 + c] * s;
        }
        for (int c = 0; c < 6; c++) {
            wa[c] += e0 * Fa[c] + e1 * Fa[6 + c];
            P.wp[6 * o + c] = e0 * Fp[c] + e1 * Fp[6 + c];
            rha[c] += Fa[c] * r0 + Fa[6 + c] * r1;
        }
        if (ca >= 0)
            for (int a = 0; a < 6; a++)
                for (int c = 0; c < 6; c++) Saa[6 * a + c] += Fa[a] * Fa[c] + Fa[6 + a] * Fa[6 + c];
        if (cp >= 0) {
            for (int a = 0; a < 6; a++) {
                atomicAdd(&P.rhs[cp + a], Fp[a] * r0 + Fp[6 + a] * r1);
                for (int c = 0; c < 6; c++) {
                    atomicAdd(&P.S[(cp + a) * NMAX + cp + c], Fp[a] * Fp[c] + Fp[6 + a] * Fp[6 + c]);
                    if (ca >= 0) {
                        const double x = Fa[a] * Fp[c] + Fa[6 + a] * Fp[6 + c];   // (anchor row a, observer col c)
                        atomicAdd(&P.S[(ca + a) * NMAX + cp + c], x);
                        atomicAdd(&P.S[(cp + c) * NMAX + ca + a], x);
                    }
                }
            }
        }
    }
    const double inv = 1.0 / ete;
    P.ete[l] = ete;
    P.etb[l] = etb;
    for (int c = 0; c < 6; c++) P.wa[6 * l + c] = wa[c];
    if (ca >= 0)
        for (int a = 0; a < 6; a++) {
            atomicAdd(&P.rhs[ca + a], rha[a] - wa[a] * inv * etb);
            for (int c = 0; c < 6; c++)
                atomicAdd(&P.S[(ca + a) * NMAX + ca + c], DENSE ? Saa[6 * a + c] : Saa[6 * a + c] - wa[a] * inv * wa[c]);
        }
    if (DENSE) {
        const double rs = sqrt(inv);
        double* row = P.Wt + (size_t)l * NMAX;
        if (ca >= 0) for (int c = 0; c < 6; c++) row[ca + c] += wa[c] * rs;
        for (int i = b; i < e; i++) {
            const int oi = P.lm_obs[i];
            const int ci = P.pose_col[P.obs_kf[oi]];
            if (ci < 0) continue;
            for (int c = 0; c < 6; c++) {
                row[ci + c] += P.wp[6 * oi + c] * rs;
                atomicAdd(&P.rhs[ci + c], -P.wp[6 * oi + c] * inv * etb);
            }
        }
        return;
    }
    // - w w' / ete over (observer, observer) and (anchor, observer) pairs
    for (int i = b; i < e; i++) {
        const int oi = P.lm_obs[i];
        const int ci = P.pose_col[P.obs_kf[oi]];
        if (ci < 0) continue;
        double wi[6];
        for (int c = 0; c < 6; c++) wi[c] = P.wp[6 * oi + c];
        for (int a = 0; a < 6; a++) atomicAdd(&P.rhs[ci + a], -wi[a] * inv * etb);
        if (ca >= 0)
            for (int a = 0; a < 6; a++)
                for (int c = 0; c < 6; c++) {
                    const double x = -wa[a] * inv * wi[c];
                    atomicAdd(&P.S[(ca + a) * NMAX + ci + c], x);
                    atomicAdd(&P.S[(ci + c) * NMAX + ca + a], x);
                }
        for (int j = b; j < e; j++) {
            const int oj = P.lm_obs[j];
            const int cj = P.pose_col[P.obs_kf[oj]];
            if (cj < 0) continue;
            for (int a = 0; a < 6; a++)
                for (int c = 0; c < 6; c++) atomicAdd(&P.S[(ci + a) * NMAX + cj + c], -wi[a] * inv * P.wp[6 * oj + c]);
        }
    }
}

template <bool DENSE>
__global__ void __launch_bounds__(128) ba_schur_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.y];
    if (P.st->done) return;
    if (!DENSE && P.st->use_gather) return;   // the gather path already assembled S
    const int l = blockIdx.x * 128 + threadIdx.x;
    if (l >= D.nlm_pad) return;
    schur_landmark<DENSE>(P, D, l);
}

// ------------------------------------------------------------------------------------------ dense Schur term on tensor cores
// S -= Wt' * Wt  with Wt [K = nlm_pad][128] row-major, FP64 tensor-core MMA (mma.sync.m8n8k4.f64 -> SASS DMMA; wgmma has
// no FP64 kind).  Grid: (16 output blocks of 32x32) x (K splits) x problems; 4 warps per CTA interleave the K steps, the
// four partial 32x32 blocks are summed in shared memory and added to S with one FP64 atomic per element.
__device__ __forceinline__ void dmma_m8n8k4(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

constexpr int SYRK_KSPLIT = 8;

__global__ void __launch_bounds__(128) ba_syrk_dmma_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.z];
    if (P.st->done) return;
    __shared__ double part[4][32][33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int bi = blockIdx.x >> 2, bj = blockIdx.x & 3;          // 4 x 4 blocks of 32 x 32
    const int i0 = bi * 32, j0 = bj * 32;
    const int n = P.st->ncols;
    if (i0 >= n || j0 >= n) return;                                // block entirely in the padding
    const int ksteps = D.nlm_pad / 4;
    const int per = (ksteps + SYRK_KSPLIT - 1) / SYRK_KSPLIT;
    const int kb = blockIdx.y * per, ke = min(ksteps, kb + per);
    double acc[4][4][2];
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b][0] = acc[a][b][1] = 0.0;
    const int kr = lane & 3, cc = lane >> 2;
    for (int ks = kb + warp; ks < ke; ks += 4) {
        const double* row = P.Wt + (size_t)(4 * ks + kr) * NMAX;
        double av[4], bv[4];
#pragma unroll
        for (int t = 0; t < 4; t++) { av[t] = __ldg(row + i0 + 8 * t + cc); bv[t] = __ldg(row + j0 + 8 * t + cc); }
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
            for (int b = 0; b < 4; b++) dmma_m8n8k4(acc[a][b][0], acc[a][b][1], av[a], bv[b]);
    }
    // C fragment: row = lane / 4, cols = 2 * (lane % 4) + {0, 1}
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) {
            part[warp][8 * a + cc][8 * b + 2 * kr] = acc[a][b][0];
            part[warp][8 * a + cc][8 * b + 2 * kr + 1] = acc[a][b][1];
        }
    __syncthreads();
    for (int t = threadIdx.x; t < 32 * 32; t += 128) {
        const int r = t >> 5, c = t & 31;
        const double v = part[0][r][c] + part[1][r][c] + part[2][r][c] + part[3][r][c];
        if (v != 0.0) atomicAdd(&P.S[(i0 + r) * NMAX + j0 + c], -v);
    }
}


// ------------------------------------------------------------------------------------------ gather-form Schur (no atomics)
// The reduced camera system is assembled block by block: S[bi][bj] = sum over the landmarks that see both poses of
//   F_u'F_v - w_u w_v' / (E'E + D^2)        (u, v = the landmark's slots holding poses bi, bj; w = F'e)
// A slot is 0 for the anchor keyframe and 1 + k for the landmark's k-th observation.  The (block -> landmark pairs)
// lists depend only on the problem's structure, so they are built once per solve (deterministically, in landmark
// order) by ba_plist_kernel; every LM iteration then runs ba_lm_kernel (per-landmark E'E, E'b, F'e) and ba_gather_kernel
// (one warp per block, fixed summation order -> bit-reproducible results, zero atomics).
// per-landmark Schur ingredients: E'E + D^2, E'b, F'e for the anchor slot (wa) and every observation slot (wp)
__device__ __forceinline__ void lm_landmark(const BaProblem& P, int l) {
    const int b = P.lm_start[l], e = P.lm_start[l + 1];
    if (e == b) return;
    const int ca = P.pose_col[P.anch_kf[l]];
    const double sce = P.sce[l];
    double ete = P.De[l] * P.De[l], etb = 0, wa[6] = {0, 0, 0, 0, 0, 0};
    for (int i = b; i < e; i++) {
        const int o = P.lm_obs[i];
        const int cp = P.pose_col[P.obs_kf[o]];
        double d[2], q[2], J[12], w[6];
        ld2<2>(P.Jd + 2 * o, d);
        ld2<2>(P.res + 2 * o, q);
        ld2<12>(P.Ja + 12 * o, J);
        const double e0 = d[0] * sce, e1 = d[1] * sce;
        ete += e0 * e0 + e1 * e1;
        etb += e0 * q[0] + e1 * q[1];
#pragma unroll
        for (int c = 0; c < 6; c++) {
            if (ca >= 0) wa[c] += (e0 * J[c] + e1 * J[6 + c]) * P.scf[ca + c];
            w[c] = cp >= 0 ? (e0 * -J[c] + e1 * -J[6 + c]) * P.scf[cp + c] : 0.0;
        }
        st2<6>(P.wp + 6 * o, w);
    }
    P.ete[l] = ete;
    P.etb[l] = etb;
    st2<6>(P.wa + 6 * l, wa);
}
// ... or, for a problem whose structure the packed lists cannot express (use_gather == 0), the whole per-landmark Schur update with
// FP64 atomics (one launch serves both paths: a problem takes exactly one of them)
__global__ void __launch_bounds__(128) ba_lm_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.y];
    if (P.st->done) return;
    const int l = blockIdx.x * 128 + threadIdx.x;
    if (P.st->use_gather) { if (l < D.nlm) lm_landmark(P, l); }
    else if (l < D.nlm) schur_landmark<false>(P, D, l);
}

// Contribution of one (landmark, slot_u, slot_v) entry to block (bi, bj):  C = F_u'F_v - w_u w_v' / (E'E + D^2)  and, for
// u == v, the right-hand side F_u'b - w_u E'b / (E'E + D^2).  TRANSPOSE adds C' instead (second half of a duplicate-pose pair).
template <bool TRANSPOSE>   // TRANSPOSE is kept for completeness; the kernel only instantiates <false>
__device__ __forceinline__ void gather_entry(const BaProblem& P, uint64_t en, const double* sci, const double* scj, double* acc,
                                             double* rh) {
    // the entry carries the observation indices of its two slots: the loads below depend on it alone (the first version looked them
    // up through lm_start -> lm_obs: two more round trips in a kernel that is nothing but dependent round trips)
    const int l = (int)(en >> 48), su = (int)(en >> 40) & 0xff, sv = (int)(en >> 32) & 0xff;
    const double inv = 1.0 / P.ete[l], etb = P.etb[l];
    const int ou = su ? (int)(en >> 16) & 0xffff : -1, ov = sv ? (int)en & 0xffff : -1;
    double wu[6], wv[6];
    ld2<6>(su ? P.wp + 6 * ou : P.wa + 6 * l, wu);
    ld2<6>(sv ? P.wp + 6 * ov : P.wa + 6 * l, wv);
#pragma unroll
    for (int c = 0; c < 6; c++) wu[c] *= inv;
#define ACC(a, c) acc[TRANSPOSE ? 6 * (c) + (a) : 6 * (a) + (c)]
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int c = 0; c < 6; c++) ACC(a, c) -= wu[a] * wv[c];
    // F_u' F_v: non-zero only when both slots share a residual row pair
    if (su == 0 && sv == 0) {                        // anchor x anchor: every observation of the landmark
        const int ob = P.lm_start[l], oe = P.lm_start[l + 1];
        for (int i = ob; i < oe; i++) {
            const int o = P.lm_obs[i];
            double F0[6], F1[6], J[12], q[2];
            ld2<12>(P.Ja + 12 * o, J);
            ld2<2>(P.res + 2 * o, q);
#pragma unroll
            for (int c = 0; c < 6; c++) { F0[c] = J[c] * sci[c]; F1[c] = J[6 + c] * sci[c]; }
            const double r0 = q[0], r1 = q[1];
#pragma unroll
            for (int a = 0; a < 6; a++) {
                if (!TRANSPOSE) rh[a] += F0[a] * r0 + F1[a] * r1;
#pragma unroll
                for (int c = 0; c < 6; c++) ACC(a, c) += F0[a] * F0[c] + F1[a] * F1[c];
            }
        }
        if (!TRANSPOSE)
#pragma unroll
            for (int a = 0; a < 6; a++) rh[a] -= wu[a] * etb;
    } else if (su == sv) {                           // observation x itself
        double F0[6], F1[6], J[12], q[2];
        ld2<12>(P.Ja + 12 * ou, J);
        ld2<2>(P.res + 2 * ou, q);
#pragma unroll
        for (int c = 0; c < 6; c++) { F0[c] = -J[c] * sci[c]; F1[c] = -J[6 + c] * sci[c]; }
        const double r0 = q[0], r1 = q[1];
#pragma unroll
        for (int a = 0; a < 6; a++) {
            if (!TRANSPOSE) rh[a] += F0[a] * r0 + F1[a] * r1 - wu[a] * etb;
#pragma unroll
            for (int c = 0; c < 6; c++) ACC(a, c) += F0[a] * F0[c] + F1[a] * F1[c];
        }
    } else if (su == 0 || sv == 0) {                 // anchor x observation (either order): rows of that observation
        const int o = su ? ou : ov;
        double A0[6], A1[6], J[12];
        ld2<12>(P.Ja + 12 * o, J);
#pragma unroll
        for (int a = 0; a < 6; a++) {
            A0[a] = (su ? -J[a] : J[a]) * sci[a];
            A1[a] = (su ? -J[6 + a] : J[6 + a]) * sci[a];
        }
#pragma unroll
        for (int c = 0; c < 6; c++) {
            const double b0 = (sv ? -J[c] : J[c]) * scj[c];
            const double b1 = (sv ? -J[6 + c] : J[6 + c]) * scj[c];
#pragma unroll
            for (int a = 0; a < 6; a++) ACC(a, c) += A0[a] * b0 + A1[a] * b1;
        }
    }
#undef ACC
}

// One CTA (2 warps) per upper-triangular 6x6 block (bi < bj) and GA_SPLIT CTAs per DIAGONAL block, whose lists are the long
// ones (every landmark the pose sees, ~600 entries against ~100): a part strides over the block's entry list, each thread
// keeps a private 6x6 (+ rhs) accumulator, then a fixed-order shuffle + shared-memory reduction.  Diagonal parts leave their
// partial sums in a scratch slot; the part that arrives last (ticket) adds the GA_SPLIT slots in slot order.  The block and its
// mirror are stored -- no floating-point atomics, bit-reproducible.
constexpr int GA_THREADS = 64, GA_SPLIT = 8;   // 2 warps per part x 8 parts (the combine loop is valid for any CTA size)
constexpr int GA_GRID = NBMAX * GA_SPLIT + (MAXKEYS - NBMAX);   // diagonal parts first, then the strictly upper blocks
__global__ void __launch_bounds__(GA_THREADS, 8) ba_gather_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.y];
    const BaState& st = *P.st;
    if (st.done || !st.use_gather) return;
    int bi, bj, part = 0, nparts = 1;
    if ((int)blockIdx.x < NBMAX * GA_SPLIT) { bi = bj = blockIdx.x / GA_SPLIT; part = blockIdx.x % GA_SPLIT; nparts = GA_SPLIT; }
    else {
        int rem = blockIdx.x - NBMAX * GA_SPLIT;     // enumerates (bi, bj > bi) over NBMAX
        bi = 0;
        while (bi < NBMAX - 1 && rem >= NBMAX - 1 - bi) { rem -= NBMAX - 1 - bi; bi++; }
        bj = bi + 1 + rem;
    }
    if (bi >= st.nb || bj >= st.nb) return;
    const int blk = bi * NBMAX + bj;
    __shared__ double red[GA_THREADS / 32][42];
    __shared__ int last_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ci = 6 * bi, cj = 6 * bj;
    const int eb = P.blk_off[blk], ee = eb + P.blk_start[blk + 1];
    double acc[36], rh[6];
#pragma unroll
    for (int i = 0; i < 36; i++) acc[i] = 0.0;
#pragma unroll
    for (int i = 0; i < 6; i++) rh[i] = 0.0;
    double sci[6], scj[6];
#pragma unroll
    for (int c = 0; c < 6; c++) { sci[c] = P.scf[ci + c]; scj[c] = P.scf[cj + c]; }
    for (int idx = eb + part * GA_THREADS + tid; idx < ee; idx += nparts * GA_THREADS) {
        const uint64_t en = P.pairs[idx];
        gather_entry<false>(P, en, sci, scj, acc, rh);   // (duplicate-pose pairs never reach this kernel: see ba_pairs_kernel)
    }
    // fixed-order reduction: butterfly inside each warp, then the warps in order
#pragma unroll
    for (int i = 0; i < 36; i++) {
#pragma unroll
        for (int off = 16; off; off >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
        if (lane == 0) red[warp][i] = acc[i];
    }
#pragma unroll
    for (int i = 0; i < 6; i++) {
#pragma unroll
        for (int off = 16; off; off >>= 1) rh[i] += __shfl_xor_sync(0xffffffffu, rh[i], off);
        if (lane == 0) red[warp][36 + i] = rh[i];
    }
    __syncthreads();
    // the 36 + 6 entries of the block are finished by threads x = tid, tid + GA_THREADS, ... (any CTA size)
    if (nparts > 1) {
        double* slot = P.ga_part + ((size_t)bi * GA_SPLIT + part) * 42;
        for (int x = tid; x < 42; x += GA_THREADS) {
            double v = 0;
#pragma unroll
            for (int wv = 0; wv < GA_THREADS / 32; wv++) v += red[wv][x];
            slot[x] = v;
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) last_s = atomicInc(reinterpret_cast<unsigned int*>(P.ga_ticket + bi), GA_SPLIT - 1) == GA_SPLIT - 1;   // wraps to 0
        __syncthreads();
        if (!last_s) return;
        __threadfence();
    }
    for (int x = tid; x < 42; x += GA_THREADS) {
        double v = 0;
        if (nparts > 1) {
            const volatile double* all = P.ga_part + (size_t)bi * GA_SPLIT * 42;
#pragma unroll
            for (int q = 0; q < GA_SPLIT; q++) v += all[q * 42 + x];
        } else {
#pragma unroll
            for (int wv = 0; wv < GA_THREADS / 32; wv++) v += red[wv][x];
        }
        if (x < 36) {
            const int a = x / 6, c = x % 6;
            if (bi == bj) P.S[(ci + a) * NMAX + ci + c] = v + (a == c ? P.Df[ci + a] * P.Df[ci + a] : 0.0);
            else { P.S[(ci + a) * NMAX + cj + c] = v; P.S[(cj + c) * NMAX + ci + a] = v; }
        } else if (bi == bj) P.rhs[ci + x - 36] = v;
    }
}

// ------------------------------------------------------------------------------------------ reduced solve (1 CTA / problem)
// Right-looking LDL' of the <= 126 x 126 reduced camera system, REGISTER-TILED: the lower triangle of the (augmented) 128 x 128
// matrix is cut into 4 x 4 tiles, one per thread (528 tiles, column-block-major, so whole warps retire as the elimination moves
// right); V = L D is built in place.  Per panel of 4 columns (one tile column), TWO barriers: the diagonal tile eliminates its
// 4 x 4 block in registers and publishes it with the 4 pivot reciprocals; the tiles below it finish their 4 columns locally and
// publish them; then every trailing tile takes the 4 rank-1 updates  a[i][c] -= V[i][j] (V[c][j] / d_j)  in column order, from
// 8 shared-memory words each -- 16 FP64 FMAs against 8 loads, where a left-looking form spends three loads per multiply-add and
// is shared-memory-bandwidth bound.  Each element gets the same products subtracted in the same order as with one barrier
// per column, so the result is the same bits.  Row n of the matrix is the right-hand side, so the
// forward substitution z = L^-1 b falls out of the same updates.  Then x = L^-T D^-1 z by warp 0 (lane-strided, registers).
// No square roots; fixed operation order (bit-reproducible).  yf = S^-1 rhs.
constexpr int CH_TILES = 32 * 33 / 2, CH_THREADS = (CH_TILES + 31) / 32 * 32;   // 528 tiles -> 544 threads
// (a CTA of exactly CH_THREADS threads; sm: (NMAX * (NMAX + 1) + NMAX) doubles of shared memory)
__device__ void ba_chol_body(const BaProblem& P, double* sm) {
    BaState& st = *P.st;
    const int n = st.ncols, tid = threadIdx.x, lane = tid & 31;
    const int ld = NMAX + 1;
    double* V = sm;                 // (n + 1) x ld, filled after the factorisation for the backward solve
    double* invd = sm + NMAX * ld;  // NMAX
    __shared__ double pcol[4][NMAX];   // the panel's columns, rows below its diagonal tile
    __shared__ double dg[4][4];        // the panel's diagonal tile, eliminated
    __shared__ double pivinv[2][4];    // the panel's pivot reciprocals, by panel parity
    __shared__ int ok_s;
    // tile of this thread: column block tj, row block ti >= tj
    int tj = 0, rem = tid;
    while (tj < 32 && rem >= 32 - tj) { rem -= 32 - tj; tj++; }
    const int ti = tj + rem;
    const bool tile = tid < CH_TILES;
    const int r0 = 4 * ti, c0 = 4 * tj;
    double a[4][4];
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const int gr = r0 + r, gc = c0 + c;
            double v = 0.0;
            if (tile && gc < n) {
                if (gr < n) v = P.S[gr * NMAX + gc];
                else if (gr == n) v = P.rhs[gc];
            }
            a[r][c] = v;
        }
    if (tid == 0) ok_s = 1;
    const int last_jb = (n - 1) >> 2;
    // One panel (tile column jb, its 4 columns j = 4 jb + jj) per pass, two barriers.  Column-block-major tile order: a warp's
    // lanes retire (tj < jb) almost together, and a retired warp only keeps arriving at the barriers.
    for (int jb = 0; jb <= last_jb; jb++) {
        const int nj = min(4, n - 4 * jb);   // columns of this panel (uniform)
        double* pinv = pivinv[jb & 1];       // the next panel's diagonal tile writes the other half while trailing tiles read this one
        // 1. the diagonal tile eliminates its 4 x 4 block in registers and publishes it with the pivot reciprocals
        if (tile && ti == jb && tj == jb) {
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
                if (jj >= nj) break;
                const double d = a[jj][jj];
                if (!(d > 0)) ok_s = 0;
                // 1 / d sits on the serial chain of the elimination (pivot j + 1 needs it): MUFU.RCP64H seed (>= 20 bits) + two
                // Newton steps = 5 dependent operations instead of the IEEE division's subroutine; error <= 1 ulp, fixed sequence
                const double dd = d > 0 ? d : 1.0;
                double inv;
                asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(inv) : "d"(dd));
                inv = fma(inv, fma(-dd, inv, 1.0), inv);
                inv = fma(inv, fma(-dd, inv, 1.0), inv);
                pinv[jj] = inv;
                invd[4 * jb + jj] = inv;
                double lc[4];
#pragma unroll
                for (int c = 0; c < 4; c++) lc[c] = a[c][jj] * inv;
#pragma unroll
                for (int r = 0; r < 4; r++)
#pragma unroll
                    for (int c = jj + 1; c < 4; c++) a[r][c] -= a[r][jj] * lc[c];
            }
#pragma unroll
            for (int r = 0; r < 4; r++)
#pragma unroll
                for (int c = 0; c < 4; c++) dg[r][c] = a[r][c];
        }
        __syncthreads();
        // 2. the panel's tiles below it apply the in-panel updates and publish their 4 finished columns
        if (tile && tj == jb && ti > jb) {
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
                if (jj >= nj) break;
                double lc[4];
#pragma unroll
                for (int c = 0; c < 4; c++) lc[c] = dg[c][jj] * pinv[jj];
#pragma unroll
                for (int r = 0; r < 4; r++)
#pragma unroll
                    for (int c = jj + 1; c < 4; c++) a[r][c] -= a[r][jj] * lc[c];
            }
#pragma unroll
            for (int jj = 0; jj < 4; jj++)
#pragma unroll
                for (int r = 0; r < 4; r++) pcol[jj][r0 + r] = a[r][jj];
        }
        __syncthreads();
        // 3. the trailing tiles take the panel's rank-1 updates  a[i][c] -= V[i][j] (V[c][j] / d_j)  in column order -- every
        // element sees the same products subtracted in the same order as a column-at-a-time elimination
        if (tile && tj > jb) {
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
                if (jj >= nj) break;
                const double inv = pinv[jj];
                double lr[4], lc[4];
#pragma unroll
                for (int r = 0; r < 4; r++) lr[r] = pcol[jj][r0 + r];
#pragma unroll
                for (int c = 0; c < 4; c++) lc[c] = pcol[jj][c0 + c] * inv;
#pragma unroll
                for (int r = 0; r < 4; r++)
#pragma unroll
                    for (int c = 0; c < 4; c++) a[r][c] -= lr[r] * lc[c];
            }
        }
    }
    // V for the backward solve (lower triangle + the augmented row)
    if (tile) {
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int gr = r0 + r, gc = c0 + c;
                if (gr <= n && gc < n) V[gr * ld + gc] = a[r][c];
            }
    }
    __syncthreads();
    // backward: x = L^-T D^-1 z, column-oriented inside one warp: lane owns entries lane, lane+32, lane+64, lane+96 in
    // registers; after x_i is final it is broadcast and eliminated from the entries above it.
    if (tid < 32) {
        double xr[4];
#pragma unroll
        for (int q = 0; q < 4; q++) { const int i = lane + 32 * q; xr[q] = i < n ? V[n * ld + i] * invd[i] : 0.0; }
        for (int i = n - 1; i >= 0; i--) {
            const int qi = i >> 5;                                             // warp-uniform
            const double own = qi == 0 ? xr[0] : qi == 1 ? xr[1] : qi == 2 ? xr[2] : xr[3];
            const double xi = __shfl_sync(0xffffffffu, own, i & 31);
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int k = lane + 32 * q;
                if (k < i) xr[q] -= V[i * ld + k] * invd[k] * xi;
            }
        }
#pragma unroll
        for (int q = 0; q < 4; q++) { const int i = lane + 32 * q; if (i < n) P.yf[i] = xr[q]; }
        if (lane == 0) st.chol_ok = ok_s;
    }
}
__global__ void __launch_bounds__(CH_THREADS) ba_chol_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    extern __shared__ double sm[];
    const BaProblem P = probs[blockIdx.x];
    if (P.st->done) return;
    ba_chol_body(P, sm);
}

// ------------------------------------------------------------------------------------------ back-substitution (thread / landmark)
// ye = (E'b - E'F yf) / (E'E + D^2), candidate inverse depths, this landmark's share of the model cost change
// -(J s)'(r + J s / 2); CTA (0, p) also builds the candidate poses Plus(x, delta).
// candidate pose of keyframe k: Plus(x, -yf * scale) for a free pose, a copy otherwise
__device__ __forceinline__ void backsub_cand_pose(const BaProblem& P, int k, double* out) {
    const int c0 = P.pose_col[k];
    if (c0 >= 0) {
        double dlt[6];
        for (int i = 0; i < 6; i++) dlt[i] = -P.yf[c0 + i] * P.scf[c0 + i];
        se3_plus(P.poses + 7 * k, dlt, out);
    } else
        for (int i = 0; i < 7; i++) out[i] = P.poses[7 * k + i];
}
// one landmark: ye, candidate inverse depth, and its share of the model cost change (returned)
__device__ __forceinline__ double backsub_landmark(const BaProblem& P, int l) {
    const int b = P.lm_start[l], e = P.lm_start[l + 1];
    double ye = 0, acc = 0;
    if (e > b) {
        double s = P.etb[l];
        const int ca = P.pose_col[P.anch_kf[l]];
        if (ca >= 0) { double w[6]; ld2<6>(P.wa + 6 * l, w); for (int c = 0; c < 6; c++) s -= w[c] * P.yf[ca + c]; }
        for (int i = b; i < e; i++) {
            const int o = P.lm_obs[i];
            const int cp = P.pose_col[P.obs_kf[o]];
            if (cp >= 0) { double w[6]; ld2<6>(P.wp + 6 * o, w); for (int c = 0; c < 6; c++) s -= w[c] * P.yf[cp + c]; }
        }
        ye = s / P.ete[l];
        const double se = -ye * P.sce[l];
        for (int i = b; i < e; i++) {
            const int o = P.lm_obs[i];
            const int cp = P.pose_col[P.obs_kf[o]];
            double d[2], r[2], J[12];
            ld2<2>(P.Jd + 2 * o, d);
            ld2<2>(P.res + 2 * o, r);
            ld2<12>(P.Ja + 12 * o, J);
            double m0 = d[0] * se, m1 = d[1] * se;
#pragma unroll
            for (int c = 0; c < 6; c++) {
                if (ca >= 0) { const double q = -P.yf[ca + c] * P.scf[ca + c]; m0 += J[c] * q; m1 += J[6 + c] * q; }
                if (cp >= 0) { const double q = -P.yf[cp + c] * P.scf[cp + c]; m0 += -J[c] * q; m1 += -J[6 + c] * q; }
            }
            acc += m0 * (r[0] + m0 / 2.0) + m1 * (r[1] + m1 / 2.0);
        }
        P.cand_invd[l] = P.invd[l] + se;
    } else
        P.cand_invd[l] = P.invd[l];
    P.ye[l] = ye;
    return acc;
}
__global__ void __launch_bounds__(BS_THREADS) ba_backsub_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.y];
    __shared__ double red[BS_THREADS];
    if (P.st->done) return;
    const int l = blockIdx.x * BS_THREADS + threadIdx.x;
    if (blockIdx.x == 0)   // every keyframe (up to 256, two per thread): ba_post_body copies all nkf candidates over the poses
        for (int k = threadIdx.x; k < D.nkf; k += BS_THREADS) backsub_cand_pose(P, k, P.cand_poses + 7 * k);
    const double acc = l < D.nlm ? backsub_landmark(P, l) : 0.0;
    const double tot = block_sum<BS_THREADS>(acc, red);
    if (threadIdx.x == 0) P.mc_part[blockIdx.x] = tot;
}

// ------------------------------------------------------------------------------------------ control: after the step
__device__ void ba_post_body(const BaProblem& P, const BaDims& D) {
    BaState& st = *P.st;
    __shared__ double red[34];
    __shared__ int accept_s;
    const int tid = threadIdx.x, NT = blockDim.x;
    if (st.done) return;
    // model cost change -(J s)'(r + J s / 2) from the back-substitution partials (fixed order)
    double mcs = 0;
    for (int i = tid; i < D.nbs; i += NT) mcs += P.mc_part[i];
    const double model_change = -block_sum_dyn(mcs, red);
    const bool valid = st.chol_ok && (model_change > 0.0);
    __syncthreads();
    if (!valid) {   // HandleInvalidStep + LevenbergMarquardtStrategy::StepIsInvalid
        if (tid == 0) {
            st.model_change = model_change;
            if (++st.invalid_steps >= 5) { st.term = 2; st.done = 1; }
            st.radius *= 0.5;
            st.reuse_diagonal = 1;
            st.push_cost = st.x_cost;
            st.chol_ok = 1;
        }
        return;
    }
    if (P.last_poses) {
        // the candidate has been evaluated (cost-only pass): from here until the next valid step it is the point the
        // reference's functors were evaluated at last, whether or not the step is accepted or a tolerance ends the solve
        for (int i = tid; i < 7 * D.nkf; i += NT) P.last_poses[i] = P.cand_poses[i];
        for (int l = tid; l < D.nlm; l += NT) P.last_invd[l] = P.cand_invd[l];
        if (tid == 0) st.has_last = 1;
    }
    double c = 0;
    for (int i = tid; i < D.nblk; i += NT) c += P.cost_part[i];
    const double cand_cost = block_sum_dyn(c, red);
    double sn = 0;
    for (int k = tid; k < D.nkf; k += NT)
        if (P.pose_col[k] >= 0)
            for (int i = 0; i < 7; i++) { const double d = P.poses[7 * k + i] - P.cand_poses[7 * k + i]; sn += d * d; }
    for (int l = tid; l < D.nlm; l += NT)
        if (P.lm_start[l + 1] > P.lm_start[l]) { const double d = P.invd[l] - P.cand_invd[l]; sn += d * d; }
    sn = block_sum_dyn(sn, red);
    if (tid == 0) {
        int accept = 0;
        st.invalid_steps = 0;
        st.cand_cost = cand_cost;
        const double step_norm = sqrt(sn);
        if (step_norm <= 1e-8 * (st.xnorm + 1e-8)) { st.term = 0; st.done = 1; }                 // ParameterToleranceReached
        else if (fabs(st.x_cost - cand_cost) <= 1e-3 * st.x_cost) { st.term = 0; st.done = 1; }  // FunctionToleranceReached
        else {
            const double mc = model_change;
            st.model_change = model_change;
            const double rel = (st.se_cur - cand_cost) / mc;
            const double hist = (st.se_ref - cand_cost) / (st.se_acc_ref + mc);
            const double quality = fmax(rel, hist);
            if (quality > 1e-3) {
                accept = 1;
                st.radius = fmin(1e16, st.radius / fmax(1.0 / 3.0, 1.0 - pow(2.0 * quality - 1.0, 3)));
                st.decrease_factor = 2.0;
                st.reuse_diagonal = 0;
                st.se_cur = cand_cost; st.se_acc_cand += mc; st.se_acc_ref += mc;
                bool nonmono = false;
                if (st.se_cur < st.se_min) { st.se_min = st.se_cur; st.se_cand = st.se_cur; st.se_acc_cand = 0; }
                else { nonmono = true; if (st.se_cur > st.se_cand) { st.se_cand = st.se_cur; st.se_acc_cand = 0; } }
                if (!nonmono) { st.se_ref = st.se_cand; st.se_acc_ref = st.se_acc_cand; }
                st.last_success = 1;
                st.relin = 1;
            } else {
                st.radius = st.radius / st.decrease_factor;
                st.decrease_factor *= 2.0;
                st.reuse_diagonal = 1;
                st.push_cost = cand_cost;
            }
        }
        accept_s = accept;
    }
    __syncthreads();
    if (accept_s) {
        for (int i = tid; i < 7 * D.nkf; i += NT) P.poses[i] = P.cand_poses[i];
        for (int l = tid; l < D.nlm; l += NT) P.invd[l] = P.cand_invd[l];
        for (int i = tid; i < NMAX; i += NT) { P.nf[i] = 0; P.gf[i] = 0; }
        for (int l = tid; l < D.nlm; l += NT) { P.ne[l] = 0; P.ge[l] = 0; }
    }
}

__global__ void __launch_bounds__(CT_THREADS) ba_post_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.x];
    ba_post_body(P, D);
}

// kernel-level dump of the linearisation (corrected residuals and local Jacobians) for parity tests
__global__ void ba_linearize_dump_kernel(const double* calib, const double* poses, const double* invd, const int32_t* anch_kf,
                                         const double* anch_uv, const int32_t* obs_kf, const int32_t* obs_lm,
                                         const double* obs_uv, int nobs, double hub, double* res, double* Ja, double* Jp,
                                         double* Jd, double* cost) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= nobs) return;
    const int l = obs_lm[o];
    double r[2] = {0, 0}, A[12], Pp[12], Dd[2];
    for (int i = 0; i < 12; i++) A[i] = Pp[i] = 0;
    Dd[0] = Dd[1] = 0;
    double c = 0;
    if (l >= 0) {
        ba_evaluate(calib, poses + 7 * anch_kf[l], poses + 7 * obs_kf[o], invd[l], obs_uv[2 * o], obs_uv[2 * o + 1],
                    anch_uv[2 * l], anch_uv[2 * l + 1], r, A, Pp, Dd);
        double rho0, rho1;
        huber(r[0] * r[0] + r[1] * r[1], hub, rho0, rho1);
        c = 0.5 * rho0;
        const double sc = sqrt(rho1);
        r[0] *= sc; r[1] *= sc; Dd[0] *= sc; Dd[1] *= sc;
        for (int i = 0; i < 12; i++) { A[i] *= sc; Pp[i] *= sc; }
    }
    res[2 * o] = r[0]; res[2 * o + 1] = r[1]; Jd[2 * o] = Dd[0]; Jd[2 * o + 1] = Dd[1];
    for (int i = 0; i < 12; i++) { Ja[12 * o + i] = A[i]; Jp[12 * o + i] = Pp[i]; }
    cost[o] = c;
}

// ------------------------------------------------------------------------------------------ localBA outlier handling
// Optimizer::localBA (optimizer.cpp:273-299, 330-356): after a solve, a residual is an outlier if the functor's LAST
// evaluation saw chi2 = |r|^2 (sigma = 1) above the threshold or a non-positive depth.
__global__ void ba_local_init_kernel(const BaProblem* __restrict__ probs, BaDims D) {
    const BaProblem P = probs[blockIdx.y];
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o < D.nobs) { P.obs_lm_w[o] = P.obs_lm_in[o]; P.flags[o] = 0; }
    if (o == 0) { P.st->nbad = 0; P.st->has_last = 0; P.st->skipped = 0; }
}

template <int MARK>
__global__ void __launch_bounds__(LIN_THREADS) ba_flag_kernel(const BaProblem* __restrict__ probs, BaDims D, double chi2_thr) {
    const BaProblem P = probs[blockIdx.y];
    BaState& st = *P.st;
    if (MARK == 2 && st.skipped) return;
    const int o = blockIdx.x * LIN_THREADS + threadIdx.x;
    const int l = o < D.nobs ? P.obs_lm_w[o] : -1;
    if (l < 0) return;
    const double* poses = st.has_last ? P.last_poses : P.poses;
    const double* invd = st.has_last ? P.last_invd : P.invd;
    double r[2];
    const bool front = ba_evaluate(P.calib, poses + 7 * P.anch_kf[l], poses + 7 * P.obs_kf[o], invd[l], P.obs_uv[2 * o],
                                   P.obs_uv[2 * o + 1], P.anch_uv[2 * l], P.anch_uv[2 * l + 1], r, nullptr, nullptr, nullptr);
    if (r[0] * r[0] + r[1] * r[1] > chi2_thr || !front) {
        P.flags[o] = MARK;
        if (MARK == 1) { P.obs_lm_w[o] = -1; atomicAdd(&st.nbad, 1); }   // RemoveResidualBlock; integer count: order-independent
    }
}

__global__ void ba_summary_local_kernel(const BaProblem* __restrict__ probs, double* __restrict__ summary, int second) {
    const BaState& st = *probs[blockIdx.x].st;
    if (threadIdx.x == 0) {
        double* s = summary + 10 * blockIdx.x + 5 * second;
        if (second && st.skipped) { s[0] = s[1] = s[2] = s[3] = s[4] = 0; return; }
        s[0] = st.initial_cost; s[1] = st.x_cost; s[2] = st.n_success; s[3] = st.n_iter; s[4] = st.term;
    }
}

__global__ void ba_summary_kernel(const BaProblem* __restrict__ probs, double* __restrict__ summary) {
    const BaState& st = *probs[blockIdx.x].st;
    if (threadIdx.x == 0) {
        double* s = summary + 8 * blockIdx.x;
        s[0] = st.initial_cost; s[1] = st.x_cost; s[2] = st.n_success; s[3] = st.n_iter; s[4] = st.term;
        s[5] = st.ncols; s[6] = st.radius; s[7] = st.iteration;
    }
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

// Workspace carving: one contiguous block per problem.
static int g_ba_dense_schur = 0;   // alva_set_option("ba_dense_schur", 1): tensor-core SYRK for the Schur term
static int g_ba_ctl_threads = CT_THREADS;   // alva_set_option("ba_ctl_threads", 256 | 512 | 1024): CTA size of the control kernels

static size_t ba_ws_bytes(int nkf, int nlm, int nobs, int nblk) {
    size_t d = 0;
    if (g_ba_dense_schur) d += (size_t)((nlm + 3) / 4 * 4) * NMAX;
    d += (size_t)nobs * (2 + 12 + 2 + 6);           // res, Ja, Jd, wp
    d += 5 * (size_t)NMAX;                           // nf gf scf diagf Df
    d += 5 * (size_t)nlm;                            // ne ge sce diage De
    d += (size_t)nlm * (1 + 1 + 6 + 1);              // ete etb wa ye
    d += (size_t)NMAX * NMAX + 2 * NMAX;             // S rhs yf
    d += (size_t)nkf * 7 + nlm;                      // cand
    d += (size_t)nblk;                               // cost partials
    d += (size_t)((nlm + BS_THREADS - 1) / BS_THREADS);   // model-cost partials
    d += (size_t)NBMAX * GA_SPLIT * 42;                   // gather partials
    d += 64;                                              // ba_prepare rounds every array to an even number of doubles
    size_t bytes = d * sizeof(double);
    bytes += align_up((size_t)nkf * 4, 8) + align_up((size_t)(nlm + 1) * 4, 8) + align_up((size_t)nobs * 4, 8);
    bytes += align_up((size_t)nobs * 4, 8) + align_up((size_t)nlm * 4, 8);                          // obs_col, anch_col
    bytes += align_up((size_t)(NBMAX + 1) * 4, 8) + align_up(((size_t)nobs + (size_t)nlm) * 4, 8);   // pstart, plist
    bytes += 2 * align_up((size_t)(NBMAX * NBMAX + 1) * 4, 8) + align_up((size_t)(8 * (size_t)nobs + 2 * (size_t)nlm) * 8, 8);   // blk_start, blk_off, pairs
    bytes += align_up((size_t)NBMAX * 4, 8);                                                        // ga_ticket
    bytes += align_up(sizeof(BaState), 8);
    return align_up(bytes, 256);
}

// Table of per-problem pointers at the head of ctx->ba_ws.  It depends only on the argument pointers and dimensions, so
// it is rebuilt (one synchronous copy) only when those change -- a steady-state solve enqueues kernels and nothing else.
// local: alva_k_ba_local's extra buffers (working obs_lm, last evaluated point) and its flags output.
static int ba_prepare(alva_ctx* ctx, int nprob, int nkf, int nlm, int nobs, const double* calib, double* poses,
                      const uint8_t* pose_const, double* invd, const int32_t* anch_kf, const double* anch_uv,
                      const int32_t* obs_kf, const int32_t* obs_lm, const double* obs_uv, int32_t* flags,
                      const BaProblem** dp_out, BaDims* D_out) {
    const bool local = flags != nullptr;
    const int nblk = (nobs + LIN_THREADS - 1) / LIN_THREADS;
    const size_t per_local = align_up((size_t)nobs * 4, 8) + (7 * (size_t)nkf + (size_t)nlm) * sizeof(double);
    const size_t per = align_up(ba_ws_bytes(nkf, nlm, nobs, nblk) + (local ? per_local : 0), 256);
    const size_t tab = align_up(sizeof(BaProblem) * nprob, 256);
    if (tab + per * nprob > ctx->ba_ws_bytes) {
        ctx->ws_epoch++;
        if (ctx->ba_ws) { ALVA_CUDA(cudaStreamSynchronize(ctx->stream)); ALVA_CUDA(cudaFree(ctx->ba_ws)); ctx->ba_ws = nullptr; ctx->ba_ws_bytes = 0; }
        ALVA_CUDA(cudaMalloc(&ctx->ba_ws, tab + per * nprob));
        ctx->ba_ws_bytes = tab + per * nprob;
        ctx->ba_table_key = 0;
    }
    uint8_t* ws = (uint8_t*)ctx->ba_ws;
    uint64_t key = 1469598103934665603ull;
    auto mix = [&](uint64_t v) { key = (key ^ v) * 1099511628211ull; };
    mix((uint64_t)(uintptr_t)ws); mix(nprob); mix(nkf); mix(nlm); mix(nobs); mix((uint64_t)g_ba_dense_schur);
    mix((uint64_t)(uintptr_t)calib); mix((uint64_t)(uintptr_t)poses); mix((uint64_t)(uintptr_t)pose_const); mix((uint64_t)(uintptr_t)invd);
    mix((uint64_t)(uintptr_t)anch_kf); mix((uint64_t)(uintptr_t)anch_uv); mix((uint64_t)(uintptr_t)obs_kf);
    mix((uint64_t)(uintptr_t)obs_lm); mix((uint64_t)(uintptr_t)obs_uv); mix((uint64_t)(uintptr_t)flags);
    if (key != ctx->ba_table_key) {
        std::string hostbuf(sizeof(BaProblem) * nprob, '\0');
        BaProblem* hp = reinterpret_cast<BaProblem*>(&hostbuf[0]);
        for (int p = 0; p < nprob; p++) {
            BaProblem& P = hp[p];
            P.calib = calib + 4 * (size_t)p; P.poses = poses + 7 * (size_t)nkf * p; P.pose_const = pose_const + (size_t)nkf * p;
            P.invd = invd + (size_t)nlm * p; P.anch_kf = anch_kf + (size_t)nlm * p; P.anch_uv = anch_uv + 2 * (size_t)nlm * p;
            P.obs_kf = obs_kf + (size_t)nobs * p; P.obs_lm = obs_lm + (size_t)nobs * p; P.obs_uv = obs_uv + 2 * (size_t)nobs * p;
            double* d = reinterpret_cast<double*>(ws + tab + per * p);
            auto take = [&](size_t n) { double* r = d; d += (n + 1) & ~(size_t)1; return r; };   // every array 16-byte aligned (ld2)
            P.res = take(2 * (size_t)nobs); P.Ja = take(12 * (size_t)nobs); P.Jd = take(2 * (size_t)nobs);
            P.wp = take(6 * (size_t)nobs);
            P.nf = take(NMAX); P.gf = take(NMAX); P.scf = take(NMAX); P.diagf = take(NMAX); P.Df = take(NMAX);
            P.ne = take(nlm); P.ge = take(nlm); P.sce = take(nlm); P.diage = take(nlm); P.De = take(nlm);
            P.ete = take(nlm); P.etb = take(nlm); P.wa = take(6 * (size_t)nlm); P.ye = take(nlm);
            P.S = take((size_t)NMAX * NMAX); P.rhs = take(NMAX); P.yf = take(NMAX);
            P.cand_poses = take(7 * (size_t)nkf); P.cand_invd = take(nlm); P.cost_part = take(nblk);
            P.Wt = g_ba_dense_schur ? take((size_t)((nlm + 3) / 4 * 4) * NMAX) : nullptr;
            P.mc_part = take((size_t)((nlm + BS_THREADS - 1) / BS_THREADS));
            P.ga_part = take((size_t)NBMAX * GA_SPLIT * 42);
            P.last_poses = local ? take(7 * (size_t)nkf) : nullptr;
            P.last_invd = local ? take(nlm) : nullptr;
            uint8_t* b = reinterpret_cast<uint8_t*>(d);
            P.pose_col = reinterpret_cast<int32_t*>(b); b += align_up((size_t)nkf * 4, 8);
            P.lm_start = reinterpret_cast<int32_t*>(b); b += align_up((size_t)(nlm + 1) * 4, 8);
            P.lm_obs = reinterpret_cast<int32_t*>(b); b += align_up((size_t)nobs * 4, 8);
            P.obs_col = reinterpret_cast<int32_t*>(b); b += align_up((size_t)nobs * 4, 8);
            P.anch_col = reinterpret_cast<int32_t*>(b); b += align_up((size_t)nlm * 4, 8);
            P.pstart = reinterpret_cast<int32_t*>(b); b += align_up((size_t)(NBMAX + 1) * 4, 8);
            P.plist = reinterpret_cast<uint32_t*>(b); b += align_up(((size_t)nobs + (size_t)nlm) * 4, 8);
            P.blk_start = reinterpret_cast<int32_t*>(b); b += align_up((size_t)(NBMAX * NBMAX + 1) * 4, 8);
            P.blk_off = reinterpret_cast<int32_t*>(b); b += align_up((size_t)(NBMAX * NBMAX + 1) * 4, 8);
            P.pairs = reinterpret_cast<uint64_t*>(b); b += align_up((size_t)(8 * (size_t)nobs + 2 * (size_t)nlm) * 8, 8);
            P.ga_ticket = reinterpret_cast<int32_t*>(b); b += align_up((size_t)NBMAX * 4, 8);
            P.obs_lm_in = nullptr; P.obs_lm_w = nullptr; P.flags = nullptr;
            if (local) {
                P.obs_lm_in = P.obs_lm;
                P.obs_lm_w = reinterpret_cast<int32_t*>(b); b += align_up((size_t)nobs * 4, 8);
                P.obs_lm = P.obs_lm_w;
                P.flags = flags + (size_t)nobs * p;
            }
            P.st = reinterpret_cast<BaState*>(b);
        }
        ALVA_CUDA(cudaMemcpyAsync(ws, hp, sizeof(BaProblem) * nprob, cudaMemcpyHostToDevice, ctx->stream));
        ALVA_CUDA(cudaStreamSynchronize(ctx->stream));   // hostbuf is pageable: the copy must finish before it dies
        ctx->ba_table_key = key;
    }
    *dp_out = reinterpret_cast<const BaProblem*>(ws);
    *D_out = BaDims{nkf, nlm, nobs, nblk, 0.0, 0, (nlm + 3) / 4 * 4, 8 * nobs + 2 * nlm, (nlm + BS_THREADS - 1) / BS_THREADS, 0};
    return 0;
}

// One trust-region solve: structure, then max_iter x (linearise, reduce, factor, back-substitute, evaluate, decide).
// Every decision is taken on the device (BaState), so the host only enqueues; kernels of a finished problem return at once.
static int ba_run_solve(alva_ctx* ctx, const BaProblem* dp, const BaDims& D, int nprob) {
    const bool dense = g_ba_dense_schur != 0;
    const size_t chol_smem = ((size_t)NMAX * (NMAX + 1) + NMAX) * sizeof(double);
    ALVA_CUDA(cudaFuncSetAttribute(ba_chol_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)chol_smem));
    ba_setup_kernel<<<nprob, SETUP_THREADS, 0, ctx->stream>>>(dp, D);
    ALVA_LAUNCH_CHECK(ctx);
    const dim3 lin_grid(D.nblk, nprob), schur_grid((D.nlm_pad + 127) / 128, nprob), syrk_grid(16, SYRK_KSPLIT, nprob);
    const dim3 key_grid(GA_GRID, nprob), bs_grid(D.nbs, nprob), stats_grid(D.nbs + NBMAX, nprob);
    bool forked = false;
    if (!dense) {   // structure of the gather-form Schur complement, once per solve -- beside the first linearisation, which
                    // does not need it (fork / join on the context's auxiliary stream; also valid inside a stream capture)
        const dim3 pr_grid(NBMAX, nprob);
        cudaStream_t ps = ctx->stream;
        if (ctx->aux_stream && cudaEventRecord(ctx->aux_fork, ctx->stream) == cudaSuccess &&
            cudaStreamWaitEvent(ctx->aux_stream, ctx->aux_fork, 0) == cudaSuccess) { ps = ctx->aux_stream; forked = true; }
        ba_pairs_kernel<0><<<pr_grid, 32, 0, ps>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
        ba_pairs_kernel<1><<<pr_grid, 32, 0, ps>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
        if (forked) ALVA_CUDA(cudaEventRecord(ctx->aux_join, ps));
    }
    for (int it = 0; it <= D.max_iter; it++) {
        ba_linearize_kernel<true><<<lin_grid, LIN_THREADS, 0, ctx->stream>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
        ba_stats_kernel<<<stats_grid, BS_THREADS, 0, ctx->stream>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
        ba_pre_kernel<<<nprob, g_ba_ctl_threads, 0, ctx->stream>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
        if (it == D.max_iter) {   // the last pass only finalises (iteration count reached)
            if (forked) { ALVA_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->aux_join, 0)); forked = false; }   // max_iter == 0
            break;
        }
        if (dense) {
            ba_schur_kernel<true><<<schur_grid, 128, 0, ctx->stream>>>(dp, D);
            ALVA_LAUNCH_CHECK(ctx);
            ba_syrk_dmma_kernel<<<syrk_grid, 128, 0, ctx->stream>>>(dp, D);
            ALVA_LAUNCH_CHECK(ctx);
        } else {
            if (forked) { ALVA_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->aux_join, 0)); forked = false; }   // use_gather is final
            ba_lm_kernel<<<schur_grid, 128, 0, ctx->stream>>>(dp, D);           // gather path (no-op if structure too large)
            ALVA_LAUNCH_CHECK(ctx);
            ba_gather_kernel<<<key_grid, GA_THREADS, 0, ctx->stream>>>(dp, D);
            ALVA_LAUNCH_CHECK(ctx);
        }
        ba_chol_kernel<<<nprob, CH_THREADS, chol_smem, ctx->stream>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
        ba_backsub_kernel<<<bs_grid, BS_THREADS, 0, ctx->stream>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
        ba_linearize_kernel<false><<<lin_grid, LIN_THREADS, 0, ctx->stream>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
        ba_post_kernel<<<nprob, g_ba_ctl_threads, 0, ctx->stream>>>(dp, D);
        ALVA_LAUNCH_CHECK(ctx);
    }
    return 0;
}

static bool ba_args_ok(alva_ctx* ctx, int nprob, int nkf, int nlm, int nobs, const void* calib, const void* poses,
                       const void* pose_const, const void* invd, const void* anch_kf, const void* anch_uv, const void* obs_kf,
                       const void* obs_lm, const void* obs_uv, int max_iter) {
    return ctx && nprob >= 1 && nkf >= 1 && nkf <= 256 && nlm >= 1 && nobs >= 1 && calib && poses && pose_const && invd &&
           anch_kf && anch_uv && obs_kf && obs_lm && obs_uv && max_iter >= 0;
}

extern "C" int alva_k_ba_solve(alva_ctx* ctx, int nprob, int nkf, int nlm, int nobs, const double* calib, double* poses,
                               const uint8_t* pose_const, double* invd, const int32_t* anch_kf, const double* anch_uv,
                               const int32_t* obs_kf, const int32_t* obs_lm, const double* obs_uv, double huber_delta,
                               int max_iter, double* summary) { AlvaDeviceGuard guard__(ctx);
    if (!ba_args_ok(ctx, nprob, nkf, nlm, nobs, calib, poses, pose_const, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv, max_iter)) {
        alva_set_error("alva_k_ba_solve: bad argument (need 1 <= nkf <= 256)");
        return ALVA_E_INVALID;
    }
    const BaProblem* dp;
    BaDims D;
    if (int e = ba_prepare(ctx, nprob, nkf, nlm, nobs, calib, poses, pose_const, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv,
                           nullptr, &dp, &D))
        return e;
    D.huber = huber_delta; D.max_iter = max_iter;
    if (int e = ba_run_solve(ctx, dp, D, nprob)) return e;
    if (summary) {
        ba_summary_kernel<<<nprob, 32, 0, ctx->stream>>>(dp, summary);
        ALVA_LAUNCH_CHECK(ctx);
    }
    return 0;
}

// Optimizer::localBA steps 2-4 (src/slam/src/optimizer.cpp:251-359) for nprob independent problems, all on the device:
// solve (Huber, <= max_iter), remove the residuals whose last evaluation was an outlier, and -- per problem, only if it
// lost residuals and the robust loss is on -- solve again (<= 5 iterations) and flag once more.
extern "C" int alva_k_ba_local(alva_ctx* ctx, int nprob, int nkf, int nlm, int nobs, const double* calib, double* poses,
                               const uint8_t* pose_const, double* invd, const int32_t* anch_kf, const double* anch_uv,
                               const int32_t* obs_kf, const int32_t* obs_lm, const double* obs_uv, double huber_delta,
                               double chi2_thr, int max_iter, int32_t* flags, double* summary) { AlvaDeviceGuard guard__(ctx);
    if (!ba_args_ok(ctx, nprob, nkf, nlm, nobs, calib, poses, pose_const, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv, max_iter) ||
        !flags) {
        alva_set_error("alva_k_ba_local: bad argument (need 1 <= nkf <= 256, flags != NULL)");
        return ALVA_E_INVALID;
    }
    const BaProblem* dp;
    BaDims D;
    if (int e = ba_prepare(ctx, nprob, nkf, nlm, nobs, calib, poses, pose_const, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv,
                           flags, &dp, &D))
        return e;
    D.huber = huber_delta; D.max_iter = max_iter;
    const dim3 obs_grid(D.nblk, nprob);
    ba_local_init_kernel<<<obs_grid, LIN_THREADS, 0, ctx->stream>>>(dp, D);
    ALVA_LAUNCH_CHECK(ctx);
    if (int e = ba_run_solve(ctx, dp, D, nprob)) return e;
    if (summary) { ba_summary_local_kernel<<<nprob, 32, 0, ctx->stream>>>(dp, summary, 0); ALVA_LAUNCH_CHECK(ctx); }
    ba_flag_kernel<1><<<obs_grid, LIN_THREADS, 0, ctx->stream>>>(dp, D, chi2_thr);
    ALVA_LAUNCH_CHECK(ctx);
    D.pass = 1; D.max_iter = 5;   // optimizer.cpp:309: the refinement is capped at 5 iterations
    if (int e = ba_run_solve(ctx, dp, D, nprob)) return e;
    ba_flag_kernel<2><<<obs_grid, LIN_THREADS, 0, ctx->stream>>>(dp, D, chi2_thr);
    ALVA_LAUNCH_CHECK(ctx);
    if (summary) { ba_summary_local_kernel<<<nprob, 32, 0, ctx->stream>>>(dp, summary, 1); ALVA_LAUNCH_CHECK(ctx); }
    return 0;
}

extern "C" int alva_k_ba_linearize(alva_ctx* ctx, int nkf, int nlm, int nobs, const double* calib, const double* poses,
                                   const double* invd, const int32_t* anch_kf, const double* anch_uv, const int32_t* obs_kf,
                                   const int32_t* obs_lm, const double* obs_uv, double huber_delta, double* res, double* Ja,
                                   double* Jp, double* Jd, double* cost_per_obs) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || nobs < 1 || !calib || !poses || !invd || !res || !Ja || !Jp || !Jd || !cost_per_obs) {
        alva_set_error("alva_k_ba_linearize: bad argument");
        return ALVA_E_INVALID;
    }
    (void)nkf; (void)nlm;
    ba_linearize_dump_kernel<<<(nobs + 127) / 128, 128, 0, ctx->stream>>>(calib, poses, invd, anch_kf, anch_uv, obs_kf, obs_lm,
                                                                         obs_uv, nobs, huber_delta, res, Ja, Jp, Jd, cost_per_obs);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// Test hook: the reduced camera system S, rhs of a solve's first LM iteration (iteration 0's linearisation, Jacobi scaling
// and diagonal), assembled by the path the solve would take -- or, with atomic != 0, by the atomic per-landmark path on the
// same linearisation.  S_out [nprob][128][128], rhs_out [nprob][128], info [nprob][2] = {reduced-system width, gather path}.
namespace {
__global__ void ba_force_atomic_kernel(const BaProblem* __restrict__ probs) { probs[blockIdx.x].st->use_gather = 0; }
__global__ void ba_dump_schur_kernel(const BaProblem* __restrict__ probs, double* S_out, double* rhs_out, double* info) {
    const BaProblem P = probs[blockIdx.x];
    for (int i = threadIdx.x; i < NMAX * NMAX; i += blockDim.x) S_out[(size_t)blockIdx.x * NMAX * NMAX + i] = P.S[i];
    for (int i = threadIdx.x; i < NMAX; i += blockDim.x) rhs_out[(size_t)blockIdx.x * NMAX + i] = P.rhs[i];
    if (threadIdx.x == 0) { info[2 * blockIdx.x] = P.st->ncols; info[2 * blockIdx.x + 1] = P.st->use_gather; }
}
}  // namespace
extern "C" int alva_k_ba_schur_dump(alva_ctx* ctx, int nprob, int nkf, int nlm, int nobs, const double* calib, const double* poses,
                                    const uint8_t* pose_const, const double* invd, const int32_t* anch_kf, const double* anch_uv,
                                    const int32_t* obs_kf, const int32_t* obs_lm, const double* obs_uv, double huber_delta,
                                    int atomic, double* S_out, double* rhs_out, double* info) { AlvaDeviceGuard guard__(ctx);
    if (!ba_args_ok(ctx, nprob, nkf, nlm, nobs, calib, poses, pose_const, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv, 1) ||
        !S_out || !rhs_out || !info || g_ba_dense_schur) {
        alva_set_error("alva_k_ba_schur_dump: bad argument (need 1 <= nkf <= 256, outputs, ba_dense_schur off)");
        return ALVA_E_INVALID;
    }
    const BaProblem* dp;
    BaDims D;
    // the first iteration writes neither the poses nor the inverse depths (only ba_post_kernel does)
    if (int e = ba_prepare(ctx, nprob, nkf, nlm, nobs, calib, const_cast<double*>(poses), pose_const, const_cast<double*>(invd),
                           anch_kf, anch_uv, obs_kf, obs_lm, obs_uv, nullptr, &dp, &D))
        return e;
    D.huber = huber_delta; D.max_iter = 1;
    const dim3 lin_grid(D.nblk, nprob), schur_grid((D.nlm_pad + 127) / 128, nprob), stats_grid(D.nbs + NBMAX, nprob);
    ba_setup_kernel<<<nprob, SETUP_THREADS, 0, ctx->stream>>>(dp, D);
    ba_pairs_kernel<0><<<dim3(NBMAX, nprob), 32, 0, ctx->stream>>>(dp, D);
    ba_pairs_kernel<1><<<dim3(NBMAX, nprob), 32, 0, ctx->stream>>>(dp, D);
    if (atomic) ba_force_atomic_kernel<<<nprob, 1, 0, ctx->stream>>>(dp);
    ba_linearize_kernel<true><<<lin_grid, LIN_THREADS, 0, ctx->stream>>>(dp, D);
    ba_stats_kernel<<<stats_grid, BS_THREADS, 0, ctx->stream>>>(dp, D);
    ba_pre_kernel<<<nprob, g_ba_ctl_threads, 0, ctx->stream>>>(dp, D);
    ba_lm_kernel<<<schur_grid, 128, 0, ctx->stream>>>(dp, D);
    ba_gather_kernel<<<dim3(GA_GRID, nprob), GA_THREADS, 0, ctx->stream>>>(dp, D);
    ba_dump_schur_kernel<<<nprob, 256, 0, ctx->stream>>>(dp, S_out, rhs_out, info);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// Library-wide options: "ba_dense_schur" = 1 routes the -(E'F)'(E'E)^-1(E'F) term of the Schur complement through the
// FP64 tensor-core SYRK (S -= Wt'Wt) instead of per-landmark atomics.  Returns 0, or ALVA_E_INVALID for an unknown name.
extern int alva_g_knn_qpw;   // hamming.cu
int alva_g_ba_overlap = 1;   // pipeline.cu: local BA on its own stream beside the frame stages

extern int alva_g_frontend_antipodal, alva_g_frontend_variant, alva_g_frontend_prefetch, alva_g_frontend_ctas;   // frontend.cu
extern int alva_g_knn_mma, alva_g_knn_mma_mode, alva_g_knn_mma_kind;
extern int alva_g_pipeline_graphs, alva_g_ba_lag;   // pipeline.cu
uint64_t alva_g_options_epoch = 0;
// a change of value bumps the options epoch: alva_pipeline then re-captures graphs that may have baked in the old choice
static int set_option(int& opt, int value) {
    if (opt != value) { opt = value; alva_g_options_epoch++; }
    return 0;
}
extern "C" int alva_set_option(const char* name, int value) {
    if (name && !strcmp(name, "ba_dense_schur")) return set_option(g_ba_dense_schur, value ? 1 : 0);
    if (name && !strcmp(name, "ba_ctl_threads") && (value == 256 || value == 512 || value == 1024)) return set_option(g_ba_ctl_threads, value);
    if (name && !strcmp(name, "frontend_antipodal")) return set_option(alva_g_frontend_antipodal, value ? 1 : 0);
    if (name && !strcmp(name, "frontend_variant") && (value == 0 || value == 2)) return set_option(alva_g_frontend_variant, value);
    if (name && !strcmp(name, "frontend_ctas") && (value == 4 || value == 5)) return set_option(alva_g_frontend_ctas, value);
    if (name && !strcmp(name, "frontend_prefetch")) return set_option(alva_g_frontend_prefetch, value ? 1 : 0);
    if (name && !strcmp(name, "pipeline_graphs")) return set_option(alva_g_pipeline_graphs, value ? 1 : 0);
    if (name && !strcmp(name, "pipeline_ba_lag")) return set_option(alva_g_ba_lag, value ? 1 : 0);
    if (name && !strcmp(name, "pipeline_ba_overlap")) return set_option(alva_g_ba_overlap, value ? 1 : 0);
    if (name && !strcmp(name, "knn_qpw") && (value == 4 || value == 8)) return set_option(alva_g_knn_qpw, value);
    if (name && !strcmp(name, "knn_mma") && value >= 0 && value <= 2) return set_option(alva_g_knn_mma, value);
    if (name && !strcmp(name, "knn_mma_kind") && value >= 0 && value <= 2) return set_option(alva_g_knn_mma_kind, value);
    if (name && !strcmp(name, "knn_mma_mode") && value >= 0 && value <= 2) return set_option(alva_g_knn_mma_mode, value);
    alva_set_error("alva_set_option: unknown option");
    return ALVA_E_INVALID;
}
