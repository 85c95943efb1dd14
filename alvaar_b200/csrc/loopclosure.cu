// loopclosure.cu -- cross-stream loop-closure detection over exchanged keyframe blocks (SURVEY 8e / 8f.4).
//
// The reference has no loop closure and no multi-stream mode (iBoW-LCD is vendored but never linked), so nothing here has a
// reference behaviour to match: PARITY UNPINNED for this stage -- it is validated stage by stage against a host model of what it
// computes (tests/lc_util.py, tests/test_gpu_loopclosure_model.py) and end to end by determinism and planted revisits
// (tests/test_gpu_loopclosure.py).  Capability model (not code): src/libs/ibow_lcd/src/lcdetector.cc -- candidate scoring,
// consecutive-detection ("island") consistency, geometric verification before a loop is reported.
//
// Per step every rank packs its K new keyframes into fixed-size KEYFRAME BLOCKS (wire format below, documented in
// include/alva_b200.h and INTEGRATION.md), the blocks are all-gathered (NCCL over NVLink: torch.distributed in the harness), and
// every rank runs on the gathered buffer, on its own stream, with no host synchronisation:
//   1. knn2_blockpair_kernel (hamming.cu): keyframe e of this rank against keyframe e of every other rank -- brute-force Hamming
//      2-NN over the live descriptors only;
//   2. lc_score_kernel: ratio test (best * ratio_den < second * ratio_num) + absolute distance gate -> putative matches, their
//      count, and the matched pairs' bearing vectors (pixel -> unit bearing with the block's own intrinsics);
//   3. alva_k_essential_5pt (32 hypotheses = one round of the five-point RANSAC) for the NEWEST keyframe of the step against every
//      remote stream with >= min_matches matches: the geometric check (every other pair has count 0 and returns at once);
//   4. one small device-to-host copy of {matches, success, inliers} per pair into page-locked memory + an event.
// alva_lc_poll() (host) consumes finished steps in order and applies the temporal rule: a loop with remote stream r is reported on
// the newest keyframe of a step when the last `min_consecutive` keyframe events against r all had >= min_matches putative matches
// and that keyframe passed the geometric check with >= min_inliers inliers.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include <deque>
#include <vector>

int alva_knn2_blockpair_launch(alva_ctx* ctx, const uint8_t* gathered, size_t block_bytes, int n_max, int K, int world, int rank,
                               int hdr_bytes, int32_t* out);

namespace {

constexpr int HDR = ALVA_LC_HEADER_BYTES;
constexpr int PAIR_CAP = ALVA_LC_PAIR_CAP;   // putative matches kept per keyframe pair (more than enough for RANSAC)

// a header count, written by another rank: live entries in [0, n_max]
__device__ __forceinline__ int live_count(int count, int n_max) { return min(max(count, 0), n_max); }

// header words: 0 magic, 1 version, 2 stream id, 3 keyframe sequence number, 4 count, 5 n_max, 6..9 fx fy cx cy (float)
__global__ void lc_pack_kernel(const uint8_t* __restrict__ desc, const float* __restrict__ pts, const int32_t* __restrict__ counts,
                               const int32_t* __restrict__ kf_frames, int cap, int n_max, int stream_id, int kf_seq0, float fx, float fy,
                               float cx, float cy, uint8_t* __restrict__ send, size_t block_bytes) {
    const int e = blockIdx.y;
    const int f = kf_frames[e];
    const int n = live_count(min(counts[f], cap), n_max);
    uint8_t* blk = send + (size_t)e * block_bytes;
    if (blockIdx.x == 0 && threadIdx.x < 16) {
        int32_t* h = reinterpret_cast<int32_t*>(blk);
        float* hf = reinterpret_cast<float*>(blk);
        const int i = threadIdx.x;
        if (i == 0) h[0] = ALVA_LC_MAGIC;
        else if (i == 1) h[1] = ALVA_LC_VERSION;
        else if (i == 2) h[2] = stream_id;
        else if (i == 3) h[3] = kf_seq0 + e;
        else if (i == 4) h[4] = n;
        else if (i == 5) h[5] = n_max;
        else if (i == 6) hf[6] = fx;
        else if (i == 7) hf[7] = fy;
        else if (i == 8) hf[8] = cx;
        else if (i == 9) hf[9] = cy;
        else h[i] = 0;
    }
    float2* px = reinterpret_cast<float2*>(blk + HDR);
    uint4* d = reinterpret_cast<uint4*>(blk + HDR + (size_t)n_max * 8);
    const float2* spx = reinterpret_cast<const float2*>(pts) + (size_t)f * cap;
    const uint4* sd = reinterpret_cast<const uint4*>(desc) + (size_t)f * cap * 2;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_max; i += gridDim.x * blockDim.x) {
        const bool live = i < n;
        px[i] = live ? spx[i] : make_float2(0.f, 0.f);
        d[2 * i] = live ? sd[2 * i] : make_uint4(0, 0, 0, 0);
        d[2 * i + 1] = live ? sd[2 * i + 1] : make_uint4(0, 0, 0, 0);
    }
}

__device__ __forceinline__ void bearing(float u, float v, float fx, float fy, float cx, float cy, double* b) {
    const double x = ((double)u - (double)cx) / (double)fx, y = ((double)v - (double)cy) / (double)fy;
    const double n = sqrt(x * x + y * y + 1.0);
    b[0] = x / n; b[1] = y / n; b[2] = 1.0 / n;
}

// one CTA per keyframe pair (e, r): ratio test over the local keyframe's 2-NN lists, ordered compaction of the survivors
__global__ void __launch_bounds__(256) lc_score_kernel(const uint8_t* __restrict__ gathered, size_t block_bytes, int n_max, int K, int rank,
                                                       const int4* __restrict__ nn, int max_dist, int ratio_num, int ratio_den,
                                                       int min_matches, int32_t* __restrict__ nmatch, int32_t* __restrict__ npair,
                                                       double* __restrict__ bv_local, double* __restrict__ bv_remote) {
    __shared__ int woff[8];
    __shared__ int base_s;
    const int r = blockIdx.x, e = blockIdx.y, world = gridDim.x;
    const int p = e * world + r;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (r == rank) { if (tid == 0) { nmatch[p] = 0; npair[p] = 0; } return; }
    const uint8_t* lb = gathered + ((size_t)rank * K + e) * block_bytes;
    const uint8_t* rb = gathered + ((size_t)r * K + e) * block_bytes;
    const int32_t* lh = reinterpret_cast<const int32_t*>(lb);
    const int32_t* rh = reinterpret_cast<const int32_t*>(rb);
    const float* lf = reinterpret_cast<const float*>(lb);
    const float* rf = reinterpret_cast<const float*>(rb);
    const bool valid = lh[0] == ALVA_LC_MAGIC && rh[0] == ALVA_LC_MAGIC && lh[1] == ALVA_LC_VERSION && rh[1] == ALVA_LC_VERSION;
    const int nq = valid ? live_count(lh[4], n_max) : 0;
    const float2* lpx = reinterpret_cast<const float2*>(lb + HDR);
    const float2* rpx = reinterpret_cast<const float2*>(rb + HDR);
    const int4* my = nn + (size_t)p * n_max;
    double* bl = bv_local + (size_t)p * PAIR_CAP * 3;
    double* br = bv_remote + (size_t)p * PAIR_CAP * 3;
    if (tid == 0) base_s = 0;
    __syncthreads();
    for (int i0 = 0; i0 < nq; i0 += 256) {
        const int i = i0 + tid;
        bool keep = false;
        int4 m = make_int4(-1, 0, -1, 0);
        if (i < nq) {
            m = my[i];
            keep = m.x >= 0 && m.y <= max_dist && (m.z < 0 || m.y * ratio_den < m.w * ratio_num);
        }
        const uint32_t bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) woff[warp] = __popc(bal);
        __syncthreads();
        int off = base_s;
        for (int w = 0; w < warp; w++) off += woff[w];
        if (keep) {
            const int d = off + __popc(bal & ((1u << lane) - 1u));
            if (d < PAIR_CAP) {
                const float2 a = lpx[i], b = rpx[m.x];
                bearing(a.x, a.y, lf[6], lf[7], lf[8], lf[9], bl + 3 * d);
                bearing(b.x, b.y, rf[6], rf[7], rf[8], rf[9], br + 3 * d);
            }
        }
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < 8; w++) t += woff[w]; base_s += t; }
        __syncthreads();
    }
    if (tid == 0) {
        const int n = base_s;
        nmatch[p] = n;
        // the geometric check is run for the NEWEST keyframe of the step only (0 -> it returns at once for this pair): one round of
        // the five-point RANSAC is serial FP64 (Sturm / Newton root isolation: dependent Horner chains) that outlasts a
        // pipeline step, and the temporal rule already asks the earlier events of the streak for match counts only
        // "enough" is relative as well: unrelated scenes still leave ~6 % of the keypoints as chance matches after the ratio test
        npair[p] = (e == K - 1 && n >= max(min_matches, nq / 8)) ? min(n, PAIR_CAP) : 0;
    }
}

// {matches, RANSAC success, inliers, remote keyframe sequence number} per pair, gathered for one small copy
// verdict: 0 = too few matches (or the geometric check failed), 1 = geometric check passed, 2 = enough matches, not checked (not the
// step's newest keyframe)
__global__ void lc_collect_kernel(const uint8_t* __restrict__ gathered, size_t block_bytes, int K, int world, int rank, int n_max, int min_matches,
                                  const int32_t* __restrict__ nmatch, const double* __restrict__ info, const double* __restrict__ Rt,
                                  double* __restrict__ out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= K * world) return;
    const int e = p / world, r = p - e * world;
    const int32_t* rh = reinterpret_cast<const int32_t*>(gathered + ((size_t)r * K + e) * block_bytes);
    const int32_t* lh = reinterpret_cast<const int32_t*>(gathered + ((size_t)rank * K + e) * block_bytes);
    const int nq = lh[0] == ALVA_LC_MAGIC ? live_count(lh[4], n_max) : 0;
    const bool enough = r != rank && nmatch[p] >= max(min_matches, nq / 8);
    double* o = out + (size_t)p * 16;
    o[0] = nmatch[p]; o[1] = e == K - 1 ? info[4 * p] : (enough ? 2.0 : 0.0); o[2] = info[4 * p + 1]; o[3] = rh[3];
    for (int i = 0; i < 12; i++) o[4 + i] = Rt[12 * p + i];
}

}  // namespace

struct alva_lc {
    alva_ctx* ctx = nullptr;
    alva_lc_config cfg{};
    size_t block_bytes = 0;
    int npair = 0;
    // device
    int32_t *nn = nullptr, *nmatch = nullptr, *npairs = nullptr;
    double *bvl = nullptr, *bvr = nullptr, *Rt = nullptr, *info = nullptr, *res_dev = nullptr;
    uint8_t* outl = nullptr;
    // page-locked result slots, one per step in flight
    static constexpr int NSLOT = 4;
    double* res_host[NSLOT] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t done[NSLOT] = {nullptr, nullptr, nullptr, nullptr};
    int local_seq0[NSLOT] = {0, 0, 0, 0};
    std::deque<int> inflight;
    int next_slot = 0, step_seq0 = 0;
    std::vector<int> consecutive;   // per remote stream: keyframe events in a row that passed the geometric check
    std::deque<alva_lc_event> ready;
};

extern "C" size_t alva_lc_block_bytes(int n_max) { return (size_t)ALVA_LC_HEADER_BYTES + (size_t)n_max * 8 + (size_t)n_max * 32; }

extern "C" void alva_lc_destroy(alva_lc* lc) {
    if (!lc) return;
    AlvaDeviceGuard guard__(lc->ctx);
    cudaStreamSynchronize(lc->ctx->stream);
    void* bufs[] = {lc->nn, lc->nmatch, lc->npairs, lc->bvl, lc->bvr, lc->Rt, lc->info, lc->res_dev, lc->outl};
    for (void* b : bufs) if (b) cudaFree(b);
    for (int s = 0; s < alva_lc::NSLOT; s++) {
        if (lc->res_host[s]) cudaFreeHost(lc->res_host[s]);
        if (lc->done[s]) cudaEventDestroy(lc->done[s]);
    }
    delete lc;
}

extern "C" alva_lc* alva_lc_create(alva_ctx* ctx, const alva_lc_config* cfg) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !cfg || cfg->n_max < 8 || cfg->n_max > 8192 || (cfg->n_max & 7) || cfg->kf_per_step < 1 || cfg->world < 1 || cfg->rank < 0 ||
        cfg->rank >= cfg->world) {
        alva_set_error("alva_lc_create: bad configuration (n_max: multiple of 8 in [8, 8192])");
        return nullptr;
    }
    alva_lc* lc = new alva_lc();
    lc->ctx = ctx;
    lc->cfg = *cfg;
    if (lc->cfg.min_matches <= 0) lc->cfg.min_matches = 30;
    if (lc->cfg.max_dist <= 0) lc->cfg.max_dist = 64;
    if (lc->cfg.ratio_num <= 0 || lc->cfg.ratio_den <= 0) { lc->cfg.ratio_num = 4; lc->cfg.ratio_den = 5; }   // best < 0.8 * second
    if (lc->cfg.min_consecutive <= 0) lc->cfg.min_consecutive = 3;
    if (lc->cfg.min_inliers <= 0) lc->cfg.min_inliers = 20;
    if (lc->cfg.err_px <= 0.f) lc->cfg.err_px = 3.0f;
    lc->block_bytes = alva_lc_block_bytes(cfg->n_max);
    lc->npair = cfg->kf_per_step * cfg->world;
    lc->consecutive.assign(cfg->world, 0);
    const size_t np = lc->npair;
    bool ok = cudaMalloc(&lc->nn, np * cfg->n_max * 16) == cudaSuccess && cudaMalloc(&lc->nmatch, np * 4) == cudaSuccess &&
              cudaMalloc(&lc->npairs, np * 4) == cudaSuccess && cudaMalloc(&lc->bvl, np * PAIR_CAP * 24) == cudaSuccess &&
              cudaMalloc(&lc->bvr, np * PAIR_CAP * 24) == cudaSuccess && cudaMalloc(&lc->Rt, np * 96) == cudaSuccess &&
              cudaMalloc(&lc->info, np * 32) == cudaSuccess && cudaMalloc(&lc->res_dev, np * 128) == cudaSuccess &&
              cudaMalloc(&lc->outl, np * PAIR_CAP) == cudaSuccess;
    for (int s = 0; ok && s < alva_lc::NSLOT; s++)
        ok = cudaHostAlloc((void**)&lc->res_host[s], np * 128, cudaHostAllocDefault) == cudaSuccess &&
             cudaEventCreateWithFlags(&lc->done[s], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) { alva_set_error("alva_lc_create: allocation failed (%s)", cudaGetErrorString(cudaGetLastError())); alva_lc_destroy(lc); return nullptr; }
    cudaMemsetAsync(lc->Rt, 0, np * 96, ctx->stream);
    cudaMemsetAsync(lc->info, 0, np * 32, ctx->stream);
    return lc;
}

// `on`: the context whose stream runs the pack kernel -- the producer of desc / pts (the per-frame context), so that packing never
// queues behind a detection on the detector's own stream; NULL = the detector's context.
extern "C" int alva_lc_pack_on(alva_lc* lc, alva_ctx* on, const uint8_t* desc, const float* pts, const int32_t* counts, int cap,
                               const int32_t* kf_frames, int kf_seq0, const float* K4, uint8_t* send) { AlvaDeviceGuard guard__(lc ? lc->ctx : nullptr);
    if (!lc || !desc || !pts || !counts || !kf_frames || !K4 || !send || cap < 1) { alva_set_error("alva_lc_pack: bad argument"); return ALVA_E_INVALID; }
    alva_ctx* ctx = on ? on : lc->ctx;
    if (ctx->device != lc->ctx->device) { alva_set_error("alva_lc_pack_on: context of another device"); return ALVA_E_INVALID; }
    const int K = lc->cfg.kf_per_step;
    lc_pack_kernel<<<dim3(4, K), 256, 0, ctx->stream>>>(desc, pts, counts, kf_frames, cap, lc->cfg.n_max, lc->cfg.rank, kf_seq0, K4[0], K4[1],
                                                        K4[2], K4[3], send, lc->block_bytes);
    ALVA_LAUNCH_CHECK(ctx);
    lc->step_seq0 = kf_seq0;
    return 0;
}
extern "C" int alva_lc_pack(alva_lc* lc, const uint8_t* desc, const float* pts, const int32_t* counts, int cap, const int32_t* kf_frames,
                            int kf_seq0, const float* K4, uint8_t* send) {
    return alva_lc_pack_on(lc, nullptr, desc, pts, counts, cap, kf_frames, kf_seq0, K4, send);
}

extern "C" int alva_lc_detect(alva_lc* lc, const uint8_t* gathered) { AlvaDeviceGuard guard__(lc ? lc->ctx : nullptr);
    if (!lc || !gathered) { alva_set_error("alva_lc_detect: bad argument"); return ALVA_E_INVALID; }
    if ((int)lc->inflight.size() >= alva_lc::NSLOT) { alva_set_error("alva_lc_detect: %d steps in flight, call alva_lc_poll", alva_lc::NSLOT); return ALVA_E_STATE; }
    const alva_lc_config& c = lc->cfg;
    alva_ctx* ctx = lc->ctx;
    const int K = c.kf_per_step, W = c.world;
    if (int e = alva_knn2_blockpair_launch(ctx, gathered, lc->block_bytes, c.n_max, K, W, c.rank, HDR, lc->nn)) return e;
    lc_score_kernel<<<dim3(W, K), 256, 0, ctx->stream>>>(gathered, lc->block_bytes, c.n_max, K, c.rank, reinterpret_cast<const int4*>(lc->nn), c.max_dist,
                                                         c.ratio_num, c.ratio_den, c.min_matches, lc->nmatch, lc->npairs, lc->bvl, lc->bvr);
    ALVA_LAUNCH_CHECK(ctx);
    // geometric check of every pair in one batch (count 0 -> immediate failure); intrinsics of the local block for the threshold
    const uint8_t* lb = gathered + (size_t)c.rank * K * lc->block_bytes;
    (void)lb;
    // 32 hypotheses = one round of the RANSAC kernel (100 outlast a pipeline step).  With ~70 %
    // inliers among the putative matches one all-inlier 8-sample turns up in 32 draws 3 times out of 4; a miss only resets the
    // temporal counter of that stream for one keyframe.
    if (int e = alva_k_essential_5pt(ctx, lc->npair, PAIR_CAP, lc->bvl, lc->bvr, lc->npairs, 32, c.err_px, 0, c.fx_hint > 0 ? c.fx_hint : 500.f,
                                     c.fy_hint > 0 ? c.fy_hint : 500.f, 12345u, lc->Rt, lc->outl, lc->info))
        return e;
    lc_collect_kernel<<<(lc->npair + 127) / 128, 128, 0, ctx->stream>>>(gathered, lc->block_bytes, K, W, c.rank, c.n_max, c.min_matches, lc->nmatch,
                                                                          lc->info, lc->Rt, lc->res_dev);
    ALVA_LAUNCH_CHECK(ctx);
    const int slot = lc->next_slot;
    ALVA_CUDA(cudaMemcpyAsync(lc->res_host[slot], lc->res_dev, (size_t)lc->npair * 128, cudaMemcpyDeviceToHost, ctx->stream));
    ALVA_CUDA(cudaEventRecord(lc->done[slot], ctx->stream));
    lc->local_seq0[slot] = lc->step_seq0;
    lc->inflight.push_back(slot);
    lc->next_slot = (slot + 1) % alva_lc::NSLOT;
    return 0;
}

// Finished steps are consumed in order.  wait != 0: block until every step in flight has finished.  Returns the number of
// events written (<= cap); events that did not fit stay queued.
extern "C" int alva_lc_poll(alva_lc* lc, alva_lc_event* out, int cap, int wait) { AlvaDeviceGuard guard__(lc ? lc->ctx : nullptr);
    if (!lc || (cap > 0 && !out)) { alva_set_error("alva_lc_poll: bad argument"); return ALVA_E_INVALID; }
    const alva_lc_config& c = lc->cfg;
    while (!lc->inflight.empty()) {
        const int slot = lc->inflight.front();
        if (wait) ALVA_CUDA(cudaEventSynchronize(lc->done[slot]));
        else {
            const cudaError_t q = cudaEventQuery(lc->done[slot]);
            if (q == cudaErrorNotReady) break;
            if (q != cudaSuccess) { alva_set_error("alva_lc_poll: %s", cudaGetErrorString(q)); return ALVA_E_CUDA; }
        }
        lc->inflight.pop_front();
        const double* res = lc->res_host[slot];
        for (int e = 0; e < c.kf_per_step; e++)
            for (int r = 0; r < c.world; r++) {
                if (r == c.rank) continue;
                const double* o = res + (size_t)(e * c.world + r) * 16;
                // streak of keyframe events with enough ratio-tested matches; on the newest keyframe of a step the geometric check
                // ran as well and must have passed -- a loop is reported there, once the streak is long enough
                const bool checked = e == c.kf_per_step - 1;
                const bool pass = checked ? (o[1] == 1.0 && (int)o[2] >= c.min_inliers) : o[1] == 2.0;
                lc->consecutive[r] = pass ? lc->consecutive[r] + 1 : 0;
                if (pass && checked && lc->consecutive[r] >= c.min_consecutive) {
                    alva_lc_event ev{};
                    ev.local_kf = lc->local_seq0[slot] + e; ev.remote_rank = r; ev.remote_kf = (int)o[3];
                    ev.n_matches = (int)o[0]; ev.n_inliers = (int)o[2]; ev.consecutive = lc->consecutive[r];
                    for (int i = 0; i < 12; i++) ev.Rt[i] = o[4 + i];
                    lc->ready.push_back(ev);
                }
            }
    }
    int n = 0;
    while (n < cap && !lc->ready.empty()) { out[n++] = lc->ready.front(); lc->ready.pop_front(); }
    return n;
}

extern "C" int alva_lc_inflight(const alva_lc* lc) { return lc ? (int)lc->inflight.size() : ALVA_E_INVALID; }

// per-pair numbers of the most recently finished step (tests / diagnostics): out [K][world][4] = matches, success, inliers, remote kf
extern "C" int alva_lc_last_scores(alva_lc* lc, double* out) { AlvaDeviceGuard guard__(lc ? lc->ctx : nullptr);
    if (!lc || !out) return ALVA_E_INVALID;
    ALVA_CUDA(cudaStreamSynchronize(lc->ctx->stream));
    std::vector<double> h((size_t)lc->npair * 16);
    ALVA_CUDA(cudaMemcpy(h.data(), lc->res_dev, h.size() * 8, cudaMemcpyDeviceToHost));
    for (int p = 0; p < lc->npair; p++) for (int i = 0; i < 4; i++) out[4 * p + i] = h[(size_t)p * 16 + i];
    return 0;
}

// the 2-NN lists, geometric-check sizes and bearing vectors of the last step (tests / diagnostics); any output may be NULL
extern "C" int alva_lc_last_matches(alva_lc* lc, int32_t* nn, int32_t* npair, double* bv_local, double* bv_remote) {
    AlvaDeviceGuard guard__(lc ? lc->ctx : nullptr);
    if (!lc) return ALVA_E_INVALID;
    const size_t np = lc->npair;
    ALVA_CUDA(cudaStreamSynchronize(lc->ctx->stream));
    if (nn) ALVA_CUDA(cudaMemcpy(nn, lc->nn, np * lc->cfg.n_max * 16, cudaMemcpyDeviceToHost));
    if (npair) ALVA_CUDA(cudaMemcpy(npair, lc->npairs, np * 4, cudaMemcpyDeviceToHost));
    if (bv_local) ALVA_CUDA(cudaMemcpy(bv_local, lc->bvl, np * PAIR_CAP * 24, cudaMemcpyDeviceToHost));
    if (bv_remote) ALVA_CUDA(cudaMemcpy(bv_remote, lc->bvr, np * PAIR_CAP * 24, cudaMemcpyDeviceToHost));
    return 0;
}
