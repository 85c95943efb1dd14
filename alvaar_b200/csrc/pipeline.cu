// pipeline.cu -- the per-frame hot path as ONE object: a batch of RGBA frames goes through
//   gray + Gaussian pyramid + FAST-9/NMS  ->  retainBest(nfeatures)  ->  ORB (blur + IC angle + rBRIEF-256)
//   ->  brute-force Hamming 2-NN against the local map's descriptors  ->  (every kf_interval-th frame) local BA
// with every intermediate resident in HBM and no host synchronisation inside a step.  This is what the reference does
// per frame / per keyframe on the CPU (SURVEY.md 3.2: System::findCameraPose -> VisualFrontend::track ->
// MapManager::createKeyframe -> Mapper::matchingToLocalMap -> Optimizer::localBA), restated for the north-star
// feature front end; `System` (system.cu) drives it one frame at a time, bench.py drives it in batches.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include <algorithm>
#include <map>
#include <tuple>
#include <vector>

// stage entry points implemented in the other translation units
extern "C" int alva_k_hamming_knn2_batch(alva_ctx*, const uint8_t* q, const int32_t* counts, int nbatch, int qcap,
                                         const uint8_t* t, int nt, int32_t* out);

namespace {

// grid-stride over the slots: a pre-selection list's capacity (the NMS bound of the frame) is far larger than its live count
__global__ void keys_to_points_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ counts, int cap,
                                      float* __restrict__ pts, int live_only) {
    const int f = blockIdx.y;
    const int n = min(counts[f], cap);
    const int end = live_only ? n : cap;   // large pre-selection lists: dead slots are never read
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < end; i += gridDim.x * blockDim.x) {
        float2 p = make_float2(0.f, 0.f);
        if (i < n) {
            const uint32_t k = keys[(size_t)f * cap + i];
            p = make_float2((float)ALVA_KEY_X(k), (float)ALVA_KEY_Y(k));
        }
        reinterpret_cast<float2*>(pts)[(size_t)f * cap + i] = p;
    }
}

static unsigned points_blocks(int cap) { return (unsigned)std::min((cap + 127) / 128, 32); }

__global__ void clamp_counts_kernel(int32_t* counts, int n, int cap) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) counts[i] = min(counts[i], cap);
}

}  // namespace

struct alva_pipeline {
    alva_ctx* ctx = nullptr;
    alva_pipeline_config cfg{};
    int w1, h1, w2, h2, w3, h3;
    int kcap = 0;       // raw FAST corners per frame: the NMS bound, so that none is ever dropped
    int fcap = 0;       // selected features per frame (slots)
    int nprob = 0;      // BA problems per step
    // device buffers
    uint8_t *l0 = nullptr, *l1 = nullptr, *l2 = nullptr, *l3 = nullptr, *blur = nullptr;
    int16_t *d0 = nullptr, *d1 = nullptr, *d2 = nullptr, *d3 = nullptr;   // Scharr derivative levels (cfg.derivatives)
    uint32_t *keys = nullptr, *sel = nullptr, *keys2 = nullptr;   // keys2 / counts2 / pts2 / resp2: ALVA_ORB_HARRIS pre-selection
    int32_t* counts2 = nullptr;
    float *pts2 = nullptr, *resp2 = nullptr;
    int32_t *counts = nullptr, *selcounts = nullptr;
    float *pts = nullptr, *angles = nullptr;
    uint8_t *desc = nullptr, *kept = nullptr, *map = nullptr;
    int32_t* matches = nullptr;
    // BA batch: pristine copies + working copies
    double *ba_calib = nullptr, *ba_poses0 = nullptr, *ba_poses = nullptr, *ba_invd0 = nullptr, *ba_invd = nullptr,
           *ba_anch_uv = nullptr, *ba_obs_uv = nullptr, *ba_summary = nullptr;
    uint8_t* ba_const = nullptr;
    int32_t *ba_anch_kf = nullptr, *ba_obs_kf = nullptr, *ba_obs_lm = nullptr;
    bool have_map = false, have_ba = false;
    // host-step staging
    // two staging slots: the upload of one submission overlaps the compute of the previous one (alva_pipeline_submit_host)
    static constexpr int NSLOT = 2;
    uint8_t* in_dev[NSLOT] = {nullptr, nullptr};
    static constexpr int NCHUNK = 4;
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t chunk_ev[NSLOT][NCHUNK] = {}, free_ev[NSLOT] = {}, done_ev[NSLOT] = {};
    bool slot_used[NSLOT] = {false, false};
    int next_slot = 0, outstanding = 0, oldest_slot = 0;
    static constexpr int NEV = 64;      // ring of event pairs around the fused front-end launch
    cudaEvent_t ev0[NEV] = {}, ev1[NEV] = {};
    // local BA runs beside the per-frame stages on its own (high-priority) stream, as the reference architecture's mapper
    // does beside the tracker: forked from / joined back into ctx->stream with events, so callers still see one stream
    // feature selection (retainBest / Harris / retainBest: small, latency-bound kernels) runs on a second stream beside the
    // pyramid, derivative and blur kernels, which do not depend on it; joined before the descriptors
    alva_ctx* sel_ctx = nullptr;
    cudaStream_t sel_stream = nullptr;
    cudaEvent_t sel_fork = nullptr, sel_join = nullptr, pyr_join = nullptr;
    // BA slots.  Slot 0: the step's BA is joined at the end of the SAME step and works in place on the public buffers
    // (ba_poses / ba_invd / ba_summary).  Slots 1, 2 ("pipeline_ba_lag" = 1): the chain of step s is joined at the end of step
    // s + 1, two chains in flight on two streams -- a chain is ~60 dependent, latency-bound launches that use a few percent of
    // the GPU but take longer than the frame stages of a step, so in-step joining makes it the critical path; the mapper of the
    // reference delivers its results asynchronously in the same way.  These slots solve in private buffers and the joined
    // result is copied to the public ones (alva_pipeline_drain joins what is still in flight).
    static constexpr int NBA = 3;
    alva_ctx* ba_ctx[NBA] = {nullptr, nullptr, nullptr};
    cudaStream_t ba_stream[NBA] = {nullptr, nullptr, nullptr};
    cudaEvent_t ba_fork[NBA] = {nullptr, nullptr, nullptr}, ba_join[NBA] = {nullptr, nullptr, nullptr};
    bool ba_forked[NBA] = {false, false, false};
    double *ba_wposes[NBA] = {nullptr, nullptr, nullptr}, *ba_winvd[NBA] = {nullptr, nullptr, nullptr}, *ba_wsummary[NBA] = {nullptr, nullptr, nullptr};
    int ba_last = -1;          // slot forked most recently (-1: none in flight or joined)
    long long ba_forks = 0;    // lagged forks so far (parity picks the slot)
    bool profile = false;
    long long step_index = 0;
    std::vector<void*> allocs;
    // CUDA graphs: the per-frame stages of a frame range (keyed by input pointer and range: the kernel arguments are baked in) and
    // the step's local-BA chain are each captured after a first direct run has sized every scratch buffer, and replayed with one
    // launch (~60 + ~50 dependent launches per step otherwise).  A graph also bakes in the workspaces of the contexts its kernels
    // run on (ctx / sel_ctx for a frame range, ba_ctx[k] for BA slot k) and the kernel variants the options chose.  Any call on
    // those contexts may grow a workspace and free the old one, and alva_set_option may pick another kernel, so a graph records
    // the contexts' workspace epochs and the options epoch it was captured under and is replayed only while they are current;
    // otherwise it is dropped, the key runs directly again and is captured anew on its next use (a capture thus always follows
    // a direct run under the same workspaces and options, and never has to grow a buffer, which would synchronise the stream
    // and end the capture).  Not used while profiling: a graph cannot carry the per-launch event pairs alva_pipeline_frontend_ms
    // reads.
    struct Epochs {
        uint64_t ws0 = 0, ws1 = 0, opt = 0;
        bool operator==(const Epochs& o) const { return ws0 == o.ws0 && ws1 == o.ws1 && opt == o.opt; }
    };
    struct Graph {
        cudaGraphExec_t exec = nullptr;
        long long launches = 0;
        int runs = 0;     // direct runs under `seen` (capture after the first)
        Epochs seen;      // epochs after the last direct run or capture
    };
    std::map<std::tuple<const uint8_t*, int, int>, Graph> frame_graphs;
    Graph ba_graph[NBA];
    bool graphs_failed = false;
    long long graph_replays = 0;
    long long graphs_captured = 0;   // cumulative: a re-capture after a workspace or option change counts again
};

static int palloc(alva_pipeline* p, void** ptr, size_t bytes) {
    cudaError_t e = cudaMalloc(ptr, bytes ? bytes : 16);
    if (e != cudaSuccess) { alva_set_error("pipeline cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e)); return ALVA_E_CUDA; }
    p->allocs.push_back(*ptr);
    return 0;
}
#define PALLOC(field, bytes) do { if (int e_ = palloc(p, (void**)&p->field, (bytes))) { alva_pipeline_destroy(p); return nullptr; } } while (0)

extern "C" void alva_pipeline_destroy(alva_pipeline* p) {
    if (!p) return;
    AlvaDeviceGuard guard__(p->ctx);
    cudaStreamSynchronize(p->ctx->stream);
    for (auto& kv : p->frame_graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    for (int k = 0; k < alva_pipeline::NBA; k++) {
        if (p->ba_stream[k]) cudaStreamSynchronize(p->ba_stream[k]);
        if (p->ba_graph[k].exec) cudaGraphExecDestroy(p->ba_graph[k].exec);
    }
    for (void* a : p->allocs) cudaFree(a);
    if (p->sel_ctx) { alva_ctx_destroy(p->sel_ctx); p->sel_ctx = nullptr; }
    if (p->sel_stream) { cudaStreamSynchronize(p->sel_stream); cudaStreamDestroy(p->sel_stream); }
    if (p->sel_fork) cudaEventDestroy(p->sel_fork);
    if (p->sel_join) cudaEventDestroy(p->sel_join);
    if (p->pyr_join) cudaEventDestroy(p->pyr_join);
    for (int k = 0; k < alva_pipeline::NBA; k++) {
        if (p->ba_ctx[k]) { alva_ctx_destroy(p->ba_ctx[k]); p->ba_ctx[k] = nullptr; }
        if (p->ba_stream[k]) { cudaStreamSynchronize(p->ba_stream[k]); cudaStreamDestroy(p->ba_stream[k]); }
        if (p->ba_fork[k]) cudaEventDestroy(p->ba_fork[k]);
        if (p->ba_join[k]) cudaEventDestroy(p->ba_join[k]);
    }
    if (p->copy_stream) {
        cudaStreamSynchronize(p->copy_stream);
        cudaStreamDestroy(p->copy_stream);
        for (int s = 0; s < alva_pipeline::NSLOT; s++) {
            for (int i = 0; i < alva_pipeline::NCHUNK; i++) if (p->chunk_ev[s][i]) cudaEventDestroy(p->chunk_ev[s][i]);
            if (p->free_ev[s]) cudaEventDestroy(p->free_ev[s]);
            if (p->done_ev[s]) cudaEventDestroy(p->done_ev[s]);
        }
    }
    for (int i = 0; i < alva_pipeline::NEV; i++) {
        if (p->ev0[i]) cudaEventDestroy(p->ev0[i]);
        if (p->ev1[i]) cudaEventDestroy(p->ev1[i]);
    }
    delete p;
}

extern "C" alva_pipeline* alva_pipeline_create(alva_ctx* ctx, const alva_pipeline_config* cfg) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !cfg || cfg->batch < 1 || cfg->w < 64 || cfg->h < 64 || cfg->w > ALVA_MAX_DIM || cfg->h > ALVA_MAX_DIM ||
        cfg->nfeatures < 1 || cfg->map_size < 0 || cfg->kf_interval < 0) {
        alva_set_error("alva_pipeline_create: bad configuration");
        return nullptr;
    }
    alva_pipeline* p = new alva_pipeline();
    p->ctx = ctx;
    p->cfg = *cfg;
    const int w = cfg->w, h = cfg->h, B = cfg->batch;
    p->w1 = (w + 1) / 2; p->h1 = (h + 1) / 2; p->w2 = (p->w1 + 1) / 2; p->h2 = (p->h1 + 1) / 2;
    p->w3 = (p->w2 + 1) / 2; p->h3 = (p->h2 + 1) / 2;
    p->fcap = ((cfg->nfeatures + cfg->nfeatures / 2 + 63) / 64) * 64;   // retainBest keeps ties: 1.5x head-room
    // FAST's 3x3 NMS is strict, so no two corners are neighbours: at most one per 2x2 block.  Every corner of a frame fits.
    p->kcap = ((w + 1) / 2) * ((h + 1) / 2);
    p->nprob = cfg->kf_interval > 0 ? (B + cfg->kf_interval - 1) / cfg->kf_interval : 0;
    PALLOC(l0, (size_t)B * w * h); PALLOC(l1, (size_t)B * p->w1 * p->h1); PALLOC(l2, (size_t)B * p->w2 * p->h2);
    PALLOC(l3, (size_t)B * p->w3 * p->h3); PALLOC(blur, (size_t)B * w * h);
    if (cfg->derivatives) {
        PALLOC(d0, (size_t)B * w * h * 4); PALLOC(d1, (size_t)B * p->w1 * p->h1 * 4);
        PALLOC(d2, (size_t)B * p->w2 * p->h2 * 4); PALLOC(d3, (size_t)B * p->w3 * p->h3 * 4);
    }
    PALLOC(keys, (size_t)B * p->kcap * 4); PALLOC(counts, (size_t)B * 4);
    PALLOC(sel, (size_t)B * p->fcap * 4); PALLOC(selcounts, (size_t)B * 4);
    if (cfg->orb_flags & ALVA_ORB_HARRIS) {
        PALLOC(keys2, (size_t)B * p->kcap * 4); PALLOC(counts2, (size_t)B * 4);
        PALLOC(pts2, (size_t)B * p->kcap * 8); PALLOC(resp2, (size_t)B * p->kcap * 4);
    }
    PALLOC(pts, (size_t)B * p->fcap * 8); PALLOC(angles, (size_t)B * p->fcap * 4);
    PALLOC(desc, (size_t)B * p->fcap * 32); PALLOC(kept, (size_t)B * p->fcap);
    PALLOC(matches, (size_t)B * p->fcap * 16);
    PALLOC(map, (size_t)(cfg->map_size > 0 ? cfg->map_size : 1) * 32);
    if (p->nprob > 0) {
        const size_t np = p->nprob, nkf = cfg->ba_nkf, nlm = cfg->ba_nlm, nobs = cfg->ba_nobs;
        if (nkf < 1 || nlm < 1 || nobs < 1) { alva_set_error("alva_pipeline_create: BA dimensions missing"); alva_pipeline_destroy(p); return nullptr; }
        PALLOC(ba_calib, np * 4 * 8); PALLOC(ba_poses0, np * nkf * 7 * 8); PALLOC(ba_poses, np * nkf * 7 * 8);
        PALLOC(ba_invd0, np * nlm * 8); PALLOC(ba_invd, np * nlm * 8); PALLOC(ba_anch_uv, np * nlm * 16);
        PALLOC(ba_obs_uv, np * nobs * 16); PALLOC(ba_summary, np * 8 * 8); PALLOC(ba_const, np * nkf);
        PALLOC(ba_anch_kf, np * nlm * 4); PALLOC(ba_obs_kf, np * nobs * 4); PALLOC(ba_obs_lm, np * nobs * 4);
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        for (int k = 0; k < alva_pipeline::NBA; k++) {
            if (cudaStreamCreateWithPriority(&p->ba_stream[k], cudaStreamNonBlocking, hi) != cudaSuccess ||
                cudaEventCreateWithFlags(&p->ba_fork[k], cudaEventDisableTiming) != cudaSuccess ||
                cudaEventCreateWithFlags(&p->ba_join[k], cudaEventDisableTiming) != cudaSuccess ||
                !(p->ba_ctx[k] = alva_ctx_create(ctx->device, (void*)p->ba_stream[k]))) {
                alva_set_error("alva_pipeline_create: BA stream setup failed");
                alva_pipeline_destroy(p);
                return nullptr;
            }
            if (k == 0) { p->ba_wposes[0] = p->ba_poses; p->ba_winvd[0] = p->ba_invd; p->ba_wsummary[0] = p->ba_summary; }
            else { PALLOC(ba_wposes[k], np * nkf * 7 * 8); PALLOC(ba_winvd[k], np * nlm * 8); PALLOC(ba_wsummary[k], np * 8 * 8); }
        }
    }
    if (cudaStreamCreateWithFlags(&p->sel_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&p->sel_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&p->sel_join, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&p->pyr_join, cudaEventDisableTiming) != cudaSuccess ||
        !(p->sel_ctx = alva_ctx_create(ctx->device, (void*)p->sel_stream))) {
        alva_set_error("alva_pipeline_create: selection stream setup failed");
        alva_pipeline_destroy(p);
        return nullptr;
    }
    for (int i = 0; i < alva_pipeline::NEV; i++)
        if (cudaEventCreate(&p->ev0[i]) != cudaSuccess || cudaEventCreate(&p->ev1[i]) != cudaSuccess) {
            alva_set_error("cudaEventCreate failed");
            alva_pipeline_destroy(p);
            return nullptr;
        }
    return p;
}

extern "C" int alva_pipeline_set_map(alva_pipeline* p, const uint8_t* desc_host, int n) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p || !desc_host || n != p->cfg.map_size) { alva_set_error("alva_pipeline_set_map: need exactly map_size descriptors"); return ALVA_E_INVALID; }
    ALVA_CUDA(cudaMemcpyAsync(p->map, desc_host, (size_t)n * 32, cudaMemcpyHostToDevice, p->ctx->stream));
    ALVA_CUDA(cudaStreamSynchronize(p->ctx->stream));
    p->have_map = true;
    return 0;
}

// One BA problem (host arrays, layout of alva_k_ba_solve) replicated into slot `slot` of the per-step BA batch.
extern "C" int alva_pipeline_set_ba(alva_pipeline* p, int slot, const double* calib, const double* poses, const uint8_t* pose_const,
                                    const double* invd, const int32_t* anch_kf, const double* anch_uv, const int32_t* obs_kf,
                                    const int32_t* obs_lm, const double* obs_uv) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p || slot < 0 || slot >= p->nprob) { alva_set_error("alva_pipeline_set_ba: bad slot"); return ALVA_E_INVALID; }
    const size_t nkf = p->cfg.ba_nkf, nlm = p->cfg.ba_nlm, nobs = p->cfg.ba_nobs, s = slot;
    cudaStream_t st = p->ctx->stream;
    ALVA_CUDA(cudaMemcpyAsync(p->ba_calib + 4 * s, calib, 32, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_poses0 + nkf * 7 * s, poses, nkf * 56, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_const + nkf * s, pose_const, nkf, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_invd0 + nlm * s, invd, nlm * 8, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_anch_kf + nlm * s, anch_kf, nlm * 4, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_anch_uv + 2 * nlm * s, anch_uv, nlm * 16, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_obs_kf + nobs * s, obs_kf, nobs * 4, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_obs_lm + nobs * s, obs_lm, nobs * 4, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_obs_uv + 2 * nobs * s, obs_uv, nobs * 16, cudaMemcpyHostToDevice, st));
    ALVA_CUDA(cudaStreamSynchronize(st));
    if (slot == p->nprob - 1) p->have_ba = true;
    return 0;
}

extern "C" int alva_pipeline_profile(alva_pipeline* p, int enable) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p) return ALVA_E_INVALID;
    p->profile = enable != 0;
    p->step_index = 0;
    return 0;
}

// Durations (ms) of the fused front-end launch (gray + pyramid L1 + FAST) of the last min(n, steps, 64) steps since
// profiling was enabled, measured with CUDA events on the launch stream.  Returns how many were written.
extern "C" int alva_pipeline_frontend_ms(alva_pipeline* p, float* ms, int n) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p || !ms || !p->profile) { alva_set_error("profiling not enabled"); return ALVA_E_STATE; }
    ALVA_CUDA(cudaStreamSynchronize(p->ctx->stream));
    const long long have = p->step_index < alva_pipeline::NEV ? p->step_index : alva_pipeline::NEV;
    const int m = n < have ? n : (int)have;
    for (int i = 0; i < m; i++) {
        const int slot = (int)((p->step_index - 1 - i) % alva_pipeline::NEV);
        ALVA_CUDA(cudaEventElapsedTime(&ms[i], p->ev0[slot], p->ev1[slot]));
    }
    return m;
}

// defined in frontend.cu: the fused launch alone (so the events bracket exactly the dominant kernel)
int alva_harris_launch(alva_ctx* ctx, const uint8_t* gray, int w, int h, int nframes, const float* pts, const int32_t* npts_per_frame,
                       int npts, float* resp, int zero_dead);
int alva_scharr_levels_launch(alva_ctx* ctx, int nlev, const uint8_t* const* src, int16_t* const* dst, const int* w, const int* h,
                              int nframes);
int alva_retain_best_f32_launch(alva_ctx* ctx, const float* pts, const float* resp, const int32_t* counts, int cap, int nframes,
                                int n_keep, float* pts_out, const uint32_t* keys_in, uint32_t* keys_out, int32_t* out_counts,
                                int out_cap);
int alva_frontend_main_launch(alva_ctx* ctx, const uint8_t* rgba, int w, int h, int nframes, uint8_t* l0, uint8_t* l1, int thr,
                              uint32_t* keys, int32_t* counts, int cap);

// Stages 1-4 on frames [f0, f0 + nf) of the batch (every buffer is frame-major, so a range is a pointer offset).
static int pipeline_ba_fork(alva_pipeline* p);

static int pipeline_frames(alva_pipeline* p, const uint8_t* rgba_dev, int f0, int nf, bool timed, bool fork_ba) {
    alva_ctx* ctx = p->ctx;
    const alva_pipeline_config& c = p->cfg;
    const int w = c.w, h = c.h;
    cudaStream_t st = ctx->stream;
    const size_t F = (size_t)f0;
    uint8_t *l0 = p->l0 + F * w * h, *l1 = p->l1 + F * p->w1 * p->h1, *l2 = p->l2 + F * p->w2 * p->h2, *l3 = p->l3 + F * p->w3 * p->h3;
    uint8_t* blur = p->blur + F * w * h;
    uint32_t *keys = p->keys + F * p->kcap, *sel = p->sel + F * p->fcap;
    int32_t *counts = p->counts + F, *selcounts = p->selcounts + F;
    // 1. fused front end (+ pyramid levels 2, 3)
    ALVA_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * nf, st));
    const int slot = (int)(p->step_index % alva_pipeline::NEV);
    if (timed && p->profile) ALVA_CUDA(cudaEventRecord(p->ev0[slot], st));
    if (int e = alva_frontend_main_launch(ctx, rgba_dev + F * w * h * 4, w, h, nf, l0, l1, c.fast_thr, keys, counts, p->kcap)) return e;
    if (timed && p->profile) { ALVA_CUDA(cudaEventRecord(p->ev1[slot], st)); p->step_index++; }
    // the step's local BA starts here, beside everything below (after the front end so that the event pair above times
    // that kernel alone)
    if (fork_ba) if (int e = pipeline_ba_fork(p)) return e;
    // 2. feature selection inside ORB's 31-px border, row-major -- on the selection stream
    alva_ctx* sc = p->sel_ctx;
    cudaStream_t ss = p->sel_stream;
    const long long sel_before = sc->launches;
    ALVA_CUDA(cudaEventRecord(p->sel_fork, st));
    ALVA_CUDA(cudaStreamWaitEvent(ss, p->sel_fork, 0));
    if (c.orb_flags & ALVA_ORB_HARRIS) {
        // ORB::detectAndCompute's own rule (orb.cpp:855-925): retainBest(2n) on the FAST score, Harris response of the
        // survivors, retainBest(n) on that
        uint32_t* keys2 = p->keys2 + F * p->kcap;
        int32_t* counts2 = p->counts2 + F;
        float *pts2 = p->pts2 + F * p->kcap * 2, *resp2 = p->resp2 + F * p->kcap;
        if (int e = alva_k_retain_best(sc, keys, counts, p->kcap, nf, w, h, 2 * c.nfeatures, 31, keys2, counts2, p->kcap)) return e;
        keys_to_points_kernel<<<dim3(points_blocks(p->kcap), nf), 128, 0, ss>>>(keys2, counts2, p->kcap, pts2, 1);
        ALVA_LAUNCH_CHECK(sc);
        if (int e = alva_harris_launch(sc, l0, w, h, nf, pts2, counts2, p->kcap, resp2, 0)) return e;
        if (int e = alva_retain_best_f32_launch(sc, pts2, resp2, counts2, p->kcap, nf, c.nfeatures, p->pts + F * p->fcap * 2, keys2, sel,
                                                selcounts, p->fcap))
            return e;
        clamp_counts_kernel<<<(nf + 127) / 128, 128, 0, ss>>>(selcounts, nf, p->fcap);
        ALVA_LAUNCH_CHECK(sc);
    } else {
        // retainBest keeps ties, so more than fcap can survive: the call keeps the first fcap of them in row-major order
        if (int e = alva_k_retain_best(sc, keys, counts, p->kcap, nf, w, h, c.nfeatures, 31, sel, selcounts, p->fcap)) return e;
        keys_to_points_kernel<<<dim3(points_blocks(p->fcap), nf), 128, 0, ss>>>(sel, selcounts, p->fcap, p->pts + F * p->fcap * 2, 0);
        ALVA_LAUNCH_CHECK(sc);
    }
    ALVA_CUDA(cudaEventRecord(p->sel_join, ss));
    // 1b. rest of the pyramid + derivative levels: bandwidth-bound, nothing in this step reads them, so they follow the
    // selection on the side stream and overlap the ALU-bound descriptor / matching kernels on the main stream
    if (int e = alva_k_pyrdown(sc, l1, l2, p->w1, p->h1, nf)) return e;
    if (int e = alva_k_pyrdown(sc, l2, l3, p->w2, p->h2, nf)) return e;
    if (c.derivatives) {   // the derivative pyramid the KLT tracker reads (buildOpticalFlowPyramid withDerivatives)
        const uint8_t* srcs[4] = {l0, l1, l2, l3};
        int16_t* dsts[4] = {p->d0 + F * w * h * 2, p->d1 + F * p->w1 * p->h1 * 2, p->d2 + F * p->w2 * p->h2 * 2,
                            p->d3 + F * p->w3 * p->h3 * 2};
        const int ws[4] = {w, p->w1, p->w2, p->w3}, hs[4] = {h, p->h1, p->h2, p->h3};
        if (int e = alva_scharr_levels_launch(sc, 4, srcs, dsts, ws, hs, nf)) return e;
    }
    ALVA_CUDA(cudaEventRecord(p->pyr_join, ss));
    ctx->launches += sc->launches - sel_before;
    // 3. ORB
    if (int e = alva_k_orb_blur(ctx, l0, blur, w, h, nf, c.orb_flags & ALVA_ORB_FMA)) return e;
    ALVA_CUDA(cudaStreamWaitEvent(st, p->sel_join, 0));
    if (int e = alva_k_orb_describe(ctx, l0, blur, w, h, nf, p->pts + F * p->fcap * 2, selcounts, p->fcap, c.orb_flags,
                                    p->desc + F * p->fcap * 32, p->kept + F * p->fcap, p->angles + F * p->fcap))
        return e;
    // 4. match against the local map
    if (c.map_size > 0)
        if (int e = alva_k_hamming_knn2_batch(ctx, p->desc + F * p->fcap * 32, selcounts, nf, p->fcap, p->map, c.map_size,
                                              p->matches + F * p->fcap * 4))
            return e;
    ALVA_CUDA(cudaStreamWaitEvent(st, p->pyr_join, 0));   // the step is complete only with its pyramid
    return 0;
}

// 5. local BA for this step's keyframes.  Forked at the start of the step onto the BA stream (its inputs do not depend on
// this step's frames), joined at the end: small dependent launches (1 CTA per problem in the factorisation) that would
// otherwise leave most SMs idle overlap the wide per-frame kernels.
extern int alva_g_ba_overlap;   // alva_set_option("pipeline_ba_overlap", 0): run BA after the frame stages instead (A/B measurement)
int alva_g_ba_lag = 0;          // alva_set_option("pipeline_ba_lag", 1): join a step's BA at the end of the NEXT step (two chains in flight)

int alva_g_pipeline_graphs = 1;   // alva_set_option("pipeline_graphs", 0): always launch kernel by kernel

static bool graphs_on(const alva_pipeline* p) { return alva_g_pipeline_graphs && !p->profile && !p->graphs_failed; }

// capture what `body` enqueues on `st` (and on streams it forks to and joins back from) into an executable graph
template <class F>
static bool capture_graph(alva_pipeline* p, cudaStream_t st, alva_pipeline::Graph& out, F&& body) {
    cudaGraph_t g = nullptr;
    const long long l0 = p->ctx->launches;
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); return false; }
    const int e = body();
    const cudaError_t ce = cudaStreamEndCapture(st, &g);
    const long long n = p->ctx->launches - l0;
    p->ctx->launches = l0;
    bool ok = ce == cudaSuccess && e == 0 && g != nullptr;
    if (ok) ok = cudaGraphInstantiate(&out.exec, g, 0) == cudaSuccess;
    if (g) cudaGraphDestroy(g);
    if (!ok) { cudaGetLastError(); out.exec = nullptr; return false; }
    out.launches = n;
    p->graphs_captured++;
    return true;
}

static alva_pipeline::Epochs epochs_now(const alva_ctx* a, const alva_ctx* b) {
    alva_pipeline::Epochs e;
    e.ws0 = a->ws_epoch;
    e.ws1 = b ? b->ws_epoch : 0;
    e.opt = alva_g_options_epoch;
    return e;
}

// drop a graph (and the direct runs it would be captured after) if a workspace or option it depends on changed since
static void graph_validate(alva_pipeline::Graph& g, const alva_pipeline::Epochs& now) {
    if (g.seen == now) return;
    if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; }   // a launch still in flight completes first
    g.runs = 0;
    g.seen = now;
}

// the BA chain itself, on slot k's stream (pristine copies -> working copies, then the solve)
static int pipeline_ba_body(alva_pipeline* p, int k) {
    const alva_pipeline_config& c = p->cfg;
    cudaStream_t st = p->ba_stream[k];
    const size_t np = p->nprob;
    ALVA_CUDA(cudaMemcpyAsync(p->ba_wposes[k], p->ba_poses0, np * c.ba_nkf * 56, cudaMemcpyDeviceToDevice, st));
    ALVA_CUDA(cudaMemcpyAsync(p->ba_winvd[k], p->ba_invd0, np * c.ba_nlm * 8, cudaMemcpyDeviceToDevice, st));
    const long long before = p->ba_ctx[k]->launches;
    const int e = alva_k_ba_solve(p->ba_ctx[k], p->nprob, c.ba_nkf, c.ba_nlm, c.ba_nobs, p->ba_calib, p->ba_wposes[k], p->ba_const,
                                  p->ba_winvd[k], p->ba_anch_kf, p->ba_anch_uv, p->ba_obs_kf, p->ba_obs_lm, p->ba_obs_uv, c.ba_huber,
                                  c.ba_max_iter, p->ba_wsummary[k]);
    p->ctx->launches += p->ba_ctx[k]->launches - before;   // one launch counter per pipeline (alva_ctx_launches)
    return e;
}

static int pipeline_ba_launch(alva_pipeline* p, int k) {
    cudaStream_t st = p->ba_stream[k];
    ALVA_CUDA(cudaEventRecord(p->ba_fork[k], p->ctx->stream));
    ALVA_CUDA(cudaStreamWaitEvent(st, p->ba_fork[k], 0));
    p->ba_forked[k] = true;
    p->ba_last = k;
    if (!graphs_on(p)) return pipeline_ba_body(p, k);
    alva_pipeline::Graph& g = p->ba_graph[k];
    graph_validate(g, epochs_now(p->ba_ctx[k], nullptr));
    if (!g.exec && g.runs >= 1 && !capture_graph(p, st, g, [&] { return pipeline_ba_body(p, k); }))
        p->graphs_failed = true;
    if (g.exec) {
        ALVA_CUDA(cudaGraphLaunch(g.exec, st));
        p->ctx->launches += g.launches;
        p->graph_replays++;
        return 0;
    }
    g.runs++;
    const int e = pipeline_ba_body(p, k);
    g.seen = epochs_now(p->ba_ctx[k], nullptr);   // what the run grew is what a capture will bake in
    return e;
}

// main stream waits for slot k's chain; a lagged slot's results go to the public buffers
static int pipeline_ba_join_slot(alva_pipeline* p, int k) {
    if (!p->ba_forked[k]) return 0;
    p->ba_forked[k] = false;
    if (p->ba_last == k) p->ba_last = -1;
    cudaStream_t st = p->ctx->stream;
    ALVA_CUDA(cudaEventRecord(p->ba_join[k], p->ba_stream[k]));
    ALVA_CUDA(cudaStreamWaitEvent(st, p->ba_join[k], 0));
    if (k != 0) {
        const alva_pipeline_config& c = p->cfg;
        const size_t np = p->nprob;
        ALVA_CUDA(cudaMemcpyAsync(p->ba_poses, p->ba_wposes[k], np * c.ba_nkf * 56, cudaMemcpyDeviceToDevice, st));
        ALVA_CUDA(cudaMemcpyAsync(p->ba_invd, p->ba_winvd[k], np * c.ba_nlm * 8, cudaMemcpyDeviceToDevice, st));
        ALVA_CUDA(cudaMemcpyAsync(p->ba_summary, p->ba_wsummary[k], np * 64, cudaMemcpyDeviceToDevice, st));
    }
    return 0;
}

static bool ba_lagged() { return alva_g_ba_overlap && alva_g_ba_lag; }

static int pipeline_ba_fork(alva_pipeline* p) {
    if (p->nprob <= 0 || !alva_g_ba_overlap) return 0;
    if (!ba_lagged()) {
        for (int k = 1; k < alva_pipeline::NBA; k++) if (int e = pipeline_ba_join_slot(p, k)) return e;   // mode switched
        return pipeline_ba_launch(p, 0);
    }
    if (int e = pipeline_ba_join_slot(p, 0)) return e;
    const int k = 1 + (int)(p->ba_forks++ & 1);
    if (int e = pipeline_ba_join_slot(p, k)) return e;   // (joined a step ago in the steady state)
    return pipeline_ba_launch(p, k);
}

// end of a step: same-step mode joins the step's own chain; lagged mode joins the PREVIOUS step's
static int pipeline_ba_join(alva_pipeline* p) {
    if (p->nprob > 0 && !alva_g_ba_overlap && !p->ba_forked[0])
        if (int e = pipeline_ba_launch(p, 0)) return e;
    if (!ba_lagged()) {
        for (int k = 0; k < alva_pipeline::NBA; k++) if (int e = pipeline_ba_join_slot(p, k)) return e;
        return 0;
    }
    const int cur = p->ba_last;
    for (int k = 0; k < alva_pipeline::NBA; k++)
        if (k != cur) if (int e = pipeline_ba_join_slot(p, k)) return e;
    p->ba_last = cur;
    return 0;
}

// joins every chain still in flight (lagged mode leaves the last step's); the public BA buffers then hold the newest result
extern "C" int alva_pipeline_drain(alva_pipeline* p) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p) { alva_set_error("alva_pipeline_drain: bad argument"); return ALVA_E_INVALID; }
    const int cur = p->ba_last;
    for (int k = 0; k < alva_pipeline::NBA; k++) if (k != cur) if (int e = pipeline_ba_join_slot(p, k)) return e;
    if (cur >= 0) if (int e = pipeline_ba_join_slot(p, cur)) return e;   // the newest last: its copy wins
    return 0;
}

static int pipeline_ready(alva_pipeline* p) {
    if (p->cfg.map_size > 0 && !p->have_map) { alva_set_error("pipeline: local map not set"); return ALVA_E_STATE; }
    if (p->nprob > 0 && !p->have_ba) { alva_set_error("pipeline: BA problems not set"); return ALVA_E_STATE; }
    return 0;
}

// the per-frame stages of frames [f0, f0 + nf): a graph replay when one exists for this (input, range) and the workspaces and
// options it baked in are current, else direct launches (the first direct run of a key sizes the scratch buffers; the next
// call captures)
static int pipeline_frames_auto(alva_pipeline* p, const uint8_t* rgba_dev, int f0, int nf, bool timed, bool fork_ba) {
    if (!graphs_on(p)) return pipeline_frames(p, rgba_dev, f0, nf, timed, fork_ba);
    if (fork_ba) if (int e = pipeline_ba_fork(p)) return e;   // the BA chain is its own graph on its own stream
    alva_pipeline::Graph& g = p->frame_graphs[std::make_tuple(rgba_dev, f0, nf)];
    graph_validate(g, epochs_now(p->ctx, p->sel_ctx));
    if (!g.exec && g.runs >= 1 &&
        !capture_graph(p, p->ctx->stream, g, [&] { return pipeline_frames(p, rgba_dev, f0, nf, false, false); }))
        p->graphs_failed = true;
    if (g.exec) {
        ALVA_CUDA(cudaGraphLaunch(g.exec, p->ctx->stream));
        p->ctx->launches += g.launches;
        p->graph_replays++;
        return 0;
    }
    g.runs++;
    const int e = pipeline_frames(p, rgba_dev, f0, nf, timed, false);
    g.seen = epochs_now(p->ctx, p->sel_ctx);
    return e;
}

extern "C" int alva_pipeline_step_dev(alva_pipeline* p, const uint8_t* rgba_dev) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p || !rgba_dev) { alva_set_error("alva_pipeline_step_dev: bad argument"); return ALVA_E_INVALID; }
    if (int e = pipeline_ready(p)) return e;
    if (int e = pipeline_frames_auto(p, rgba_dev, 0, p->cfg.batch, true, true)) { pipeline_ba_join(p); return e; }
    return pipeline_ba_join(p);
}

// {graphs captured so far (re-captures included), graph launches so far, 1 if a capture failed and the pipeline fell back to
// direct launches}
extern "C" int alva_pipeline_graph_stats(alva_pipeline* p, int32_t* out3) {
    if (!p || !out3) return ALVA_E_INVALID;
    out3[0] = (int32_t)p->graphs_captured; out3[1] = (int32_t)p->graph_replays; out3[2] = p->graphs_failed ? 1 : 0;
    return 0;
}

// Host-buffer step (the e2e leg).  alva_pipeline_submit_host enqueues one batch and returns at once: the batch is uploaded in
// chunks on a dedicated copy stream into one of two staging slots while the compute stream works on the chunks that have
// landed (event-ordered) -- and while the PREVIOUS submission is still computing -- then the per-frame results are copied
// back.  alva_pipeline_wait blocks until the oldest outstanding submission (at most two) has delivered its results.
// alva_pipeline_step_host = submit + wait.
extern "C" int alva_pipeline_submit_host(alva_pipeline* p, const uint8_t* rgba_host, int32_t* nfeat_host, int32_t* matches_host,
                                         double* ba_poses_host, double* ba_summary_host) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p || !rgba_host) { alva_set_error("alva_pipeline_submit_host: bad argument"); return ALVA_E_INVALID; }
    if (int e = pipeline_ready(p)) return e;
    if (p->outstanding >= alva_pipeline::NSLOT) { alva_set_error("alva_pipeline_submit_host: two submissions outstanding, call alva_pipeline_wait"); return ALVA_E_STATE; }
    const alva_pipeline_config& c = p->cfg;
    const size_t frame_bytes = (size_t)c.w * c.h * 4;
    const int slot = p->next_slot;
    if (!p->in_dev[slot]) { if (int e = palloc(p, (void**)&p->in_dev[slot], frame_bytes * c.batch)) return e; }
    if (!p->copy_stream) {
        ALVA_CUDA(cudaStreamCreateWithFlags(&p->copy_stream, cudaStreamNonBlocking));
        for (int s = 0; s < alva_pipeline::NSLOT; s++) {
            for (int i = 0; i < alva_pipeline::NCHUNK; i++) ALVA_CUDA(cudaEventCreateWithFlags(&p->chunk_ev[s][i], cudaEventDisableTiming));
            ALVA_CUDA(cudaEventCreateWithFlags(&p->free_ev[s], cudaEventDisableTiming));
            ALVA_CUDA(cudaEventCreateWithFlags(&p->done_ev[s], cudaEventDisableTiming));
        }
    }
    cudaStream_t st = p->ctx->stream;
    const int nchunk = c.batch >= 4 * alva_pipeline::NCHUNK ? alva_pipeline::NCHUNK : 1;
    const int per = (c.batch + nchunk - 1) / nchunk;
    // the upload may not overwrite frames an earlier submission that used this slot is still reading
    if (p->slot_used[slot]) ALVA_CUDA(cudaStreamWaitEvent(p->copy_stream, p->free_ev[slot], 0));
    for (int i = 0; i < nchunk; i++) {
        const int f0 = i * per, nf = (f0 + per <= c.batch) ? per : c.batch - f0;
        if (nf <= 0) break;
        ALVA_CUDA(cudaMemcpyAsync(p->in_dev[slot] + frame_bytes * f0, rgba_host + frame_bytes * f0, frame_bytes * nf, cudaMemcpyHostToDevice, p->copy_stream));
        ALVA_CUDA(cudaEventRecord(p->chunk_ev[slot][i], p->copy_stream));
    }
    for (int i = 0; i < nchunk; i++) {
        const int f0 = i * per, nf = (f0 + per <= c.batch) ? per : c.batch - f0;
        if (nf <= 0) break;
        ALVA_CUDA(cudaStreamWaitEvent(st, p->chunk_ev[slot][i], 0));
        if (int e = pipeline_frames_auto(p, p->in_dev[slot], f0, nf, false, i == 0)) { pipeline_ba_join(p); return e; }
    }
    if (int e = pipeline_ba_join(p)) return e;
    ALVA_CUDA(cudaEventRecord(p->free_ev[slot], st));   // the staged frames have been consumed
    if (nfeat_host) ALVA_CUDA(cudaMemcpyAsync(nfeat_host, p->selcounts, sizeof(int32_t) * c.batch, cudaMemcpyDeviceToHost, st));
    if (matches_host && c.map_size > 0)
        ALVA_CUDA(cudaMemcpyAsync(matches_host, p->matches, (size_t)c.batch * p->fcap * 16, cudaMemcpyDeviceToHost, st));
    if (p->nprob > 0) {
        if (ba_poses_host) ALVA_CUDA(cudaMemcpyAsync(ba_poses_host, p->ba_poses, (size_t)p->nprob * c.ba_nkf * 56, cudaMemcpyDeviceToHost, st));
        if (ba_summary_host) ALVA_CUDA(cudaMemcpyAsync(ba_summary_host, p->ba_summary, (size_t)p->nprob * 64, cudaMemcpyDeviceToHost, st));
    }
    ALVA_CUDA(cudaEventRecord(p->done_ev[slot], st));
    p->slot_used[slot] = true;
    if (p->outstanding == 0) p->oldest_slot = slot;
    p->outstanding++;
    p->next_slot = (slot + 1) % alva_pipeline::NSLOT;
    return 0;
}

extern "C" int alva_pipeline_wait(alva_pipeline* p) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p) { alva_set_error("alva_pipeline_wait: bad argument"); return ALVA_E_INVALID; }
    if (p->outstanding == 0) return 0;
    ALVA_CUDA(cudaEventSynchronize(p->done_ev[p->oldest_slot]));
    p->outstanding--;
    p->oldest_slot = (p->oldest_slot + 1) % alva_pipeline::NSLOT;
    return 0;
}

extern "C" int alva_pipeline_step_host(alva_pipeline* p, const uint8_t* rgba_host, int32_t* nfeat_host, int32_t* matches_host,
                                       double* ba_poses_host, double* ba_summary_host) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p) { alva_set_error("alva_pipeline_step_host: bad argument"); return ALVA_E_INVALID; }
    while (p->outstanding) if (int e = alva_pipeline_wait(p)) return e;
    if (int e = alva_pipeline_submit_host(p, rgba_host, nfeat_host, matches_host, ba_poses_host, ba_summary_host)) return e;
    return alva_pipeline_wait(p);
}

extern "C" int alva_pipeline_info(const alva_pipeline* p, int32_t* out /* [4]: fcap, kcap, nprob, map_size */) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p || !out) return ALVA_E_INVALID;
    out[0] = p->fcap; out[1] = p->kcap; out[2] = p->nprob; out[3] = p->cfg.map_size;
    return 0;
}

// device pointer of an intermediate (tests): 0 l0, 1 l1, 2 l2, 3 l3, 4 blur, 5 keys, 6 counts, 7 sel, 8 selcounts, 9 pts,
// 10 angles, 11 desc, 12 kept, 13 matches, 14 ba_poses, 15 ba_invd, 16 ba_summary
extern "C" void* alva_pipeline_buffer(alva_pipeline* p, int which) { AlvaDeviceGuard guard__(p ? p->ctx : nullptr);
    if (!p) return nullptr;
    void* t[] = {p->l0, p->l1, p->l2, p->l3, p->blur, p->keys, p->counts, p->sel, p->selcounts, p->pts, p->angles, p->desc,
                 p->kept, p->matches, p->ba_poses, p->ba_invd, p->ba_summary, p->d0, p->d1, p->d2, p->d3};
    return (which >= 0 && which < 21) ? t[which] : nullptr;
}
