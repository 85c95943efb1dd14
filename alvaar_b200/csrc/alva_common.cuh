// alva_common.cuh -- shared device helpers (PTX wrappers for mbarrier / TMA, SWAR byte math) and the
// host-side context for libalva_b200.so.  sm_90a only.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

// ---------------------------------------------------------------- host side
struct alva_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int num_sms = 132;
    long long launches = 0;
    // scratch (grown on demand)
    void* scratch = nullptr;
    size_t scratch_bytes = 0;
    // staging for the host-buffer (alva_h_*) entry points
    void* dev_stage = nullptr;
    size_t dev_stage_bytes = 0;
    // BA: fingerprint of the per-problem pointer table currently resident at the head of `scratch`
    uint64_t ba_table_key = 0;
    void* ba_ws = nullptr;          // BA workspace (own allocation: the table must survive other stages' scratch use)
    size_t ba_ws_bytes = 0;
    void* det_ws = nullptr;         // alva_k_orb_detect's intermediate lists (own allocation, same reason)
    size_t det_ws_bytes = 0;
    void* p3p_tab = nullptr;        // P3P-LMedS sampler table (depends on seed and length only): resident across calls
    int p3p_tab_len = 0;
    uint32_t p3p_tab_seed = 0;
    void* init_tab = nullptr;       // five-point RANSAC sampler table, likewise (the loop-closure detector runs it every step)
    int init_tab_len = 0;
    uint32_t init_tab_seed = 0;
    void* knn_ws = nullptr;         // tensor-core matcher: expanded int8 operand tiles, row map (hamming_mma.cu)
    size_t knn_ws_bytes = 0;
    void* clahe_ws = nullptr;       // alva_k_clahe's per-tile LUTs [frames][tiles_y][tiles_x][256] (clahe.cu)
    size_t clahe_ws_bytes = 0;
    // bumped whenever one of the workspace pointers above changes (a grown buffer frees the old one): a CUDA graph that
    // baked in this context's workspaces is replayed only while the epoch it was captured at is current (pipeline.cu)
    uint64_t ws_epoch = 0;
    // fork / join inside one entry point (BA: the structure kernels run beside the first linearisation).  Created with the
    // context so that nothing is allocated while a caller captures `stream` into a CUDA graph.
    cudaStream_t aux_stream = nullptr;
    cudaEvent_t aux_fork = nullptr, aux_join = nullptr;
};

// Every public entry point runs on the context's device whatever the caller's current device is (two Systems on two GPUs
// driven from one thread; a System driven from a thread that did not create it) and restores the caller's device on exit.
struct AlvaDeviceGuard {
    int prev = -1;
    bool switched = false;
    explicit AlvaDeviceGuard(int dev) {
        if (dev < 0) return;
        if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = (cudaSetDevice(dev) == cudaSuccess);
    }
    explicit AlvaDeviceGuard(const alva_ctx* c) : AlvaDeviceGuard(c ? c->device : -1) {}
    ~AlvaDeviceGuard() { if (switched) cudaSetDevice(prev); }
    AlvaDeviceGuard(const AlvaDeviceGuard&) = delete;
    AlvaDeviceGuard& operator=(const AlvaDeviceGuard&) = delete;
};

void alva_set_error(const char* fmt, ...);
void* alva_scratch(alva_ctx* ctx, size_t bytes);   // device scratch, valid until the next call
extern uint64_t alva_g_options_epoch;   // bumped whenever alva_set_option changes a value (ba.cu)
bool alva_make_tmap(CUtensorMap* map, CUtensorMapDataType dt, int rank, const void* base,
                    const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box);

#define ALVA_CUDA(call)                                                                         \
    do {                                                                                        \
        cudaError_t e__ = (call);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            alva_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return -2;                                                                          \
        }                                                                                       \
    } while (0)

#define ALVA_LAUNCH_CHECK(ctx)                                                                  \
    do {                                                                                        \
        (ctx)->launches++;                                                                      \
        cudaError_t e__ = cudaGetLastError();                                                   \
        if (e__ != cudaSuccess) {                                                               \
            alva_set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
            return -2;                                                                          \
        }                                                                                       \
    } while (0)

// ---------------------------------------------------------------- device side
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a TMA copy that never completes (bad descriptor) traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    for (uint32_t spin = 0; !mbar_try_wait(bar, parity); spin++)
        if (spin > (1u << 26)) __trap();
}
// TMA: 3-D tiled bulk tensor load global -> shared, completion on an mbarrier (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)),
        "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// TMA: the same box pulled into L2 only (no shared-memory destination, no barrier): a later CTA's tile (SASS: UTMAPF)
__device__ __forceinline__ void tma_prefetch_l2_3d(const CUtensorMap* map, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"((uint64_t)map), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}

// ---- SWAR helpers on 4 packed unsigned bytes ------------------------------------------------
#define ALVA_H 0x80808080u
#define ALVA_L 0x7f7f7f7fu

// per-byte a >= b, result in bit 7 of each byte (other bits are garbage)
__device__ __forceinline__ uint32_t swar_ge_raw(uint32_t a, uint32_t b) {
    uint32_t t = (a | ALVA_H) - (b & ALVA_L);
    // bit7: (a7 & ~b7) | (~(a7 ^ b7) & t7)
    return (a & ~b) | (~(a ^ b) & t);
}
__device__ __forceinline__ uint32_t swar_ge(uint32_t a, uint32_t b) { return swar_ge_raw(a, b) & ALVA_H; }
// per-byte saturating add / sub of a replicated constant
__device__ __forceinline__ uint32_t swar_addus(uint32_t a, uint32_t b) { return __vaddus4(a, b); }
__device__ __forceinline__ uint32_t swar_subus(uint32_t a, uint32_t b) { return __vsubus4(a, b); }

__device__ __forceinline__ int reflect101(int p, int n) {
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = p < 0 ? -p : 2 * (n - 1) - p;
    return p;
}

#endif  // __CUDACC__
