// api.cu -- context management, error reporting and TMA descriptor creation for libalva_b200.so.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include <stdarg.h>
#include <string.h>
#include <mutex>

static thread_local char g_err[512] = "";

void alva_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}

extern "C" const char* alva_last_error(void) { return g_err; }
extern "C" int alva_version(void) { return 100; }

// cuTensorMapEncodeTiled through the runtime's driver entry point: no link-time dependency on libcuda,
// so the library also loads (for symbol checks) on a machine without a driver.
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)p;
    });
    return fn;
}

bool alva_make_tmap(CUtensorMap* map, CUtensorMapDataType dt, int rank, const void* base, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return false;
    cuuint64_t d[5];
    cuuint64_t s[4];
    cuuint32_t b[5], es[5];
    for (int i = 0; i < rank; i++) { d[i] = dims[i]; b[i] = box[i]; es[i] = 1; }
    for (int i = 0; i + 1 < rank; i++) s[i] = strides_bytes[i];
    CUresult r = enc(map, dt, (cuuint32_t)rank, const_cast<void*>(base), d, s, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

void* alva_scratch(alva_ctx* ctx, size_t bytes) {
    if (bytes > ctx->scratch_bytes) {
        ctx->ws_epoch++;
        if (ctx->scratch) {
            cudaStreamSynchronize(ctx->stream);
            cudaFree(ctx->scratch);
            ctx->scratch = nullptr;
            ctx->scratch_bytes = 0;
        }
        size_t want = bytes + bytes / 4 + 4096;
        cudaError_t e = cudaMalloc(&ctx->scratch, want);
        if (e != cudaSuccess) {
            alva_set_error("scratch cudaMalloc(%zu) -> %s", want, cudaGetErrorString(e));
            ctx->scratch = nullptr;
            return nullptr;
        }
        ctx->scratch_bytes = want;
    }
    return ctx->scratch;
}

extern "C" alva_ctx* alva_ctx_create(int device, void* stream) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        alva_set_error("alva_ctx_create: no CUDA device (%s) -- libalva_b200 has no CPU fallback",
                       e != cudaSuccess ? cudaGetErrorString(e) : "count = 0");
        return nullptr;
    }
    if (device < 0 || device >= n) { alva_set_error("alva_ctx_create: device %d out of range (%d)", device, n); return nullptr; }
    AlvaDeviceGuard guard__(device);   // the caller's current device is left as it was
    int curdev = -1;
    if ((e = cudaGetDevice(&curdev)) != cudaSuccess || curdev != device) { alva_set_error("cudaSetDevice(%d): %s", device, cudaGetErrorString(e)); return nullptr; }
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) { alva_set_error("props: %s", cudaGetErrorString(e)); return nullptr; }
    if (prop.major != 9 || prop.minor != 0) {
        alva_set_error("alva_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
        return nullptr;
    }
    alva_ctx* ctx = new alva_ctx();
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    if (stream) ctx->stream = (cudaStream_t)stream;
    else {
        if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) {
            alva_set_error("cudaStreamCreate: %s", cudaGetErrorString(e));
            delete ctx;
            return nullptr;
        }
        ctx->own_stream = true;
    }
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if (cudaStreamCreateWithPriority(&ctx->aux_stream, cudaStreamNonBlocking, hi) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->aux_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->aux_join, cudaEventDisableTiming) != cudaSuccess) {
        alva_set_error("alva_ctx_create: auxiliary stream / events: %s", cudaGetErrorString(cudaGetLastError()));
        alva_ctx_destroy(ctx);
        return nullptr;
    }
    return ctx;
}

extern "C" void alva_ctx_destroy(alva_ctx* ctx) {
    if (!ctx) return;
    AlvaDeviceGuard guard__(ctx);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->dev_stage) cudaFree(ctx->dev_stage);
    if (ctx->ba_ws) cudaFree(ctx->ba_ws);
    if (ctx->det_ws) cudaFree(ctx->det_ws);
    if (ctx->knn_ws) cudaFree(ctx->knn_ws);
    if (ctx->clahe_ws) cudaFree(ctx->clahe_ws);
    if (ctx->p3p_tab) cudaFree(ctx->p3p_tab);
    if (ctx->init_tab) cudaFree(ctx->init_tab);
    if (ctx->aux_stream) { cudaStreamSynchronize(ctx->aux_stream); cudaStreamDestroy(ctx->aux_stream); }
    if (ctx->aux_fork) cudaEventDestroy(ctx->aux_fork);
    if (ctx->aux_join) cudaEventDestroy(ctx->aux_join);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

extern "C" int alva_ctx_sync(alva_ctx* ctx) { AlvaDeviceGuard guard__(ctx);
    if (!ctx) { alva_set_error("null ctx"); return ALVA_E_INVALID; }
    ALVA_CUDA(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" long long alva_ctx_launches(const alva_ctx* ctx) { return ctx ? ctx->launches : 0; }
