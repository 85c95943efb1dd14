// clahe.cu -- CLAHE (contrast-limited adaptive histogram equalisation) of 8-bit gray frames, bit-exact with
// cv::createCLAHE(clip, Size(tiles_x, tiles_y))->apply as VisualFrontend::preprocessImage runs it before it builds the KLT
// pyramid (visual_frontend.cpp:16-18, 672-698 -> opencv imgproc/src/clahe.cpp:142-313, 349-429).  Two launches:
//   clahe_lut_kernel    one CTA per (tile, frame): per-warp shared histograms of the tile (the reflect-101 extension of a
//                       non-dividing grid is read by index, never built), clip + redistribution, 256-bin block scan, LUT
//   clahe_apply_kernel  one CTA per band of rows: the two LUT rows the band interpolates between staged in shared memory,
//                       4 pixels per thread (u8x4 loads / stores), bilinear blend in float
// Built with -fmad=false and written with __fmul_rn / __fadd_rn: the reference OpenCV is an SSE build without FMA, and every
// float step below (LUT scale, tile coordinates, the blend) must round exactly as its scalar code does.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include <math.h>

namespace {

constexpr int kLutThreads = 256;     // one thread per histogram bin
constexpr int kLutWarps = kLutThreads / 32;
constexpr int kApplyThreads = 256;
constexpr int kBand = 16;            // rows per apply CTA
constexpr int kStageMaxTiles = 64;   // 2 x 64 x 256 B = 32 KB of staged LUT rows; wider grids read the LUTs from global

__device__ __forceinline__ int reflect101_ext(int p, int n) { return p < n ? p : reflect101(p, n); }

__device__ __forceinline__ uint8_t sat_round(float v) {
    const int r = __float2int_rn(v);   // cvRound: round half to even
    return (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
}

__global__ void __launch_bounds__(kLutThreads) clahe_lut_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ lut, int w, int h,
                                                                int tx, int ntiles, int tw, int th, int clip, float scale) {
    __shared__ int hist[kLutWarps][256];
    __shared__ int part[kLutWarps];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int f = blockIdx.x / ntiles, k = blockIdx.x % ntiles;
    for (int i = tid; i < kLutWarps * 256; i += kLutThreads) (&hist[0][0])[i] = 0;
    __syncthreads();
    const uint8_t* s = src + (size_t)f * w * h;
    const int x0 = (k % tx) * tw, y0 = (k / tx) * th;
    for (int r = warp; r < th; r += kLutWarps) {   // a warp per row, lanes along it; rows / columns past the image reflect
        const uint8_t* row = s + (size_t)reflect101_ext(y0 + r, h) * w;
        for (int c = lane; c < tw; c += 32) atomicAdd(&hist[warp][row[reflect101_ext(x0 + c, w)]], 1);
    }
    __syncthreads();
    int v = 0;
#pragma unroll
    for (int q = 0; q < kLutWarps; q++) v += hist[q][tid];
    if (clip > 0) {   // clahe.cpp:183-208
        int ex = v > clip ? v - clip : 0;
        v -= ex;
#pragma unroll
        for (int o = 16; o; o >>= 1) ex += __shfl_xor_sync(0xffffffffu, ex, o);
        if (lane == 0) part[warp] = ex;
        __syncthreads();
        int clipped = 0;
#pragma unroll
        for (int q = 0; q < kLutWarps; q++) clipped += part[q];
        const int batch = clipped / 256, residual = clipped - batch * 256;
        v += batch;
        if (residual) {   // one count to every step-th bin from bin 0, `residual` of them
            const int step = max(256 / residual, 1);
            if (tid % step == 0 && tid / step < residual) v++;
        }
        __syncthreads();
    }
    // inclusive scan over the 256 bins
    int sum = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, sum, o);
        if (lane >= o) sum += t;
    }
    if (lane == 31) part[warp] = sum;
    __syncthreads();
    for (int q = 0; q < warp; q++) sum += part[q];
    lut[(size_t)blockIdx.x * 256 + tid] = sat_round(__fmul_rn(__int2float_rn(sum), scale));   // clahe.cpp:211-219
}

__device__ __forceinline__ uint8_t blend(const uint8_t* L1, const uint8_t* L2, int x, int v, float inv_tw, int tx, float ya, float ya1) {
    const float txf = __fsub_rn(__fmul_rn(__int2float_rn(x), inv_tw), 0.5f);
    int tx1 = __float2int_rd(txf);
    const float xa = __fsub_rn(txf, __int2float_rn(tx1)), xa1 = __fsub_rn(1.0f, xa);
    const int tx2 = min(tx1 + 1, tx - 1);
    tx1 = max(tx1, 0);
    const int i1 = tx1 * 256 + v, i2 = tx2 * 256 + v;
    const float a = __fadd_rn(__fmul_rn(__int2float_rn(L1[i1]), xa1), __fmul_rn(__int2float_rn(L1[i2]), xa));
    const float b = __fadd_rn(__fmul_rn(__int2float_rn(L2[i1]), xa1), __fmul_rn(__int2float_rn(L2[i2]), xa));
    return sat_round(__fadd_rn(__fmul_rn(a, ya1), __fmul_rn(b, ya)));   // clahe.cpp:305-308, in that order
}

template <bool kStage, bool kVec>
__global__ void __launch_bounds__(kApplyThreads) clahe_apply_kernel(const uint8_t* src, uint8_t* dst, const uint8_t* __restrict__ lut, int w,
                                                                    int h, int tx, int ty, int nbands, float inv_tw, float inv_th) {
    __shared__ __align__(16) uint8_t sl[kStage ? 2 * kStageMaxTiles * 256 : 16];
    const int f = blockIdx.x / nbands, band = blockIdx.x % nbands;
    const uint8_t* s = src + (size_t)f * w * h;
    uint8_t* d = dst + (size_t)f * w * h;
    const uint8_t* L = lut + (size_t)f * tx * ty * 256;
    const int rowbytes = tx * 256;
    int staged = INT32_MIN;
    const int y1 = min(h, (band + 1) * kBand);
    for (int y = band * kBand; y < y1; y++) {
        const float tyf = __fsub_rn(__fmul_rn(__int2float_rn(y), inv_th), 0.5f);   // clahe.cpp:287-297
        const int ty1 = __float2int_rd(tyf);
        const float ya = __fsub_rn(tyf, __int2float_rn(ty1)), ya1 = __fsub_rn(1.0f, ya);
        const int t1 = max(ty1, 0), t2 = min(ty1 + 1, ty - 1);
        const uint8_t *L1 = L + (size_t)t1 * rowbytes, *L2 = L + (size_t)t2 * rowbytes;
        if (kStage) {
            if (ty1 != staged) {   // uniform over the CTA: y is
                __syncthreads();
                const uint4* g1 = (const uint4*)L1;
                const uint4* g2 = (const uint4*)L2;
                uint4* s4 = (uint4*)sl;
                const int n16 = rowbytes / 16;
                for (int i = threadIdx.x; i < n16; i += kApplyThreads) { s4[i] = g1[i]; s4[n16 + i] = g2[i]; }
                __syncthreads();
                staged = ty1;
            }
            L1 = sl; L2 = sl + rowbytes;
        }
        const uint8_t* srow = s + (size_t)y * w;
        uint8_t* drow = d + (size_t)y * w;
        if (kVec) {
            for (int j = threadIdx.x; j < (w >> 2); j += kApplyThreads) {
                const uchar4 p = ((const uchar4*)srow)[j];
                const int x = 4 * j;
                uchar4 o;
                o.x = blend(L1, L2, x, p.x, inv_tw, tx, ya, ya1);
                o.y = blend(L1, L2, x + 1, p.y, inv_tw, tx, ya, ya1);
                o.z = blend(L1, L2, x + 2, p.z, inv_tw, tx, ya, ya1);
                o.w = blend(L1, L2, x + 3, p.w, inv_tw, tx, ya, ya1);
                ((uchar4*)drow)[j] = o;
            }
        } else {
#pragma unroll 1
            for (int x = threadIdx.x; x < w; x += kApplyThreads) drow[x] = blend(L1, L2, x, srow[x], inv_tw, tx, ya, ya1);
        }
    }
}

}  // namespace

// clip as clahe.cpp:387-394 computes it: (int)(clip_limit * area / 256) in double, at least 1 (0 = no clipping).  A product past
// the int range converts to INT_MIN on x86 (cvttsd2si), which the max() then turns into 1: restated here without the UB.
static int clahe_clip(double clip_limit, int area) {
    if (!(clip_limit > 0.0)) return 0;
    const double v = clip_limit * area / 256;
    const int c = v >= 2147483648.0 ? INT32_MIN : (int)v;
    return c > 1 ? c : 1;
}

// both launches on ctx->stream; `lut` holds [nframes][tiles_y][tiles_x][256] bytes.  No allocation, no synchronisation: the
// System captures it into its pyramid graph.
int alva_clahe_launch(alva_ctx* ctx, const uint8_t* src, uint8_t* dst, int w, int h, int nframes, double clip_limit, int tiles_x,
                      int tiles_y, uint8_t* lut) {
    const bool even = w % tiles_x == 0 && h % tiles_y == 0;
    const int tw = even ? w / tiles_x : (w + tiles_x - w % tiles_x) / tiles_x;   // clahe.cpp:362-385
    const int th = even ? h / tiles_y : (h + tiles_y - h % tiles_y) / tiles_y;
    const int ntiles = tiles_x * tiles_y;
    const float scale = 255.0f / (float)(tw * th);
    clahe_lut_kernel<<<ntiles * nframes, kLutThreads, 0, ctx->stream>>>(src, lut, w, h, tiles_x, ntiles, tw, th, clahe_clip(clip_limit, tw * th), scale);
    ALVA_LAUNCH_CHECK(ctx);
    const int nbands = (h + kBand - 1) / kBand;
    const float inv_tw = 1.0f / (float)tw, inv_th = 1.0f / (float)th;
    const bool stage = tiles_x <= kStageMaxTiles, vec = (w & 3) == 0 && ((uintptr_t)src & 3) == 0 && ((uintptr_t)dst & 3) == 0;
    auto k = stage ? (vec ? clahe_apply_kernel<true, true> : clahe_apply_kernel<true, false>)
                   : (vec ? clahe_apply_kernel<false, true> : clahe_apply_kernel<false, false>);
    k<<<nbands * nframes, kApplyThreads, 0, ctx->stream>>>(src, dst, lut, w, h, tiles_x, tiles_y, nbands, inv_tw, inv_th);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_clahe(alva_ctx* ctx, const uint8_t* src, uint8_t* dst, int w, int h, int nframes, double clip_limit, int tiles_x,
                            int tiles_y) {
    AlvaDeviceGuard guard__(ctx);
    if (!ctx || !src || !dst || w < 1 || h < 1 || nframes < 1 || tiles_x < 1 || tiles_y < 1 || tiles_x > w || tiles_y > h ||
        !(clip_limit >= 0.0)) {
        alva_set_error("alva_k_clahe: bad argument (%dx%d, %d frames, %dx%d tiles, clip %g)", w, h, nframes, tiles_x, tiles_y, clip_limit);
        return ALVA_E_INVALID;
    }
    const size_t bytes = (size_t)nframes * tiles_x * tiles_y * 256;
    if (bytes > ctx->clahe_ws_bytes) {
        ctx->ws_epoch++;
        if (ctx->clahe_ws) {
            ALVA_CUDA(cudaStreamSynchronize(ctx->stream));
            cudaFree(ctx->clahe_ws);
            ctx->clahe_ws = nullptr;
            ctx->clahe_ws_bytes = 0;
        }
        ALVA_CUDA(cudaMalloc(&ctx->clahe_ws, bytes));
        ctx->clahe_ws_bytes = bytes;
    }
    return alva_clahe_launch(ctx, src, dst, w, h, nframes, clip_limit, tiles_x, tiles_y, (uint8_t*)ctx->clahe_ws);
}
