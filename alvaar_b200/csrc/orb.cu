// orb.cu -- ORB pre-blur and steered-BRIEF (rBRIEF-256) descriptors at given points, sm_90a.
//
// Reference behaviour (bit-exact; CPU restatement in oracle/alva_oracle.c):
//   FeatureExtractor::describeFeaturePoints   src/slam/src/feature_extractor.cpp:160-214
//     -> ORB::create(500, 1., 0)->compute      opencv features2d/src/orb.cpp:970-1218
//        border rule (31 px, rounded)          orb.cpp:1130, keypoint.cpp:92-117
//        GaussianBlur(7x7, sigma 2) float path orb.cpp:1188 -> imgproc/src/filter.simd.hpp:468-510, 1163-1215
//        computeOrbDescriptors                 orb.cpp:219-350 (pattern orb.cpp:380-638)
//        ICAngles + fastAtan2 (detect mode)    orb.cpp:181-215, core/src/mathfuncs_core.simd.hpp:34-71
//
// The blur is order- and fusion-sensitive float arithmetic: every product and sum below is an explicit
// __fmul_rn/__fadd_rn (or one __fmaf_rn in ALVA_ORB_FMA mode) so nvcc cannot re-associate or contract it.
#include "alva_common.cuh"
#include <algorithm>
#include "../../include/alva_b200.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

namespace {

__constant__ __align__(16) int8_t c_pattern[1024] = {
#include "orb_pattern.inc"
};
// getGaussianKernel(7, 2, CV_32F) (imgproc/src/smooth.dispatch.cpp:76-190): k[3], k[2]=k[4], k[1]=k[5], k[0]=k[6]
__constant__ uint32_t c_gauss_bits[4] = {0x3e5d4ae0u, 0x3e434a39u, 0x3e06387eu, 0x3d8fafb1u};

constexpr int BTW = 128, BTH = 64;          // blur tile (outputs)
constexpr int BIP = BTW + 32;               // input smem pitch in bytes: image x0-16 at byte 0 (x0-3 .. x0+BTW+2 are used);
                                            // 16 halo bytes so that a TMA box starts 16-byte aligned
constexpr int BIX = 16;                     // byte of image column x0
constexpr int BIR = BTH + 6;                // input rows y0-3 .. y0+BTH+2

// u8 -> f32 without the conversion pipe: 0x4B000000 | b is the float 2^23 + b; one PRMT + one FADD (exact)
__device__ __forceinline__ float byte_to_float(uint32_t word, uint32_t sel) {
    return __fsub_rn(__uint_as_float(__byte_perm(word, 0x4B000000u, sel)), 8388608.f);
}

// Separable 7x7 Gaussian exactly as OpenCV's float path evaluates it (see file header): row pass then column pass.
// The (BTW+32) x (BTH+6) input tile arrives by ONE TMA bulk-tensor copy (out-of-image bytes come back as zeros and the
// reflect-101 border is patched in shared memory); geometries TMA cannot address take a plain-load path.
// Thread = 4 adjacent pixels: the row pass reads three packed words and produces a float4; the column pass walks an
// 8-row strip with a rolling 7-row window of float4, packs 4 results and stores one 32-bit word.
template <bool FMA>
__global__ void __launch_bounds__(256) orb_blur_kernel(const __grid_constant__ CUtensorMap tmap, int use_tma,
                                                       const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int w, int h) {
    __shared__ __align__(128) uint8_t in_s[BIR][BIP];
    __shared__ __align__(16) float row_s[BIR][BTW];
    __shared__ uint64_t bar;
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * BTW, y0 = blockIdx.y * BTH;
    const size_t fo = (size_t)blockIdx.z * w * h;
    const uint8_t* s = src + fo;
    float k[4];
#pragma unroll
    for (int i = 0; i < 4; i++) k[i] = __uint_as_float(c_gauss_bits[i]);   // k[j] = weight at distance j

    if (use_tma) {
        if (tid == 0) { mbar_init(&bar, 1); fence_barrier_init(); }
        __syncthreads();
        if (tid == 0) {
            mbar_arrive_expect_tx(&bar, BIP * BIR);
            tma_load_3d(&in_s[0][0], &tmap, &bar, x0 - BIX, y0 - 3, blockIdx.z);
        }
        mbar_wait(&bar, 0);
        // reflect-101 patch of what lies outside the image: columns first (rows inside the image), then whole rows
        const bool el = (x0 == 0), er = (x0 + BTW + 3 > w);
        if (el || er) {
            for (int r = tid; r < BIR; r += 256) {
                const int y = y0 - 3 + r;
                if (y < 0 || y >= h) continue;
                uint8_t* row = &in_s[r][0];
                if (el) { row[BIX - 1] = row[BIX + 1]; row[BIX - 2] = row[BIX + 2]; row[BIX - 3] = row[BIX + 3]; }
                if (er) {
                    const int cw = w - x0 + BIX;   // byte of image column w
                    if (cw + 2 < BIP) { row[cw] = row[cw - 2]; row[cw + 1] = row[cw - 3]; row[cw + 2] = row[cw - 4]; }
                }
            }
            __syncthreads();
        }
        if (y0 == 0 || y0 + BTH + 3 > h) {
            for (int i = tid; i < 6 * (BIP / 4); i += 256) {
                const int j = i / (BIP / 4), c4 = i - j * (BIP / 4);
                // j = 0..2: image rows -1, -2, -3 (top);  j = 3..5: rows h, h+1, h+2 (bottom)
                const int y = j < 3 ? -1 - j : h + (j - 3);
                const int ys = j < 3 ? 1 + j : h - 2 - (j - 3);
                const int r = y - y0 + 3, rs = ys - y0 + 3;
                if (r >= 0 && r < BIR && rs >= 0 && rs < BIR && ys >= 0 && ys < h)
                    reinterpret_cast<uint32_t*>(&in_s[r][0])[c4] = reinterpret_cast<const uint32_t*>(&in_s[rs][0])[c4];
            }
        }
    } else {
        for (int i = tid; i < BIR * BIP; i += 256) {
            const int r = i / BIP, c = i - r * BIP;
            const int x = reflect101(max(min(x0 + c - BIX, w + 7), -8), w), y = reflect101(min(y0 + r - 3, h + 3), h);
            in_s[r][c] = __ldg(s + (size_t)y * w + x);
        }
    }
    __syncthreads();
    // row filter: s = k0*S[0]; s += k[i]*S[i], left to right (RowFilter<uchar,float>, filter.simd.hpp:2477-2487)
    for (int i = tid; i < BIR * (BTW / 4); i += 256) {
        const int r = i >> 5, g = i & 31;                      // BTW / 4 == 32 groups per row
        const uint32_t* wp = reinterpret_cast<const uint32_t*>(&in_s[r][0]) + BIX / 4 - 1 + g;   // W0 = x-4..x-1, W1 = x..x+3, W2 = x+4..x+7
        const uint32_t W0 = wp[0], W1 = wp[1], W2 = wp[2];
        float f[10];                                            // pixels x-3 .. x+6
        f[0] = byte_to_float(W0, 0x7651); f[1] = byte_to_float(W0, 0x7652); f[2] = byte_to_float(W0, 0x7653);
        f[3] = byte_to_float(W1, 0x7650); f[4] = byte_to_float(W1, 0x7651); f[5] = byte_to_float(W1, 0x7652);
        f[6] = byte_to_float(W1, 0x7653); f[7] = byte_to_float(W2, 0x7650); f[8] = byte_to_float(W2, 0x7651);
        f[9] = byte_to_float(W2, 0x7652);
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            float acc;
            if (FMA) {
                acc = 0.f;
#pragma unroll
                for (int t = 0; t < 7; t++) acc = __fmaf_rn(f[j + t], k[t < 3 ? 3 - t : t - 3], acc);
            } else {
                acc = __fmul_rn(k[3], f[j]);
#pragma unroll
                for (int t = 1; t < 7; t++) acc = __fadd_rn(acc, __fmul_rn(k[t < 3 ? 3 - t : t - 3], f[j + t]));
            }
            o[j] = acc;
        }
        *reinterpret_cast<float4*>(&row_s[r][4 * g]) = make_float4(o[0], o[1], o[2], o[3]);
    }
    __syncthreads();
    // column filter: s = k3*R[0]; s += k[3+j]*(R[+j] + R[-j]) (SymmColumnFilter, filter.simd.hpp:2697-2790), cvRound
    {
        const int g = tid & 31, strip = tid >> 5;              // 32 column groups x 8 strips of 8 rows
        const int x = x0 + 4 * g;
        float4 win[7];
#pragma unroll
        for (int r = 0; r < 6; r++) win[r] = *reinterpret_cast<const float4*>(&row_s[8 * strip + r][4 * g]);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            win[(i + 6) % 7] = *reinterpret_cast<const float4*>(&row_s[8 * strip + i + 6][4 * g]);
            const int y = y0 + 8 * strip + i;
            uint32_t packed = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) {
#define WV(d) (reinterpret_cast<const float*>(&win[(i + 3 + (d)) % 7])[j])
                float acc = FMA ? __fmaf_rn(k[0], WV(0), 0.f) : __fmul_rn(k[0], WV(0));
#pragma unroll
                for (int d = 1; d <= 3; d++) {
                    const float ab = __fadd_rn(WV(d), WV(-d));
                    acc = FMA ? __fmaf_rn(k[d], ab, acc) : __fadd_rn(acc, __fmul_rn(k[d], ab));
                }
#undef WV
                int v = __float2int_rn(acc);
                v = max(0, min(255, v));
                packed |= (uint32_t)v << (8 * j);
            }
            if (y < h && x < w) {
                uint8_t* d = dst + fo + (size_t)y * w + x;
                if (x + 3 < w && ((w & 3) == 0)) *reinterpret_cast<uint32_t*>(d) = packed;
                else
                    for (int j = 0; j < 4 && x + j < w; j++) d[j] = (uint8_t)(packed >> (8 * j));
            }
        }
    }
}

// cv::fastAtan2 (degrees), baseline arithmetic: no contraction
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float p1 = 0.9997878412794807f * (float)(180 / 3.1415926535897932384626433832795);
    const float p3 = -0.3258083974640975f * (float)(180 / 3.1415926535897932384626433832795);
    const float p5 = 0.1555786518463281f * (float)(180 / 3.1415926535897932384626433832795);
    const float p7 = -0.04432655554792128f * (float)(180 / 3.1415926535897932384626433832795);
    const float ax = fabsf(x), ay = fabsf(y);
    const float eps = (float)2.2204460492503131e-16;
    float a, c, c2;
    if (ax >= ay) {
        c = __fdiv_rn(ay, __fadd_rn(ax, eps));
        c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = __fdiv_rn(ax, __fadd_rn(ay, eps));
        c2 = __fmul_rn(c, c);
        a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

// umax of computeKeyPoints (orb.cpp:819-834) for halfPatchSize 15
__constant__ int8_t c_umax[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};

// one warp per keypoint; lane j produces descriptor byte j
__global__ void __launch_bounds__(256) orb_describe_kernel(const uint8_t* __restrict__ gray, const uint8_t* __restrict__ blurred,
                                                           int w, int h, const float* __restrict__ pts,
                                                           const int32_t* __restrict__ npts_per_frame, int npts, int flags,
                                                           uint8_t* __restrict__ desc, uint8_t* __restrict__ kept,
                                                           float* __restrict__ angles_out) {
    // the 256 test pairs as words (x0, y0, x1, y1), TRANSPOSED: pair 8 * lane + t sits at [t][lane], so the 8 loads of a warp are
    // conflict-free (pair-major order puts the lanes 32 bytes apart: 4 byte loads per pair, each 8-way bank conflicted)
    __shared__ uint32_t pat_s[8][32];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) pat_s[i & 7][i >> 3] = reinterpret_cast<const uint32_t*>(c_pattern)[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int f = blockIdx.y;
    const int kp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int n = npts_per_frame ? min(npts_per_frame[f], npts) : npts;
    if (kp >= npts) return;
    const size_t o = (size_t)f * npts + kp;
    if (kp >= n) {   // unused slot
        if (lane == 0) kept[o] = 0;
        desc[o * 32 + lane] = 0;
        if (angles_out && lane == 0) angles_out[o] = -1.f;
        return;
    }
    const float px = pts[o * 2], py = pts[o * 2 + 1];
    const int cx = __float2int_rn(px), cy = __float2int_rn(py);
    const bool keep = (w > 62 && h > 62) && cx >= 31 && cx < w - 31 && cy >= 31 && cy < h - 31;
    if (!keep) {
        if (lane == 0) kept[o] = 0;
        desc[o * 32 + lane] = 0;
        if (angles_out && lane == 0) angles_out[o] = -1.f;
        return;
    }
    const size_t fo = (size_t)f * w * h;
    float angle = -1.f;   // KeyPoint::convert default (core/src/types.cpp:93-101)
    if (flags & ALVA_ORB_IC_ANGLE) {
        // intensity-centroid moments over the circular patch r = 15 (exact integers), warp-reduced
        const uint8_t* c = gray + fo + (size_t)cy * w + cx;
        int m01 = 0, m10 = 0;
        // lanes split the 31 columns u = -15..15 (lane 31 idle)
        const int u = lane - 15;
        if (lane < 31) {
            m10 += u * c[u];   // v = 0 row
            for (int v = 1; v <= 15; v++) {
                if (abs(u) <= c_umax[v]) {
                    const int vp = c[u + v * w], vm = c[u - v * w];
                    m01 += v * (vp - vm);
                    m10 += u * (vp + vm);
                }
            }
        }
#pragma unroll
        for (int off = 16; off; off >>= 1) {
            m01 += __shfl_xor_sync(0xffffffffu, m01, off);
            m10 += __shfl_xor_sync(0xffffffffu, m10, off);
        }
        angle = fast_atan2_deg((float)m01, (float)m10);
    }
    // orb.cpp:232-235: angle *= (float)(CV_PI/180.f); a = (float)cos(angle), b = (float)sin(angle)
    const float ang = __fmul_rn(angle, (float)(3.1415926535897932384626433832795 / 180.f));
    const float a = (float)cos((double)ang), b = (float)sin((double)ang);
    const uint8_t* center = blurred + fo + (size_t)cy * w + cx;
    int val = 0;
#pragma unroll
    for (int t = 0; t < 8; t++) {
        const uint32_t pw = pat_s[t][lane];
        const float p0x = (float)(int8_t)pw, p0y = (float)(int8_t)(pw >> 8), p1x = (float)(int8_t)(pw >> 16), p1y = (float)(int8_t)(pw >> 24);
        const int x0 = __float2int_rn(__fsub_rn(__fmul_rn(p0x, a), __fmul_rn(p0y, b)));
        const int y0 = __float2int_rn(__fadd_rn(__fmul_rn(p0x, b), __fmul_rn(p0y, a)));
        const int x1 = __float2int_rn(__fsub_rn(__fmul_rn(p1x, a), __fmul_rn(p1y, b)));
        const int y1 = __float2int_rn(__fadd_rn(__fmul_rn(p1x, b), __fmul_rn(p1y, a)));
        const int t0 = center[y0 * w + x0], t1 = center[y1 * w + x1];
        val |= (t0 < t1) << t;
    }
    desc[o * 32 + lane] = (uint8_t)val;
    if (lane == 0) {
        kept[o] = 1;
        if (angles_out) angles_out[o] = angle;
    }
}

// ---- HarrisResponses (features2d/src/orb.cpp:130-177): blockSize 7, k = 0.04; one warp per keypoint ----------------
// Integer Sobel sums over the 7x7 block (exact), then the float formula in the reference's operation order.
__global__ void __launch_bounds__(256) harris_kernel(const uint8_t* __restrict__ gray, int w, int h, const float* __restrict__ pts,
                                                     const int32_t* __restrict__ npts_per_frame, int npts,
                                                     float* __restrict__ resp, int zero_dead) {
    const int lane = threadIdx.x & 31, f = blockIdx.y;
    const int n = npts_per_frame ? min(npts_per_frame[f], npts) : npts;
    // grid-stride over the slots: the slot capacity can be far larger than the live count (pre-selection lists), and a
    // grid sized by capacity would be launch-bound
    for (int kp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); kp < npts; kp += gridDim.x * (blockDim.x >> 5)) {
        const size_t o = (size_t)f * npts + kp;
        if (kp >= n) {
            if (zero_dead && lane == 0) resp[o] = 0.f;
            if (!zero_dead) break;
            continue;
        }
        const int x0 = __float2int_rn(pts[2 * o]), y0 = __float2int_rn(pts[2 * o + 1]);
        if (x0 < 4 || y0 < 4 || x0 >= w - 4 || y0 >= h - 4) { if (lane == 0) resp[o] = 0.f; continue; }
        const uint8_t* c = gray + (size_t)f * w * h + (size_t)y0 * w + x0;
        int a = 0, b = 0, cc = 0;
        for (int i = lane; i < 49; i += 32) {
            const int dy = i / 7 - 3, dx = i % 7 - 3;
            const uint8_t* p = c + dy * w + dx;
            const int tl = p[-w - 1], tc = p[-w], tr = p[-w + 1], ml = p[-1], mr = p[1], bl = p[w - 1], bc = p[w], br = p[w + 1];
            const int Ix = (mr - ml) * 2 + (tr - tl) + (br - bl);
            const int Iy = (bc - tc) * 2 + (bl - tl) + (br - tr);
            a += Ix * Ix; b += Iy * Iy; cc += Ix * Iy;
        }
#pragma unroll
        for (int off = 16; off; off >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, off);
            b += __shfl_xor_sync(0xffffffffu, b, off);
            cc += __shfl_xor_sync(0xffffffffu, cc, off);
        }
        if (lane == 0) {
            // scale = 1.f/((1 << 2) * blockSize * 255.f); scale_sq_sq = scale*scale*scale*scale (orb.cpp:145-146)
            const float scale = __fdiv_rn(1.f, 7140.f);
            const float s4 = __fmul_rn(__fmul_rn(__fmul_rn(scale, scale), scale), scale);
            const float fa = (float)a, fb = (float)b, fc = (float)cc;
            const float sum = __fadd_rn(fa, fb);
            // ((float)a * b - (float)c * c - harris_k * ((float)a + b) * ((float)a + b)) * scale_sq_sq   (orb.cpp:173-174)
            const float v = __fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, sum), sum));
            resp[o] = __fmul_rn(v, s4);
        }
    }
}

// ---- KeyPointsFilter::retainBest(n) on float responses (keypoint.cpp:69-90), one CTA per frame ----------------------
// Radix-select the n-th largest response, keep every keypoint with response >= it, in input (row-major) order.
// Writes (x, y, response, 0) rows + the (x, y) list the describe kernel reads.
__device__ __forceinline__ uint32_t float_key(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__global__ void __launch_bounds__(1024) retain_best_f32_kernel(const float* __restrict__ pts, const float* __restrict__ resp,
                                                               const int32_t* __restrict__ counts, int cap, int n_keep,
                                                               float* __restrict__ kp_out, float* __restrict__ pts_out,
                                                               const uint32_t* __restrict__ keys_in, uint32_t* __restrict__ keys_out,
                                                               int32_t* __restrict__ out_counts, int out_cap) {
    __shared__ int hist[256];
    __shared__ uint32_t prefix_s, mask_s;
    __shared__ int krem_s, wsum[32], base_s;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = min(counts[f], cap);
    const float* r = resp + (size_t)f * cap;
    float thr = -INFINITY;
    if (n_keep >= 0 && n > n_keep) {
        if (n_keep == 0) thr = INFINITY;
        else {
            if (tid == 0) { prefix_s = 0; mask_s = 0; krem_s = n_keep; }
            for (int pass = 3; pass >= 0; pass--) {
                for (int i = tid; i < 256; i += 1024) hist[i] = 0;
                __syncthreads();
                const uint32_t prefix = prefix_s, mask = mask_s;
                for (int i = tid; i < n; i += 1024) {
                    const uint32_t k = float_key(r[i]);
                    if ((k & mask) == prefix) atomicAdd(&hist[(k >> (8 * pass)) & 255], 1);
                }
                __syncthreads();
                if (tid == 0) {
                    int acc = 0, k = krem_s, bsel = 0;
                    for (int bkt = 255; bkt >= 0; bkt--) {
                        if (acc + hist[bkt] >= k) { bsel = bkt; break; }
                        acc += hist[bkt];
                    }
                    krem_s = k - acc;
                    prefix_s = prefix | ((uint32_t)bsel << (8 * pass));
                    mask_s = mask | (0xffu << (8 * pass));
                }
                __syncthreads();
            }
            const uint32_t k = prefix_s;
            thr = __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
        }
    }
    if (tid == 0) base_s = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += 1024) {   // ordered compaction
        const int i = i0 + tid;
        const bool keep = i < n && r[i] >= thr;
        const uint32_t m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) wsum[warp] = __popc(m);
        __syncthreads();
        int off = base_s;
        for (int wv = 0; wv < warp; wv++) off += wsum[wv];
        const int pos = off + __popc(m & ((1u << lane) - 1));
        if (keep && pos < out_cap) {
            const size_t src = (size_t)f * cap + i, dst = (size_t)f * out_cap + pos;
            const float x = pts[2 * src], y = pts[2 * src + 1];
            if (kp_out) { kp_out[4 * dst] = x; kp_out[4 * dst + 1] = y; kp_out[4 * dst + 2] = r[i]; kp_out[4 * dst + 3] = 0.f; }
            pts_out[2 * dst] = x; pts_out[2 * dst + 1] = y;
            if (keys_out) keys_out[dst] = keys_in[src];
        }
        __syncthreads();
        if (tid == 0) { int t = 0; for (int wv = 0; wv < 32; wv++) t += wsum[wv]; base_s += t; }
        __syncthreads();
    }
    if (tid == 0) out_counts[f] = base_s;
}

__global__ void detect_finish_kernel(const float* __restrict__ angles, const int32_t* __restrict__ counts, int out_cap,
                                     float* __restrict__ kp_out) {
    const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < min(counts[f], out_cap)) kp_out[4 * ((size_t)f * out_cap + i) + 3] = angles[(size_t)f * out_cap + i];
}

__global__ void keys_to_pts_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ counts, int cap,
                                   float* __restrict__ pts) {
    const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(counts[f], cap)) return;
    const uint32_t k = keys[(size_t)f * cap + i];
    reinterpret_cast<float2*>(pts)[(size_t)f * cap + i] = make_float2((float)ALVA_KEY_X(k), (float)ALVA_KEY_Y(k));
}

}  // namespace

extern "C" int alva_k_orb_blur(alva_ctx* ctx, const uint8_t* gray, uint8_t* blurred, int w, int h, int nframes, int flags) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !gray || !blurred || w < 8 || h < 8 || nframes < 1 || gray == blurred) {
        alva_set_error("alva_k_orb_blur: bad argument (in-place not supported)");
        return ALVA_E_INVALID;
    }
    dim3 grid((w + BTW - 1) / BTW, (h + BTH - 1) / BTH, nframes);
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof tmap);
    const uint64_t dims[3] = {(uint64_t)w, (uint64_t)h, (uint64_t)nframes};
    const uint64_t strides[2] = {(uint64_t)w, (uint64_t)w * h};
    const uint32_t box[3] = {BIP, BIR, 1};
    static const bool no_tma = getenv("ALVA_DISABLE_TMA") != nullptr;   // debugging aid: force the plain-load path
    const int use_tma = (!no_tma && (w % 16) == 0 && w >= BIP && h >= 8 && ((uintptr_t)gray % 16) == 0 &&
                         alva_make_tmap(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, gray, dims, strides, box))
                            ? 1 : 0;
    if (flags & ALVA_ORB_FMA) orb_blur_kernel<true><<<grid, 256, 0, ctx->stream>>>(tmap, use_tma, gray, blurred, w, h);
    else orb_blur_kernel<false><<<grid, 256, 0, ctx->stream>>>(tmap, use_tma, gray, blurred, w, h);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_orb_describe(alva_ctx* ctx, const uint8_t* gray, const uint8_t* blurred, int w, int h, int nframes,
                                   const float* pts, const int32_t* npts_per_frame, int npts, int flags, uint8_t* desc,
                                   uint8_t* kept, float* angles_out) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !blurred || !pts || !desc || !kept || w < 1 || h < 1 || nframes < 1 || npts < 1 ||
        ((flags & ALVA_ORB_IC_ANGLE) && !gray)) {
        alva_set_error("alva_k_orb_describe: bad argument");
        return ALVA_E_INVALID;
    }
    dim3 grid((npts + 7) / 8, nframes);
    orb_describe_kernel<<<grid, 256, 0, ctx->stream>>>(gray, blurred, w, h, pts, npts_per_frame, npts, flags, desc, kept,
                                                       angles_out);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// internal (pipeline.cu): KeyPointsFilter::retainBest(n) on float responses, order-preserving; optional packed keys
int alva_retain_best_f32_launch(alva_ctx* ctx, const float* pts, const float* resp, const int32_t* counts, int cap, int nframes,
                                int n_keep, float* pts_out, const uint32_t* keys_in, uint32_t* keys_out, int32_t* out_counts,
                                int out_cap) {
    retain_best_f32_kernel<<<nframes, 1024, 0, ctx->stream>>>(pts, resp, counts, cap, n_keep, nullptr, pts_out, keys_in, keys_out,
                                                              out_counts, out_cap);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// zero_dead = 0 (internal callers with huge slot capacities): slots past the live count are left untouched
int alva_harris_launch(alva_ctx* ctx, const uint8_t* gray, int w, int h, int nframes, const float* pts, const int32_t* npts_per_frame,
                       int npts, float* resp, int zero_dead) {
    dim3 grid(std::min((npts + 7) / 8, 256), nframes);
    harris_kernel<<<grid, 256, 0, ctx->stream>>>(gray, w, h, pts, npts_per_frame, npts, resp, zero_dead);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_harris(alva_ctx* ctx, const uint8_t* gray, int w, int h, int nframes, const float* pts,
                             const int32_t* npts_per_frame, int npts, float* resp) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !gray || !pts || !resp || w < 9 || h < 9 || nframes < 1 || npts < 1) {
        alva_set_error("alva_k_harris: bad argument");
        return ALVA_E_INVALID;
    }
    return alva_harris_launch(ctx, gray, w, h, nframes, pts, npts_per_frame, npts, resp, 1);
}

// ORB::detectAndCompute, nlevels = 1 (orb.cpp:970-1218 with computeKeyPoints :785-958): FAST(thr, nms) -> border 31 ->
// retainBest(2n) by FAST score -> Harris -> retainBest(n) by Harris -> IC angle -> blur -> steered rBRIEF.
// Composition of this library's own stage kernels; intermediate lists live in a context-owned workspace.
extern "C" int alva_k_orb_detect(alva_ctx* ctx, const uint8_t* gray, int w, int h, int nframes, int nfeatures, int fast_thr,
                                 int flags, float* kp_out, uint8_t* desc, int32_t* counts, int out_cap) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !gray || !kp_out || !desc || !counts || w < 64 || h < 64 || nframes < 1 || nfeatures < 1 || out_cap < 1) {
        alva_set_error("alva_k_orb_detect: bad argument (need w, h >= 64)");
        return ALVA_E_INVALID;
    }
    const int kcap = (int)std::min<size_t>(std::max<size_t>(8192, (size_t)w * h / 24), 1u << 20);
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    const size_t b_keys = al((size_t)nframes * kcap * 4), b_pts = al((size_t)nframes * kcap * 8), b_resp = al((size_t)nframes * kcap * 4);
    const size_t b_cnt = al((size_t)nframes * 4), b_img = al((size_t)nframes * w * h);
    const size_t b_pts2 = al((size_t)nframes * out_cap * 8), b_ang = al((size_t)nframes * out_cap * 4), b_kept = al((size_t)nframes * out_cap);
    const size_t need = 2 * b_keys + b_pts + b_resp + 2 * b_cnt + b_img + b_pts2 + b_ang + b_kept;
    if (need > ctx->det_ws_bytes) {
        if (ctx->det_ws) { ALVA_CUDA(cudaStreamSynchronize(ctx->stream)); ALVA_CUDA(cudaFree(ctx->det_ws)); ctx->det_ws = nullptr; ctx->det_ws_bytes = 0; }
        ALVA_CUDA(cudaMalloc(&ctx->det_ws, need));
        ctx->det_ws_bytes = need;
    }
    uint8_t* b = (uint8_t*)ctx->det_ws;
    uint32_t* keys0 = (uint32_t*)b; b += b_keys;
    uint32_t* keys1 = (uint32_t*)b; b += b_keys;
    float* pts1 = (float*)b; b += b_pts;
    float* resp = (float*)b; b += b_resp;
    int32_t* cnt0 = (int32_t*)b; b += b_cnt;
    int32_t* cnt1 = (int32_t*)b; b += b_cnt;
    uint8_t* blurred = b; b += b_img;
    float* pts2 = (float*)b; b += b_pts2;
    float* ang = (float*)b; b += b_ang;
    uint8_t* kept = b;
    if (int e = alva_k_fast9(ctx, gray, w, h, nframes, fast_thr, keys0, cnt0, kcap, 1)) return e;
    if (int e = alva_k_retain_best(ctx, keys0, cnt0, kcap, nframes, w, h, 2 * nfeatures, 31, keys1, cnt1, kcap)) return e;
    dim3 kgrid((kcap + 255) / 256, nframes);
    keys_to_pts_kernel<<<kgrid, 256, 0, ctx->stream>>>(keys1, cnt1, kcap, pts1);
    ALVA_LAUNCH_CHECK(ctx);
    if (int e = alva_harris_launch(ctx, gray, w, h, nframes, pts1, cnt1, kcap, resp, 0)) return e;
    retain_best_f32_kernel<<<nframes, 1024, 0, ctx->stream>>>(pts1, resp, cnt1, kcap, nfeatures, kp_out, pts2, nullptr, nullptr, counts, out_cap);
    ALVA_LAUNCH_CHECK(ctx);
    if (int e = alva_k_orb_blur(ctx, gray, blurred, w, h, nframes, flags)) return e;
    if (int e = alva_k_orb_describe(ctx, gray, blurred, w, h, nframes, pts2, counts, out_cap, flags | ALVA_ORB_IC_ANGLE, desc, kept, ang))
        return e;
    dim3 fgrid((out_cap + 255) / 256, nframes);
    detect_finish_kernel<<<fgrid, 256, 0, ctx->stream>>>(ang, counts, out_cap, kp_out);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}
