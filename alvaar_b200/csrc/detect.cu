// detect.cu -- the reference's keyframe corner detector on the GPU: per-grid-cell Shi-Tomasi maxima with a shared
// suppression mask, adaptive quality threshold, then cornerSubPix.  Batched over frames.
//
// What is computed (bit-exact with the reference: integer cell maxima, their order and count, the adapted quality, and the
// sub-pixel positions as float bit patterns; the CPU restatement is oracle/detect_oracle.c):
//   FeatureExtractor::detectFeaturePoints          src/slam/src/feature_extractor.cpp:11-158 (caller map_manager.cpp:193-222)
//   cv::GaussianBlur(3x3) on the cell ROI          opencv imgproc/src/smooth.dispatch.cpp:611-755 -> 8-bit fixed-point sepFilter2D
//       whose SIMD body rounds half-to-even (filter.simd.hpp:1010-1099) and whose scalar tail (last cell & 3 columns) rounds
//       half-up (FixedPtCastEx)
//   cv::cornerMinEigenVal(block 3, Sobel 3)        imgproc/src/corner.cpp:237-330, 52-103; float filters filter.simd.hpp:2094-2165
//   cv::circle / cv::minMaxLoc                     imgproc/src/drawing.cpp:1476-1610; first maximum in row-major order
//   cv::cornerSubPix(3, 30 it, 0.01)               imgproc/src/cornersubpix.cpp:44-160, getRectSubPix_8u32f samplers.cpp:219-268
//
// How: the arithmetic is per cell and embarrassingly parallel (one CTA per cell and frame: blur, Sobel, covariance box sums
// and minimum eigenvalue through shared memory, the float expressions in the reference's operation order, -fmad=false);
// only the suppression mask couples cells, and only neighbouring ones, in the reference's serial cell order.  That order is
// kept exactly by a wavefront: cell (r, c) needs (r, c-1) and (r-1, c+1) -> step t = c + 2r, all cells of a step in
// parallel (one warp each, one CTA per frame), a bit mask in HBM standing in for the reference's float mask image.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include <float.h>
#include <math.h>
#include <vector>
#include <stdlib.h>

namespace {

constexpr int MAX_CELL = 64;
constexpr int MAX_RADIUS = MAX_CELL / 4;

struct DetectParams {
    const uint8_t* img;      // [nframes][h][w]
    int w, h, nframes, cs, rad, nch, ncw;
    const float* cur;        // [nframes][cur_cap][2]
    const int32_t* ncur;     // [nframes]
    int cur_cap;
    int roi[4];
    int hw[MAX_RADIUS + 1];  // cv::circle disk half-widths per |row offset|
    uint8_t* occ;            // [nframes][(nch+1)*(ncw+1)]
    float* hmap;             // [nframes][ncells][cs*cs]
    float4* cand;            // [nframes][ncells]: {best, index, second best (outside the best's disc), index} under the static mask
    uint32_t* mask;          // [nframes][h][mw] bit = 1: allowed
    int mw;
    double* quality;         // [nframes] in/out
    float* out;              // [nframes][out_cap][2]
    int32_t* out_int;        // optional [nframes][out_cap][2]
    int32_t* counts;         // [nframes]
    int out_cap;
    float sp_mask[49];       // cornerSubPix Gaussian window (host expf)
    int32_t* dbg;            // optional [8] counters (ALVA_DETECT_DEBUG): why the select kernel re-scanned a cell
    uint8_t* sel;            // [nframes][sel_bytes]: the select kernel's prim / sec / cell states when they do not fit in shared memory
    size_t sel_bytes;
};

__device__ __forceinline__ int refl(int p, int n) {
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = p < 0 ? -p : 2 * (n - 1) - p;
    return p;
}

// ---- D0: occupancy + mask init + disks of the current keypoints (one CTA per frame)
__device__ void clear_disk(uint32_t* mask, int mw, int w, int h, int cx, int cy, int rad, const int* hw, int lane, int nl) {
    for (int r = -rad + lane; r <= rad; r += nl) {
        const int y = cy + r, half = hw[r < 0 ? -r : r];
        if (y < 0 || y >= h || half < 0) continue;
        int xa = cx - half, xb = cx + half;
        xa = xa < 0 ? 0 : xa; xb = xb > w - 1 ? w - 1 : xb;
        if (xa > xb) continue;
        uint32_t* row = mask + (size_t)y * mw;
        for (int wd = xa >> 5; wd <= xb >> 5; wd++) {
            const int lo = max(xa, wd * 32) & 31, hi = min(xb, wd * 32 + 31) & 31;
            const uint32_t bits = (hi == 31 ? 0xffffffffu : ((1u << (hi + 1)) - 1u)) & ~((1u << lo) - 1u);
            atomicAnd(row + wd, ~bits);
        }
    }
}

__global__ void __launch_bounds__(512) detect_prepare_kernel(const DetectParams P) {
    const int f = blockIdx.x, tid = threadIdx.x;
    uint8_t* occ = P.occ + (size_t)f * (P.nch + 1) * (P.ncw + 1);
    uint32_t* mask = P.mask + (size_t)f * P.h * P.mw;
    for (int i = tid; i < (P.nch + 1) * (P.ncw + 1); i += blockDim.x) occ[i] = 0;
    for (int i = tid; i < P.h * P.mw; i += blockDim.x) mask[i] = 0xffffffffu;
    __syncthreads();
    const int n = P.ncur ? min(P.ncur[f], P.cur_cap) : 0;
    const float* cur = P.cur + (size_t)f * P.cur_cap * 2;
    const int lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    for (int i = wid; i < n; i += nw) {
        const float px = cur[2 * i], py = cur[2 * i + 1];
        // occupiedCells[px.y / cellSize][px.x / cellSize] (float division, truncation to size_t: a quotient in (-1, 0), i.e. a
        // coordinate in (-cell, 0), truncates to row / column 0; below that the conversion is undefined and nothing is marked)
        const float fr = py / (float)P.cs, fc = px / (float)P.cs;
        if (lane == 0 && fr > -1.f && fc > -1.f) {
            const long long r = (long long)fr, c = (long long)fc;
            if (r <= P.nch && c <= P.ncw) occ[r * (P.ncw + 1) + c] = 1;
        }
        clear_disk(mask, P.mw, P.w, P.h, __float2int_rn(px), __float2int_rn(py), P.rad, P.hw, lane, 32);
    }
}

// ---- D1: minimum-eigenvalue map of one cell (one CTA per cell and frame)
__global__ void __launch_bounds__(256) detect_mineig_kernel(const DetectParams P) {
    extern __shared__ float smf[];
    const int cs = P.cs, f = blockIdx.y, cell = blockIdx.x, tid = threadIdx.x;
    const int r = cell / P.ncw, c = cell - r * P.ncw;
    const int x0 = c * cs, y0 = r * cs;
    if (P.occ[(size_t)f * (P.nch + 1) * (P.ncw + 1) + r * (P.ncw + 1) + c]) return;
    if (!(x0 + cs < P.w - 1 && y0 + cs < P.h - 1)) return;
    float* rd = smf;                        // cs x (cs + 2): row-filtered [-1 0 1], rows -1..cs
    float* rs = rd + cs * (cs + 2);         // row-filtered [s 2s s]
    float* dx = rs + cs * (cs + 2);         // cs x cs
    float* dy = dx + cs * cs;
    uint8_t* blur = reinterpret_cast<uint8_t*>(dy + cs * cs);
    const uint8_t* img = P.img + (size_t)f * P.w * P.h;
    const int simd_cols = cs & ~3;
    for (int i = tid; i < cs * cs; i += blockDim.x) {
        const int y = i / cs, x = i - y * cs;
        int s = 0;
#pragma unroll
        for (int j = -1; j <= 1; j++) {
            const uint8_t* row = img + (size_t)refl(y0 + y + j, P.h) * P.w;
            const int hs = __ldg(row + refl(x0 + x - 1, P.w)) + 2 * __ldg(row + refl(x0 + x, P.w)) + __ldg(row + refl(x0 + x + 1, P.w));
            s += (j == 0 ? 2 : 1) * hs;
        }
        int q;
        if (x < simd_cols) { q = s >> 4; const int rr = s & 15; if (rr > 8 || (rr == 8 && (q & 1))) q++; }
        else q = (s + 8) >> 4;
        blur[i] = (uint8_t)q;
    }
    __syncthreads();
    const float s = (float)(1.0 / (4.0 * 3.0 * 255.0)), s2 = 2.0f * s;
    for (int i = tid; i < cs * (cs + 2); i += blockDim.x) {
        const int yy = i / cs - 1, x = i - (yy + 1) * cs;
        const uint8_t* row = blur + refl(yy, cs) * cs;
        const float a = (float)row[refl(x - 1, cs)], b = (float)row[x], cc = (float)row[refl(x + 1, cs)];
        float d = -1.0f * a; d += 0.0f * b; d += 1.0f * cc;
        float m = s * a; m += s2 * b; m += s * cc;
        rd[i] = d; rs[i] = m;
    }
    __syncthreads();
    for (int i = tid; i < cs * cs; i += blockDim.x) {
        const int y = i / cs, x = i - y * cs;
        const float d0 = rd[y * cs + x], d1 = rd[(y + 1) * cs + x], d2 = rd[(y + 2) * cs + x];
        const float t1 = d1 * s2 + 0.0f;
        dx[i] = (d0 + d2) * s + t1;
        dy[i] = rs[(y + 2) * cs + x] - rs[y * cs + x] + 0.0f;
    }
    __syncthreads();
    float* hmap = P.hmap + ((size_t)f * P.nch * P.ncw + cell) * cs * cs;
    float* hs = rd;   // the row-filter buffer is free again: keep the masked values for the two arg-max passes
    const uint32_t* mask = P.mask + (size_t)f * P.h * P.mw;
    __syncthreads();
    for (int i = tid; i < cs * cs; i += blockDim.x) {
        const int y = i / cs, x = i - y * cs;
        double A = 0, B = 0, C = 0;
#pragma unroll
        for (int j = -1; j <= 1; j++)
#pragma unroll
            for (int k = -1; k <= 1; k++) {
                const int yy = refl(y + j, cs), xx = refl(x + k, cs);
                const float gx = dx[yy * cs + xx], gy = dy[yy * cs + xx];
                A += (double)(gx * gx); B += (double)(gx * gy); C += (double)(gy * gy);
            }
        const float a = (float)A * 0.5f, b = (float)B, cc = (float)C * 0.5f;
        const float t = a - cc;
        const float v = (a + cc) - __fsqrt_rn(b * b + t * t);
        const int X = x0 + x, Y = y0 + y;
        const bool allowed = (mask[(size_t)Y * P.mw + (X >> 5)] >> (X & 31)) & 1u;   // static mask: discs of the current keypoints
        hs[i] = allowed ? v : 0.0f;
        hmap[i] = hs[i];   // stored already multiplied by the static mask (hMap.mul(mask), feature_extractor.cpp:77)
    }
    __syncthreads();
    // best and second-best (outside the best's disc) under the static mask, first index on ties -- what the reference's two
    // minMaxLoc calls return whenever no neighbouring cell's detection reaches into this cell (checked in the select kernel)
    __shared__ float red_v[8];
    __shared__ int red_i[8];
    __shared__ int s_p1;
    float4 res;
    for (int pass = 0; pass < 2; pass++) {
        const int p1 = pass ? s_p1 : -1;
        const int p1y = p1 >= 0 ? p1 / cs : 0, p1x = p1 >= 0 ? p1 - p1y * cs : 0;
        float best = -FLT_MAX;
        int bidx = 0x7fffffff;
        for (int i = tid; i < cs * cs; i += blockDim.x) {
            float v = hs[i];
            if (pass) {
                const int y = i / cs, x = i - y * cs;
                const int ady = abs(y - p1y), adx = abs(x - p1x);
                if (ady <= P.rad && adx <= P.hw[ady]) v = 0.0f;
            }
            if (v > best) { best = v; bidx = i; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, off);
            const int oi = __shfl_xor_sync(0xffffffffu, bidx, off);
            if (ob > best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
        }
        if ((tid & 31) == 0) { red_v[tid >> 5] = best; red_i[tid >> 5] = bidx; }
        __syncthreads();
        if (tid == 0) {
            for (int k = 1; k < 8; k++)
                if (red_v[k] > best || (red_v[k] == best && red_i[k] < bidx)) { best = red_v[k]; bidx = red_i[k]; }
            if (pass == 0) { s_p1 = bidx; res.x = best; res.y = __int_as_float(bidx); }
            else { res.z = best; res.w = __int_as_float(bidx); P.cand[(size_t)f * P.nch * P.ncw + cell] = res; }
        }
        __syncthreads();
    }
}

// ---- D2: serial-order selection by wavefront (one CTA per frame, one warp per cell of the current step).
// Everything a cell needs in the common case is in shared memory: its two pre-computed maxima and the detections of the
// four neighbours processed before it.  Only when a neighbour's disc covers a pre-computed maximum is the cell re-scanned
// (static bit mask AND the neighbouring / own discs); nothing is written to HBM until the final list.
// A grid too large for shared memory (kGlobalSel) keeps prim / sec / cell states in the workspace (P.sel) and reads the
// pre-computed maxima where the cell kernel left them; the arithmetic and the order are the same.
template <bool kGlobalSel>
__global__ void __launch_bounds__(512) detect_select_kernel(const DetectParams P) {
    extern __shared__ int32_t sel[];      // prim[ncells], sec[ncells]  (x | y << 16, -1 = none), then float4 cand[ncells], occ bytes
    __shared__ int s_nocc;
    __shared__ int shw[MAX_RADIUS + 1];
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    const int cs = P.cs, ncells = P.nch * P.ncw;
    if (tid <= MAX_RADIUS) shw[tid] = P.hw[tid];
    int32_t* const base = kGlobalSel ? reinterpret_cast<int32_t*>(P.sel + (size_t)f * P.sel_bytes) : sel;
    int32_t* prim = base;
    int32_t* sec = base + ncells;
    float4* scand = reinterpret_cast<float4*>(sel + 2 * ncells + ((2 * ncells) & 3 ? 4 - ((2 * ncells) & 3) : 0));
    const float4* cand = kGlobalSel ? P.cand + (size_t)f * ncells : scand;
    uint8_t* socc = kGlobalSel ? reinterpret_cast<uint8_t*>(base + 2 * ncells) : reinterpret_cast<uint8_t*>(scand + ncells);
    const uint8_t* occ = P.occ + (size_t)f * (P.nch + 1) * (P.ncw + 1);
    const double q = P.quality[f];
    if (tid == 0) s_nocc = 0;
    __syncthreads();
    int myocc = 0;
    for (int i = tid; i < ncells; i += blockDim.x) {
        const int r = i / P.ncw, c = i - r * P.ncw;
        const uint8_t o = occ[r * (P.ncw + 1) + c];
        const int x0 = c * cs, y0 = r * cs;
        const bool searched = !o && (x0 + cs < P.w - 1 && y0 + cs < P.h - 1);
        socc[i] = o ? 1 : (searched ? 0 : 2);
        myocc += o ? 1 : 0;
        prim[i] = -1; sec[i] = -1;
        if (!kGlobalSel && searched) scand[i] = P.cand[(size_t)f * ncells + i];
    }
    if (myocc) atomicAdd(&s_nocc, myocc);
    __syncthreads();
    const int nsteps = (P.ncw - 1) + 2 * (P.nch - 1) + 1;
    for (int t = 0; t < nsteps; t++) {
        const int rlo = max(0, (t - (P.ncw - 1) + 1) / 2), rhi = min(P.nch - 1, t / 2);
        for (int r = rlo + wid; r <= rhi; r += nw) {
            const int c = t - 2 * r;
            if (c < 0 || c >= P.ncw) continue;
            const int cell = r * P.ncw + c;
            if (socc[cell]) continue;
            const int x0 = c * cs, y0 = r * cs;
            // discs that can reach into this cell: detections of W, NW, N, NE (processed in earlier steps), later the own primary.
            // Fixed register slots (an absent detection sits far away), half-widths from shared memory: the test is on the
            // wavefront's critical path.
            int dcx[9], dcy[9];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int rr = r + (k == 0 ? 0 : -1), c2 = c + (k == 0 ? -1 : k - 2);
                const bool in = !(rr < 0 || c2 < 0 || c2 >= P.ncw);
#pragma unroll
                for (int which = 0; which < 2; which++) {
                    const int32_t v = in ? (which ? sec : prim)[rr * P.ncw + c2] : -1;
                    dcx[2 * k + which] = v >= 0 ? (v & 0xffff) : -30000;
                    dcy[2 * k + which] = v >= 0 ? (v >> 16) : -30000;
                }
            }
            dcx[8] = dcy[8] = -30000;
            auto covered = [&](int X, int Y) {
                bool cov = false;
#pragma unroll
                for (int k = 0; k < 9; k++) {
                    const int ady = abs(Y - dcy[k]), adx = abs(X - dcx[k]);
                    if (ady <= P.rad && adx <= shw[ady]) cov = true;
                }
                return cov;
            };
            const float4 cd = cand[cell];
            int P1idx = -1;
            for (int pass = 0; pass < 2; pass++) {
                float best;
                int bidx;
                // fast path: the pre-computed static-mask maximum stands unless a neighbour's disc covers it (the second one
                // also needs the primary to be exactly the pre-computed one: it was taken outside THAT disc)
                const float fm = pass ? cd.z : cd.x;
                const int fi = __float_as_int(pass ? cd.w : cd.y);
                bool fast = fm > 0.0f && (pass == 0 || P1idx == __float_as_int(cd.y));
                if (fast) {
                    const int fy = fi / cs, fx = fi - fy * cs;
                    fast = !covered(x0 + fx, y0 + fy);
                }
                if (P.dbg && lane == 0) {
                    atomicAdd(P.dbg + 0, 1);
                    if (!fast) atomicAdd(P.dbg + 1 + (fm > 0.0f ? (pass == 0 || P1idx == __float_as_int(cd.y) ? 2 : 1) : 0), 1);
                }
                if (fast) { best = fm; bidx = fi; }
                else {
                    // re-scan: the statically masked map (from the cell kernel) with the neighbouring / own discs applied.  Loads
                    // are issued eight deep: the scan sits on the wavefront's critical path, so its latency is what counts
                    const float* hmap = P.hmap + ((size_t)f * ncells + cell) * cs * cs;
                    best = -FLT_MAX;
                    bidx = 0x7fffffff;
                    for (int e0 = lane; e0 < cs * cs; e0 += 32 * 8) {
                        float hv[8];
#pragma unroll
                        for (int k = 0; k < 8; k++) { const int e = e0 + 32 * k; hv[k] = e < cs * cs ? __ldg(hmap + e) : -FLT_MAX; }
#pragma unroll
                        for (int k = 0; k < 8; k++) {
                            const int e = e0 + 32 * k;
                            // a disc can only lower a value to 0, so only values that could still win (or any value while the
                            // running best is negative) need the disc test
                            if (e < cs * cs && (hv[k] > best || best < 0.0f)) {
                                const int y = e / cs, x = e - y * cs;
                                const float v = covered(x0 + x, y0 + y) ? 0.0f : hv[k];
                                if (v > best) { best = v; bidx = e; }
                            }
                        }
                    }
#pragma unroll
                    for (int off = 16; off > 0; off >>= 1) {
                        const float ob = __shfl_xor_sync(0xffffffffu, best, off);
                        const int oi = __shfl_xor_sync(0xffffffffu, bidx, off);
                        if (ob > best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
                    }
                }
                const int by = bidx / cs, bx = bidx - by * cs;
                const int X = bx + x0, Y = by + y0;
                if (X < P.roi[0] || Y < P.roi[1] || X >= P.roi[0] + P.roi[2] || Y >= P.roi[1] + P.roi[3]) break;
                if (!((double)best >= q)) break;   // nothing is drawn, so the second search would repeat this one and fail alike
                if (pass == 0) { P1idx = bidx; dcx[8] = X; dcy[8] = Y; }
                if (lane == 0) (pass == 0 ? prim : sec)[cell] = X | (Y << 16);
            }
        }
        __syncthreads();
    }
    // feature_extractor.cpp:107-145: primaries in cell order, then secondaries while cells remain, quality adaptation
    if (tid == 0) {
        float* out = P.out + (size_t)f * P.out_cap * 2;
        int32_t* oi = P.out_int ? P.out_int + (size_t)f * P.out_cap * 2 : nullptr;
        int n = 0;
        auto put = [&](int32_t v) {
            if (n < P.out_cap) {
                out[2 * n] = (float)(v & 0xffff); out[2 * n + 1] = (float)(v >> 16);
                if (oi) { oi[2 * n] = v & 0xffff; oi[2 * n + 1] = v >> 16; }
            }
            n++;
        };
        for (int i = 0; i < ncells; i++) if (prim[i] >= 0) put(prim[i]);
        const int nk = n, nocc = s_nocc;
        if (nk + nocc < ncells) {
            const int nsec = ncells - (nk + nocc);
            int k = 0;
            for (int i = 0; i < ncells && k < nsec; i++) if (sec[i] >= 0) { put(sec[i]); k++; }
        }
        if ((double)n < 0.33 * (double)(ncells - nocc)) P.quality[f] = q * 0.5;
        else if ((double)n > 0.9 * (double)(ncells - nocc)) P.quality[f] = q * 1.5;
        P.counts[f] = n;
    }
}

// ---- D3: cornerSubPix, one thread per point (the reference's double sums are order-sensitive; one thread keeps the order)
__device__ void rect_subpix9(const uint8_t* __restrict__ img, int w, int h, float cx, float cy, float* out /* 9x9 */) {
    const int pw = 9;
    cx -= (pw - 1) * 0.5f; cy -= (pw - 1) * 0.5f;
    const int ipx = (int)floorf(cx), ipy = (int)floorf(cy);
    if (0 <= ipx && ipx + pw < w && 0 <= ipy && ipy + pw < h) {
        float a = cx - (float)ipx;
        const float b = cy - (float)ipy;
        a = a > 0.0001f ? a : 0.0001f;
        const float a12 = a * (1.f - b), a22 = a * b, b1 = 1.f - b, b2 = b;
        const double s = (1. - (double)a) / (double)a;
        for (int i = 0; i < pw; i++) {
            const uint8_t* r0 = img + (size_t)(ipy + i) * w + ipx;
            const uint8_t* r1 = r0 + w;
            float prev = (1 - a) * (b1 * (float)__ldg(r0) + b2 * (float)__ldg(r1));
            for (int j = 0; j < pw; j++) {
                const float t = a12 * (float)__ldg(r0 + j + 1) + a22 * (float)__ldg(r1 + j + 1);
                out[i * pw + j] = prev + t;
                prev = (float)((double)t * s);
            }
        }
    } else {
        const float a = cx - (float)ipx, b = cy - (float)ipy;
        const float a11 = (1.f - a) * (1.f - b), a12 = a * (1.f - b), a21 = (1.f - a) * b, a22 = a * b, b1 = 1.f - b, b2 = b;
        for (int i = 0; i < pw; i++) {
            int y0 = ipy + i, y1 = y0 + 1;
            y0 = y0 < 0 ? 0 : (y0 > h - 1 ? h - 1 : y0); y1 = y1 < 0 ? 0 : (y1 > h - 1 ? h - 1 : y1);
            const uint8_t* r0 = img + (size_t)y0 * w;
            const uint8_t* r1 = img + (size_t)y1 * w;
            for (int j = 0; j < pw; j++) {
                const int x0 = ipx + j, x1 = x0 + 1;
                if (x0 < 0 || x1 > w - 1) {
                    const int xc = x0 < 0 ? 0 : w - 1;
                    out[i * pw + j] = (float)r0[xc] * b1 + (float)r1[xc] * b2;
                } else
                    out[i * pw + j] = (float)r0[x0] * a11 + (float)r0[x1] * a12 + (float)r1[x0] * a21 + (float)r1[x1] * a22;
            }
        }
    }
}

__global__ void __launch_bounds__(64) corner_subpix_kernel(const DetectParams P, float* pts, const int32_t* counts, int cap,
                                                           int max_iter, double eps2) {
    const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(counts[f], cap);
    if (i >= n) return;
    const uint8_t* img = P.img + (size_t)f * P.w * P.h;
    float* p = pts + ((size_t)f * cap + i) * 2;
    const float cTx = p[0], cTy = p[1];
    float cx = cTx, cy = cTy;
    float buf[81];
    int iter = 0;
    double err = 0;
    do {
        double a = 0, b = 0, c = 0, bb1 = 0, bb2 = 0;
        rect_subpix9(img, P.w, P.h, cx, cy, buf);
        for (int ii = 0, k = 0; ii < 7; ii++) {
            const float* sp = buf + (ii + 1) * 9 + 1;
            const double py = ii - 3;
            for (int j = 0; j < 7; j++, k++) {
                const double m = P.sp_mask[k];
                const double tgx = sp[j + 1] - sp[j - 1];
                const double tgy = sp[j + 9] - sp[j - 9];
                const double gxx = tgx * tgx * m, gxy = tgx * tgy * m, gyy = tgy * tgy * m;
                const double px = j - 3;
                a += gxx; b += gxy; c += gyy;
                bb1 += gxx * px + gxy * py;
                bb2 += gxy * px + gyy * py;
            }
        }
        const double det = a * c - b * b;
        if (fabs(det) <= DBL_EPSILON * DBL_EPSILON) break;
        const double scale = 1.0 / det;
        const float nx = (float)((double)cx + c * scale * bb1 - b * scale * bb2);
        const float ny = (float)((double)cy - b * scale * bb1 + a * scale * bb2);
        err = (double)((nx - cx) * (nx - cx) + (ny - cy) * (ny - cy));
        cx = nx; cy = ny;
        if (cx < 0 || cx >= (float)P.w || cy < 0 || cy >= (float)P.h) break;
    } while (++iter < max_iter && err > eps2);
    if (fabsf(cx - cTx) > 3.f || fabsf(cy - cTy) > 3.f) { cx = cTx; cy = cTy; }
    p[0] = cx; p[1] = cy;
}

void circle_halfwidths(int radius, int* hw) {   // cv::circle's filled disk (drawing.cpp:1483-1610)
    for (int i = 0; i <= MAX_RADIUS; i++) hw[i] = -1;
    int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
    while (dx >= dy) {
        if (dx > hw[dy]) hw[dy] = dx;
        if (dy > hw[dx]) hw[dx] = dy;
        dy++;
        err += plus;
        plus += 2;
        const int mask = (err <= 0) - 1;
        err -= minus & mask;
        dx += mask;
        minus -= mask & 2;
    }
}

void subpix_mask(float* m) {   // cornersubpix.cpp:72-81 with win = 3
    for (int i = 0; i < 7; i++) {
        const float y = (float)(i - 3) / 3;
        const float vy = std::exp(-y * y);
        for (int j = 0; j < 7; j++) {
            const float x = (float)(j - 3) / 3;
            m[i * 7 + j] = (float)(vy * std::exp(-x * x));
        }
    }
}

}  // namespace

extern "C" int alva_k_corner_subpix(alva_ctx* ctx, const uint8_t* gray, int w, int h, int nframes, float* pts,
                                    const int32_t* counts, int cap) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !gray || !pts || !counts || nframes < 1 || cap < 1 || w < 11 || h < 11) { alva_set_error("alva_k_corner_subpix: bad argument"); return ALVA_E_INVALID; }
    DetectParams P{};
    P.img = gray; P.w = w; P.h = h; P.nframes = nframes;
    subpix_mask(P.sp_mask);
    corner_subpix_kernel<<<dim3((cap + 63) / 64, nframes), 64, 0, ctx->stream>>>(P, pts, counts, cap, 30, 0.01 * 0.01);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_detect_grid(alva_ctx* ctx, const uint8_t* gray, int w, int h, int nframes, int cell, const float* cur,
                                  const int32_t* ncur, int cur_cap, const int32_t* roi, double* quality, float* out,
                                  int32_t* out_int, int32_t* counts, int out_cap) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !gray || !roi || !quality || !out || !counts || nframes < 1 || out_cap < 1 || (ncur && (!cur || cur_cap < 1))) {
        alva_set_error("alva_k_detect_grid: bad argument");
        return ALVA_E_INVALID;
    }
    if (cell < 8 || cell > MAX_CELL || w < cell || h < cell || w > ALVA_MAX_DIM || h > ALVA_MAX_DIM) {
        alva_set_error("alva_k_detect_grid: cell %d (8..%d) / frame %dx%d not supported", cell, MAX_CELL, w, h);
        return ALVA_E_INVALID;
    }
    DetectParams P{};
    P.img = gray; P.w = w; P.h = h; P.nframes = nframes; P.cs = cell; P.rad = cell / 4;
    P.nch = h / cell; P.ncw = w / cell;
    P.cur = cur; P.ncur = ncur; P.cur_cap = cur_cap;
    for (int i = 0; i < 4; i++) P.roi[i] = roi[i];
    circle_halfwidths(P.rad, P.hw);
    subpix_mask(P.sp_mask);
    P.mw = (w + 31) / 32;
    const int ncells = P.nch * P.ncw;
    const size_t occ_b = (((size_t)nframes * (P.nch + 1) * (P.ncw + 1)) + 255) & ~(size_t)255;
    const size_t hmap_b = (size_t)nframes * ncells * cell * cell * sizeof(float);
    const size_t mask_b = (size_t)nframes * h * P.mw * sizeof(uint32_t);
    const size_t cand_b = (size_t)nframes * ncells * sizeof(float4);
    // the select kernel keeps its per-cell state in shared memory up to 200 KB (8 191 cells), in the workspace past that
    const size_t sm2 = (size_t)2 * ncells * sizeof(int32_t) + 16 + (size_t)ncells * (sizeof(float4) + 1);
    const bool sel_global = sm2 > 200 * 1024;
    P.sel_bytes = sel_global ? ((size_t)ncells * (2 * sizeof(int32_t) + 1) + 15) & ~(size_t)15 : 0;
    const size_t sel_b = (size_t)nframes * P.sel_bytes;
    const size_t need = occ_b + hmap_b + mask_b + cand_b + 1024 + (sel_global ? sel_b + 256 : 0);
    if (need > ctx->det_ws_bytes) {
        ctx->ws_epoch++;
        if (ctx->det_ws) { ALVA_CUDA(cudaStreamSynchronize(ctx->stream)); ALVA_CUDA(cudaFree(ctx->det_ws)); ctx->det_ws = nullptr; ctx->det_ws_bytes = 0; }
        ALVA_CUDA(cudaMalloc(&ctx->det_ws, need));
        ctx->det_ws_bytes = need;
    }
    uint8_t* ws = (uint8_t*)ctx->det_ws;
    P.occ = ws; P.hmap = (float*)(ws + occ_b); P.mask = (uint32_t*)(ws + occ_b + hmap_b);
    P.cand = (float4*)(ws + ((occ_b + hmap_b + mask_b + 255) & ~(size_t)255));
    if (sel_global) P.sel = ws + ((((occ_b + hmap_b + mask_b + 255) & ~(size_t)255) + cand_b + 255) & ~(size_t)255);
    P.quality = quality; P.out = out; P.out_int = out_int; P.counts = counts; P.out_cap = out_cap;
    static int32_t* dbg_dev = nullptr;
    static const bool dbg_on = getenv("ALVA_DETECT_DEBUG") != nullptr;
    if (dbg_on) {
        if (!dbg_dev) { ALVA_CUDA(cudaMalloc(&dbg_dev, 32)); }
        ALVA_CUDA(cudaMemsetAsync(dbg_dev, 0, 32, ctx->stream));
        P.dbg = dbg_dev;
    }
    detect_prepare_kernel<<<nframes, 512, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    const size_t sm1 = (size_t)(2 * cell * (cell + 2) + 2 * cell * cell) * sizeof(float) + (size_t)cell * cell;
    ALVA_CUDA(cudaFuncSetAttribute(detect_mineig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1));
    detect_mineig_kernel<<<dim3(ncells, nframes), 256, sm1, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    if (sel_global) detect_select_kernel<true><<<nframes, 512, 0, ctx->stream>>>(P);
    else {
        ALVA_CUDA(cudaFuncSetAttribute(detect_select_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
        detect_select_kernel<false><<<nframes, 512, sm2, ctx->stream>>>(P);
    }
    ALVA_LAUNCH_CHECK(ctx);
    corner_subpix_kernel<<<dim3((out_cap + 63) / 64, nframes), 64, 0, ctx->stream>>>(P, out, counts, out_cap, 30, 0.01 * 0.01);
    ALVA_LAUNCH_CHECK(ctx);
    if (dbg_on) {
        int32_t hdbg[8];
        ALVA_CUDA(cudaMemcpyAsync(hdbg, dbg_dev, 32, cudaMemcpyDeviceToHost, ctx->stream));
        ALVA_CUDA(cudaStreamSynchronize(ctx->stream));
        fprintf(stderr, "[detect] searches %d, re-scans: max<=0 %d, primary differs %d, covered %d\n", hdbg[0], hdbg[1], hdbg[2], hdbg[3]);
    }
    return 0;
}
