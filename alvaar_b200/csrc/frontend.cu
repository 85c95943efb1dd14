// frontend.cu -- RGBA->gray, Gaussian pyramid and FAST-9 (+score, +3x3 NMS) for sm_90a.
//
// What is computed (bit-exact with the reference; the CPU restatement is oracle/alva_oracle.c):
//   gray   : cv::cvtColor(RGBA2GRAY)           reference call site src/slam/src/system.cpp:111-112
//   pyramid: cv::pyrDown per level             src/slam/src/visual_frontend.cpp:696 -> opencv
//                                              video/src/lkpyramid.cpp:726-822, imgproc/src/pyramids.cpp:783-900
//   FAST   : cv::FAST(thr, nms, TYPE_9_16)     opencv features2d/src/fast.cpp:57-292, fast_score.cpp:119-210
//
// How (HBM-bound integer/byte work -- no tensor cores here):
//   * one CTA per 120x62 pixel tile; the RGBA box (128x70 px, 35 KB) arrives by ONE TMA bulk-tensor
//     copy (cp.async.bulk.tensor.3d, zero-filled out of bounds) signalled on an mbarrier;
//   * gray is produced once into shared memory (4 px / thread, 128-bit LDS, 32-bit STS) and streamed
//     to HBM with coalesced 32-bit stores; L1 of the pyramid is produced from the same shared tile with
//     16x2-lane SWAR arithmetic, so the input is read from HBM exactly once;
//   * FAST runs bit-sliced on 4 pixels per register (SWAR): per-byte threshold compares via the
//     borrow trick, the 9-of-16 contiguity test as 3-input LOP3 networks -- branch-free, no divergence;
//   * corners are compacted with warp ballots into per-warp shared-memory queues and scored 32 at a time
//     with packed 16x2 min/max (VIMNMX.U16x2); NMS is again SWAR over the shared score tile;
//   * keypoints leave as packed keys (y<<20 | x<<8 | score); a row-bucket pass restores cv::FAST's
//     row-major order when the caller asks for it.
#include "alva_common.cuh"
#include "fast_swar.h"
#include "../../include/alva_b200.h"
#include <stdlib.h>
#include <algorithm>

namespace {

constexpr int TW = 120, TH = 62;          // tile interior
constexpr int BW = TW + 8, BH = TH + 8;   // loaded box (halo 4)
constexpr int GP = 144;                   // gray smem pitch (bytes); image x0 sits at byte 8
constexpr int GPW = GP / 4;
constexpr int SP = 128;                   // score smem pitch; image x0-4 sits at byte 0
constexpr int SPW = SP / 4;
constexpr int SR = TH + 2;                // score rows: image y0-1 .. y0+TH
constexpr int NTHREADS = 256;
constexpr int NWARPS = NTHREADS / 32;
constexpr int QCAP = 1024;                // per-warp candidate queue (32 lanes x 8 rows x 4 px): lives in the idle RGBA staging buffer
constexpr int KPCAP = 1888;               // >= TW*TH/4 (NMS leaves at most one keypoint per 2x2)

struct FrontendParams {
    const uint8_t* src;   // rgba (RGBA mode) or gray (gray mode), tightly packed frames
    uint8_t* l0;          // gray out (RGBA mode), may be null
    uint8_t* l1;          // first pyramid level out, may be null
    uint32_t* keys;       // may be null (no FAST)
    int32_t* counts;
    int w, h, nframes, tiles_x, tiles_y;
    int thr, cap, use_tma;
    int prefetch;         // variant 2: frames ahead whose tile (same position) is pulled into L2 while this one is processed; 0 = off
    uint32_t mul[7];      // 2^(25+i): kept as run-time data so the row-packing multiply-high stays an FMA-pipe IMAD.HI
};

struct __align__(128) SmemLayout {
    uint8_t rgba[BW * BH * 4];     // TMA destination (RGBA mode); after the gray pass it is reused for the per-warp queues
                                   // (first NWARPS*QCAP*2 bytes) and the tile's keypoint list (KPCAP words after them)
    uint8_t gray[GP * BH];         // TMA destination (gray mode)
    uint8_t score[SP * SR];
    uint64_t bar;
    int kpcount;
    int kpbase;
};

// ---- gray conversion of 4 RGBA pixels (uint4 = 4 x RGBA8) ------------------------------------------
// Y = (9798 R + 19235 G + 3735 B + 2^14) >> 15.  With every term doubled the result is byte 2 of the accumulator, so
// two 16x8-bit dot-product instructions (IDP.2A, FMA pipe) per pixel and three PRMT per four pixels do the whole job.
__device__ __forceinline__ uint32_t gray_acc(uint32_t px) {
    return __dp2a_hi(7470u, px, __dp2a_lo(19596u | (38470u << 16), px, 32768u));
}
__device__ __forceinline__ uint32_t gray1(uint32_t px) { return gray_acc(px) >> 16; }
__device__ __forceinline__ uint32_t gray4(uint4 p) {
    const uint32_t lo = __byte_perm(gray_acc(p.x), gray_acc(p.y), 0x0062);
    const uint32_t hi = __byte_perm(gray_acc(p.z), gray_acc(p.w), 0x0062);
    return __byte_perm(lo, hi, 0x5410);
}

// ---- FAST-9 candidate test, bit-sliced over 4 pixels x 8 rows --------------------------------------
// A pixel can only be a FAST-9 corner if 9 contiguous ring pixels differ from the centre by more than t (either sign).
// |ring - c| comes from one VABSDIFF4 per ring element and four pixels, "> t" from the add-and-carry trick, and the
// resulting bit-7 flags of EIGHT rows are packed into one 32-bit word per ring element (a 64-bit multiply-add on the
// FMA pipe does the shift-and-accumulate), so the 9-of-16 contiguity network (40 LOP3) runs once per 32 pixels.
// Candidates then get their exact score (both polarities) in fast_strength2(); score > t decides cornerness exactly
// as cornerScore / the ring test do in the reference.
template <bool HI_THR>
__device__ __forceinline__ uint32_t absdiff_gt(uint32_t ring, uint32_t c, uint32_t K) {
    const uint32_t a = __vabsdiffu4(ring, c);
    const uint32_t sum = (a & ALVA_L) + K;
    return HI_THR ? (sum & a & ALVA_H) : ((sum | a) & ALVA_H);
}

// exact corner strength of one pixel: max over the 16 arcs of min over the arc of (ring - c) [bright] or (c - ring) [dark]
__device__ __forceinline__ int fast_strength2(const uint8_t* p) {
    constexpr int o[16] = {3 * GP,      3 * GP + 1,  2 * GP + 2,  GP + 3,      3,           -GP + 3,
                           -2 * GP + 2, -3 * GP + 1, -3 * GP,     -3 * GP - 1, -2 * GP - 2, -GP - 3,
                           -3,          GP - 3,      2 * GP - 2,  3 * GP - 1};
    const uint32_t c = p[0];
    const uint32_t bias = 0x01000100u - (c | (c << 16));
    // e[k] = (ring_k - c + 256, ring_{k+8} - c + 256) as two unsigned 16-bit lanes; es = halves swapped
    uint32_t e[8], es[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        e[k] = ((uint32_t)p[o[k]] | ((uint32_t)p[o[k + 8]] << 16)) + bias;
        es[k] = __byte_perm(e[k], 0, 0x1032);
    }
    // register k of a 16-long circular sequence holds elements (k, k + 8); index m >= 8 is the swapped register m - 8
#define CIRC(arr, sw, m) ((m) < 8 ? arr[(m)] : sw[(m) - 8])
    uint32_t tn[8], tx[8], tns[8], txs[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        tn[k] = __vimin3_u16x2(e[k], CIRC(e, es, k + 1), CIRC(e, es, k + 2));
        tx[k] = __vimax3_u16x2(e[k], CIRC(e, es, k + 1), CIRC(e, es, k + 2));
    }
#pragma unroll
    for (int k = 0; k < 6; k++) { tns[k] = __byte_perm(tn[k], 0, 0x1032); txs[k] = __byte_perm(tx[k], 0, 0x1032); }
    uint32_t bmax = 0, dmin = 0xffffffffu;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t a9n = __vimin3_u16x2(tn[k], CIRC(tn, tns, k + 3), CIRC(tn, tns, k + 6));
        const uint32_t a9x = __vimax3_u16x2(tx[k], CIRC(tx, txs, k + 3), CIRC(tx, txs, k + 6));
        bmax = __vmaxu2(bmax, a9n);
        dmin = __vminu2(dmin, a9x);
    }
#undef CIRC
    const int sb = (int)max(bmax & 0xffffu, bmax >> 16) - 256;     // bright: max_arc min(ring - c)
    const int sd = 256 - (int)min(dmin & 0xffffu, dmin >> 16);     // dark:   max_arc min(c - ring)
    return max(sb, sd);
}

// Candidate mask of one lane's 4-pixel column over 8 rows (bit 8j + i = pixel j, row i): 9 contiguous ring pixels differ
// from the centre by more than t.  g0 points at the word of the lane's pixels in the first of the 14 gray rows involved.
template <bool HI_THR>
__device__ __forceinline__ uint32_t fast_candidates8(const uint32_t* g0, uint32_t K, const uint32_t* mul) {
    // gray rows needed: centre rows r0 .. r0+7 with r0 = 8*warp + 3, i.e. rows 8*warp .. 8*warp + 13 (< BH = 70)
    uint32_t Lw[7], Mw[7], Rw[7];   // rolling 7-row window: slot (row % 7)
    uint32_t mulreg[7];
#pragma unroll
    for (int i = 0; i < 7; i++) mulreg[i] = mul[i];
#pragma unroll
    for (int r = 0; r < 6; r++) { Lw[r] = g0[r * GPW - 1]; Mw[r] = g0[r * GPW]; Rw[r] = g0[r * GPW + 1]; }
    uint32_t acc[16];
#pragma unroll
    for (int k = 0; k < 16; k++) acc[k] = 0u;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        {   // bring in window row i + 6
            const int r = i + 6;
            Lw[r % 7] = g0[r * GPW - 1]; Mw[r % 7] = g0[r * GPW]; Rw[r % 7] = g0[r * GPW + 1];
        }
        // window rows i .. i+6 <-> dy = -3 .. +3
#define WL(dy) Lw[(i + 3 + (dy)) % 7]
#define WM(dy) Mw[(i + 3 + (dy)) % 7]
#define WR(dy) Rw[(i + 3 + (dy)) % 7]
        uint32_t ring[16];
        ring[0] = WM(3);
        ring[1] = __byte_perm(WM(3), WR(3), 0x4321);
        ring[15] = __byte_perm(WL(3), WM(3), 0x6543);
        ring[2] = __byte_perm(WM(2), WR(2), 0x5432);
        ring[14] = __byte_perm(WL(2), WM(2), 0x5432);
        ring[3] = __byte_perm(WM(1), WR(1), 0x6543);
        ring[13] = __byte_perm(WL(1), WM(1), 0x4321);
        ring[4] = __byte_perm(WM(0), WR(0), 0x6543);
        ring[12] = __byte_perm(WL(0), WM(0), 0x4321);
        ring[5] = __byte_perm(WM(-1), WR(-1), 0x6543);
        ring[11] = __byte_perm(WL(-1), WM(-1), 0x4321);
        ring[6] = __byte_perm(WM(-2), WR(-2), 0x5432);
        ring[10] = __byte_perm(WL(-2), WM(-2), 0x5432);
        ring[7] = __byte_perm(WM(-3), WR(-3), 0x4321);
        ring[8] = WM(-3);
        ring[9] = __byte_perm(WL(-3), WM(-3), 0x6543);
        const uint32_t c = WM(0);
#undef WL
#undef WM
#undef WR
        // flag (bit 7 of byte j) -> bit 8j + i of the packed word: hi32(U * 2^(25+i)) == U >> (7 - i).  mad.hi keeps the
        // shift-and-accumulate on the FMA pipe (a plain shift would be strength-reduced onto the saturated ALU pipe);
        // row 7 needs no shift at all.
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const uint32_t U = absdiff_gt<HI_THR>(ring[k], c, K);
            if (i < 7) asm("mad.hi.u32 %0, %1, %2, %0;" : "+r"(acc[k]) : "r"(U), "r"(mulreg[i]));
            else acc[k] += U;
        }
    }
    uint32_t T[16];
#pragma unroll
    for (int k = 0; k < 16; k++) T[k] = acc[k] & acc[(k + 1) & 15] & acc[(k + 2) & 15];
    uint32_t cand = 0;
#pragma unroll
    for (int k = 0; k < 16; k++) cand |= T[k] & T[(k + 3) & 15] & T[(k + 6) & 15];
    return cand;
}

template <bool RGBA, bool ANTI = false>
__global__ void __launch_bounds__(NTHREADS, 4)
frontend_tile_kernel(const __grid_constant__ CUtensorMap tmap, const FrontendParams P) {
    extern __shared__ uint8_t smem_raw[];
    // TMA destinations must be 128-byte aligned: align the dynamic window by hand (128 spare bytes are allocated)
    SmemLayout& S = *reinterpret_cast<SmemLayout*>(smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u));

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int t = blockIdx.x;
    const int tiles_per_frame = P.tiles_x * P.tiles_y;
    const int f = t / tiles_per_frame;
    t -= f * tiles_per_frame;
    const int ty = t / P.tiles_x, tx = t - ty * P.tiles_x;
    const int x0 = tx * TW, y0 = ty * TH;
    const int w = P.w, h = P.h;
    // TMA needs the box start 16-byte aligned along the innermost dimension.  RGBA: (x0-4)*4 B is always a multiple of 16.
    // Gray (u8): x0-8 is 0 or 8 mod 16, so the box starts `sh` bytes earlier and the tile sits `sh` bytes further right
    // in the shared rows (pitch 144 still covers x0-8 .. x0+TW+7).
    const int sh = RGBA ? 0 : ((x0 - 8) & 15);
    const int cbw = 1 + (sh >> 2);   // word index (within a gray smem row) of image column x0-4

    // ------------------------------------------------------------------ A. load the tile
    if (P.use_tma) {
        if (tid == 0) {
            mbar_init(&S.bar, 1);
            fence_barrier_init();
        }
        __syncthreads();
        if (tid == 0) {
            if (RGBA) {
                mbar_arrive_expect_tx(&S.bar, BW * BH * 4);
                tma_load_3d(S.rgba, &tmap, &S.bar, x0 - 4, y0 - 4, f);
            } else {
                mbar_arrive_expect_tx(&S.bar, GP * BH);
                tma_load_3d(S.gray, &tmap, &S.bar, x0 - 8 - sh, y0 - 4, f);
            }
        }
    } else {
        if (RGBA) {
            const uint32_t* src = reinterpret_cast<const uint32_t*>(P.src) + (size_t)f * w * h;
            uint32_t* dst = reinterpret_cast<uint32_t*>(S.rgba);
            for (int i = tid; i < BW * BH; i += NTHREADS) {
                const int by = i / BW, bx = i - by * BW;
                const int x = x0 - 4 + bx, y = y0 - 4 + by;
                dst[i] = (x >= 0 && x < w && y >= 0 && y < h) ? __ldg(src + (size_t)y * w + x) : 0u;
            }
        } else {
            const uint8_t* src = P.src + (size_t)f * w * h;
            for (int i = tid; i < GP * BH; i += NTHREADS) {
                const int by = i / GP, bx = i - by * GP;
                const int x = x0 - 8 - sh + bx, y = y0 - 4 + by;
                S.gray[i] = (x >= 0 && x < w && y >= 0 && y < h) ? __ldg(src + (size_t)y * w + x) : 0;
            }
        }
    }
    // zero the score tile and counters while the copy is in flight
    {
        uint32_t* sc = reinterpret_cast<uint32_t*>(S.score);
        for (int i = tid; i < SP * SR / 4; i += NTHREADS) sc[i] = 0;
        if (tid == 0) S.kpcount = 0;
    }
    if (P.use_tma) mbar_wait(&S.bar, 0);
    else __syncthreads();

    // ------------------------------------------------------------------ B. gray
    if (RGBA) {
        const uint4* src4 = reinterpret_cast<const uint4*>(S.rgba);
        uint32_t* gw = reinterpret_cast<uint32_t*>(S.gray);
        uint8_t* l0 = P.l0 ? P.l0 + (size_t)f * w * h : nullptr;
        const bool w4 = (w & 3) == 0;
        const int g = lane;                                   // BW/4 == 32 groups per row: lane = group
        const int x = x0 + 4 * (g - 1);
        const bool colstore = l0 && g >= 1 && g <= 30 && x < w;
        // warp `warp` converts box rows warp, warp + 8, ... (9 rounds, the last one only for rows < BH).  Fully unrolled with
        // pointer increments: all loads of a warp are in flight together and the per-row index arithmetic disappears.
        constexpr int ROUNDS = (BH + NWARPS - 1) / NWARPS;
        const uint4* sp = src4 + warp * 32 + g;
        uint32_t* gp = gw + warp * GPW + 1 + g;             // image x0-4+4g at gray byte 4+4g
        uint4 px[ROUNDS];
#pragma unroll
        for (int it = 0; it < ROUNDS; it++)
            if (it < ROUNDS - 1 || warp + NWARPS * it < BH) px[it] = sp[it * NWARPS * 32];
        uint8_t* d = l0 ? l0 + (size_t)(y0 + warp - 4) * w + x : nullptr;
        const size_t dstep = (size_t)NWARPS * w;
        if (ANTI && w4) {
            // experimental instantiation: the same conversion and stores with the row / width tests hoisted out of the rounds
            // (the default loop below re-tests w % 4 and carries the byte-store fallback in every round: more predicate and
            // branch scaffolding than arithmetic)
            const int by_end = min(4 + TH, h - y0 + 4);   // box rows [4, by_end) are image rows of this tile
#pragma unroll
            for (int it = 0; it < ROUNDS; it++) {
                const int by = warp + NWARPS * it;
                if (it < ROUNDS - 1 || by < BH) {
                    const uint32_t v = gray4(px[it]);
                    gp[it * NWARPS * GPW] = v;
                    if (colstore && (it > 0 || by >= 4) && by < by_end) *reinterpret_cast<uint32_t*>(d + it * dstep) = v;
                }
            }
        } else
#pragma unroll
        for (int it = 0; it < ROUNDS; it++) {
            const int by = warp + NWARPS * it;
            if (it < ROUNDS - 1 || by < BH) {
                const uint32_t v = gray4(px[it]);
                gp[it * NWARPS * GPW] = v;
                const int y = y0 + by - 4;
                if (colstore && by >= 4 && by < 4 + TH && y < h) {
                    uint8_t* dd = d + it * dstep;
                    if (w4) *reinterpret_cast<uint32_t*>(dd) = v;  // x % 4 == 0 and w % 4 == 0 -> aligned, in range
                    else
                        for (int j = 0; j < 4 && x + j < w; j++) dd[j] = (uint8_t)(v >> (8 * j));
                }
            }
        }
        // columns x0-8..x0-5 and x0+TW+4..x0+TW+7 are never written: only garbage lanes read them
    }
    __syncthreads();

    // reflect-101 fix-up of the 2-px halo outside the image (pyrDown borders).  FAST never reads it:
    // its candidates lie >= 3 px inside the image.
    const bool edge_l = (x0 == 0), edge_r = (x0 + TW >= w), edge_t = (y0 == 0), edge_b = (y0 + TH >= h);
    if (P.l1 && (edge_l || edge_r || edge_t || edge_b)) {
        if (edge_l || edge_r) {
            for (int r = tid; r < BH; r += NTHREADS) {
                uint8_t* row = S.gray + r * GP;
                if (edge_l) { row[7 + sh] = row[9 + sh]; row[6 + sh] = row[10 + sh]; }
                if (edge_r) {
                    const int cw = w - x0 + 8 + sh;   // gray byte of image column w
                    row[cw] = row[cw - 2];
                    row[cw + 1] = row[cw - 3];
                }
            }
            __syncthreads();
        }
        if (edge_t || edge_b) {
            for (int c = tid; c < GP; c += NTHREADS) {
                if (edge_t) { S.gray[3 * GP + c] = S.gray[5 * GP + c]; S.gray[2 * GP + c] = S.gray[6 * GP + c]; }
                if (edge_b) {
                    const int rh = h - y0 + 4;   // gray row of image row h
                    S.gray[rh * GP + c] = S.gray[(rh - 2) * GP + c];
                    S.gray[(rh + 1) * GP + c] = S.gray[(rh - 3) * GP + c];
                }
            }
            __syncthreads();
        }
    }

    const uint32_t* G = reinterpret_cast<const uint32_t*>(S.gray);

    // ------------------------------------------------------------------ C. pyramid level 1
    // [1 4 6 4 1] x [1 4 6 4 1] / 256 on even pixels.  Horizontal taps are 8-bit dot products (IDP.4A, FMA pipe) on the
    // packed gray words; a thread owns two adjacent outputs and four output rows (11 input rows, rolling).
    if (P.l1) {
        const int w1 = (w + 1) >> 1, h1 = (h + 1) >> 1;
        uint8_t* l1 = P.l1 + (size_t)f * w1 * h1;
        const int pc = tid % 30, sg = tid / 30;   // 30 pair-columns x 8 row segments (threads 240..255 idle)
        if (sg < 8) {
            const int lx = (x0 >> 1) + 2 * pc;
            const int ly0 = (y0 >> 1) + 4 * sg;
            if (lx < w1 && ly0 < h1) {
                const uint32_t* base = G + (8 * sg + 2) * GPW + cbw + pc;   // gray row 2j+2 for j = 4*sg
                uint32_t hA[11], hB[11];
#pragma unroll
                for (int r = 0; r < 11; r++) {
                    const uint32_t L = base[r * GPW], M = base[r * GPW + 1], R = base[r * GPW + 2];
                    // output A centred on M0: L2 L3 M0 M1 M2 ; output B centred on M2: M0 M1 M2 M3 R0
                    hA[r] = __dp4a(__byte_perm(L, M, 0x5432), 0x04060401u, __dp4a(M, 0x00010000u, 0u));
                    hB[r] = __dp4a(M, 0x04060401u, __dp4a(R, 0x00000001u, 0u));
                }
                const bool pair_ok = (lx + 1 < w1), al16 = ((w1 & 1) == 0);
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int ly = ly0 + j;
                    if (ly < h1 && 4 * sg + j < TH / 2) {
                        const uint32_t vA = hA[2 * j] + hA[2 * j + 4] + (hA[2 * j + 1] + hA[2 * j + 3]) * 4u + hA[2 * j + 2] * 6u + 128u;
                        const uint32_t vB = hB[2 * j] + hB[2 * j + 4] + (hB[2 * j + 1] + hB[2 * j + 3]) * 4u + hB[2 * j + 2] * 6u + 128u;
                        const uint32_t o = __byte_perm(vA, vB, 0x0051);   // (vA >> 8) & 255 | ((vB >> 8) & 255) << 8
                        uint8_t* d = l1 + (size_t)ly * w1 + lx;
                        if (pair_ok && al16) *reinterpret_cast<uint16_t*>(d) = (uint16_t)o;
                        else { d[0] = (uint8_t)o; if (pair_ok) d[1] = (uint8_t)(o >> 8); }
                    }
                }
            }
        }
    }

    // ------------------------------------------------------------------ D. FAST candidates + exact score
    // warp w owns score rows 8w .. 8w+7 (image rows y0-1+8w ..); lane = 4-pixel group column (image x0-4+4*lane ..)
    uint16_t* Q = reinterpret_cast<uint16_t*>(S.rgba) + warp * QCAP;   // the RGBA staging buffer is idle from here on
    uint32_t* kplist = reinterpret_cast<uint32_t*>(S.rgba + NWARPS * QCAP * 2);
    static_assert(NWARPS * QCAP * 2 + KPCAP * 4 <= BW * BH * 4, "queues + keypoint list must fit the staging buffer");
    int qn = 0;   // candidates in this warp's queue (phase D fills it, phase E walks it again)
    if (P.keys) {
        const int thr = P.thr;
        const bool hi_thr = thr >= 128;
        const uint32_t K = (uint32_t)(hi_thr ? 255 - thr : 127 - thr) * 0x01010101u;
        // validity of this lane's 4 pixels (columns) and of the warp's 8 rows, as a (8j + i) bit mask
        uint32_t vm;
        {
            const int xlo = max(3, x0 - 1), xhi = min(w - 4, x0 + TW);
            const int ylo = max(3, y0 - 1), yhi = min(h - 4, y0 + TH);
            const int yb = y0 - 1 + 8 * warp;                 // image row of bit 0
            const int r0v = max(ylo - yb, 0), r1v = min(yhi - yb, 7);   // valid row bits [r0v, r1v]
            const uint32_t rowbits = r1v >= r0v ? ((0xffu >> (7 - r1v)) & (0xffu << r0v)) & 0xffu : 0u;
            const int xb = x0 - 4 + 4 * lane;                 // image column of byte 0
            const int c0v = max(xlo - xb, 0), c1v = min(xhi - xb, 3);   // valid bytes [c0v, c1v]
            const uint32_t colbytes = c1v >= c0v ? ((0x01010101u >> (8 * (3 - c1v))) & (0x01010101u << (8 * c0v))) : 0u;
            vm = colbytes * rowbits;                          // rowbits replicated into every valid byte
        }
        if (__any_sync(0xffffffffu, vm != 0)) {
            // gray rows needed: centre rows 8*warp+3 .. 8*warp+10, i.e. rows 8*warp .. 8*warp + 13 (< BH = 70)
            const uint32_t* g0 = G + (8 * warp) * GPW + cbw + lane;
            uint32_t cand;
            if (ANTI) {
                // experimental (alva_set_option("frontend_antipodal", 1)): 8 of the 16 ring flag words are assembled from their
                // antipodal partners instead of recomputed -- fast_swar.h; its host emulation is checked in the CPU suite
                uint32_t acc[16];
                if (hi_thr) fast_swar::phase1<true, GPW>(g0, K, P.mul, acc); else fast_swar::phase1<false, GPW>(g0, K, P.mul, acc);
#define ALVA_ASM_LEFT(M)  { const uint32_t o_ = acc[fast_swar::source_of(M)]; acc[M] = fast_swar::assemble<M>(o_, __shfl_up_sync(0xffffffffu, o_, 1), 0u, acc[M]); }
#define ALVA_ASM_RIGHT(M) { const uint32_t o_ = acc[fast_swar::source_of(M)]; acc[M] = fast_swar::assemble<M>(o_, 0u, __shfl_down_sync(0xffffffffu, o_, 1), acc[M]); }
                ALVA_ASM_RIGHT(5) ALVA_ASM_RIGHT(6) ALVA_ASM_RIGHT(7)       // sources 13, 14, 15: dx < 0 -> pixels to the right
                acc[8] = fast_swar::assemble<8>(acc[0], 0u, 0u, acc[8]);    // source 0: dx = 0
                ALVA_ASM_LEFT(9) ALVA_ASM_LEFT(10) ALVA_ASM_LEFT(11) ALVA_ASM_LEFT(12)   // sources 1..4: dx > 0 -> pixels to the left
#undef ALVA_ASM_LEFT
#undef ALVA_ASM_RIGHT
                cand = fast_swar::contiguous9(acc);
            } else {
                cand = hi_thr ? fast_candidates8<true>(g0, K, P.mul) : fast_candidates8<false>(g0, K, P.mul);
            }
            cand &= vm;
            // ordered compaction of the candidate pixels into the warp queue (one prefix sum per 8 rows)
            const int mine = __popc(cand);
            int incl = mine;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += v; }
            int pos = incl - mine;
            qn = __shfl_sync(0xffffffffu, incl, 31);
            const int pixbase = (8 * warp + 3) * GP + 4 * (cbw + lane);
            while (cand) {
                const int b = __ffs(cand) - 1;
                cand &= cand - 1;
                Q[pos++] = (uint16_t)(pixbase + (b & 7) * GP + (b >> 3));
            }
            __syncwarp();
            for (int q0 = 0; q0 < qn; q0 += 32) {
                if (q0 + lane < qn) {
                    const int pix = Q[q0 + lane];
                    const int sc = fast_strength2(S.gray + pix);
                    if (sc > thr) {
                        const int pr = pix / GP, pcg = pix - pr * GP;
                        S.score[(pr - 3) * SP + (pcg - 4 * cbw)] = (uint8_t)(sc - 1);
                    }
                }
            }
        }
    }
    __syncthreads();

    // ------------------------------------------------------------------ E. 3x3 NMS (strict >) + emit
    // The warp's candidate queue is walked a second time: a candidate that became a corner (non-zero score, inside the tile
    // interior) is compared with its 8 neighbours in the shared score tile.  Only corners pay for the neighbour loads
    // (~4 % of the pixels); nothing scans the score tile.
    if (P.keys) {
        for (int q0 = 0; q0 < qn; q0 += 32) {
            bool iskp = false;
            uint32_t key = 0;
            if (q0 + lane < qn) {
                const int pix = Q[q0 + lane];
                const int pr = pix / GP, pcg = pix - pr * GP;
                const int sr = pr - 3, scol = pcg - 4 * cbw;          // score-tile row / column (column 4 = image x0)
                if (sr >= 1 && sr <= TH && scol >= 4 && scol < 4 + TW) {
                    const uint8_t* sp = S.score + sr * SP + scol;
                    const uint32_t v = sp[0];
                    if (v) {
                        const uint32_t m = max(max(max((uint32_t)sp[-SP - 1], (uint32_t)sp[-SP]), max((uint32_t)sp[-SP + 1], (uint32_t)sp[-1])),
                                               max(max((uint32_t)sp[1], (uint32_t)sp[SP - 1]), max((uint32_t)sp[SP], (uint32_t)sp[SP + 1])));
                        iskp = v > m;
                        key = ((uint32_t)(y0 + sr - 1) << 20) | ((uint32_t)(x0 + scol - 4) << 8) | v;
                    }
                }
            }
            const uint32_t mk = __ballot_sync(0xffffffffu, iskp);
            if (mk) {
                int base = 0;
                if (lane == 0) base = atomicAdd(&S.kpcount, __popc(mk));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (iskp) {
                    const int kp = base + __popc(mk & ((1u << lane) - 1u));
                    if (kp < KPCAP) kplist[kp] = key;
                }
            }
        }
        __syncthreads();
        const int n = min(S.kpcount, KPCAP);
        if (tid == 0) S.kpbase = n ? atomicAdd(P.counts + f, n) : 0;
        __syncthreads();
        const int base = S.kpbase;
        uint32_t* out = P.keys + (size_t)f * P.cap;
        for (int i = tid; i < n; i += NTHREADS)
            if (base + i < P.cap) out[base + i] = kplist[i];
    }
}

// ======================================================================================== variant 2
// Same tile geometry, same results; what changed against frontend_tile_kernel:
//   * gray: row / width tests hoisted out of the rounds (the conversion is little arithmetic and much scaffolding);
//   * pyramid L1: a thread owns 4 adjacent outputs x 2 rows (7 gray rows x {LDS.32, LDS.64, LDS.32}) instead of 2 x 4;
//   * FAST pre-test with antipodal flag sharing (fast_swar.h);
//   * candidate compaction on the TRANSPOSED bit matrix: a lane's 4 x 8 pixel block is either empty or crowded (corner
//     clusters), so the per-lane emit loop runs with few active lanes; after a 32 x 32 bit transpose across the warp (2 PRMT + 3
//     mask stages on SHFL.BFLY) lane b owns bit position b = (pixel j, row i) of all 32 lanes -- pixels 4 apart in one row,
//     which no cluster fills -- and the loop is balanced.  The queue order that results (same row, distinct words) also makes
//     the 16 ring loads of the scoring phase almost bank-conflict free;
//   * the scoring loop compacts the true corners of the tile interior in place (queue prefix), so the NMS / emit phase walks
//     ~4 % of the pixels with full lanes instead of re-walking every candidate; the score tile has a 33-word pitch.
//   * 120 x 60 tiles (720 and 1080 are multiples of 60: no ragged bottom row) and the score tile folded into the idle RGBA
//     staging buffer: 44.8 KB of shared memory per CTA instead of 54.4 -> 5 CTAs per SM (40 warps) instead of 4.
//   * a (tiles_x, tiles_y, frames) grid instead of two run-time divisions per warp; each warp sends its keypoints straight to the frame's list (one global
//     atomic per warp) instead of a tile list + two barriers + a copy loop; the pyramid's edge words come from the neighbour
//     lanes (instead of 2-way bank-conflicted 32-bit loads); 128-bit score clears;
//     optionally the tile `prefetch` frames ahead is pulled into L2 by TMA.
constexpr int TH2 = 60, BH2 = TH2 + 8;    // tile interior rows / loaded box rows
constexpr int SR2 = TH2 + 2;              // score rows: image y0-1 .. y0+TH2
constexpr int SP2 = 132;                  // score pitch: 33 words -> rows rotate through the banks
struct __align__(128) SmemLayout2 {
    // TMA destination (RGBA mode).  After the gray pass: per-warp queues (NWARPS * QCAP u16) and the score tile (SP2 bytes x
    // 8 rows per warp)
    uint8_t rgba[BW * BH2 * 4];
    uint8_t gray[GP * (BH2 + 2)];  // TMA destination (gray mode); + 2 rows: the last warp's pre-test window (8 * 7 + 14 rows) reads
                                   // two rows past the box -- they only feed pixels its validity mask drops
    uint64_t bar;
};
constexpr int V2_SCORE_OFF = NWARPS * QCAP * 2;
static_assert(V2_SCORE_OFF % 16 == 0 && (8 * SP2) % 16 == 0 && V2_SCORE_OFF + SP2 * 8 * NWARPS <= BW * BH2 * 4,
              "queues + score tile must fit the staging buffer; 128-bit clears");
static_assert(NWARPS * 8 >= SR2, "8 score rows per warp");

template <bool RGBA>
__global__ void __launch_bounds__(NTHREADS, 5)
frontend_tile_kernel_v2(const __grid_constant__ CUtensorMap tmap, const FrontendParams P) {
    extern __shared__ uint8_t smem_raw[];
    SmemLayout2& S = *reinterpret_cast<SmemLayout2*>(smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u));

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tx = blockIdx.x, ty = blockIdx.y, f = blockIdx.z;
    const int x0 = tx * TW, y0 = ty * TH2;
    const int w = P.w, h = P.h;
    const int sh = RGBA ? 0 : ((x0 - 8) & 15);
    const int cbw = 1 + (sh >> 2);   // word index (within a gray smem row) of image column x0-4

    // ------------------------------------------------------------------ A. load the tile (TMA only: the launcher falls back
    // to the baseline kernel for geometries the tensor map cannot express)
    if (tid == 0) {
        mbar_init(&S.bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (tid == 0) {
        if (RGBA) {
            mbar_arrive_expect_tx(&S.bar, BW * BH2 * 4);
            tma_load_3d(S.rgba, &tmap, &S.bar, x0 - 4, y0 - 4, f);
        } else {
            mbar_arrive_expect_tx(&S.bar, GP * BH2);
            tma_load_3d(S.gray, &tmap, &S.bar, x0 - 8 - sh, y0 - 4, f);
        }
        if (P.prefetch && f + P.prefetch < P.nframes) {
            if (RGBA) tma_prefetch_l2_3d(&tmap, x0 - 4, y0 - 4, f + P.prefetch);
            else tma_prefetch_l2_3d(&tmap, x0 - 8 - sh, y0 - 4, f + P.prefetch);
        }
    }
    mbar_wait(&S.bar, 0);

    // ------------------------------------------------------------------ B. gray (w % 4 == 0 guaranteed by the TMA path)
    if (RGBA) {
        const uint4* src4 = reinterpret_cast<const uint4*>(S.rgba);
        uint32_t* gw = reinterpret_cast<uint32_t*>(S.gray);
        uint8_t* l0 = P.l0 ? P.l0 + (size_t)f * w * h : nullptr;
        const int g = lane;
        const int x = x0 + 4 * (g - 1);
        const bool colstore = l0 && g >= 1 && g <= 30 && x < w;
        constexpr int ROUNDS = (BH2 + NWARPS - 1) / NWARPS;
        const uint4* sp = src4 + warp * 32 + g;
        uint32_t* gp = gw + warp * GPW + 1 + g;
        uint4 px[ROUNDS];
#pragma unroll
        for (int it = 0; it < ROUNDS; it++)
            if (it < ROUNDS - 1 || warp + NWARPS * it < BH2) px[it] = sp[it * NWARPS * 32];
        uint8_t* d = l0 ? l0 + (ptrdiff_t)(y0 + warp - 4) * w + x : nullptr;
        const size_t dstep = (size_t)NWARPS * w;
        const int by_end = min(4 + TH2, h - y0 + 4);   // box rows [4, by_end) are image rows of this tile
#pragma unroll
        for (int it = 0; it < ROUNDS; it++) {
            const int by = warp + NWARPS * it;
            if (it < ROUNDS - 1 || by < BH2) {
                const uint32_t v = gray4(px[it]);
                gp[it * NWARPS * GPW] = v;
                if (colstore && (it > 0 || by >= 4) && by < by_end) *reinterpret_cast<uint32_t*>(d + it * dstep) = v;
            }
        }
    }
    __syncthreads();

    // the staging buffer is idle from here on: every warp clears the 8 score rows it will write in phase D
    uint8_t* const score = S.rgba + V2_SCORE_OFF;
    {
        uint4* sc = reinterpret_cast<uint4*>(score + warp * 8 * SP2);
#pragma unroll
        for (int i = 0; i < (8 * SP2 / 16 + 31) / 32; i++)
            if (lane + 32 * i < 8 * SP2 / 16) sc[lane + 32 * i] = make_uint4(0u, 0u, 0u, 0u);
    }

    const bool edge_l = (x0 == 0), edge_r = (x0 + TW >= w), edge_t = (y0 == 0), edge_b = (y0 + TH2 >= h);
    if (P.l1 && (edge_l || edge_r || edge_t || edge_b)) {
        if (edge_l || edge_r) {
            for (int r = tid; r < BH2; r += NTHREADS) {
                uint8_t* row = S.gray + r * GP;
                if (edge_l) { row[7 + sh] = row[9 + sh]; row[6 + sh] = row[10 + sh]; }
                if (edge_r) {
                    const int cw = w - x0 + 8 + sh;
                    row[cw] = row[cw - 2];
                    row[cw + 1] = row[cw - 3];
                }
            }
            __syncthreads();
        }
        if (edge_t || edge_b) {
            for (int c = tid; c < GP; c += NTHREADS) {
                if (edge_t) { S.gray[3 * GP + c] = S.gray[5 * GP + c]; S.gray[2 * GP + c] = S.gray[6 * GP + c]; }
                if (edge_b) {
                    const int rh = h - y0 + 4;
                    S.gray[rh * GP + c] = S.gray[(rh - 2) * GP + c];
                    S.gray[(rh + 1) * GP + c] = S.gray[(rh - 3) * GP + c];
                }
            }
            __syncthreads();
        }
    }

    const uint32_t* G = reinterpret_cast<const uint32_t*>(S.gray);

    // ------------------------------------------------------------------ C. pyramid level 1: 4 outputs x 2 rows per thread
    if (P.l1) {
        const int w1 = (w + 1) >> 1, h1 = (h + 1) >> 1;
        uint8_t* l1 = P.l1 + (size_t)f * w1 * h1;
        const int pc = tid % 15, sg = tid / 15;   // 15 quad-columns x 16 row pairs (threads 240..255 idle)
        const int lx = (x0 >> 1) + 4 * pc;
        const int ly0 = (y0 >> 1) + 2 * sg;
        // Every lane loads its two middle words of the 7 rows; the edge words W0 (2 bytes used) / W3 (1 byte) are the
        // neighbour lanes' W2 / W1 -- only the first / last quad of a row group and the warp's end lanes load them.  All 32
        // lanes run this part (shuffles), whether or not their outputs exist (idle lanes read row group 15 again).
        const uint32_t* base = G + (4 * min(sg, 15) + 2) * GPW + cbw + 2 * pc;   // gray row 2j+2 for output row j = 2*sg
        const bool ld0 = pc == 0 || lane == 0, ld3 = pc == 14 || lane == 31;
        uint32_t hs[7][4];
#pragma unroll
        for (int r = 0; r < 7; r++) {
            const uint32_t W1 = base[r * GPW + 1], W2 = base[r * GPW + 2];
            uint32_t W0 = __shfl_up_sync(0xffffffffu, W2, 1), W3 = __shfl_down_sync(0xffffffffu, W1, 1);
            if (ld0) W0 = base[r * GPW];
            if (ld3) W3 = base[r * GPW + 3];
            hs[r][0] = __dp4a(__byte_perm(W0, W1, 0x5432), 0x04060401u, __dp4a(W1, 0x00010000u, 0u));
            hs[r][1] = __dp4a(W1, 0x04060401u, __dp4a(W2, 0x00000001u, 0u));
            hs[r][2] = __dp4a(__byte_perm(W1, W2, 0x5432), 0x04060401u, __dp4a(W2, 0x00010000u, 0u));
            hs[r][3] = __dp4a(W2, 0x04060401u, __dp4a(W3, 0x00000001u, 0u));
        }
        if (sg < 16 && lx < w1 && ly0 < h1) {
            const bool quad_ok = (lx + 3 < w1) && ((w1 & 3) == 0) && ((reinterpret_cast<uintptr_t>(P.l1) & 3) == 0);
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int ly = ly0 + j;
                if (ly < h1 && 2 * sg + j < TH2 / 2) {
                    uint32_t v[4];
#pragma unroll
                    for (int i = 0; i < 4; i++)
                        v[i] = hs[2 * j][i] + hs[2 * j + 4][i] + (hs[2 * j + 1][i] + hs[2 * j + 3][i]) * 4u + hs[2 * j + 2][i] * 6u + 128u;
                    // byte 1 of each sum
                    const uint32_t o = __byte_perm(__byte_perm(v[0], v[1], 0x0051), __byte_perm(v[2], v[3], 0x0051), 0x5410);
                    uint8_t* d = l1 + (size_t)ly * w1 + lx;
                    if (quad_ok) *reinterpret_cast<uint32_t*>(d) = o;
                    else
                        for (int i = 0; i < 4 && lx + i < w1; i++) d[i] = (uint8_t)(o >> (8 * i));
                }
            }
        }
    }

    // ------------------------------------------------------------------ D. FAST candidates + exact score
    uint16_t* Q = reinterpret_cast<uint16_t*>(S.rgba) + warp * QCAP;
    int cn = 0;   // corners of this warp inside the tile interior: prefix of Q after this phase
    if (P.keys) {
        const int thr = P.thr;
        const bool hi_thr = thr >= 128;
        const uint32_t K = (uint32_t)(hi_thr ? 255 - thr : 127 - thr) * 0x01010101u;
        uint32_t vm;
        {
            const int xlo = max(3, x0 - 1), xhi = min(w - 4, x0 + TW);
            const int ylo = max(3, y0 - 1), yhi = min(h - 4, y0 + TH2);
            const int yb = y0 - 1 + 8 * warp;
            const int r0v = max(ylo - yb, 0), r1v = min(yhi - yb, 7);
            const uint32_t rowbits = r1v >= r0v ? ((0xffu >> (7 - r1v)) & (0xffu << r0v)) & 0xffu : 0u;
            const int xb = x0 - 4 + 4 * lane;
            const int c0v = max(xlo - xb, 0), c1v = min(xhi - xb, 3);
            const uint32_t colbytes = c1v >= c0v ? ((0x01010101u >> (8 * (3 - c1v))) & (0x01010101u << (8 * c0v))) : 0u;
            vm = colbytes * rowbits;
        }
        if (__any_sync(0xffffffffu, vm != 0)) {
            const uint32_t* g0 = G + (8 * warp) * GPW + cbw + lane;
            uint32_t acc[16];
            if (hi_thr) fast_swar::phase1<true, GPW>(g0, K, P.mul, acc); else fast_swar::phase1<false, GPW>(g0, K, P.mul, acc);
#define ALVA_ASM_LEFT(M)  { const uint32_t o_ = acc[fast_swar::source_of(M)]; acc[M] = fast_swar::assemble<M>(o_, __shfl_up_sync(0xffffffffu, o_, 1), 0u, acc[M]); }
#define ALVA_ASM_RIGHT(M) { const uint32_t o_ = acc[fast_swar::source_of(M)]; acc[M] = fast_swar::assemble<M>(o_, 0u, __shfl_down_sync(0xffffffffu, o_, 1), acc[M]); }
            ALVA_ASM_RIGHT(5) ALVA_ASM_RIGHT(6) ALVA_ASM_RIGHT(7)
            acc[8] = fast_swar::assemble<8>(acc[0], 0u, 0u, acc[8]);
            ALVA_ASM_LEFT(9) ALVA_ASM_LEFT(10) ALVA_ASM_LEFT(11) ALVA_ASM_LEFT(12)
#undef ALVA_ASM_LEFT
#undef ALVA_ASM_RIGHT
            uint32_t u = fast_swar::contiguous9(acc) & vm;
            // 32 x 32 bit transpose across the warp: afterwards lane b holds, in bit l, lane l's flag for bit position b
            {
                uint32_t x = __shfl_xor_sync(0xffffffffu, u, 16);
                u = __byte_perm(u, x, (lane & 16) ? 0x3276u : 0x5410u);
                x = __shfl_xor_sync(0xffffffffu, u, 8);
                u = __byte_perm(u, x, (lane & 8) ? 0x3715u : 0x6240u);
                x = __shfl_xor_sync(0xffffffffu, u, 4);
                u = (lane & 4) ? ((u & 0xf0f0f0f0u) | ((x >> 4) & 0x0f0f0f0fu)) : ((u & 0x0f0f0f0fu) | ((x & 0x0f0f0f0fu) << 4));
                x = __shfl_xor_sync(0xffffffffu, u, 2);
                u = (lane & 2) ? ((u & 0xccccccccu) | ((x >> 2) & 0x33333333u)) : ((u & 0x33333333u) | ((x & 0x33333333u) << 2));
                x = __shfl_xor_sync(0xffffffffu, u, 1);
                u = (lane & 1) ? ((u & 0xaaaaaaaau) | ((x >> 1) & 0x55555555u)) : ((u & 0x55555555u) | ((x & 0x55555555u) << 1));
            }
            const int mine = __popc(u);
            int incl = mine;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += v; }
            int pos = incl - mine;
            const int qn = __shfl_sync(0xffffffffu, incl, 31);
            // queue entry = (gray row << 8) | gray byte column; this lane's bit position is pixel j = lane >> 3, row i = lane & 7
            const uint32_t e0 = ((uint32_t)(8 * warp + 3 + (lane & 7)) << 8) | (uint32_t)(4 * cbw + (lane >> 3));
            while (u) {
                const int l = __ffs(u) - 1;
                u &= u - 1;
                Q[pos++] = (uint16_t)(e0 + 4 * l);
            }
            __syncwarp();
            const uint32_t lt = (1u << lane) - 1u;
            for (int q0 = 0; q0 < qn; q0 += 32) {
                bool corner_in = false;
                uint32_t centry = 0;
                if (q0 + lane < qn) {
                    const uint32_t e = Q[q0 + lane];
                    const int pr = e >> 8, pcg = e & 255;
                    const int sc = fast_strength2(S.gray + pr * GP + pcg);
                    if (sc > thr) {
                        const int sr = pr - 3, scol = pcg - 4 * cbw;   // score-tile row / column (column 4 = image x0)
                        score[sr * SP2 + scol] = (uint8_t)(sc - 1);
                        corner_in = sr >= 1 && sr <= TH2 && scol >= 4 && scol < 4 + TW;
                        centry = ((uint32_t)sr << 7) | (uint32_t)scol;
                    }
                }
                const uint32_t mk = __ballot_sync(0xffffffffu, corner_in);
                if (corner_in) Q[cn + __popc(mk & lt)] = (uint16_t)centry;   // cn + rank <= q0 + lane: never ahead of the reads
                cn += __popc(mk);
            }
        }
    }
    __syncthreads();

    // ------------------------------------------------------------------ E. 3x3 NMS (strict >) over the corners + emit
    // A warp's first four rounds (128 corners; ~40 is typical) keep their keys in registers: ONE global atomic takes the warp's
    // range of the frame's list, then the rounds store.  No tile-level list, no further barrier (order_keys_kernel sorts the
    // frame's list anyway).  Corners beyond 128 take one atomic per round.
    if (P.keys) {
        const uint32_t lt = (1u << lane) - 1u;
        auto nms_key = [&](int c, uint32_t& key) -> bool {
            if (c >= cn) return false;
            const uint32_t e = Q[c];
            const int sr = e >> 7, scol = e & 127;
            const uint8_t* sp = score + sr * SP2 + scol;
            const uint32_t v = sp[0];
            const uint32_t m = max(max(max((uint32_t)sp[-SP2 - 1], (uint32_t)sp[-SP2]), max((uint32_t)sp[-SP2 + 1], (uint32_t)sp[-1])),
                                   max(max((uint32_t)sp[1], (uint32_t)sp[SP2 - 1]), max((uint32_t)sp[SP2], (uint32_t)sp[SP2 + 1])));
            key = ((uint32_t)(y0 + sr - 1) << 20) | ((uint32_t)(x0 + scol - 4) << 8) | v;
            return v > m;
        };
        uint32_t* const out = P.keys + (size_t)f * P.cap;
        uint32_t keyr[4] = {0u, 0u, 0u, 0u}, mkr[4] = {0u, 0u, 0u, 0u};
        bool isr[4] = {false, false, false, false};
#pragma unroll
        for (int r = 0; r < 4; r++)
            if (32 * r < cn) {   // warp-uniform
                isr[r] = nms_key(32 * r + lane, keyr[r]);
                mkr[r] = __ballot_sync(0xffffffffu, isr[r]);
            }
        const int total = __popc(mkr[0]) + __popc(mkr[1]) + __popc(mkr[2]) + __popc(mkr[3]);
        if (total) {
            int base = 0;
            if (lane == 0) base = atomicAdd(P.counts + f, total);
            base = __shfl_sync(0xffffffffu, base, 0);
#pragma unroll
            for (int r = 0; r < 4; r++) {
                const int pos = base + __popc(mkr[r] & lt);
                if (isr[r] && pos < P.cap) out[pos] = keyr[r];
                base += __popc(mkr[r]);
            }
        }
        for (int c0 = 128; c0 < cn; c0 += 32) {
            uint32_t key = 0;
            const bool iskp = nms_key(c0 + lane, key);
            const uint32_t mk = __ballot_sync(0xffffffffu, iskp);
            if (mk) {
                int base = 0;
                if (lane == 0) base = atomicAdd(P.counts + f, __popc(mk));
                base = __shfl_sync(0xffffffffu, base, 0) + __popc(mk & lt);
                if (iskp && base < P.cap) out[base] = key;
            }
        }
    }
}

// ---- standalone RGBA -> gray (alva_k_gray) ---------------------------------------------------------
__global__ void gray_kernel(const uint8_t* __restrict__ rgba, uint8_t* __restrict__ gray, size_t npix) {
    const size_t i4 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i4 + 3 < npix) {
        const uint4 p = __ldg(reinterpret_cast<const uint4*>(rgba) + i4 / 4);
        *reinterpret_cast<uint32_t*>(gray + i4) = gray4(p);
    } else {
        for (size_t i = i4; i < npix; i++) gray[i] = (uint8_t)gray1(reinterpret_cast<const uint32_t*>(rgba)[i]);
    }
}

// ---- generic pyrDown (any size; used for levels >= 2 and alva_k_pyrdown) ----------------------------
// one output, any position: 25 byte loads with reflect-101 (borders, odd geometries)
__device__ __forceinline__ uint8_t pyrdown_one(const uint8_t* __restrict__ s, int w, int h, int x, int y) {
    int xs[5], acc = 0;
#pragma unroll
    for (int i = 0; i < 5; i++) xs[i] = reflect101(2 * x + i - 2, w);
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const uint8_t* row = s + (size_t)reflect101(2 * y + j - 2, h) * w;
        const int hsum = __ldg(row + xs[0]) + __ldg(row + xs[4]) + 4 * (__ldg(row + xs[1]) + __ldg(row + xs[3])) +
                         6 * __ldg(row + xs[2]);
        const int kj = (j == 0 || j == 4) ? 1 : (j == 2 ? 6 : 4);
        acc += kj * hsum;
    }
    return (uint8_t)((acc + 128) >> 8);
}
// A thread owns 4 adjacent outputs x 4 output rows: 11 source rows x 4 aligned words, horizontal taps as IDP.4A on the
// packed words (as in the fused kernel), vertical taps in registers -- 2.75 word loads per output instead of 25 byte loads.
// Threads whose footprint touches the image border (or unaligned geometries) take the per-output path.
constexpr int PD_ROWS = 4;
__global__ void __launch_bounds__(256) pyrdown_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int w, int h,
                                                      int nframes) {
    const int dw = (w + 1) >> 1, dh = (h + 1) >> 1;
    const int x = 4 * (blockIdx.x * 32 + threadIdx.x);
    const int y0 = (blockIdx.y * 8 + threadIdx.y) * PD_ROWS;
    if (x >= dw || y0 >= dh) return;
    const uint8_t* s = src + (size_t)blockIdx.z * w * h;
    uint8_t* d = dst + (size_t)blockIdx.z * dw * dh;
    // fast path: aligned rows and a full group of 4 outputs.  The left / right image border costs nothing here: the two
    // reflected columns are bytes of the neighbouring word (cols -2,-1 = cols 2,1; col w = col w-2), rows reflect by index.
    const bool left = (x == 0), right = (2 * x + 12 > w);
    const bool fast = (w & 3) == 0 && (((uintptr_t)src) & 3) == 0 && x + 3 < dw && y0 + PD_ROWS <= dh && 2 * x + 8 <= w && h >= 4;
    if (!fast) {
        for (int j = 0; j < PD_ROWS && y0 + j < dh; j++)
            for (int i = 0; i < 4 && x + i < dw; i++) d[(size_t)(y0 + j) * dw + x + i] = pyrdown_one(s, w, h, x + i, y0 + j);
        return;
    }
    uint32_t hs[2 * PD_ROWS + 3][4];   // horizontal sums of source rows 2*y0-2 .. 2*y0+2*PD_ROWS
#pragma unroll
    for (int r = 0; r < 2 * PD_ROWS + 3; r++) {
        const uint32_t* row = reinterpret_cast<const uint32_t*>(s + (size_t)reflect101(2 * y0 - 2 + r, h) * w + 2 * x);
        const uint32_t W1 = __ldg(row), W2 = __ldg(row + 1);
        const uint32_t W0 = left ? __byte_perm(W1, W1, 0x1200) : __ldg(row - 1);    // bytes 2, 3 = cols 2x-2, 2x-1
        const uint32_t W3 = right ? (W2 >> 16) : __ldg(row + 2);                     // byte 0 = col 2x+8
        // out0 centred on W1[0]: W0[2] W0[3] W1[0] W1[1] W1[2];  out1 on W1[2]: W1[0..3] W2[0];  out2 on W2[0];  out3 on W2[2]
        hs[r][0] = __dp4a(__byte_perm(W0, W1, 0x5432), 0x04060401u, __dp4a(W1, 0x00010000u, 0u));
        hs[r][1] = __dp4a(W1, 0x04060401u, __dp4a(W2, 0x00000001u, 0u));
        hs[r][2] = __dp4a(__byte_perm(W1, W2, 0x5432), 0x04060401u, __dp4a(W2, 0x00010000u, 0u));
        hs[r][3] = __dp4a(W2, 0x04060401u, __dp4a(W3, 0x00000001u, 0u));
    }
    const bool al = (dw & 3) == 0 && (((uintptr_t)dst) & 3) == 0;
#pragma unroll
    for (int j = 0; j < PD_ROWS; j++) {
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint32_t v = hs[2 * j][i] + hs[2 * j + 4][i] + (hs[2 * j + 1][i] + hs[2 * j + 3][i]) * 4u + hs[2 * j + 2][i] * 6u + 128u;
            o |= ((v >> 8) & 0xffu) << (8 * i);
        }
        uint8_t* p = d + (size_t)(y0 + j) * dw + x;
        if (al) *reinterpret_cast<uint32_t*>(p) = o;
        else { p[0] = (uint8_t)o; p[1] = (uint8_t)(o >> 8); p[2] = (uint8_t)(o >> 16); p[3] = (uint8_t)(o >> 24); }
    }
}

// ---- restore cv::FAST's row-major order: bucket by row, then sort each row's few keys by x ---------
// The first min(counts[f], cap) keys of `in` are ordered into `work` (same stride cap).  When `out` is another buffer, the
// first out_cap of the ordered keys are then copied there (stride out_cap): a truncation in row-major order, the same on every
// run.  out_counts (optional, may alias counts) receives min(count, cap, out_cap).
__global__ void __launch_bounds__(1024) order_keys_kernel(const uint32_t* __restrict__ in, uint32_t* work, const int32_t* counts,
                                                          int cap, int h, uint32_t* out, int32_t* out_counts, int out_cap) {
    extern __shared__ int osm[];   // rowstart[h+1], rowfill[h]
    int* rowstart = osm;
    int* rowfill = osm + h + 1;
    const int f = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int n = min(counts[f], cap);
    const uint32_t* kin = in + (size_t)f * cap;
    uint32_t* kout = work + (size_t)f * cap;
    for (int i = tid; i <= h; i += nt) rowstart[i] = 0;
    for (int i = tid; i < h; i += nt) rowfill[i] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += nt) atomicAdd(&rowstart[(kin[i] >> 20) + 1], 1);
    __syncthreads();
    // inclusive scan of rowstart[1..h] (h <= 4096): chunked serial + cross-chunk
    {
        __shared__ int part[1024];
        const int chunk = (h + nt) / nt;
        const int b = tid * chunk + 1, e = min(b + chunk, h + 1);
        int s = 0;
        for (int i = b; i < e; i++) s += rowstart[i];
        part[tid] = s;
        __syncthreads();
        for (int off = 1; off < nt; off <<= 1) {
            int v = tid >= off ? part[tid - off] : 0;
            __syncthreads();
            part[tid] += v;
            __syncthreads();
        }
        int run = tid ? part[tid - 1] : 0;
        for (int i = b; i < e; i++) { run += rowstart[i]; rowstart[i] = run; }
        __syncthreads();
    }
    for (int i = tid; i < n; i += nt) {
        const uint32_t k = kin[i];
        const int y = k >> 20;
        kout[rowstart[y] + atomicAdd(&rowfill[y], 1)] = k;
    }
    __syncthreads();
    for (int y = tid; y < h; y += nt) {   // insertion sort within the row (keys of one row differ in x)
        const int b = rowstart[y], e = rowstart[y + 1];
        for (int i = b + 1; i < e; i++) {
            const uint32_t k = kout[i];
            int j = i - 1;
            while (j >= b && kout[j] > k) { kout[j + 1] = kout[j]; j--; }
            kout[j + 1] = k;
        }
    }
    const int nout = min(n, out_cap);
    if (out != work) {
        __syncthreads();
        uint32_t* dst = out + (size_t)f * out_cap;
        for (int i = tid; i < nout; i += nt) dst[i] = kout[i];
    }
    if (out_counts && tid == 0) out_counts[f] = nout;   // every thread read counts[f] before the first barrier
}

// ---- KeyPointsFilter::retainBest on packed keys (one CTA per frame) --------------------------------
// Every kept key is written (out has the input's stride cap, and at most min(count, cap) keys are kept), in atomic order;
// out_counts[f] = the kept count.  order_keys_kernel then orders them and truncates.
__global__ void __launch_bounds__(1024) retain_best_kernel(const uint32_t* __restrict__ in, const int32_t* __restrict__ counts,
                                                           int cap, int w, int h, int n_keep, int edge,
                                                           uint32_t* __restrict__ out, int32_t* __restrict__ out_counts) {
    __shared__ int hist[256];
    __shared__ int thr_s, cnt_s;
    const int f = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int n = min(counts[f], cap);
    const uint32_t* kin = in + (size_t)f * cap;
    for (int i = tid; i < 256; i += nt) hist[i] = 0;
    if (tid == 0) cnt_s = 0;
    __syncthreads();
    auto inside = [&](uint32_t k) {
        if (edge <= 0) return true;
        const int x = ALVA_KEY_X(k), y = ALVA_KEY_Y(k);
        return x >= edge && x < w - edge && y >= edge && y < h - edge;
    };
    int local = 0;
    for (int i = tid; i < n; i += nt) {
        const uint32_t k = kin[i];
        if (inside(k)) { atomicAdd(&hist[k & 255], 1); local++; }
    }
    __syncthreads();
    if (tid == 0) {
        int total = 0;
        for (int s = 0; s < 256; s++) total += hist[s];
        int thr = 0;
        if (n_keep >= 0 && total > n_keep) {
            if (n_keep == 0) thr = 256;
            else {
                int acc = 0;
                for (int s = 255; s >= 0; s--) { acc += hist[s]; if (acc >= n_keep) { thr = s; break; } }
            }
        }
        thr_s = thr;
    }
    __syncthreads();
    const int thr = thr_s;
    uint32_t* kout = out + (size_t)f * cap;
    for (int i = tid; i < n; i += nt) {
        const uint32_t k = kin[i];
        if (inside(k) && (int)(k & 255) >= thr) kout[atomicAdd(&cnt_s, 1)] = k;
    }
    __syncthreads();
    if (tid == 0) out_counts[f] = cnt_s;
}

// ---- Scharr derivative image of a pyramid level (cv::buildOpticalFlowPyramid withDerivatives, lkpyramid.cpp:57-150) ----
// HBM-bound streaming: W*H bytes in, 4*W*H out (int16 dx, dy interleaved).  A thread owns a 4-pixel column strip of
// SCH_ROWS rows with a rolling 3-row window, so every input row is read once per strip (+2 halo rows) and every output
// is one 128-bit store.  Reflect-101 in both directions, exactly as the reference picks its neighbour rows / columns.
constexpr int SCH_ROWS = 8;
__device__ __forceinline__ void scharr_load6(const uint8_t* __restrict__ row, int x, int w, bool fast, int v[6]) {
    if (fast && x >= 4 && x + 8 <= w) {
        const uint32_t L = __ldg(reinterpret_cast<const uint32_t*>(row + x - 4));
        const uint32_t M = __ldg(reinterpret_cast<const uint32_t*>(row + x));
        const uint32_t R = __ldg(reinterpret_cast<const uint32_t*>(row + x + 4));
        v[0] = L >> 24; v[1] = M & 255; v[2] = (M >> 8) & 255; v[3] = (M >> 16) & 255; v[4] = M >> 24; v[5] = R & 255;
    } else {
#pragma unroll
        for (int c = 0; c < 6; c++) {
            int xx = x - 1 + c;
            if (xx < 0) xx = w > 1 ? 1 : 0;                       // trow[-1] = trow[1]
            else if (xx >= w) xx = (xx == w) ? (w > 1 ? w - 2 : 0) : w - 1;   // trow[w] = trow[w-2]; beyond: unused lanes
            v[c] = __ldg(row + xx);
        }
    }
}
struct ScharrLevels {   // up to 4 pyramid levels in one launch: blockIdx.y runs through the levels' row blocks
    const uint8_t* src[4];
    int16_t* dst[4];
    int w[4], h[4], yb0[5];   // yb0[k] = first blockIdx.y of level k, yb0[nlev] = gridDim.y
    int nlev;
};
__global__ void __launch_bounds__(256) scharr_kernel(const ScharrLevels L) {
    int lev = 0;
#pragma unroll
    for (int k = 1; k < 4; k++) if (k < L.nlev && (int)blockIdx.y >= L.yb0[k]) lev = k;
    const int w = L.w[lev], h = L.h[lev];
    const uint8_t* src = L.src[lev];
    int16_t* dst = L.dst[lev];
    const int gx = blockIdx.x * 32 + threadIdx.x, x = 4 * gx;
    const int ys = ((blockIdx.y - L.yb0[lev]) * 8 + threadIdx.y) * SCH_ROWS;
    if (x >= w || ys >= h) return;
    const uint8_t* img = src + (size_t)blockIdx.z * w * h;
    int16_t* out = dst + (size_t)blockIdx.z * w * h * 2;
    const bool fast = (w & 3) == 0 && ((uintptr_t)src & 3) == 0;
    auto rrow = [&](int y) { return y < 0 ? (h > 1 ? 1 : 0) : (y >= h ? (h > 1 ? h - 2 : 0) : y); };
    int a[6], b[6], c[6];
    scharr_load6(img + (size_t)rrow(ys - 1) * w, x, w, fast, a);
    scharr_load6(img + (size_t)rrow(ys) * w, x, w, fast, b);
#pragma unroll
    for (int i = 0; i < SCH_ROWS; i++) {
        const int y = ys + i;
        if (y >= h) break;
        scharr_load6(img + (size_t)rrow(y + 1) * w, x, w, fast, c);
        int t0[6], t1[6];
#pragma unroll
        for (int k = 0; k < 6; k++) { t0[k] = (a[k] + c[k]) * 3 + b[k] * 10; t1[k] = c[k] - a[k]; }
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int dx = t0[k + 2] - t0[k];
            const int dy = (t1[k] + t1[k + 2]) * 3 + t1[k + 1] * 10;
            o[k] = ((uint32_t)dx & 0xffffu) | ((uint32_t)dy << 16);
        }
        uint32_t* d = reinterpret_cast<uint32_t*>(out) + (size_t)y * w + x;
        if (fast && ((uintptr_t)dst & 15) == 0) *reinterpret_cast<uint4*>(d) = make_uint4(o[0], o[1], o[2], o[3]);
        else
            for (int k = 0; k < 4 && x + k < w; k++) d[k] = o[k];
#pragma unroll
        for (int k = 0; k < 6; k++) { a[k] = b[k]; b[k] = c[k]; }
    }
}

}  // namespace

// =================================================================================== host launchers
int alva_g_frontend_antipodal = 0;   // alva_set_option("frontend_antipodal", 1): experimental pre-test variant (RGBA path only)
int alva_g_frontend_prefetch = 0;    // alva_set_option("frontend_prefetch", 1): variant 2 pulls a later frame's tile into L2 (TMA prefetch)
int alva_g_frontend_ctas = 5;        // alva_set_option("frontend_ctas", 4 | 5): resident CTAs per SM of variant 2
int alva_g_frontend_variant = 2;     // alva_set_option("frontend_variant", 0 | 2): 0 = the round-1 kernel, 2 = frontend_tile_kernel_v2

static int launch_frontend(alva_ctx* ctx, bool rgba_mode, const uint8_t* src, int w, int h, int nframes, uint8_t* l0,
                           uint8_t* l1, int thr, uint32_t* keys, int32_t* counts, int cap) {
    FrontendParams P{};
    P.src = src; P.l0 = l0; P.l1 = l1; P.keys = keys; P.counts = counts;
    P.w = w; P.h = h; P.nframes = nframes;
    static const bool no_tma = getenv("ALVA_DISABLE_TMA") != nullptr;   // debugging aid: force the plain-load path
    const bool tma_geom = rgba_mode ? (w % 4 == 0) && ((uintptr_t)src % 16 == 0)
                                    : (w % 16 == 0) && (((size_t)w * h) % 16 == 0) && ((uintptr_t)src % 16 == 0);
    const bool v2 = tma_geom && !no_tma && alva_g_frontend_variant == 2 && !alva_g_frontend_antipodal;
    const int th = v2 ? TH2 : TH, bh = v2 ? BH2 : BH;
    P.tiles_x = (w + TW - 1) / TW; P.tiles_y = (h + th - 1) / th;
    P.thr = thr < 0 ? 0 : (thr > 255 ? 255 : thr); P.cap = cap;
    for (int i = 0; i < 7; i++) P.mul[i] = 1u << (25 + i);
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof tmap);
    bool tma_ok;
    if (rgba_mode) {
        uint64_t dims[3] = {(uint64_t)w, (uint64_t)h, (uint64_t)nframes};
        uint64_t strides[2] = {(uint64_t)w * 4, (uint64_t)w * h * 4};
        uint32_t box[3] = {BW, (uint32_t)bh, 1};
        tma_ok = tma_geom && alva_make_tmap(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, src, dims, strides, box);
    } else {
        uint64_t dims[3] = {(uint64_t)w, (uint64_t)h, (uint64_t)nframes};
        uint64_t strides[2] = {(uint64_t)w, (uint64_t)w * h};
        uint32_t box[3] = {GP, (uint32_t)bh, 1};
        tma_ok = tma_geom && alva_make_tmap(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, src, dims, strides, box);
    }
    if (v2 && !tma_ok) { alva_set_error("front end: cuTensorMapEncodeTiled failed"); return ALVA_E_CUDA; }
    P.use_tma = (tma_ok && !no_tma) ? 1 : 0;
    const int grid = P.tiles_x * P.tiles_y * nframes;
    const size_t smem = sizeof(SmemLayout) + 128;
    if (v2) {
        // "frontend_ctas" = 4: pad the request so that only 4 CTAs fit an SM (5 by default) -- leaves registers and shared memory
        // for the small kernels of a concurrent stream (the pipeline's BA chain)
        const size_t smem2 = sizeof(SmemLayout2) + 128 + (alva_g_frontend_ctas == 4 ? 11 * 1024 : 0);
        if (P.tiles_y > 65535 || nframes > 65535) { alva_set_error("front end: more than 65535 frames / tile rows in one launch"); return ALVA_E_INVALID; }
        const dim3 grid3(P.tiles_x, P.tiles_y, nframes);
        // L2 prefetch distance: the tile at the same position this many frames ahead starts about one residency later
        // (5 CTAs per SM in flight, tiles dispatched frame-major)
        P.prefetch = alva_g_frontend_prefetch ? (5 * ctx->num_sms + P.tiles_x * P.tiles_y - 1) / (P.tiles_x * P.tiles_y) + 1 : 0;
        if (rgba_mode) {
            ALVA_CUDA(cudaFuncSetAttribute(frontend_tile_kernel_v2<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
            frontend_tile_kernel_v2<true><<<grid3, NTHREADS, smem2, ctx->stream>>>(tmap, P);
        } else {
            ALVA_CUDA(cudaFuncSetAttribute(frontend_tile_kernel_v2<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
            frontend_tile_kernel_v2<false><<<grid3, NTHREADS, smem2, ctx->stream>>>(tmap, P);
        }
    } else if (rgba_mode && alva_g_frontend_antipodal) {
        ALVA_CUDA(cudaFuncSetAttribute(frontend_tile_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        frontend_tile_kernel<true, true><<<grid, NTHREADS, smem, ctx->stream>>>(tmap, P);
    } else if (rgba_mode) {
        ALVA_CUDA(cudaFuncSetAttribute(frontend_tile_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        frontend_tile_kernel<true><<<grid, NTHREADS, smem, ctx->stream>>>(tmap, P);
    } else {
        ALVA_CUDA(cudaFuncSetAttribute(frontend_tile_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        frontend_tile_kernel<false><<<grid, NTHREADS, smem, ctx->stream>>>(tmap, P);
    }
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// the fused launch alone (pipeline.cu brackets it with CUDA events for the roofline measurement)
int alva_frontend_main_launch(alva_ctx* ctx, const uint8_t* rgba, int w, int h, int nframes, uint8_t* l0, uint8_t* l1, int thr,
                              uint32_t* keys, int32_t* counts, int cap) {
    return launch_frontend(ctx, true, rgba, w, h, nframes, l0, l1, thr, keys, counts, cap);
}

static int launch_pyrdown(alva_ctx* ctx, const uint8_t* src, uint8_t* dst, int w, int h, int nframes) {
    const int dw = (w + 1) / 2, dh = (h + 1) / 2;
    dim3 block(32, 8), grid(((dw + 3) / 4 + 31) / 32, (dh + 8 * PD_ROWS - 1) / (8 * PD_ROWS), nframes);
    pyrdown_kernel<<<grid, block, 0, ctx->stream>>>(src, dst, w, h, nframes);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// in -> work (both stride cap) in row-major order; then, if out != work, its first out_cap keys -> out (stride out_cap).
// out_counts (optional) = the counts clamped to cap and out_cap.
static int launch_order(alva_ctx* ctx, const uint32_t* in, uint32_t* work, const int32_t* counts, int cap, int h, int nframes,
                        uint32_t* out, int32_t* out_counts, int out_cap) {
    const size_t smem = (size_t)(2 * h + 1) * sizeof(int);
    order_keys_kernel<<<nframes, 1024, smem, ctx->stream>>>(in, work, counts, cap, h, out, out_counts, out_cap);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

static int check_dims(int w, int h, int nframes) {
    if (w < 16 || h < 16 || w > ALVA_MAX_DIM || h > ALVA_MAX_DIM || nframes < 1) {
        alva_set_error("invalid frame geometry %dx%d x%d (need 16..%d)", w, h, nframes, ALVA_MAX_DIM);
        return ALVA_E_INVALID;
    }
    return 0;
}

extern "C" int alva_k_gray(alva_ctx* ctx, const uint8_t* rgba, uint8_t* gray, int w, int h, int nframes) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !rgba || !gray || w < 1 || h < 1 || nframes < 1) { alva_set_error("alva_k_gray: bad argument"); return ALVA_E_INVALID; }
    const size_t npix = (size_t)w * h * nframes;
    const size_t nthr = (npix + 3) / 4;
    gray_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, ctx->stream>>>(rgba, gray, npix);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

// internal (pipeline.cu): the derivative images of up to 4 levels in ONE launch (the small levels are launch-bound alone)
int alva_scharr_levels_launch(alva_ctx* ctx, int nlev, const uint8_t* const* src, int16_t* const* dst, const int* w, const int* h,
                              int nframes) {
    ScharrLevels L{};
    L.nlev = nlev;
    int yb = 0, gx = 1;
    for (int k = 0; k < nlev; k++) {
        L.src[k] = src[k]; L.dst[k] = dst[k]; L.w[k] = w[k]; L.h[k] = h[k]; L.yb0[k] = yb;
        yb += (h[k] + 8 * SCH_ROWS - 1) / (8 * SCH_ROWS);
        gx = std::max(gx, ((w[k] + 3) / 4 + 31) / 32);
    }
    for (int k = nlev; k < 5; k++) L.yb0[k] = yb;
    scharr_kernel<<<dim3(gx, yb, nframes), dim3(32, 8), 0, ctx->stream>>>(L);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

extern "C" int alva_k_scharr(alva_ctx* ctx, const uint8_t* gray, int16_t* deriv, int w, int h, int nframes) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !gray || !deriv || w < 1 || h < 1 || nframes < 1 || ((uintptr_t)deriv & 3)) {
        alva_set_error("alva_k_scharr: bad argument");
        return ALVA_E_INVALID;
    }
    return alva_scharr_levels_launch(ctx, 1, &gray, &deriv, &w, &h, nframes);
}

extern "C" int alva_k_pyrdown(alva_ctx* ctx, const uint8_t* src, uint8_t* dst, int w, int h, int nframes) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !src || !dst || w < 1 || h < 1 || nframes < 1) { alva_set_error("alva_k_pyrdown: bad argument"); return ALVA_E_INVALID; }
    return launch_pyrdown(ctx, src, dst, w, h, nframes);
}

static int fast_common(alva_ctx* ctx, bool rgba_mode, const uint8_t* src, int w, int h, int nframes, uint8_t* l0,
                       uint8_t* l1, uint8_t* l2, uint8_t* l3, int thr, uint32_t* keys, int32_t* counts, int cap,
                       int sorted) {
    if (int e = check_dims(w, h, nframes)) return e;
    if (keys && (!counts || cap < 1)) { alva_set_error("keys given without counts/cap"); return ALVA_E_INVALID; }
    uint32_t* raw = keys;
    if (keys && sorted) {
        raw = (uint32_t*)alva_scratch(ctx, (size_t)nframes * cap * sizeof(uint32_t));
        if (!raw) return ALVA_E_CUDA;
    }
    if (keys) ALVA_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * nframes, ctx->stream));
    if (int e = launch_frontend(ctx, rgba_mode, src, w, h, nframes, l0, l1, thr, raw, counts, cap)) return e;
    if (l1 && l2) {
        const int w1 = (w + 1) / 2, h1 = (h + 1) / 2;
        if (int e = launch_pyrdown(ctx, l1, l2, w1, h1, nframes)) return e;
        if (l3) {
            const int w2 = (w1 + 1) / 2, h2 = (h1 + 1) / 2;
            if (int e = launch_pyrdown(ctx, l2, l3, w2, h2, nframes)) return e;
        }
    }
    if (keys && sorted)
        if (int e = launch_order(ctx, raw, keys, counts, cap, h, nframes, keys, nullptr, cap)) return e;
    return 0;
}

extern "C" int alva_k_fast9(alva_ctx* ctx, const uint8_t* gray, int w, int h, int nframes, int thr, uint32_t* keys,
                            int32_t* counts, int cap, int sorted) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !gray || !keys) { alva_set_error("alva_k_fast9: bad argument"); return ALVA_E_INVALID; }
    return fast_common(ctx, false, gray, w, h, nframes, nullptr, nullptr, nullptr, nullptr, thr, keys, counts, cap, sorted);
}

extern "C" int alva_k_frontend(alva_ctx* ctx, const uint8_t* rgba, int w, int h, int nframes, uint8_t* l0, uint8_t* l1,
                               uint8_t* l2, uint8_t* l3, int thr, uint32_t* keys, int32_t* counts, int cap, int sorted) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !rgba) { alva_set_error("alva_k_frontend: bad argument"); return ALVA_E_INVALID; }
    return fast_common(ctx, true, rgba, w, h, nframes, l0, l1, l2, l3, thr, keys, counts, cap, sorted);
}

extern "C" int alva_k_retain_best(alva_ctx* ctx, const uint32_t* keys, const int32_t* counts, int cap, int nframes, int w,
                                  int h, int n, int edge, uint32_t* out_keys, int32_t* out_counts, int out_cap) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !keys || !counts || !out_keys || !out_counts || nframes < 1 || cap < 1 || out_cap < 1) {
        alva_set_error("alva_k_retain_best: bad argument");
        return ALVA_E_INVALID;
    }
    // select every kept key (up to cap of them) into tmp, order them all, then keep the first out_cap: the truncation never
    // depends on the order in which the selection's atomics land.  With out_cap == cap the ordering writes out_keys directly.
    const bool direct = out_cap == cap;
    const size_t words = (size_t)nframes * cap;
    uint32_t* tmp = (uint32_t*)alva_scratch(ctx, (direct ? 1 : 2) * words * sizeof(uint32_t));
    if (!tmp) return ALVA_E_CUDA;
    uint32_t* work = direct ? out_keys : tmp + words;
    retain_best_kernel<<<nframes, 1024, 0, ctx->stream>>>(keys, counts, cap, w, h, n, edge, tmp, out_counts);
    ALVA_LAUNCH_CHECK(ctx);
    return launch_order(ctx, tmp, work, out_counts, cap, h, nframes, out_keys, out_counts, out_cap);
}

// Host-buffer front end: pinned/pageable host RGBA in, packed keys + counts out.  The copies are part of the call
// (bench.py's e2e leg; also what a host without device pointers binds).
extern "C" int alva_h_frontend(alva_ctx* ctx, const uint8_t* rgba_host, int w, int h, int nframes, int thr,
                               uint32_t* keys_host, int32_t* counts_host, int cap) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !rgba_host || !keys_host || !counts_host) { alva_set_error("alva_h_frontend: bad argument"); return ALVA_E_INVALID; }
    if (int e = check_dims(w, h, nframes)) return e;
    const size_t in_bytes = (size_t)w * h * 4 * nframes;
    const size_t key_bytes = (size_t)cap * nframes * sizeof(uint32_t);
    const size_t cnt_bytes = ((size_t)nframes * sizeof(int32_t) + 255) & ~(size_t)255;
    const size_t need = in_bytes + key_bytes + cnt_bytes + 512;
    if (need > ctx->dev_stage_bytes) {
        ctx->ws_epoch++;
        if (ctx->dev_stage) { ALVA_CUDA(cudaStreamSynchronize(ctx->stream)); ALVA_CUDA(cudaFree(ctx->dev_stage)); ctx->dev_stage = nullptr; }
        ALVA_CUDA(cudaMalloc(&ctx->dev_stage, need));
        ctx->dev_stage_bytes = need;
    }
    uint8_t* d_in = (uint8_t*)ctx->dev_stage;
    uint32_t* d_keys = (uint32_t*)(d_in + ((in_bytes + 255) & ~(size_t)255));
    int32_t* d_cnt = (int32_t*)((uint8_t*)d_keys + ((key_bytes + 255) & ~(size_t)255));
    ALVA_CUDA(cudaMemcpyAsync(d_in, rgba_host, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (int e = fast_common(ctx, true, d_in, w, h, nframes, nullptr, nullptr, nullptr, nullptr, thr, d_keys, d_cnt, cap, 0)) return e;
    ALVA_CUDA(cudaMemcpyAsync(counts_host, d_cnt, sizeof(int32_t) * nframes, cudaMemcpyDeviceToHost, ctx->stream));
    ALVA_CUDA(cudaMemcpyAsync(keys_host, d_keys, key_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    ALVA_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int f = 0; f < nframes; f++)
        if (counts_host[f] > cap) { alva_set_error("frame %d: %d corners exceed cap %d", f, counts_host[f], cap); return ALVA_E_CAPACITY; }
    return 0;
}
