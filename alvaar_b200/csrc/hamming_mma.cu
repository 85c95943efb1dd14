// hamming_mma.cu -- brute-force Hamming 2-NN on the Hopper tensor cores (warpgroup wgmma, sm_90a).
//
// Reference behaviour (exact, same as hamming.cu): cv::BFMatcher(NORM_HAMMING).knnMatch(k = 2)
//   opencv features2d/src/matchers.cpp:757 -> core/src/batch_distance.cpp:103-123 (batchDistHamming),
//   k-NN insertion :235-248 (strict '<': ties keep the lowest train index).
//
// Why tensor cores: brute-force Hamming IS a contraction.  With every descriptor bit b expanded to the 8-bit value
// 2b - 1 (+1 / -1), the dot product of two 256-element rows is  256 - 2 * hamming,  exactly (an int32, or a float whose
// partial sums are all integers of magnitude <= 256).  So the N_q x N_t distance matrix is one 8-bit GEMM with K = 256, and the
// integer pipes (which bound the LOP3/POPC kernel of hamming.cu) are left with nothing but the top-2 selection.  Two operand
// kinds are built: int8 (+-1 as s8, s32 accumulators; the default) and E4M3 (+-1.0, f32 accumulators); the results are
// bit-identical (every value involved is an exactly representable integer).
//
// Shape of the kernel (one CTA per 256 query rows, 1 CTA / SM, 17 warps):
//   warps 0-15  consumers: 4 warpgroups, one per 64 query rows.  Per train tile each warpgroup issues 8
//                       wgmma.mma_async m64n128k32 (K = 256) with both operands read from shared memory, waits for them,
//                       hands the ring stage back, and runs the top-2 selection on the accumulators in its own registers
//                       while the other warpgroups' MMAs keep the tensor cores busy.  In the accumulator fragment a thread
//                       holds 32 columns of two rows; it reduces every 8 dot products of a row to their maximum and compares
//                       it with the dot product of its current second best; only the groups that hit run the top-2
//                       insertion, on packed keys hamming << 22 | index (one multiply-add builds a key, three min / max insert
//                       it: OpenCV's strict '<' with ties to the lowest train index is the unsigned order of those keys).  The
//                       four threads that share a row merge their pairs by shuffles at the end.
//   warp 16     producer: bulk async copies (cp.async.bulk, the TMA engine's 1-D mode) of pre-tiled 32 KB operand blobs into
//                       a 4-stage shared-memory ring, completion on mbarriers.
// The operands are expanded from the packed 256-bit descriptors by knn2_expand_kernel straight into the shared-memory
// image of a tile (canonical K-major layout), so the producer needs no tensor map and no swizzle pattern has to be
// matched by hand anywhere else.  Live queries of a batch are compacted on the way ([nbatch][qcap] slots, counts[b] live).
#include "alva_common.cuh"
#include "../../include/alva_b200.h"

namespace {

constexpr int TM = 128;                 // query rows per A tile (two wgmma M = 64 blocks)
constexpr int TN = 128;                 // train rows per B tile (wgmma N)
constexpr int WM = 64;                  // query rows per consumer warpgroup (wgmma M)
constexpr int KBYTES = 256;             // int8 elements per expanded descriptor
constexpr int BLOB = TM * KBYTES;       // one operand tile in shared memory: 32 KB
constexpr int NSTAGE = 4;               // train-tile ring
constexpr int CONS_WARPS = 16;          // 4 warpgroups x 64 query rows = 256 rows per CTA
constexpr int PROD_WARP = CONS_WARPS;
constexpr int NTHREADS = (CONS_WARPS + 1) * 32;   // + the producer warp
constexpr uint32_t NONE = 0xffffffffu;
constexpr int NEG = -(1 << 20);         // "no candidate yet" dot product

// wgmma shared-memory matrix descriptor pieces, per layout mode (host-filled; kernel parameters so that a debugging run can
// try a variant without a rebuild)
struct MmaLayout {
    uint32_t desc_hi;     // bits 32..63: stride byte offset >> 4 (bits 32..45) | layout type (bits 62..63: 1 = 128-byte swizzle)
    uint32_t lbo16;       // leading byte offset >> 4 (bits 16..29)
    uint32_t koff[8];     // byte offset of K step j (32 int8 each) inside a tile
    uint32_t moff;        // byte offset of query row 64 (the second warpgroup's rows) inside a tile
    int mode;             // 0: no swizzle ("interleaved" 8 x 16 B core matrices)   1: 128-byte swizzle
                          // 2: as 0 with the two offsets exchanged (debugging aid for the descriptor convention)
};

// byte offset of (row r, 16-byte K chunk c) inside a 128-row tile
__host__ __device__ __forceinline__ uint32_t tile_offset(int mode, int r, int c) {
    if (mode != 1) return (uint32_t)c * (TM * 16) + (uint32_t)r * 16;   // core matrix = 8 rows x 16 B contiguous
    return (uint32_t)(c >> 3) * (TM * 128) + (uint32_t)r * 128 + (uint32_t)(((c & 7) ^ (r & 7)) << 4);
}

// ---------------------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 128] (+)= A[64 x 32] * B[128 x 32]^T, both K-major in shared memory; the accumulator fragment stays in registers
__device__ __forceinline__ void wgmma_i8(int (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
        "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n"
        "}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
          "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]),
          "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
          "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]),
          "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]),
          "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]),
          "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]),
          "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_e4m3(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
        "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}

// ---------------------------------------------------------------------------------------------- operand expansion
// offsets[b] = number of live queries in batches < b  (counts clamped to [0, qcap]); one small CTA
__global__ void __launch_bounds__(256) knn2_offsets_kernel(const int32_t* __restrict__ counts, int nbatch, int qcap,
                                                           int32_t* __restrict__ offsets) {
    __shared__ int part[256];
    const int tid = threadIdx.x;
    const int per = (nbatch + 255) / 256;
    const int b0 = tid * per, b1 = min(nbatch, b0 + per);
    int s = 0;
    for (int b = b0; b < b1; b++) s += max(0, min(counts[b], qcap));
    part[tid] = s;
    __syncthreads();
    for (int off = 1; off < 256; off <<= 1) {
        const int v = tid >= off ? part[tid - off] : 0;
        __syncthreads();
        part[tid] += v;
        __syncthreads();
    }
    int run = tid ? part[tid - 1] : 0;
    for (int b = b0; b < b1; b++) { offsets[b] = run; run += max(0, min(counts[b], qcap)); }
    if (tid == 255) offsets[nbatch] = part[255];
}

// 16 descriptor bits -> 16 bytes (+1 for a set bit, -1 for a clear one), LSB first.  int8: 0x01 / 0xFF; E4M3: 0x38 / 0xB8
__device__ __forceinline__ uint4 expand16(uint32_t v, int kind) {
    uint32_t w[4];
#pragma unroll
    for (int g = 0; g < 4; g++) {
        const uint32_t nib = (v >> (4 * g)) & 15u;
        const uint32_t b01 = (nib * 0x00204081u) & 0x01010101u;   // bit i of the nibble -> byte i
        w[g] = kind ? (0xB8B8B8B8u ^ (b01 * 0x80u)) : ~(b01 * 0xFEu);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// One thread per (tile row, 16-byte K chunk).  blockIdx.x < a_blocks: query side (compacting live slots through
// `offsets`), else train side.  Rows past the end of either side are written as zeros (their dot products are masked
// / never stored).  rowmap[compact row] = query slot, or -1.
__global__ void __launch_bounds__(256) knn2_expand_kernel(const uint8_t* __restrict__ q, const int32_t* __restrict__ offsets,
                                                          int nbatch, int qcap, int nq_slots, uint8_t* __restrict__ Aexp,
                                                          int32_t* __restrict__ rowmap, int a_blocks, const uint8_t* __restrict__ t,
                                                          int nt, uint8_t* __restrict__ Bexp, int mode, int kind) {
    const bool is_a = (int)blockIdx.x < a_blocks;
    const int idx = (is_a ? blockIdx.x : blockIdx.x - a_blocks) * 256 + threadIdx.x;
    const int tile = idx >> 11, wi = idx & 2047, c = wi >> 7, r = wi & 127;
    const int R = tile * TM + r;
    const uint8_t* src = nullptr;
    if (is_a) {
        const int total = offsets ? offsets[nbatch] : nq_slots;
        if (R >= ((total + 255) & ~255)) return;   // beyond the last 256-row group any CTA will touch
        int slot = -1;
        if (R < total) {
            if (offsets) {
                int lo = 0, hi = nbatch;
                while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (offsets[mid] <= R) lo = mid; else hi = mid; }
                slot = lo * qcap + (R - offsets[lo]);
            } else slot = R;
            src = q + (size_t)slot * 32;
        }
        if (c == 0) rowmap[R] = slot;
    } else {
        if (R < nt) src = t + (size_t)R * 32;
    }
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (src) o = expand16(*reinterpret_cast<const uint16_t*>(src + 2 * c), kind);
    uint8_t* dst = (is_a ? Aexp : Bexp) + (size_t)tile * BLOB + tile_offset(mode, r, c);
    *reinterpret_cast<uint4*>(dst) = o;
}

// ---------------------------------------------------------------------------------------------- the matcher
struct SmemBars {
    uint64_t full[NSTAGE], empty[NSTAGE], afull;
};

__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, const MmaLayout& L) {
    const uint32_t lo = ((saddr >> 4) & 0x3FFFu) | ((L.lbo16 & 0x3FFFu) << 16);
    return (uint64_t)lo | ((uint64_t)L.desc_hi << 32);
}

// accumulator value type per operand kind, and the value <-> key conversions of the epilogue
template <int KIND> struct Acc;
template <> struct Acc<0> {
    using T = int;
    static __device__ __forceinline__ int neg() { return NEG; }
    static __device__ __forceinline__ int to_int(int v) { return v; }
    // (256 - dot) << 21 | idx as one multiply-add: dot * -(2^21) + ((256 << 21) + idx)  (idx < 2^22, (256 - dot) even)
    static __device__ __forceinline__ uint32_t key(int v, int idx) { return (uint32_t)v * 0xFFE00000u + ((256u << 21) + (uint32_t)idx); }
    static __device__ __forceinline__ int dot_of_key(uint32_t k) { return 256 - (int)(k >> 21); }   // NONE -> -1791: below every dot product
    static __device__ __forceinline__ void mma(int (&d)[64], uint64_t da, uint64_t db, uint32_t acc) { wgmma_i8(d, da, db, acc); }
};
template <> struct Acc<1> {
    using T = float;
    static __device__ __forceinline__ float neg() { return (float)NEG; }
    // the accumulators are integer-valued floats of magnitude <= 256: adding 1.5 * 2^23 leaves the integer in the low mantissa bits
    static __device__ __forceinline__ int to_int(float v) { return __float_as_int(v + 12582912.0f) - 0x4B400000; }
    static __device__ __forceinline__ uint32_t key(float v, int idx) { return (uint32_t)to_int(v) * 0xFFE00000u + ((256u << 21) + (uint32_t)idx); }
    static __device__ __forceinline__ float dot_of_key(uint32_t k) { return (float)(256 - (int)(k >> 21)); }
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) { wgmma_e4m3(d, da, db, acc); }
};

// the pair (k0, k1) of two smallest keys absorbs the pair (o0, o1)
__device__ __forceinline__ void merge2(uint32_t& k0, uint32_t& k1, uint32_t o0, uint32_t o1) {
    const uint32_t hi = max(k0, o0);
    k0 = min(k0, o0);
    k1 = min(min(k1, o1), hi);
}

template <int KIND>
__global__ void __launch_bounds__(NTHREADS, 1)
knn2_mma_kernel(const uint8_t* __restrict__ Aexp, const uint8_t* __restrict__ Bexp, const int32_t* __restrict__ rowmap,
                const int32_t* __restrict__ total_ptr, int nrows, int nt, int ntiles, int tiles_per_chunk, int nchunks,
                uint2* __restrict__ partial, const MmaLayout L, int32_t* __restrict__ dbg) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = sm;
    uint8_t* sB = sm + 2 * BLOB;
    SmemBars& B = *reinterpret_cast<SmemBars*>(sm + (2 + NSTAGE) * BLOB);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int total = total_ptr ? *total_ptr : nrows;
    const int pair = blockIdx.x, chunk = blockIdx.y;
    if (pair * 2 * TM >= total) return;                       // no live query in this group (uniform: before any barrier)
    const int tile0 = chunk * tiles_per_chunk;
    const int nit = min(tiles_per_chunk, ntiles - tile0);     // >= 1 by construction of nchunks

    if (threadIdx.x == 0) {
        for (int s = 0; s < NSTAGE; s++) { mbar_init(&B.full[s], 1); mbar_init(&B.empty[s], CONS_WARPS); }
        mbar_init(&B.afull, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == PROD_WARP) {
        // ---------------------------------------------------------------- producer
        if (lane == 0) {
            mbar_arrive_expect_tx(&B.afull, 2 * BLOB);
            bulk_g2s(sA, Aexp + (size_t)pair * 2 * BLOB, BLOB, &B.afull);
            bulk_g2s(sA + BLOB, Aexp + (size_t)pair * 2 * BLOB + BLOB, BLOB, &B.afull);
        }
        for (int it = 0; it < nit; it++) {
            const int s = it % NSTAGE, ph = (it / NSTAGE) & 1;
            mbar_wait(&B.empty[s], ph ^ 1);
            if (lane == 0) {
                mbar_arrive_expect_tx(&B.full[s], BLOB);
                bulk_g2s(sB + s * BLOB, Bexp + (size_t)(tile0 + it) * BLOB, BLOB, &B.full[s]);
            }
            __syncwarp();
        }
        return;
    }

    // -------------------------------------------------------------------- consumers: MMA + top-2 per query row
    using A = Acc<KIND>;
    using T = typename A::T;
    const int g = warp >> 2;                                  // warpgroup: query rows [64 g, 64 g + 64) of the CTA
    const int t = g >> 1;                                     // A tile
    const int quad = lane & 3;
    const int trow = (g & 1) * WM + (warp & 3) * 16 + (lane >> 2);   // row inside the A tile of accumulator row r0; r1 = r0 + 8
    const uint32_t a0 = smem_u32(sA) + (uint32_t)t * BLOB + (uint32_t)(g & 1) * L.moff;
    // Per thread and row: the two smallest keys seen, key = hamming << 22 | index = (256 - dot) << 21 | index -- the
    // lexicographic (distance, index) order of OpenCV's insertion as ONE unsigned compare, so the insertion itself is three
    // min / max and needs no order of arrival.  thr = the dot product of the current second best: a candidate can only
    // matter if its dot product is strictly above it (its index is larger than everything this thread has seen).
    uint32_t k0[2] = {NONE, NONE}, k1[2] = {NONE, NONE};
    T thr[2] = {A::neg(), A::neg()};
    T d[64];
#pragma unroll
    for (int i = 0; i < 64; i++) d[i] = T(0);

    mbar_wait(&B.afull, 0);
    for (int it = 0; it < nit; it++) {
        const int s = it % NSTAGE, ph = (it / NSTAGE) & 1;
        mbar_wait(&B.full[s], ph);                            // the train tile has landed
        const uint32_t b0 = smem_u32(sB + s * BLOB);
        wg_fence();
#pragma unroll
        for (int j = 0; j < 8; j++) A::mma(d, make_desc(a0 + L.koff[j], L), make_desc(b0 + L.koff[j], L), j > 0 ? 1u : 0u);
        wg_commit();
        wg_wait_all();
        // the accumulators are in registers: hand the stage back to the producer before the selection work
        __syncwarp();
        if (lane == 0) mbar_arrive(&B.empty[s]);

        // fragment: d[4c + 2h + e] = D[r0 + 8h][8c + 2 quad + e], c < 16
        if (dbg && pair == 0 && chunk == 0 && it == 0 && t == 0) {   // the raw dot products, before the tail is masked
#pragma unroll
            for (int i = 0; i < 64; i++) dbg[(trow + 8 * ((i >> 1) & 1)) * TN + 8 * (i >> 2) + 2 * quad + (i & 1)] = A::to_int(d[i]);
        }
        const int n0 = (tile0 + it) * TN + 2 * quad;
        if (n0 - 2 * quad + TN > nt) {                        // only the last train tile: columns past nt hold zero rows
#pragma unroll
            for (int i = 0; i < 64; i++) if (n0 + 8 * (i >> 2) + (i & 1) >= nt) d[i] = A::neg();   // never opens a group
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int k = 0; k < 4; k++) {                     // 8 columns of row r0 + 8h: c = 4k .. 4k + 3, e = 0, 1
                T gmax = d[16 * k + 2 * h];
#pragma unroll
                for (int c = 0; c < 4; c++)
#pragma unroll
                    for (int e = 0; e < 2; e++) gmax = max(gmax, d[16 * k + 4 * c + 2 * h + e]);
                if (gmax > thr[h]) {
#pragma unroll
                    for (int c = 0; c < 4; c++) {
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const int col = n0 + 8 * (4 * k + c) + e;
                            const uint32_t key = col < nt ? A::key(d[16 * k + 4 * c + 2 * h + e], col) : NONE;
                            const uint32_t hi = max(k0[h], key);
                            k0[h] = min(k0[h], key);
                            k1[h] = min(k1[h], hi);
                        }
                    }
                    thr[h] = A::dot_of_key(k1[h]);
                }
            }
        }
    }
    // merge the four threads of a row (lanes 4 j .. 4 j + 3 hold disjoint columns of the same two rows)
#pragma unroll
    for (int h = 0; h < 2; h++) {
#pragma unroll
        for (int x = 1; x <= 2; x <<= 1)
            merge2(k0[h], k1[h], __shfl_xor_sync(0xffffffffu, k0[h], x), __shfl_xor_sync(0xffffffffu, k1[h], x));
        const int row = pair * 2 * TM + t * TM + trow + 8 * h;
        if (quad == 0 && row < total) {
            const int slot = rowmap ? rowmap[row] : row;
            if (slot >= 0) partial[(size_t)slot * nchunks + chunk] = make_uint2(k0[h], k1[h]);
        }
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------- host side
int alva_g_knn_mma = 1;        // alva_set_option("knn_mma", 0 never | 1 automatic (large query sets) | 2 always)
int alva_g_knn_mma_kind = 0;   // alva_set_option("knn_mma_kind", 0 int8 operands / int32 accumulators | 1 E4M3 operands / fp32 accumulators)
int alva_g_knn_mma_mode = 0;   // alva_set_option("knn_mma_mode", 0 no swizzle | 1 128-byte swizzle | 2 debugging variant of 0)

int alva_knn2_merge_launch(alva_ctx* ctx, const uint2* partial, int nq, int nchunks, int32_t* out, const int32_t* counts, int qcap);

static MmaLayout make_layout(int mode) {
    MmaLayout L{};
    L.mode = mode;
    if (mode != 1) {
        // K-major, no swizzle: ((8, n), 2) : ((1, SBO), LBO) in 16-byte units -- core matrices of 8 rows x 16 B
        L.lbo16 = (TM * 16) >> 4;                 // LBO = next 16-byte K chunk
        L.desc_hi = 128u >> 4;                    // SBO = next 8-row group; layout 0
        for (int j = 0; j < 8; j++) L.koff[j] = (uint32_t)j * 2 * TM * 16;
        L.moff = WM * 16;
        if (mode == 2) { L.lbo16 = 128u >> 4; L.desc_hi = (TM * 16u) >> 4; }
    } else {
        // K-major, 128-byte swizzle: rows of 128 B, 8-row groups of 1024 B, two 128-byte K atoms per tile (LBO unused)
        L.lbo16 = 1;
        L.desc_hi = (1024u >> 4) | (1u << 30);
        for (int j = 0; j < 8; j++) L.koff[j] = (uint32_t)(j >> 2) * TM * 128 + (uint32_t)(j & 3) * 32;
        L.moff = WM * 128;
    }
    return L;
}

// true if the tensor-core path should serve this problem.  Measured on H100 (CUDA events, both paths on the same inputs): the
// LOP3/POPC kernel is as fast or faster below ~4 M query x train pairs (2048 x 1024: 12.7 vs 13.6 us), the tensor cores win above
// (4096 x 1024: 13.9 vs 14.6 us; 2048 x 10 000: 31 vs 46 us; 65 536 x 10 000: 317 vs 928 us).
bool alva_knn2_mma_wanted(int nq, int nt) {
    if (alva_g_knn_mma == 2) return true;
    if (alva_g_knn_mma == 0) return false;
    return nq >= 1024 && nt >= 1024 && (long long)nq * nt >= (1LL << 22);
}

// q: [nq][32] (or [nbatch][qcap][32] with counts), t: [nt][32]; out: [nq][4] int32 as alva_k_hamming_knn2
int alva_knn2_mma_launch(alva_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out, const int32_t* counts,
                         int nbatch, int qcap, int32_t* dbg_out) {
    const int a_tiles = 2 * ((nq + 2 * TM - 1) / (2 * TM));
    const int b_tiles = (nt + TN - 1) / TN;
    const int npairs = a_tiles / 2;
    int nchunks = 1;
    if (npairs < ctx->num_sms) {
        nchunks = (2 * ctx->num_sms + npairs - 1) / npairs;
        if (nchunks > b_tiles) nchunks = b_tiles;
    }
    const int tiles_per_chunk = (b_tiles + nchunks - 1) / nchunks;
    nchunks = (b_tiles + tiles_per_chunk - 1) / tiles_per_chunk;

    // workspace: offsets | rowmap | A tiles | B tiles | dbg
    const size_t off_bytes = (((size_t)(counts ? nbatch + 1 : 1) * 4) + 255) & ~(size_t)255;
    const size_t map_bytes = (((size_t)a_tiles * TM * 4) + 255) & ~(size_t)255;
    const size_t a_bytes = (size_t)a_tiles * BLOB, b_bytes = (size_t)b_tiles * BLOB;
    const size_t need = off_bytes + map_bytes + a_bytes + b_bytes;
    if (need > ctx->knn_ws_bytes) {
        if (ctx->knn_ws) { ALVA_CUDA(cudaStreamSynchronize(ctx->stream)); ALVA_CUDA(cudaFree(ctx->knn_ws)); ctx->knn_ws = nullptr; ctx->knn_ws_bytes = 0; }
        ALVA_CUDA(cudaMalloc(&ctx->knn_ws, need + need / 8));
        ctx->knn_ws_bytes = need + need / 8;
    }
    uint8_t* ws = (uint8_t*)ctx->knn_ws;
    int32_t* offsets = counts ? (int32_t*)ws : nullptr;
    int32_t* rowmap = (int32_t*)(ws + off_bytes);
    uint8_t* Aexp = ws + off_bytes + map_bytes;
    uint8_t* Bexp = Aexp + a_bytes;
    uint2* partial = (uint2*)alva_scratch(ctx, (size_t)nq * nchunks * sizeof(uint2));
    if (!partial) return ALVA_E_CUDA;

    const MmaLayout L = make_layout(alva_g_knn_mma_mode);
    if (counts) {
        knn2_offsets_kernel<<<1, 256, 0, ctx->stream>>>(counts, nbatch, qcap, offsets);
        ALVA_LAUNCH_CHECK(ctx);
    }
    const int a_blocks = a_tiles * 8, b_blocks = b_tiles * 8;
    const int kind = alva_g_knn_mma_kind ? 1 : 0;
    knn2_expand_kernel<<<a_blocks + b_blocks, 256, 0, ctx->stream>>>(q, offsets, nbatch, qcap, nq, Aexp, rowmap, a_blocks, t, nt, Bexp, L.mode, kind);
    ALVA_LAUNCH_CHECK(ctx);

    const size_t smem = (size_t)(2 + NSTAGE) * BLOB + sizeof(SmemBars) + 1024;
    const dim3 grid(npairs, nchunks);
    const int32_t* total_ptr = counts ? offsets + nbatch : nullptr;
    if (kind) {
        ALVA_CUDA(cudaFuncSetAttribute(knn2_mma_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        knn2_mma_kernel<1><<<grid, NTHREADS, smem, ctx->stream>>>(Aexp, Bexp, rowmap, total_ptr, nq, nt, b_tiles, tiles_per_chunk, nchunks, partial, L, dbg_out);
    } else {
        ALVA_CUDA(cudaFuncSetAttribute(knn2_mma_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        knn2_mma_kernel<0><<<grid, NTHREADS, smem, ctx->stream>>>(Aexp, Bexp, rowmap, total_ptr, nq, nt, b_tiles, tiles_per_chunk, nchunks, partial, L, dbg_out);
    }
    ALVA_LAUNCH_CHECK(ctx);
    return alva_knn2_merge_launch(ctx, partial, nq, nchunks, out, counts, qcap);
}

// Debugging aid (tools/gpu_knn_mma_check.py): run the tensor-core path unconditionally and also return the raw dot
// products of the first 128 x 128 tile (dbg_dev: 16384 int32, device memory).
extern "C" int alva_debug_knn2_mma(alva_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out, int32_t* dbg_dev) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !q || !t || !out || nq < 1 || nt < 1 || nt >= (1 << 22)) { alva_set_error("alva_debug_knn2_mma: bad argument"); return ALVA_E_INVALID; }
    return alva_knn2_mma_launch(ctx, q, nq, t, nt, out, nullptr, 0, 0, dbg_dev);
}
