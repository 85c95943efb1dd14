// hamming.cu -- brute-force Hamming 2-NN over 256-bit descriptors, sm_90a.
//
// Reference behaviour (exact): cv::BFMatcher(NORM_HAMMING).knnMatch(k = 2)
//   opencv features2d/src/matchers.cpp:757 -> core/src/batch_distance.cpp:103-123 (batchDistHamming),
//   k-NN insertion :235-248 (strict '<': ties keep the lowest train index), popcount core/src/stat.simd.hpp:81-128.
// The same primitive serves MapPoint::computeMinDescDist (src/slam/src/map_point.cpp:204-222).
//
// Integer-ALU bound (xor + popc), not HBM: 8 queries live in registers per warp, every lane streams its own train
// descriptors with two 128-bit loads, candidates are packed as (dist << 22 | index) so the lexicographic
// (distance, index) order OpenCV's insertion produces is a plain unsigned min; the 32 per-lane top-2 lists are merged
// with warp shuffles, chunk partials with a tiny second kernel.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"

namespace {

constexpr int QPW_MAX = 8;      // queries per warp: 8 (128 registers, 16 warps/SM) or 4 (<= 80 registers, 24 warps/SM); the batch
                                // entry point requires qcap % 8 == 0 so that either grouping never straddles two frames
constexpr int WPC = 8;          // warps per CTA
constexpr int MIN_CHUNK = 512;  // never split the train set finer than this
constexpr uint32_t NONE = 0xffffffffu;

__device__ __forceinline__ void top2_insert(uint32_t& k0, uint32_t& k1, uint32_t key) {
    if (key < k1) {
        if (key < k0) { k1 = k0; k0 = key; }
        else k1 = key;
    }
}

__device__ __forceinline__ uint32_t xor2(uint32_t a, uint32_t b) {
    uint32_t d;
    asm("xor.b32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t csa_sum(uint32_t a, uint32_t b, uint32_t c) {     // a ^ b ^ c
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ uint32_t csa_carry(uint32_t a, uint32_t b, uint32_t c) {   // majority(a, b, c)
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0xe8;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// exact warp-wide top-2 of the 32 per-lane (best, second) key pairs with three REDUX (keys are unique: the index is in them)
__device__ __forceinline__ void warp_top2(uint32_t k0, uint32_t k1, uint32_t& m0, uint32_t& m1) {
    m0 = __reduce_min_sync(0xffffffffu, k0);
    const uint32_t s = __reduce_min_sync(0xffffffffu, k0 == m0 ? NONE : k0);
    m1 = min(s, __reduce_min_sync(0xffffffffu, k1));
}

// one train descriptor per lane against the warp's QPW queries
template <int QPW, bool TAIL>
__device__ __forceinline__ void knn_step(const uint4 (&qa)[QPW], const uint4 (&qb)[QPW], uint32_t (&k0)[QPW], uint32_t (&k1)[QPW],
                                         uint32_t (&tk)[QPW], const uint4* __restrict__ t, int j, int te, uint32_t mul22,
                                         uint32_t mul23, uint32_t mul24) {
    const bool valid = !TAIL || j < te;
    const int jl = valid ? j : te - 1;
    const uint4 a = __ldg(t + 2 * jl), b = __ldg(t + 2 * jl + 1);
    uint32_t key[QPW];
    bool hit = false;
#pragma unroll
    for (int i = 0; i < QPW; i++) {
        // 256-bit popcount with 4 POPC instead of 8: three carry-save adders (sum = a^b^c, carry = maj(a,b,c): one LOP3
        // each) compress the eight xor words into ones / twos / fours planes:
        //   d = popc(ones) + popc(w7) + 2 popc(twos) + 4 popc(fours).
        // (opaque asm: left to itself the compiler re-associates the xors into the adders and ends up with ~21 LOP3
        //  per distance instead of the 16 written here)
        const uint32_t x0 = xor2(qa[i].x, a.x), x1 = xor2(qa[i].y, a.y), x2 = xor2(qa[i].z, a.z), x3 = xor2(qa[i].w, a.w);
        const uint32_t x4 = xor2(qb[i].x, b.x), x5 = xor2(qb[i].y, b.y), x6 = xor2(qb[i].z, b.z), x7 = xor2(qb[i].w, b.w);
        const uint32_t s1 = csa_sum(x0, x1, x2), c1 = csa_carry(x0, x1, x2);
        const uint32_t s2 = csa_sum(x3, x4, x5), c2 = csa_carry(x3, x4, x5);
        const uint32_t s3 = csa_sum(s1, s2, x6), c3 = csa_carry(s1, s2, x6);
        const uint32_t s4 = csa_sum(c1, c2, c3), c4 = csa_carry(c1, c2, c3);
        // key = (d << 22) + j, as a chain of multiply-adds
        uint32_t k = (uint32_t)(__popc(s3) + __popc(x7)) * mul22 + (uint32_t)j;
        k = (uint32_t)__popc(s4) * mul23 + k;
        k = (uint32_t)__popc(c4) * mul24 + k;
        key[i] = (TAIL && !valid) ? NONE : k;
        hit |= key[i] < tk[i];
    }
    if (__any_sync(0xffffffffu, hit)) {
#pragma unroll
        for (int i = 0; i < QPW; i++) {
            if (__any_sync(0xffffffffu, key[i] < tk[i])) {
                top2_insert(k0[i], k1[i], key[i]);
                uint32_t m0;
                warp_top2(k0[i], k1[i], m0, tk[i]);
            }
        }
    }
}

// counts != nullptr: the queries are [nbatch][qcap] slots of which only the first counts[b] are live; warps that hold
// no live query leave immediately (their partials are never read).
//
// Selection costs almost nothing: every warp keeps, per query, the key of the warp-wide SECOND best seen so far (tk).  A
// candidate can only change the final answer if its key is below tk, so the common path per distance is one compare; the
// rare path (about 2 ln N times per query) inserts into the lane's private pair and refreshes tk with three REDUX.
// mul = {2^22, 2^23, 2^24} as run-time data: weights and key packing become IMADs on the FMA pipe instead of shifts /
// LEAs on the ALU pipe, which the 16 LOP3 per distance already saturate.
template <int QPW>
__global__ void __launch_bounds__(WPC * 32, QPW == 8 ? 2 : 3) knn2_partial_kernel(const uint4* __restrict__ q, int nq, const uint4* __restrict__ t,
                                                                int nt, uint2* __restrict__ partial, int nchunks, int chunk_len,
                                                                const int32_t* __restrict__ counts, int qcap, uint32_t mul22,
                                                                uint32_t mul23, uint32_t mul24) {
    // One CTA = 8 warps x 8 queries against one chunk of the train set.  CTAs are deliberately short-lived (tens of
    // microseconds): the step's local BA and pyramid kernels run beside this one on other streams and can only get SM
    // resources when a CTA retires -- a persistent variant of this kernel starved them and cost 25 % of the step.
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    {
        const int q0 = (blockIdx.x * WPC + warp) * QPW;
        if (q0 >= nq) return;
        if (counts) { const int b = q0 / qcap; if (q0 - b * qcap >= counts[b]) return; }
        const int chunk = blockIdx.y;
        const int tb = chunk * chunk_len, te = min(nt, tb + chunk_len);
        uint4 qa[QPW], qb[QPW];
#pragma unroll
        for (int i = 0; i < QPW; i++) {
            const int qi = min(q0 + i, nq - 1);
            qa[i] = __ldg(q + 2 * qi);
            qb[i] = __ldg(q + 2 * qi + 1);
        }
        uint32_t k0[QPW], k1[QPW], tk[QPW];
#pragma unroll
        for (int i = 0; i < QPW; i++) k0[i] = k1[i] = tk[i] = NONE;
        const int full_steps = (te - tb) >> 5;   // warp-uniform trip count (the rare path votes)
        for (int sidx = 0; sidx < full_steps; sidx++)
            knn_step<QPW, false>(qa, qb, k0, k1, tk, t, tb + 32 * sidx + lane, te, mul22, mul23, mul24);
        if (tb + 32 * full_steps < te)   // ragged tail: lanes past the end contribute nothing
            knn_step<QPW, true>(qa, qb, k0, k1, tk, t, tb + 32 * full_steps + lane, te, mul22, mul23, mul24);
#pragma unroll
        for (int i = 0; i < QPW; i++) {
            uint32_t m0, m1;
            warp_top2(k0[i], k1[i], m0, m1);
            if (lane == 0 && q0 + i < nq) partial[(size_t)(q0 + i) * nchunks + chunk] = make_uint2(m0, m1);
        }
    }
}

__global__ void knn2_merge_kernel(const uint2* __restrict__ partial, int nq, int nchunks, int32_t* __restrict__ out,
                                  const int32_t* __restrict__ counts, int qcap) {
    const int qi = blockIdx.x * blockDim.x + threadIdx.x;
    if (qi >= nq) return;
    uint32_t k0 = NONE, k1 = NONE;
    bool live = true;
    if (counts) { const int b = qi / qcap; live = (qi - b * qcap) < counts[b]; }
    for (int c = 0; live && c < nchunks; c++) {
        const uint2 p = partial[(size_t)qi * nchunks + c];
        top2_insert(k0, k1, p.x);
        top2_insert(k0, k1, p.y);
    }
    int4 r;
    r.x = k0 == NONE ? -1 : (int)(k0 & 0x3fffff);
    r.y = k0 == NONE ? -1 : (int)(k0 >> 22);
    r.z = k1 == NONE ? -1 : (int)(k1 & 0x3fffff);
    r.w = k1 == NONE ? -1 : (int)(k1 >> 22);
    reinterpret_cast<int4*>(out)[qi] = r;
}


// ---- block-pair matching for the cross-stream loop-closure search (loopclosure.cu) --------------------------------------------
// gathered: [world][K] keyframe blocks of `block_bytes` each (wire format: include/alva_b200.h, "keyframe block"); this rank's
// keyframe e is matched against keyframe e of every other rank r: 2-NN of each live local descriptor among the live remote
// ones.  grid (query tiles, world, K); out [K][world][n_max] int4 = (idx0, dist0, idx1, dist1), -1 where there is none.
__global__ void __launch_bounds__(WPC * 32, 3) knn2_blockpair_kernel(const uint8_t* __restrict__ gathered, size_t block_bytes, int n_max, int K,
                                                                      int rank, int hdr_bytes, int4* __restrict__ out, uint32_t mul22,
                                                                      uint32_t mul23, uint32_t mul24) {
    constexpr int QPW = 4;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = blockIdx.y, e = blockIdx.z;
    if (r == rank) return;
    const uint8_t* lb = gathered + ((size_t)rank * K + e) * block_bytes;
    const uint8_t* rb = gathered + ((size_t)r * K + e) * block_bytes;
    // header counts come from other ranks: clamped to [0, n_max] (a negative train count would step the tail before the array)
    const int nq = min(max(reinterpret_cast<const int32_t*>(lb)[4], 0), n_max);
    const int nt = min(max(reinterpret_cast<const int32_t*>(rb)[4], 0), n_max);
    const int q0 = (blockIdx.x * WPC + warp) * QPW;
    if (q0 >= nq) return;
    const uint4* q = reinterpret_cast<const uint4*>(lb + hdr_bytes + (size_t)n_max * 8);
    const uint4* t = reinterpret_cast<const uint4*>(rb + hdr_bytes + (size_t)n_max * 8);
    int4* o = out + ((size_t)e * gridDim.y + r) * n_max;
    uint4 qa[QPW], qb[QPW];
#pragma unroll
    for (int i = 0; i < QPW; i++) {
        const int qi = min(q0 + i, nq - 1);
        qa[i] = __ldg(q + 2 * qi);
        qb[i] = __ldg(q + 2 * qi + 1);
    }
    uint32_t k0[QPW], k1[QPW], tk[QPW];
#pragma unroll
    for (int i = 0; i < QPW; i++) k0[i] = k1[i] = tk[i] = NONE;
    const int full_steps = nt >> 5;
    for (int sidx = 0; sidx < full_steps; sidx++) knn_step<QPW, false>(qa, qb, k0, k1, tk, t, 32 * sidx + lane, nt, mul22, mul23, mul24);
    if (32 * full_steps < nt) knn_step<QPW, true>(qa, qb, k0, k1, tk, t, 32 * full_steps + lane, nt, mul22, mul23, mul24);
#pragma unroll
    for (int i = 0; i < QPW; i++) {
        uint32_t m0, m1;
        warp_top2(k0[i], k1[i], m0, m1);
        if (lane == 0 && q0 + i < nq)
            o[q0 + i] = make_int4(m0 == NONE ? -1 : (int)(m0 & 0x3fffff), m0 == NONE ? -1 : (int)(m0 >> 22), m1 == NONE ? -1 : (int)(m1 & 0x3fffff),
                                  m1 == NONE ? -1 : (int)(m1 >> 22));
    }
}

}  // namespace

// Chunking of the train set.  Long chunks make the selection filter effective (its rare path runs ~2 ln(chunk) times per
// query); short CTAs keep the launch tail small and let concurrent streams in.  Aim at ~16 waves.
static void knn_chunks(const alva_ctx* ctx, int nq, int nt, int QPW, int* nchunks, int* chunk_len) {
    const int ctas_q = (nq + QPW * WPC - 1) / (QPW * WPC);
    const int target = (QPW == 8 ? 2 : 3) * ctx->num_sms * 16;   // ~16 waves of the 2 resident CTAs per SM: short CTAs, negligible tail
    int n = (target + ctas_q - 1) / ctas_q;
    const int nmax = (nt + MIN_CHUNK - 1) / MIN_CHUNK;
    if (n > nmax) n = nmax;
    if (n < 1) n = 1;
    int len = ((nt + n - 1) / n + 31) & ~31;
    *nchunks = (nt + len - 1) / len;
    *chunk_len = len;
}

int alva_g_knn_qpw = 4;   // alva_set_option("knn_qpw", 4 | 8)

// hamming_mma.cu: the tensor-core formulation (large query sets)
bool alva_knn2_mma_wanted(int nq, int nt);
int alva_knn2_mma_launch(alva_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out, const int32_t* counts,
                         int nbatch, int qcap, int32_t* dbg_out);
int alva_knn2_merge_launch(alva_ctx* ctx, const uint2* partial, int nq, int nchunks, int32_t* out, const int32_t* counts, int qcap) {
    knn2_merge_kernel<<<(nq + 127) / 128, 128, 0, ctx->stream>>>(partial, nq, nchunks, out, counts, qcap);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

static int knn_launch(alva_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out, const int32_t* counts, int qcap) {
    if (alva_knn2_mma_wanted(nq, nt)) return alva_knn2_mma_launch(ctx, q, nq, t, nt, out, counts, counts ? nq / qcap : 0, qcap, nullptr);
    int nchunks, chunk_len;
    const int QPW = alva_g_knn_qpw == 4 ? 4 : 8;
    knn_chunks(ctx, nq, nt, QPW, &nchunks, &chunk_len);
    uint2* partial = (uint2*)alva_scratch(ctx, (size_t)nq * nchunks * sizeof(uint2));
    if (!partial) return ALVA_E_CUDA;
    dim3 grid((nq + QPW * WPC - 1) / (QPW * WPC), nchunks);
    if (QPW == 8)
        knn2_partial_kernel<8><<<grid, WPC * 32, 0, ctx->stream>>>((const uint4*)q, nq, (const uint4*)t, nt, partial, nchunks, chunk_len,
                                                                   counts, qcap, 1u << 22, 1u << 23, 1u << 24);
    else
        knn2_partial_kernel<4><<<grid, WPC * 32, 0, ctx->stream>>>((const uint4*)q, nq, (const uint4*)t, nt, partial, nchunks, chunk_len,
                                                                   counts, qcap, 1u << 22, 1u << 23, 1u << 24);
    ALVA_LAUNCH_CHECK(ctx);
    return alva_knn2_merge_launch(ctx, partial, nq, nchunks, out, counts, qcap);
}

extern "C" int alva_k_hamming_knn2(alva_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !q || !t || !out || nq < 1 || nt < 1 || nt >= (1 << 22) || ((uintptr_t)q & 15) || ((uintptr_t)t & 15) ||
        ((uintptr_t)out & 15)) {
        alva_set_error("alva_k_hamming_knn2: bad argument (need 16-byte aligned buffers, 1 <= nt < 2^22)");
        return ALVA_E_INVALID;
    }
    return knn_launch(ctx, q, nq, t, nt, out, nullptr, 0);
}

extern "C" int alva_k_hamming_knn2_batch(alva_ctx* ctx, const uint8_t* q, const int32_t* counts, int nbatch, int qcap,
                                         const uint8_t* t, int nt, int32_t* out) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !q || !counts || !t || !out || nbatch < 1 || qcap < 1 || (qcap % QPW_MAX) != 0 || nt < 1 || nt >= (1 << 22) ||
        ((uintptr_t)q & 15) || ((uintptr_t)t & 15) || ((uintptr_t)out & 15)) {
        alva_set_error("alva_k_hamming_knn2_batch: bad argument (qcap must be a multiple of %d)", QPW_MAX);
        return ALVA_E_INVALID;
    }
    const int nq = nbatch * qcap;
    return knn_launch(ctx, q, nbatch * qcap, t, nt, out, counts, qcap);
}

// internal (loopclosure.cu)
int alva_knn2_blockpair_launch(alva_ctx* ctx, const uint8_t* gathered, size_t block_bytes, int n_max, int K, int world, int rank,
                               int hdr_bytes, int32_t* out) {
    dim3 grid((n_max + 4 * WPC - 1) / (4 * WPC), world, K);
    knn2_blockpair_kernel<<<grid, WPC * 32, 0, ctx->stream>>>(gathered, block_bytes, n_max, K, rank, hdr_bytes, reinterpret_cast<int4*>(out),
                                                               1u << 22, 1u << 23, 1u << 24);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}
