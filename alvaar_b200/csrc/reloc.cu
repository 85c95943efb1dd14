// reloc.cu -- the matching half of System's relocalisation (system_core.h: a lost frame's ORB descriptors straight against
// every map point, no pose prior); the pose half is alva_k_p3p_ransac + PnP in pose.cu.  The CPU restatement is
// oracle/reloc_oracle.c.
//
//   alva_k_hamming_knn2_grouped   2-NN over GROUPS of descriptors (a map point keeps one descriptor per keyframe that described
//                                 it; its distance to a query is the minimum over them, as MapPoint::computeMinDescDist in the
//                                 reference's matcher).  The table is CSR: desc_start[n_grp + 1] -> desc[rows][32].
//   alva_reloc_compact_launch     (internal) distance gate, ratio test, one query per map point; writes the RANSAC / PnP inputs.
//
// How: a group's rows are contiguous, so a thread that holds one query in registers walks the rows in order, keeps the running
// minimum of the current group and folds it into its top-2 at each group boundary (the boundaries are the same for every
// thread of a CTA: no divergence).  The rows are split over CTAs in chunks of CHUNK_ROWS nominal rows; a group belongs to the
// chunk its first row falls in, so a chunk ends on a group boundary (it may run up to one group past its nominal end).
// Top-2 partials of disjoint groups, taken in ascending group order, merge exactly: a last kernel folds the chunks' partials.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"

namespace {

constexpr int KNN_THREADS = 128;     // queries per CTA (one per thread)
constexpr int CHUNK_ROWS = 2048;     // nominal table rows per CTA
constexpr int TILE_ROWS = 256;       // rows staged in shared memory at a time
constexpr int NONE = 0x7fffffff;

struct Top2 { int g0, d0, g1, d1; };

__device__ __forceinline__ void top2_fold(Top2& t, int g, int d) {   // groups arrive in ascending order: ties keep the earlier
    if (d < t.d0) { t.g1 = t.g0; t.d1 = t.d0; t.g0 = g; t.d0 = d; }
    else if (d < t.d1) { t.g1 = g; t.d1 = d; }
}

// first index in [0, n) with a[i] >= v (n if none)
__device__ __forceinline__ int lower_bound(const int32_t* __restrict__ a, int n, int v) {
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(a + mid) < v) lo = mid + 1; else hi = mid; }
    return lo;
}

// grid (ceil(nq / KNN_THREADS), chunks): partial[chunk][nq] = the top-2 of the chunk's groups
__global__ void __launch_bounds__(KNN_THREADS) knn2_grouped_chunk_kernel(const uint8_t* __restrict__ q, int nq,
                                                                         const int32_t* __restrict__ ds, int n_grp,
                                                                         const uint8_t* __restrict__ desc, int4* __restrict__ partial) {
    __shared__ uint4 rows[TILE_ROWS][2];
    const int qi = blockIdx.x * KNN_THREADS + threadIdx.x, chunk = blockIdx.y;
    uint32_t qw[8];
    if (qi < nq) {
        const uint4* qp = (const uint4*)(q + 32 * (size_t)qi);
        const uint4 a = qp[0], b = qp[1];
        qw[0] = a.x; qw[1] = a.y; qw[2] = a.z; qw[3] = a.w; qw[4] = b.x; qw[5] = b.y; qw[6] = b.z; qw[7] = b.w;
    } else {
        for (int k = 0; k < 8; k++) qw[k] = 0;
    }
    const int g_lo = lower_bound(ds, n_grp, chunk * CHUNK_ROWS), g_hi = lower_bound(ds, n_grp, (chunk + 1) * CHUNK_ROWS);
    Top2 t{-1, NONE, -1, NONE};
    if (g_lo < g_hi) {
        const int r0 = __ldg(ds + g_lo), r1 = __ldg(ds + g_hi);
        int g = g_lo, gend = __ldg(ds + g_lo + 1), cur = NONE;
        for (int t0 = r0; t0 < r1; t0 += TILE_ROWS) {
            const int tn = min(TILE_ROWS, r1 - t0);
            for (int i = threadIdx.x; i < 2 * tn; i += KNN_THREADS) rows[i >> 1][i & 1] = ((const uint4*)(desc + 32 * (size_t)t0))[i];
            __syncthreads();
            for (int r = 0; r < tn; r++) {
                while (t0 + r >= gend) {   // group g is complete (empty groups fold NONE: never a candidate)
                    if (cur != NONE) top2_fold(t, g, cur);
                    cur = NONE; g++; gend = __ldg(ds + g + 1);
                }
                const uint4 a = rows[r][0], b = rows[r][1];
                const int d = __popc(qw[0] ^ a.x) + __popc(qw[1] ^ a.y) + __popc(qw[2] ^ a.z) + __popc(qw[3] ^ a.w) +
                              __popc(qw[4] ^ b.x) + __popc(qw[5] ^ b.y) + __popc(qw[6] ^ b.z) + __popc(qw[7] ^ b.w);
                cur = min(cur, d);
            }
            __syncthreads();
        }
        if (cur != NONE) top2_fold(t, g, cur);
    }
    if (qi < nq) partial[(size_t)chunk * nq + qi] = make_int4(t.g0, t.d0, t.g1, t.d1);
}

__global__ void __launch_bounds__(256) knn2_grouped_merge_kernel(const int4* __restrict__ partial, int nq, int nchunks,
                                                                 int32_t* __restrict__ out) {
    const int qi = blockIdx.x * blockDim.x + threadIdx.x;
    if (qi >= nq) return;
    Top2 t{-1, NONE, -1, NONE};
    for (int c = 0; c < nchunks; c++) {
        const int4 p = partial[(size_t)c * nq + qi];
        if (p.x >= 0) top2_fold(t, p.x, p.y);
        if (p.z >= 0) top2_fold(t, p.z, p.w);
    }
    reinterpret_cast<int4*>(out)[qi] = make_int4(t.g0, t.g0 >= 0 ? t.d0 : -1, t.g1, t.g1 >= 0 ? t.d1 : -1);
}

// the gate and the ratio test (5 d0 < 4 d1: d0 < 0.8 d1 exactly; one candidate group passes), and each group's best survivor:
// key[g] = min over its survivors of (d0 << 16 | query index) -- the smallest distance, then the lowest query index
__device__ __forceinline__ bool reloc_pass(const int4 k, int max_dist) { return k.x >= 0 && k.y <= max_dist && (k.z < 0 || 5 * k.y < 4 * k.w); }

__global__ void __launch_bounds__(256) reloc_best_kernel(const int4* __restrict__ knn, int nq, int max_dist, uint32_t* __restrict__ key) {
    const int qi = blockIdx.x * blockDim.x + threadIdx.x;
    if (qi >= nq) return;
    const int4 k = knn[qi];
    if (reloc_pass(k, max_dist)) atomicMin(key + k.x, ((uint32_t)k.y << 16) | (uint32_t)qi);
}

// one CTA: the kept matches in ascending query order -> bearing / world point / uv lists, (query, group) pairs, count
__global__ void __launch_bounds__(256) reloc_compact_kernel(const int4* __restrict__ knn, int nq, int max_dist, const uint32_t* __restrict__ key,
                                                            const double* __restrict__ q_bv, const double* __restrict__ q_uv,
                                                            const double* __restrict__ grp_wpt, double* __restrict__ bv, double* __restrict__ X,
                                                            double* __restrict__ uv, int32_t* __restrict__ mq, int32_t* __restrict__ mg,
                                                            int32_t* __restrict__ count) {
    __shared__ int woff[8];
    __shared__ int base_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) base_s = 0;
    __syncthreads();
    for (int i0 = 0; i0 < nq; i0 += 256) {
        const int i = i0 + tid;
        bool keep = false;
        int4 k = make_int4(-1, -1, -1, -1);
        if (i < nq) {
            k = knn[i];
            keep = reloc_pass(k, max_dist) && key[k.x] == (((uint32_t)k.y << 16) | (uint32_t)i);
        }
        const uint32_t m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) woff[warp] = __popc(m);
        __syncthreads();
        int off = base_s;
        for (int w = 0; w < warp; w++) off += woff[w];
        if (keep) {
            const int d = off + __popc(m & ((1u << lane) - 1u));
            for (int c = 0; c < 3; c++) { bv[3 * d + c] = q_bv[3 * i + c]; X[3 * d + c] = grp_wpt[3 * (size_t)k.x + c]; }
            uv[2 * d] = q_uv[2 * i]; uv[2 * d + 1] = q_uv[2 * i + 1];
            mq[d] = i; mg[d] = k.x;
        }
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < 8; w++) t += woff[w]; base_s += t; }
        __syncthreads();
    }
    if (tid == 0) count[0] = base_s;
}

int knn2_grouped_launch(alva_ctx* ctx, const uint8_t* q, int nq, const int32_t* desc_start, int n_grp, const uint8_t* desc, int n_rows,
                        int32_t* out) {
    if (nq == 0) return 0;
    const int nchunks = n_rows > 0 ? (n_rows + CHUNK_ROWS - 1) / CHUNK_ROWS : 1;
    int4* partial = (int4*)alva_scratch(ctx, (size_t)nchunks * nq * sizeof(int4) + 256);
    if (!partial) return ALVA_E_CUDA;
    knn2_grouped_chunk_kernel<<<dim3((nq + KNN_THREADS - 1) / KNN_THREADS, nchunks), KNN_THREADS, 0, ctx->stream>>>(q, nq, desc_start, n_grp,
                                                                                                                   desc, partial);
    ALVA_LAUNCH_CHECK(ctx);
    knn2_grouped_merge_kernel<<<(nq + 255) / 256, 256, 0, ctx->stream>>>(partial, nq, nchunks, out);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}

}  // namespace

extern "C" int alva_k_hamming_knn2_grouped(alva_ctx* ctx, const uint8_t* q, int nq, const int32_t* desc_start, int n_grp,
                                           const uint8_t* desc, int n_rows, int32_t* out) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || nq < 0 || n_grp < 0 || n_rows < 0 || (nq > 0 && (!q || !out)) || !desc_start || (n_rows > 0 && !desc)) {
        alva_set_error("alva_k_hamming_knn2_grouped: bad argument");
        return ALVA_E_INVALID;
    }
    if (nq > 65535) { alva_set_error("alva_k_hamming_knn2_grouped: at most 65535 queries (got %d)", nq); return ALVA_E_INVALID; }
    return knn2_grouped_launch(ctx, q, nq, desc_start, n_grp, desc, n_rows, out);
}

// internal (system.cu): knn [nq][4] of alva_k_hamming_knn2_grouped -> the correspondences relocalisation keeps, in ascending
// query order: bv / X [cap][3], uv [cap][2], mq / mg [cap] (query, group), count[1].  q_bv [nq][3] / q_uv [nq][2]: the
// queries' bearings and undistorted pixels; grp_wpt [n_grp][3]: the groups' world points; key [n_grp]: scratch.
int alva_reloc_compact_launch(alva_ctx* ctx, const int32_t* knn, int nq, int n_grp, int max_dist, const double* q_bv, const double* q_uv,
                              const double* grp_wpt, uint32_t* key, double* bv, double* X, double* uv, int32_t* mq, int32_t* mg,
                              int32_t* count) {
    if (n_grp > 0) {
        if (cudaMemsetAsync(key, 0xff, (size_t)n_grp * 4, ctx->stream) != cudaSuccess) { alva_set_error("reloc: memset failed"); return ALVA_E_CUDA; }
    }
    if (nq > 0 && n_grp > 0) {
        reloc_best_kernel<<<(nq + 255) / 256, 256, 0, ctx->stream>>>((const int4*)knn, nq, max_dist, key);
        ALVA_LAUNCH_CHECK(ctx);
    }
    reloc_compact_kernel<<<1, 256, 0, ctx->stream>>>((const int4*)knn, n_grp > 0 ? nq : 0, max_dist, key, q_bv, q_uv, grp_wpt, bv, X, uv, mq,
                                                     mg, count);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}
