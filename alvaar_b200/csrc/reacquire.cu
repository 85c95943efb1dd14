// reacquire.cu -- projection-gated matching of a tracked frame's fresh detections against the frozen map
// (alva_system_set_localisation_only: the map is never changed, so points lost by KLT come back through this match instead of
// through a keyframe).  The CPU restatement is oracle/reacquire_oracle.c; every output equals it exactly.
//
// It restates the gates of the reference's Mapper::matchToMap (src/slam/src/mapper.cpp:354-587) for queries that have no map
// point of their own: per map point of the table (RelocTable layout, ascending id)
//   skip mask -> c = Tcw X, c_z >= 0.1, |c_z| / |c| >= view_th (:425-432) -> projection through the lens (map_geom.cuh, the
//   local-map matcher's code) inside the image -> candidates = the kept queries within `radius` px of the projection ->
//   distance = the minimum Hamming distance over the point's keyframe descriptors (computeMinDescDist with one query
//   descriptor) -> best / second best with the reference's `<=` updates from 51.2 -> ratio test 0.9 (:525-546)
// and per query the map point with the smallest distance, the highest row (= id) among equal ones (the reference's `<=` in
// ascending id order, :565-585).  Candidates are taken in ascending query order; that order decides only which of several
// queries at the same smallest distance is the best (the last one), so it is computed directly as the highest query index.
//
// Unlike Frame::getSurroundingKeypoints (frame.cpp:313-341), which scans only the projection's cell and its upper-left
// neighbours and so misses a query across the right or lower border of the cell, every cell the radius disc touches is
// scanned (the disc widened by 1 px, so that float rounding of the cell index can never drop a query the distance test keeps).
//
// Launches: one CTA builds the query grid (counting sort by cell) and clears the per-query keys; one thread per map point
// applies the gates and posts its best query with a 64-bit atomicMin on (distance, reversed row); one thread per query
// writes the result.
#include "alva_common.cuh"
#include "../../include/alva_b200.h"
#include "map_geom.cuh"
#include <math.h>

namespace {

struct ReacqParams {
    int w, h, cell, ncw, nch;
    double K4[4], D4[4];
    const double* Twc;
    int n_mp;
    const double* wpt;
    const int32_t* desc_start;
    const uint8_t* desc;
    const uint8_t* skip;
    int nq;
    const float* q_px;
    const uint8_t* q_desc;
    const uint8_t* q_kept;
    float radius, view_th, min_dist;
    // scratch
    int32_t* q_cell;      // [nq] cell of a candidate query, -1 otherwise
    int32_t* q_slot;      // [nq] its position inside the cell
    int32_t* cell_start;  // [ncells + 1]
    int32_t* cell_q;      // [nq]
    unsigned long long* qbest;
    // out
    int32_t* q_row;
    int32_t* q_dist;
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// one CTA of 1024 threads: queries -> cells (kept, finite positions only; positions outside the image go to the border cell),
// an exclusive scan of the cell counts, the scatter; the per-query keys are cleared on the way
__global__ void __launch_bounds__(1024) reacq_grid_kernel(const ReacqParams P) {
    __shared__ int warp_sum[32];
    const int tid = threadIdx.x, nt = blockDim.x, ncells = P.ncw * P.nch;
    for (int c = tid; c <= ncells; c += nt) P.cell_start[c] = 0;
    for (int q = tid; q < P.nq; q += nt) P.qbest[q] = 0xffffffffffffffffull;
    __syncthreads();
    for (int q = tid; q < P.nq; q += nt) {
        const float x = P.q_px[2 * q], y = P.q_px[2 * q + 1];
        int cell = -1;
        if (P.q_kept[q] && isfinite(x) && isfinite(y)) {
            const float fx = fminf(fmaxf(x, -1.f), (float)P.w), fy = fminf(fmaxf(y, -1.f), (float)P.h);
            cell = clampi((int)floorf(fy / (float)P.cell), 0, P.nch - 1) * P.ncw + clampi((int)floorf(fx / (float)P.cell), 0, P.ncw - 1);
            P.q_slot[q] = atomicAdd(&P.cell_start[cell + 1], 1);
        }
        P.q_cell[q] = cell;
    }
    __syncthreads();
    // inclusive scan of cell_start[1..ncells]: each thread owns a contiguous chunk
    const int chunk = (ncells + nt - 1) / nt, c0 = 1 + tid * chunk, c1 = min(ncells + 1, c0 + chunk);
    int s = 0;
    for (int c = c0; c < c1; c++) s += P.cell_start[c];
    const int lane = tid & 31, wid = tid >> 5;
    int inc = s;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, off); if (lane >= off) inc += v; }
    if (lane == 31) warp_sum[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        int v = lane < nt / 32 ? warp_sum[lane] : 0;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { const int u = __shfl_up_sync(0xffffffffu, v, off); if (lane >= off) v += u; }
        warp_sum[lane] = v;
    }
    __syncthreads();
    int run = inc - s + (wid > 0 ? warp_sum[wid - 1] : 0);
    for (int c = c0; c < c1; c++) { run += P.cell_start[c]; P.cell_start[c] = run; }
    __syncthreads();
    for (int q = tid; q < P.nq; q += nt) {
        const int cell = P.q_cell[q];
        if (cell >= 0) P.cell_q[P.cell_start[cell] + P.q_slot[q]] = q;
    }
}

template <int LENS>
__global__ void __launch_bounds__(128) reacq_match_kernel(const ReacqParams P) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= P.n_mp) return;
    if (P.skip && P.skip[m]) return;
    const int d0 = P.desc_start[m], nd = P.desc_start[m + 1] - d0;
    if (nd <= 0) return;
    const double X[3] = {P.wpt[3 * m], P.wpt[3 * m + 1], P.wpt[3 * m + 2]};
    double c[3];
    alva_geom::world_to_cam(P.Twc, X, c);
    if (c[2] < 0.1) return;                                                            // mapper.cpp:425
    const float view_angle = (float)(c[2] / sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]));
    if (fabs((double)view_angle) < (double)P.view_th) return;                          // :432
    float proj[2];
    alva_geom::project_cam<LENS>(P.K4, P.D4, c, proj);
    if (!(proj[0] >= 0 && proj[1] >= 0 && (double)proj[0] < (double)P.w && (double)proj[1] < (double)P.h)) return;
    const float r = P.radius;
    const int cx0 = max(0, (int)floorf((proj[0] - r - 1.f) / (float)P.cell)), cx1 = min(P.ncw - 1, (int)floorf((proj[0] + r + 1.f) / (float)P.cell));
    const int cy0 = max(0, (int)floorf((proj[1] - r - 1.f) / (float)P.cell)), cy1 = min(P.nch - 1, (int)floorf((proj[1] + r + 1.f) / (float)P.cell));
    // best: the smallest distance (the highest query index among equal ones); second: the second smallest value; n: candidates
    // within min_dist -- what the `<=` updates in ascending query order leave
    int bestD = 1 << 20, secD = 1 << 20, bestQ = -1, n = 0;
    for (int cy = cy0; cy <= cy1; cy++)
        for (int cx = cx0; cx <= cx1; cx++) {
            const int cell = cy * P.ncw + cx;
            for (int s = P.cell_start[cell]; s < P.cell_start[cell + 1]; s++) {
                const int q = P.cell_q[s];
                const float ddx = proj[0] - P.q_px[2 * q], ddy = proj[1] - P.q_px[2 * q + 1];
                const float pxDist = (float)sqrt((double)ddx * (double)ddx + (double)ddy * (double)ddy);
                if (!(pxDist <= r)) continue;                                          // :454
                const uint4* Q = reinterpret_cast<const uint4*>(P.q_desc + 32 * (size_t)q);
                const uint4 q0 = __ldg(Q), q1 = __ldg(Q + 1);
                int dmin = 1000;
                for (int a = 0; a < nd; a++) {
                    const uint4* A = reinterpret_cast<const uint4*>(P.desc + 32 * (size_t)(d0 + a));
                    const uint4 a0 = __ldg(A), a1 = __ldg(A + 1);
                    const int hd = __popc(a0.x ^ q0.x) + __popc(a0.y ^ q0.y) + __popc(a0.z ^ q0.z) + __popc(a0.w ^ q0.w) +
                                   __popc(a1.x ^ q1.x) + __popc(a1.y ^ q1.y) + __popc(a1.z ^ q1.z) + __popc(a1.w ^ q1.w);
                    dmin = min(dmin, hd);
                }
                if (!((float)dmin <= P.min_dist)) continue;
                n++;
                if (dmin < bestD) { secD = bestD; bestD = dmin; bestQ = q; }
                else if (dmin == bestD) { secD = dmin; bestQ = max(bestQ, q); }
                else if (dmin < secD) secD = dmin;
            }
        }
    if (bestQ < 0) return;
    if (n >= 2 && 0.9 * (double)(float)secD < (double)(float)bestD) return;           // :540-546
    const unsigned long long key = ((unsigned long long)(unsigned)bestD << 32) | (unsigned)(0xffffffffu - (unsigned)m);
    atomicMin(P.qbest + bestQ, key);
}

__global__ void reacq_finalize_kernel(const ReacqParams P) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= P.nq) return;
    const unsigned long long key = P.qbest[q];
    if (key == 0xffffffffffffffffull) { P.q_row[q] = -1; P.q_dist[q] = -1; return; }
    P.q_row[q] = (int32_t)(0xffffffffu - (unsigned)(key & 0xffffffffu));
    P.q_dist[q] = (int32_t)(key >> 32);
}

}  // namespace

extern "C" int alva_k_match_frame_to_map(alva_ctx* ctx, int w, int h, int cell, double fx, double fy, double cx, double cy, int lens,
                                         const double* coef4, const double* Twc, int n_mp, const double* wpt, const int32_t* desc_start,
                                         const uint8_t* desc, const uint8_t* skip, int nq, const float* q_px, const uint8_t* q_desc,
                                         const uint8_t* q_kept, float radius, int32_t* q_row, int32_t* q_dist) { AlvaDeviceGuard guard__(ctx);
    if (!ctx || !Twc || n_mp < 0 || nq < 0 || w < 1 || h < 1 || cell < 1 || lens < alva_geom::LENS_NONE || lens > alva_geom::LENS_FISHEYE ||
        (n_mp > 0 && (!wpt || !desc_start || !desc)) || (nq > 0 && (!q_px || !q_desc || !q_kept || !q_row || !q_dist)) ||
        !(radius >= 0.f) || !(fx > 0) || !(fy > 0)) {
        alva_set_error("alva_k_match_frame_to_map: bad argument");
        return ALVA_E_INVALID;
    }
    if (lens != alva_geom::LENS_NONE) {
        if (!coef4) { alva_set_error("alva_k_match_frame_to_map: coef4 is required with a lens"); return ALVA_E_INVALID; }
        for (int i = 0; i < 4; i++)
            if (!isfinite(coef4[i])) { alva_set_error("alva_k_match_frame_to_map: non-finite lens coefficient"); return ALVA_E_INVALID; }
    }
    if ((n_mp > 0 && ((uintptr_t)desc & 15) != 0) || (nq > 0 && ((uintptr_t)q_desc & 15) != 0)) {
        alva_set_error("alva_k_match_frame_to_map: desc and q_desc must be 16-byte aligned");
        return ALVA_E_INVALID;
    }
    if (nq == 0) return 0;
    ReacqParams P{};
    P.w = w; P.h = h; P.cell = cell;
    P.ncw = (int)ceilf((float)w / (float)cell); P.nch = (int)ceilf((float)h / (float)cell);   // frame.cpp:14-15
    P.K4[0] = fx; P.K4[1] = fy; P.K4[2] = cx; P.K4[3] = cy;
    if (lens != alva_geom::LENS_NONE) for (int i = 0; i < 4; i++) P.D4[i] = coef4[i];
    P.Twc = Twc; P.n_mp = n_mp; P.wpt = wpt; P.desc_start = desc_start; P.desc = desc; P.skip = skip;
    P.nq = nq; P.q_px = q_px; P.q_desc = q_desc; P.q_kept = q_kept;
    // mapper.cpp:365-385, 436: the thresholds in the reference's float arithmetic (on the host, as match.cu)
    const float fovV = (float)(0.5 * h / fy), fovH = (float)(0.5 * w / fx);
    P.view_th = cosf(fovH > fovV ? atanf(fovH) : atanf(fovV));
    P.radius = radius;
    P.min_dist = (float)(32 * 0.2f * 8.);
    const int ncells = P.ncw * P.nch;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t b0 = al((size_t)nq * 4), b1 = al((size_t)(ncells + 1) * 4), b2 = al((size_t)nq * 8);
    uint8_t* ws = (uint8_t*)alva_scratch(ctx, 3 * b0 + b1 + b2);
    if (!ws) return ALVA_E_CUDA;
    P.q_cell = (int32_t*)ws; P.q_slot = (int32_t*)(ws + b0); P.cell_q = (int32_t*)(ws + 2 * b0); P.cell_start = (int32_t*)(ws + 3 * b0);
    P.qbest = (unsigned long long*)(ws + 3 * b0 + b1);
    P.q_row = q_row; P.q_dist = q_dist;
    reacq_grid_kernel<<<1, 1024, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    if (n_mp > 0) {
        const int nb = (n_mp + 127) / 128;
        if (lens == alva_geom::LENS_RADTAN) reacq_match_kernel<alva_geom::LENS_RADTAN><<<nb, 128, 0, ctx->stream>>>(P);
        else if (lens == alva_geom::LENS_FISHEYE) reacq_match_kernel<alva_geom::LENS_FISHEYE><<<nb, 128, 0, ctx->stream>>>(P);
        else reacq_match_kernel<alva_geom::LENS_NONE><<<nb, 128, 0, ctx->stream>>>(P);
        ALVA_LAUNCH_CHECK(ctx);
    }
    reacq_finalize_kernel<<<(nq + 255) / 256, 256, 0, ctx->stream>>>(P);
    ALVA_LAUNCH_CHECK(ctx);
    return 0;
}
