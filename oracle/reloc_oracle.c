/* oracle/reloc_oracle.c -- CPU restatement of System's relocalisation against its map (alvaar_b200/csrc/reloc.cu and
 * alva_k_p3p_ransac in pose.cu; the state machine around it is system_core.h):
 *   grouped Hamming 2-NN   every query against a table of map points, each a group of 256-bit descriptors (one per keyframe
 *                          that described it); a point's distance is the minimum over its rows (the rule of
 *                          MapPoint::computeMinDescDist in the reference's matcher)
 *   compaction             the distance gate, the ratio test and one query per map point, into correspondence lists
 *   P3P-RANSAC             the sampler and the Kneip P3P hypotheses of orc_p3p_lmeds (pose_oracle.c), scored by inlier count
 *
 * TEST INFRASTRUCTURE ONLY: only tests/ build and call this (tests/reloc_util.py links it against libalva_oracle.so for
 * orc_sac_rnd / orc_p3p_sample_model).  The product never links or executes it.  Plain C, FP64, no FMA contraction.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

void orc_sac_rnd(uint32_t seed, int n, int32_t* out);                                     /* pose_oracle.c */
int orc_p3p_sample_model(const double* bvs, const double* wpts, const int* idx, double* T);  /* pose_oracle.c */

static int ham256(const uint8_t* a, const uint8_t* b)
{
    int d = 0;
    for (int i = 0; i < 32; i++) d += __builtin_popcount((unsigned)(a[i] ^ b[i]));
    return d;
}

/* q [nq][32]; desc_start [n_grp + 1] row offsets into desc [..][32].  out [nq][4] = {grp0, d0, grp1, d1}: the nearest and
 * second-nearest groups by their minimum row distance, ties to the lower group index, -1 / -1 where there is none.  Groups
 * without rows are never candidates. */
void orc_hamming_knn2_grouped(const uint8_t* q, int nq, const int32_t* desc_start, int n_grp, const uint8_t* desc, int32_t* out)
{
    for (int i = 0; i < nq; i++) {
        int g0 = -1, d0 = 0x7fffffff, g1 = -1, d1 = 0x7fffffff;
        for (int g = 0; g < n_grp; g++) {
            int m = 0x7fffffff;
            for (int r = desc_start[g]; r < desc_start[g + 1]; r++) {
                const int d = ham256(q + 32 * (size_t)i, desc + 32 * (size_t)r);
                if (d < m) m = d;
            }
            if (m == 0x7fffffff) continue;
            if (m < d0) { g1 = g0; d1 = d0; g0 = g; d0 = m; }
            else if (m < d1) { g1 = g; d1 = m; }
        }
        out[4 * i] = g0; out[4 * i + 1] = g0 >= 0 ? d0 : -1;
        out[4 * i + 2] = g1; out[4 * i + 3] = g1 >= 0 ? d1 : -1;
    }
}

/* The matches relocalisation keeps, in ascending query order: query i survives when d0 <= max_dist and d0 < 0.8 d1 (evaluated
 * exactly as 5 d0 < 4 d1; a query with one candidate group passes the ratio test), and it is the survivor of its group with
 * the smallest d0 (the lowest query index on ties).  mq / mg [nq]: query and group of each kept match; returns their count. */
int orc_reloc_select(const int32_t* knn, int nq, int n_grp, int max_dist, int32_t* mq, int32_t* mg)
{
    uint32_t* key = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(n_grp > 0 ? n_grp : 1));
    for (int g = 0; g < n_grp; g++) key[g] = 0xffffffffu;
    uint8_t* pass = (uint8_t*)malloc((size_t)(nq > 0 ? nq : 1));
    for (int i = 0; i < nq; i++) {
        const int g0 = knn[4 * i], d0 = knn[4 * i + 1], g1 = knn[4 * i + 2], d1 = knn[4 * i + 3];
        pass[i] = g0 >= 0 && d0 <= max_dist && (g1 < 0 || 5 * d0 < 4 * d1);
        if (pass[i]) {
            const uint32_t k = ((uint32_t)d0 << 16) | (uint32_t)i;
            if (k < key[g0]) key[g0] = k;
        }
    }
    int n = 0;
    for (int i = 0; i < nq; i++)
        if (pass[i] && key[knn[4 * i]] == (((uint32_t)knn[4 * i + 1] << 16) | (uint32_t)i)) { mq[n] = i; mg[n] = knn[4 * i]; n++; }
    free(key); free(pass);
    return n;
}

/* 1 - f . normalise(R^T (X - t)), as pose_oracle.c */
static double bearing_dist(const double* T, const double* X, const double* f)
{
    double q[3];
    for (int i = 0; i < 3; i++) {
        const double tr = -(T[i] * T[3] + T[4 + i] * T[7] + T[8 + i] * T[11]);
        q[i] = T[i] * X[0] + T[4 + i] * X[1] + T[8 + i] * X[2] + tr;
    }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    return 1.0 - (q[0] / n * f[0] + q[1] / n * f[1] + q[2] / n * f[2]);
}

/* P3P-RANSAC: the draws and hypotheses of orc_p3p_lmeds (max_iter successful draws, at most 10 max_iter degenerate ones),
 * each scored by its number of inliers (bearing distance <= 1 - cos(atan(err_px / focal)) in float, as orc_p3p_lmeds); the
 * first hypothesis with the strictly largest count wins.  Twc_out 3x4 row-major [R | t]; outlier [n].  Returns 1 on success
 * (>= 5 inliers and an orthogonal R), else 0.  info[0] = #inliers, [1] = index of the selected hypothesis (-1: none), [2] = #draws. */
int orc_p3p_ransac(const double* bvs, const double* wpts, int n, int max_iter, float err_px, float fx, float fy, uint32_t seed,
                   double* Twc_out, uint8_t* outlier, double* info)
{
    if (info) { info[0] = 0; info[1] = -1; info[2] = 0; }
    if (n < 4) { for (int i = 0; i < n; i++) outlier[i] = 1; return 0; }
    float focal = fx + fy;
    focal = (float)(focal / 2.);
    const double threshold = 1.0 - cosf(atanf(err_px / focal));
    const int max_skip = max_iter * 10, len = 4 * (max_iter + max_skip);
    int32_t* rnd = (int32_t*)malloc(sizeof(int32_t) * (size_t)len);
    orc_sac_rnd(seed, len, rnd);
    int* sh = (int*)malloc(sizeof(int) * (size_t)n);
    for (int i = 0; i < n; i++) sh[i] = i;
    double bestT[12];
    int best = 0, bi = -1, iterations = 0, skipped = 0, draws = 0;
    while (iterations < max_iter && skipped < max_skip) {
        int idx[4];
        for (int i = 0; i < 4; i++) {
            const int j = i + (int)((uint32_t)rnd[4 * draws + i] % (uint32_t)(n - i));
            const int t = sh[i]; sh[i] = sh[j]; sh[j] = t;
        }
        for (int i = 0; i < 4; i++) idx[i] = sh[i];
        draws++;
        double T[12];
        if (!orc_p3p_sample_model(bvs, wpts, idx, T)) { skipped++; continue; }
        int cnt = 0;
        for (int i = 0; i < n; i++) cnt += bearing_dist(T, wpts + 3 * i, bvs + 3 * i) <= threshold;
        if (cnt > best) { best = cnt; bi = iterations; memcpy(bestT, T, sizeof bestT); }
        iterations++;
    }
    int ninl = 0, ok = 0;
    if (bi >= 0) {
        for (int i = 0; i < n; i++) {
            outlier[i] = !(bearing_dist(bestT, wpts + 3 * i, bvs + 3 * i) <= threshold);
            ninl += !outlier[i];
        }
        double e = 0;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                const double v = bestT[4 * i] * bestT[4 * j] + bestT[4 * i + 1] * bestT[4 * j + 1] + bestT[4 * i + 2] * bestT[4 * j + 2] - (i == j);
                e += v * v;
            }
        ok = ninl >= 5 && sqrt(e) < 1e-10;
        memcpy(Twc_out, bestT, sizeof bestT);
    } else {
        for (int i = 0; i < n; i++) outlier[i] = 1;
    }
    if (info) { info[0] = ninl; info[1] = bi; info[2] = draws; }
    free(rnd); free(sh);
    return ok;
}
