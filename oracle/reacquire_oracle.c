/* oracle/reacquire_oracle.c -- CPU restatement of alva_k_match_frame_to_map (alvaar_b200/csrc/reacquire.cu): the frozen map's
 * re-acquisition of a tracked frame's fresh detections (alva_system_set_localisation_only).
 *
 * TEST INFRASTRUCTURE ONLY (see alva_oracle.c's header): the tests and the CPU System backend of the test suite
 * (tests/host/system_cpu_localisation.cpp) call it; the product never links it.  Built with camera_oracle.c and
 * fisheye_oracle.c (the lens projections) by tests/localisation_util.py.
 *
 * The gates of the reference's Mapper::matchToMap (src/slam/src/mapper.cpp:354-587) for queries without a map point of their
 * own, per table row m in ascending order:
 *   skip[m] -> no descriptor rows -> c = Tcw X (the normalised quaternion, Frame::projWorldToCam) with c_z >= 0.1 -> the view
 *   gate |c_z| / |c| >= cos(atan(max(w / 2fx, h / 2fy))) in float -> the lens projection inside the image -> candidates: the
 *   kept queries with finite positions whose float pixel distance is <= radius, in ascending query order -> distance = the
 *   minimum Hamming distance over the row's keyframe descriptors -> `<=` best / second best from 51.2 -> reject the best if
 *   a second exists and 0.9 * second < best (double)
 * then per query: `<=` over the rows in ascending order, i.e. the smallest distance, the highest row among equal ones.
 * The grid below is only a faster way to find the same candidates: the distance test alone decides.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void orc_project_cam_dist(const double* K4, const double* D4, const double* p, float* out);      /* camera_oracle.c */
void orc_fisheye_project_cam(const double* K4, const double* D4, const double* p, float* out);   /* fisheye_oracle.c */

static void r_quat_R(const double* q, double* R)
{
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
static void r_world_to_cam(const double* Twc, const double* X, double* c)
{
    double R[9], ti[3];
    r_quat_R(Twc + 3, R);
    for (int i = 0; i < 3; i++) ti[i] = -(R[i] * Twc[0] + R[3 + i] * Twc[1] + R[6 + i] * Twc[2]);
    for (int i = 0; i < 3; i++) c[i] = (R[i] * X[0] + R[3 + i] * X[1] + R[6 + i] * X[2]) + ti[i];
}
static void r_project(int lens, const double* K4, const double* D4, const double* c, float* px)
{
    if (lens == 1) { orc_project_cam_dist(K4, D4, c, px); return; }
    if (lens == 2) { orc_fisheye_project_cam(K4, D4, c, px); return; }
    const double iz = 1. / c[2];
    const double x = (double)(float)(c[0] * iz), y = (double)(float)(c[1] * iz);
    px[0] = (float)(x * K4[0] + K4[2]);
    px[1] = (float)(y * K4[1] + K4[3]);
}
static int r_hamming32(const uint8_t* a, const uint8_t* b)
{
    int s = 0;
    for (int i = 0; i < 32; i++) s += __builtin_popcount((unsigned)(a[i] ^ b[i]));
    return s;
}
static int r_clamp(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
static int r_cmp_int(const void* a, const void* b) { const int x = *(const int*)a, y = *(const int*)b; return (x > y) - (x < y); }

/* Returns the number of matched queries, or -1 for a bad argument.  q_row [nq]: the matched table row or -1; q_dist [nq]: its
 * Hamming distance or -1.  lens: 0 pinhole, 1 radial-tangential, 2 fisheye (coef4 its four coefficients). */
int orc_match_frame_to_map(int w, int h, int cell, double fx, double fy, double cx, double cy, int lens, const double* coef4,
                           const double* Twc, int n_mp, const double* wpt, const int32_t* desc_start, const uint8_t* desc,
                           const uint8_t* skip, int nq, const float* q_px, const uint8_t* q_desc, const uint8_t* q_kept, float radius,
                           int32_t* q_row, int32_t* q_dist)
{
    if (w < 1 || h < 1 || cell < 1 || n_mp < 0 || nq < 0 || lens < 0 || lens > 2 || !(radius >= 0.f)) return -1;
    const double K4[4] = {fx, fy, cx, cy};
    double D4[4] = {0, 0, 0, 0};
    if (lens) for (int i = 0; i < 4; i++) D4[i] = coef4[i];
    const int ncw = (int)ceilf((float)w / (float)cell), nch = (int)ceilf((float)h / (float)cell), ncells = ncw * nch;
    const float fovV = (float)(0.5 * h / fy), fovH = (float)(0.5 * w / fx);
    const float view_th = cosf(fovH > fovV ? atanf(fovH) : atanf(fovV));
    const float min_dist = (float)(32 * 0.2f * 8.);
    for (int q = 0; q < nq; q++) { q_row[q] = -1; q_dist[q] = -1; }
    if (nq == 0) return 0;
    /* the query grid: candidates only, positions outside the image in the border cell */
    int* q_cell = (int*)malloc(sizeof(int) * (size_t)nq);
    int* start = (int*)calloc((size_t)ncells + 1, sizeof(int));
    int* cell_q = (int*)malloc(sizeof(int) * (size_t)nq);
    int* fill = (int*)calloc((size_t)ncells + 1, sizeof(int));
    for (int q = 0; q < nq; q++) {
        const float x = q_px[2 * q], y = q_px[2 * q + 1];
        q_cell[q] = -1;
        if (!q_kept[q] || !isfinite(x) || !isfinite(y)) continue;
        const float fx_ = fminf(fmaxf(x, -1.f), (float)w), fy_ = fminf(fmaxf(y, -1.f), (float)h);
        q_cell[q] = r_clamp((int)floorf(fy_ / (float)cell), 0, nch - 1) * ncw + r_clamp((int)floorf(fx_ / (float)cell), 0, ncw - 1);
        start[q_cell[q] + 1]++;
    }
    for (int c = 0; c < ncells; c++) start[c + 1] += start[c];
    for (int q = 0; q < nq; q++) if (q_cell[q] >= 0) cell_q[start[q_cell[q]] + fill[q_cell[q]]++] = q;
    int* qd = (int*)malloc(sizeof(int) * (size_t)nq);            /* per query: best distance so far (1024 = none) */
    for (int q = 0; q < nq; q++) qd[q] = 1024;
    int* cand = (int*)malloc(sizeof(int) * (size_t)nq);
    for (int m = 0; m < n_mp; m++) {
        if (skip && skip[m]) continue;
        const int d0 = desc_start[m], nd = desc_start[m + 1] - d0;
        if (nd <= 0) continue;
        double c[3];
        r_world_to_cam(Twc, wpt + 3 * (size_t)m, c);
        if (c[2] < 0.1) continue;
        const float view_angle = (float)(c[2] / sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]));
        if (fabs((double)view_angle) < (double)view_th) continue;
        float proj[2];
        r_project(lens, K4, D4, c, proj);
        if (!(proj[0] >= 0 && proj[1] >= 0 && (double)proj[0] < (double)w && (double)proj[1] < (double)h)) continue;
        /* the cells the radius disc (widened by 1 px) touches */
        const int cx0 = r_clamp((int)floorf((proj[0] - radius - 1.f) / (float)cell), 0, ncw - 1);
        const int cx1 = r_clamp((int)floorf((proj[0] + radius + 1.f) / (float)cell), 0, ncw - 1);
        const int cy0 = r_clamp((int)floorf((proj[1] - radius - 1.f) / (float)cell), 0, nch - 1);
        const int cy1 = r_clamp((int)floorf((proj[1] + radius + 1.f) / (float)cell), 0, nch - 1);
        int nc = 0;
        for (int gy = cy0; gy <= cy1; gy++)
            for (int gx = cx0; gx <= cx1; gx++)
                for (int s = start[gy * ncw + gx]; s < start[gy * ncw + gx + 1]; s++) cand[nc++] = cell_q[s];
        qsort(cand, (size_t)nc, sizeof(int), r_cmp_int);
        int bestQ = -1, secQ = -1;
        float bestDist = min_dist, secDist = min_dist;
        for (int i = 0; i < nc; i++) {
            const int q = cand[i];
            const float dx = proj[0] - q_px[2 * q], dy = proj[1] - q_px[2 * q + 1];
            const float pxDist = (float)sqrt((double)dx * dx + (double)dy * dy);
            if (!(pxDist <= radius)) continue;
            float dist = 1000.0f;
            for (int a = 0; a < nd; a++) {
                const float dd = (float)r_hamming32(desc + 32 * (size_t)(d0 + a), q_desc + 32 * (size_t)q);
                if (dd < dist) dist = dd;
            }
            if (dist <= bestDist) { secDist = bestDist; secQ = bestQ; bestDist = dist; bestQ = q; }
            else if (dist <= secDist) { secDist = dist; secQ = q; }
        }
        if (bestQ != -1 && secQ != -1 && 0.9 * (double)secDist < (double)bestDist) bestQ = -1;
        if (bestQ < 0) continue;
        if ((int)bestDist <= qd[bestQ]) { qd[bestQ] = (int)bestDist; q_row[bestQ] = m; }
    }
    int n = 0;
    for (int q = 0; q < nq; q++) if (q_row[q] >= 0) { q_dist[q] = qd[q]; n++; }
    free(q_cell); free(start); free(cell_q); free(fill); free(qd); free(cand);
    return n;
}
