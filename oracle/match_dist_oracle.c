/* oracle/match_dist_oracle.c -- CPU restatement of the reference's projection-gated matching of the local map to a keyframe,
 * through a lens with distortion: orc_match_to_map_dist.  The same procedure as orc_match_to_map (match_oracle.c), with the
 * map point's projection and the co-projection errors taken through CameraCalibration::projectCamToImageDist with the given
 * k1 k2 p1 p2 (orc_project_cam_dist, camera_oracle.c), as the reference does at mapper.cpp:425 and :504.  Built with
 * camera_oracle.c into tests/_build/libcamera_oracle.so by the tests (tests/camera_util.py).
 *
 * TEST INFRASTRUCTURE ONLY (see alva_oracle.c's header): only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may call this.  The product (alvaar_b200/) never links or executes it.
 *
 * Reference (paths under /root/reference):
 *   Mapper::matchToMap                     src/slam/src/mapper.cpp:354-587   (caller matchingToLocalMap :293-352)
 *   MapPoint::computeMinDescDist           src/slam/src/map_point.cpp:204-222  (cv::norm(NORM_HAMMING))
 *   Frame::getSurroundingKeypoints         src/slam/src/frame.cpp:313-341      (2x2 cells {r-1, r} x {c-1, c})
 *   Frame::projWorldToCam / isInImage      src/slam/src/frame.cpp:447-467
 *   CameraCalibration::projectCamToImageDist  src/slam/src/camera_calibration.cpp:34-55 (cv::projectPoints on a FLOAT point;
 *                                             with lens distortion: orc_project_cam_dist, camera_oracle.c)
 *
 * The map is passed as flat arrays (the same contract as ref_match_to_map in oracle/ref_system.cpp, which rebuilds the
 * reference's own Frame / MapPoint / MapManager objects from them and calls the unmodified Mapper::matchToMap):
 *   current frame: T_wc = [t, q(x,y,z,w)], keypoints (id, px) in grid insertion order, nkp3d
 *   keyframes: id, T_wc;  map points: id, world point, is3d, observations (keyframe index, px) sorted by keyframe id,
 *   descriptors per keyframe;  local_ids: the local map in the reference's iteration order (an unordered_set: the order is an
 *   INPUT here -- it decides `<=` ties)
 * PINNED: tests/test_gpu_distortion.py: identical maps from alva_k_match_to_map_dist; with zero coefficients it is
 * orc_match_to_map's procedure, pinned by tests/test_oracle_match.py.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

typedef struct {
    int w, h, cell, ncw, nch;
    double fx, fy, cx, cy;
    const double* dist;   /* k1 k2 p1 p2, or NULL: zero distortion */
} m_cam;

void orc_project_cam_dist(const double* K4, const double* D4, const double* p, float* out);   /* camera_oracle.c */

static void m_quat_R(const double* q, double* R)   /* normalised (x,y,z,w) -> rotation, Eigen's toRotationMatrix */
{
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
/* Tcw * X with Tcw = Twc.inverse() = (R^T, -R^T t) */
static void m_world_to_cam(const double* Twc, const double* X, double* c)
{
    double R[9], ti[3];
    m_quat_R(Twc + 3, R);
    for (int i = 0; i < 3; i++) ti[i] = -(R[i] * Twc[0] + R[3 + i] * Twc[1] + R[6 + i] * Twc[2]);
    for (int i = 0; i < 3; i++) c[i] = (R[i] * X[0] + R[3 + i] * X[1] + R[6 + i] * X[2]) + ti[i];
}
/* CameraCalibration::projectCamToImageDist: with distortion camera_oracle.c's restatement of cv::projectPoints; with zero
 * distortion the normalised point goes through a cv::Point3f */
static void m_project(const m_cam* C, const double* c, float* px)
{
    if (C->dist) {
        const double K4[4] = {C->fx, C->fy, C->cx, C->cy};
        orc_project_cam_dist(K4, C->dist, c, px);
        return;
    }
    const double iz = 1. / c[2];
    const double x = (double)(float)(c[0] * iz), y = (double)(float)(c[1] * iz);
    px[0] = (float)(x * C->fx + C->cx);
    px[1] = (float)(y * C->fy + C->cy);
}
static float m_norm2f(float ax, float ay, float bx, float by)   /* (float) cv::norm(Point2f a - b) */
{
    const float dx = ax - bx, dy = ay - by;
    return (float)sqrt((double)dx * dx + (double)dy * dy);
}
static int m_hamming32(const uint8_t* a, const uint8_t* b)
{
    int s = 0;
    for (int i = 0; i < 32; i++) s += __builtin_popcount((unsigned)(a[i] ^ b[i]));
    return s;
}

/* Returns the number of (keypoint id -> map point id) pairs written to match_kp / match_mp, ascending keypoint id.
 * dist4: k1 k2 p1 p2 of the projections (mapper.cpp:425, 504), or NULL / all zero: zero distortion. */
int orc_match_to_map_dist(int w, int h, double fx, double fy, double cx, double cy, const double* Twc_cur, int n_kp,
                          const int32_t* kp_id, const float* kp_px, int nkp3d, int n_kf, const int32_t* kf_id, const double* kf_Twc,
                          int n_mp, const int32_t* mp_id, const double* mp_wpt, const uint8_t* mp_is3d, const int32_t* obs_start,
                          const int32_t* obs_kf, const float* obs_px, const int32_t* desc_start, const int32_t* desc_kf,
                          const uint8_t* desc, int n_local, const int32_t* local_ids, float max_proj_err, float dist_ratio,
                          int32_t* match_kp, int32_t* match_mp, const double* dist4)
{
    (void)desc_kf; (void)kf_id;
    m_cam C = {w, h, 40, 0, 0, fx, fy, cx, cy, NULL};
    if (dist4 && (dist4[0] != 0 || dist4[1] != 0 || dist4[2] != 0 || dist4[3] != 0)) C.dist = dist4;
    C.ncw = (int)ceilf((float)w / C.cell); C.nch = (int)ceilf((float)h / C.cell);
    /* id -> map point index */
    int maxid = 0;
    for (int m = 0; m < n_mp; m++) if (mp_id[m] > maxid) maxid = mp_id[m];
    int* idx_of = (int*)malloc(sizeof(int) * (maxid + 2));
    for (int i = 0; i <= maxid + 1; i++) idx_of[i] = -1;
    for (int m = 0; m < n_mp; m++) idx_of[mp_id[m]] = m;
    /* grid of the current frame: cell -> keypoint indices in insertion order */
    const int ncells = C.ncw * C.nch;
    int* cell_cnt = (int*)calloc(ncells + 1, sizeof(int));
    int* kp_cell = (int*)malloc(sizeof(int) * (n_kp + 1));
    for (int i = 0; i < n_kp; i++) {
        const int r = (int)floorf(kp_px[2 * i + 1] / (float)C.cell), c = (int)floorf(kp_px[2 * i] / (float)C.cell);
        kp_cell[i] = r * C.ncw + c;
        cell_cnt[kp_cell[i]]++;
    }
    int* cell_start = (int*)malloc(sizeof(int) * (ncells + 1));
    cell_start[0] = 0;
    for (int i = 0; i < ncells; i++) cell_start[i + 1] = cell_start[i] + cell_cnt[i];
    int* cell_kp = (int*)malloc(sizeof(int) * (n_kp + 1));
    memset(cell_cnt, 0, sizeof(int) * (ncells + 1));
    for (int i = 0; i < n_kp; i++) cell_kp[cell_start[kp_cell[i]] + cell_cnt[kp_cell[i]]++] = i;
    uint8_t* observed = (uint8_t*)calloc(maxid + 2, 1);
    for (int i = 0; i < n_kp; i++) if (kp_id[i] >= 0 && kp_id[i] <= maxid) observed[kp_id[i]] = 1;

    const float fovV = (float)(0.5 * h / fy), fovH = (float)(0.5 * w / fx);
    const float maxRadFov = fovH > fovV ? atanf(fovH) : atanf(fovV);
    const float view_th = cosf(maxRadFov);
    float maxPxDist = max_proj_err;
    if (nkp3d < 30) maxPxDist = (float)(maxPxDist * 2.);
    /* per keypoint: the (map point, dist) candidates in processing order -> keep the last smallest (`<=`, mapper.cpp:565-585) */
    float* kbest = (float*)malloc(sizeof(float) * (n_kp + 1));
    int* kbest_mp = (int*)malloc(sizeof(int) * (n_kp + 1));
    for (int i = 0; i < n_kp; i++) { kbest[i] = 1024.f; kbest_mp[i] = -1; }

    for (int li = 0; li < n_local; li++) {
        const int id = local_ids[li];
        if (id >= 0 && id <= maxid && observed[id]) continue;
        const int m = (id >= 0 && id <= maxid) ? idx_of[id] : -1;
        if (m < 0) continue;
        if (!mp_is3d[m] || desc_start[m + 1] == desc_start[m]) continue;
        const double* wpt = mp_wpt + 3 * m;
        double campt[3];
        m_world_to_cam(Twc_cur, wpt, campt);
        if (campt[2] < 0.1) continue;
        const float view_angle = (float)(campt[2] / sqrt(campt[0] * campt[0] + campt[1] * campt[1] + campt[2] * campt[2]));
        if (fabs(view_angle) < view_th) continue;
        float proj[2];
        m_project(&C, campt, proj);
        if (!(proj[0] >= 0 && proj[1] >= 0 && proj[0] < (double)w && proj[1] < (double)h)) continue;
        const float minDist = (float)(32 * dist_ratio * 8.);
        int bestId = -1, secId = -1, bestKp = -1;
        float bestDist = minDist, secDist = minDist;
        const int rkp = (int)floorf(proj[1] / (float)C.cell), ckp = (int)floorf(proj[0] / (float)C.cell);
        for (int r = rkp - 1; r < rkp + 1; r++)
            for (int c = ckp - 1; c < ckp + 1; c++) {
                const int idx = r * C.ncw + c;
                if (r < 0 || c < 0 || idx >= ncells) continue;
                for (int s = cell_start[idx]; s < cell_start[idx + 1]; s++) {
                    const int k = cell_kp[s];
                    if (kp_id[k] < 0) continue;
                    const float pxDist = m_norm2f(proj[0], proj[1], kp_px[2 * k], kp_px[2 * k + 1]);
                    if (pxDist > maxPxDist) continue;
                    const int km = idx_of[kp_id[k]];
                    if (km < 0) continue;
                    if (desc_start[km + 1] == desc_start[km]) continue;
                    /* never both observed in one keyframe */
                    int cand = 1;
                    for (int a = obs_start[km]; a < obs_start[km + 1] && cand; a++)
                        for (int b = obs_start[m]; b < obs_start[m + 1]; b++)
                            if (obs_kf[a] == obs_kf[b]) { cand = 0; break; }
                    if (!cand) continue;
                    /* mean distance between the keypoint's pixels in its keyframes and the map point projected there */
                    float co = 0.f;
                    size_t nco = 0;
                    for (int a = obs_start[km]; a < obs_start[km + 1]; a++) {
                        double cc[3];
                        float pp[2];
                        m_world_to_cam(kf_Twc + 7 * obs_kf[a], wpt, cc);
                        m_project(&C, cc, pp);
                        const float dx = obs_px[2 * a] - pp[0], dy = obs_px[2 * a + 1] - pp[1];
                        co = (float)(co + sqrt((double)dx * dx + (double)dy * dy));
                        nco++;
                    }
                    if (co / nco > maxPxDist) continue;
                    float dist = 1000.0f;
                    for (int a = desc_start[m]; a < desc_start[m + 1]; a++)
                        for (int b = desc_start[km]; b < desc_start[km + 1]; b++) {
                            const float dd = (float)m_hamming32(desc + 32 * (size_t)a, desc + 32 * (size_t)b);
                            if (dd < dist) dist = dd;
                        }
                    if (dist <= bestDist) { secDist = bestDist; secId = bestId; bestDist = dist; bestId = kp_id[k]; bestKp = k; }
                    else if (dist <= secDist) { secDist = dist; secId = kp_id[k]; }
                }
            }
        if (bestId != -1 && secId != -1)
            if (0.9 * secDist < bestDist) bestId = -1;
        if (bestId < 0) continue;
        if (bestDist <= kbest[bestKp]) { kbest[bestKp] = bestDist; kbest_mp[bestKp] = id; }
    }
    /* std::map<int,int>: ascending keypoint id */
    int n = 0;
    int* ord = (int*)malloc(sizeof(int) * (n_kp + 1));
    for (int i = 0; i < n_kp; i++) ord[i] = i;
    for (int i = 1; i < n_kp; i++) {   /* insertion sort by id (test sizes) */
        const int v = ord[i];
        int j = i - 1;
        while (j >= 0 && kp_id[ord[j]] > kp_id[v]) { ord[j + 1] = ord[j]; j--; }
        ord[j + 1] = v;
    }
    for (int i = 0; i < n_kp; i++) {
        const int k = ord[i];
        if (kbest_mp[k] >= 0) { match_kp[n] = kp_id[k]; match_mp[n] = kbest_mp[k]; n++; }
    }
    free(idx_of); free(cell_cnt); free(kp_cell); free(cell_start); free(cell_kp); free(observed); free(kbest); free(kbest_mp); free(ord);
    return n;
}
