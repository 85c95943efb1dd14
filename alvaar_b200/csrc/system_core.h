// system_core.h -- the host-side state machine of `System`: what the reference keeps in Frame / MapPoint / MapManager /
// VisualFrontend / Mapper, re-hosted around the GPU stages.  It owns no pixels and does no arithmetic of the hot path: every
// image / solver stage is a call into a Backend (system.cu: the alva_k_* CUDA kernels; tests/host/system_cpu_backend.cpp: the
// CPU oracle, TEST ONLY, so that this logic can be checked against the reference's own System in the GPU-less CPU suite).
//
// Reference behaviour restated here (file:line under /root/reference/src/slam/src):
//   system.cpp:156-175                       System::processCameraPose (status 1 / 2 / 3, reset on request)
//   visual_frontend.cpp:21-101               VisualFrontend::track / process
//   visual_frontend.cpp:103-243              kltTrackingFromMotionPrior (3-D keypoints: projected prior, 1 pyramid level first)
//   visual_frontend.cpp:245-417              computePose (P3P-LMedS, outlier removal, Ceres PnP, failure handling)
//   visual_frontend.cpp:419-552              checkReadyForInit (median parallax, rotation-compensated mean parallax, 5-point)
//   visual_frontend.cpp:554-594              checkNewKeyframeRequired
//   visual_frontend.cpp:596-670              computeParallax
//   visual_frontend.hpp:17-56                MotionModel (constant velocity in se(3))
//   map_manager.cpp:12-66,183-253            createKeyframe = prepareFrame + extractKeypoints + addKeyframe
//   map_manager.cpp:68-150                   updateFrameCovisibility
//   map_manager.cpp:352-405,560-650          updateMapPoint, removeMapPointObs, removeObsFromCurrFrameById
//   mapper.cpp:9-64                          Mapper::processNewKeyframe (reset rules after a bad initialisation)
//   mapper.cpp:157-291                       triangulateTemporal
//   frame.cpp / map_point.cpp                keypoint, grid and observation bookkeeping
// The reference iterates std::unordered_map<int, Keypoint> wherever it collects points (RANSAC sample indices, Ceres residual
// order, detector masks), so the iteration ORDER is part of its behaviour; the same container type with the same sequence of
// insertions / erasures / copies is used here (libstdc++ is deterministic for equal histories).
//
//   mapper.cpp:66-155, 293-352               Mapper::optimize (local BA from keyframe 2, keyframe filtering from 20), matchingToLocalMap
//   optimizer.cpp:4-531                      Optimizer::localBA: assembly, write-back, culling (the solves: Backend::ba_local)
//   map_manager.cpp:407-575                  mergeMapPoints, removeKeyframe, removeMapPoint
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <type_traits>
#include <utility>
#include <map>
#include <memory>
#include <set>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include <random>
#include "camera_model.h"

namespace alva_sys {

// ------------------------------------------------------------------------------------------------ SE(3), Sophus conventions
struct Se3 {
    double q[4] = {0, 0, 0, 1};   // x y z w
    double t[3] = {0, 0, 0};

    void R(double* M) const {
        const double x = q[0], y = q[1], z = q[2], w = q[3];
        M[0] = 1 - 2 * (y * y + z * z); M[1] = 2 * (x * y - z * w); M[2] = 2 * (x * z + y * w);
        M[3] = 2 * (x * y + z * w); M[4] = 1 - 2 * (x * x + z * z); M[5] = 2 * (y * z - x * w);
        M[6] = 2 * (x * z - y * w); M[7] = 2 * (y * z + x * w); M[8] = 1 - 2 * (x * x + y * y);
    }
    void setR(const double* M) {   // Eigen's matrix -> quaternion
        double tr = M[0] + M[4] + M[8];
        if (tr > 0) {
            tr = sqrt(tr + 1.0);
            q[3] = 0.5 * tr; tr = 0.5 / tr;
            q[0] = (M[7] - M[5]) * tr; q[1] = (M[2] - M[6]) * tr; q[2] = (M[3] - M[1]) * tr;
        } else {
            int i = 0;
            if (M[4] > M[0]) i = 1;
            if (M[8] > M[4 * i]) i = 2;
            const int j = (i + 1) % 3, k = (j + 1) % 3;
            tr = sqrt(M[4 * i] - M[4 * j] - M[4 * k] + 1.0);
            q[i] = 0.5 * tr; tr = 0.5 / tr;
            q[3] = (M[3 * k + j] - M[3 * j + k]) * tr;
            q[j] = (M[3 * j + i] + M[3 * i + j]) * tr;
            q[k] = (M[3 * k + i] + M[3 * i + k]) * tr;
        }
        normalize();
    }
    void normalize() {
        const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        for (int i = 0; i < 4; i++) q[i] /= n;
    }
    void rot(const double* p, double* o) const {
        double M[9];
        R(M);
        for (int i = 0; i < 3; i++) o[i] = M[3 * i] * p[0] + M[3 * i + 1] * p[1] + M[3 * i + 2] * p[2];
    }
    void apply(const double* p, double* o) const { rot(p, o); for (int i = 0; i < 3; i++) o[i] += t[i]; }
    Se3 inverse() const {
        Se3 r;
        r.q[0] = -q[0]; r.q[1] = -q[1]; r.q[2] = -q[2]; r.q[3] = q[3];
        double v[3];
        r.rot(t, v);
        for (int i = 0; i < 3; i++) r.t[i] = -v[i];
        return r;
    }
    Se3 operator*(const Se3& b) const {
        Se3 r;
        const double* a = q;
        r.q[3] = a[3] * b.q[3] - a[0] * b.q[0] - a[1] * b.q[1] - a[2] * b.q[2];
        r.q[0] = a[3] * b.q[0] + a[0] * b.q[3] + a[1] * b.q[2] - a[2] * b.q[1];
        r.q[1] = a[3] * b.q[1] - a[0] * b.q[2] + a[1] * b.q[3] + a[2] * b.q[0];
        r.q[2] = a[3] * b.q[2] + a[0] * b.q[1] - a[1] * b.q[0] + a[2] * b.q[3];
        r.normalize();
        apply(b.t, r.t);
        return r;
    }
    static Se3 exp(const double* xi) {   // xi = [upsilon, omega]
        Se3 r;
        const double* om = xi + 3;
        const double th2 = om[0] * om[0] + om[1] * om[1] + om[2] * om[2], th = sqrt(th2);
        double imag, real;
        if (th < 1e-10) { const double th4 = th2 * th2; imag = 0.5 - th2 / 48. + th4 / 3840.; real = 1 - th2 / 8. + th4 / 384.; }
        else { imag = sin(0.5 * th) / th; real = cos(0.5 * th); }
        r.q[0] = imag * om[0]; r.q[1] = imag * om[1]; r.q[2] = imag * om[2]; r.q[3] = real;
        double V[9];
        const double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0};
        double O2[9];
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) O2[3 * i + j] = O[3 * i] * O[j] + O[3 * i + 1] * O[3 + j] + O[3 * i + 2] * O[6 + j];
        if (th < 1e-10) r.R(V);
        else {
            const double a = (1 - cos(th)) / th2, b = (th - sin(th)) / (th2 * th);
            for (int i = 0; i < 9; i++) V[i] = (i % 4 == 0) + a * O[i] + b * O2[i];
        }
        for (int i = 0; i < 3; i++) r.t[i] = V[3 * i] * xi[0] + V[3 * i + 1] * xi[1] + V[3 * i + 2] * xi[2];
        return r;
    }
    void log(double* xi) const {
        const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2], n = sqrt(n2), w = q[3];
        double two_atan;
        if (n < 1e-10) two_atan = 2. / w - 2. * n2 / (w * w * w);
        else if (fabs(w) < 1e-10) two_atan = (w > 0 ? M_PI : -M_PI) / n;
        else two_atan = 2. * atan(n / w) / n;
        const double th = two_atan * n;
        double om[3] = {two_atan * q[0], two_atan * q[1], two_atan * q[2]};
        const double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0};
        double O2[9], Vi[9];
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) O2[3 * i + j] = O[3 * i] * O[j] + O[3 * i + 1] * O[3 + j] + O[3 * i + 2] * O[6 + j];
        double c;
        if (fabs(th) < 1e-10) c = 1. / 12.;
        else { const double h = 0.5 * th; c = (1 - th * cos(h) / (2 * sin(h))) / (th * th); }
        for (int i = 0; i < 9; i++) Vi[i] = (i % 4 == 0) - 0.5 * O[i] + c * O2[i];
        for (int i = 0; i < 3; i++) { xi[i] = Vi[3 * i] * t[0] + Vi[3 * i + 1] * t[1] + Vi[3 * i + 2] * t[2]; xi[3 + i] = om[i]; }
    }
    void to7(double* p) const { for (int i = 0; i < 3; i++) p[i] = t[i]; for (int i = 0; i < 4; i++) p[3 + i] = q[i]; }
    static Se3 from7(const double* p) { Se3 r; for (int i = 0; i < 3; i++) r.t[i] = p[i]; for (int i = 0; i < 4; i++) r.q[i] = p[3 + i]; r.normalize(); return r; }
};

// ------------------------------------------------------------------------------------------------ camera
struct Camera {
    double fx = 1, fy = 1, cx = 0, cy = 0;
    int w = 0, h = 0;
    // lens distortion k1 k2 p1 p2 (CameraCalibration::D_); has_dist = any of them non-zero.  Without it the two functions that
    // apply it below take their pinhole forms, which give the same bits as the radial-tangential model with zero coefficients.
    double dist[4] = {0, 0, 0, 0};
    bool has_dist = false;
    void setDistortion(const double* d) {
        has_dist = false;
        for (int i = 0; i < 4; i++) { dist[i] = d[i]; has_dist = has_dist || d[i] != 0.0; }
    }
    void K4(double* k) const { k[0] = fx; k[1] = fy; k[2] = cx; k[3] = cy; }
    // CameraCalibration::undistortImagePoint: cv::undistortPoints(..., K, D, K) (camera_model.h); with zero distortion it
    // evaluates fx * ((u - cx) * (1 / fx)) + cx in double and rounds to float (calib3d/src/undistort.dispatch.cpp)
    double ifx = 1, ify = 1, k00 = 1, k02 = 0, k11 = 1, k12 = 0, k22 = 1;   // loop invariants of the two functions below
    void prepare() {
        ifx = 1. / fx; ify = 1. / fy;
        const double id = 1. / (fx * fy);
        k00 = fy * id; k02 = (-(cx * fy)) * id; k11 = fx * id; k12 = (-(fx * cy)) * id; k22 = (fx * fy) * id;
    }
    void undistort(float u, float v, float& ux, float& uy) const {
        if (has_dist) {
            double k[4];
            float o[2];
            K4(k);
            alva_cam::undistort_point(k, dist, u, v, o);
            ux = o[0]; uy = o[1];
            return;
        }
        const double x = ((double)u - cx) * ifx, y = ((double)v - cy) * ify;
        ux = (float)(fx * x + cx); uy = (float)(fy * y + cy);
    }
    // inverseK_ * [unpx, 1], normalised (frame.cpp:110-118).  inverseK_ = K_.inverse() is Eigen's 3x3 cofactor inverse
    // (cofactor * (1 / det), det = fx * fy), and the initialisation's refinement amplifies a 1-ulp change of a bearing vector to
    // 1e-4 in the pose, so the same expression tree is used here
    void bearing(float ux, float uy, double* bv) const {
        bv[0] = (k00 * (double)ux + 0.0 * (double)uy) + k02 * 1.0;
        bv[1] = (0.0 * (double)ux + k11 * (double)uy) + k12 * 1.0;
        bv[2] = (0.0 * (double)ux + 0.0 * (double)uy) + k22 * 1.0;
        const double n = sqrt((bv[0] * bv[0] + bv[1] * bv[1]) + bv[2] * bv[2]);
        bv[0] /= n; bv[1] /= n; bv[2] /= n;
    }
    void inverseK(float ux, float uy, double* b) const {   // inverseK_ * [unpx, 1] (not normalised)
        b[0] = (k00 * (double)ux + 0.0 * (double)uy) + k02 * 1.0;
        b[1] = (0.0 * (double)ux + k11 * (double)uy) + k12 * 1.0;
        b[2] = (0.0 * (double)ux + 0.0 * (double)uy) + k22 * 1.0;
    }
    void projCamToImage(const double* p, float& u, float& v) const {   // camera_calibration.cpp:26-32
        const double iz = 1. / p[2];
        u = (float)(fx * (p[0] * iz) + cx); v = (float)(fy * (p[1] * iz) + cy);
    }
    void projCamToImageDist(const double* p, float& u, float& v) const {   // :34-55: cv::projectPoints on a FLOAT point
        if (has_dist) {
            double k[4];
            float o[2];
            K4(k);
            alva_cam::project_dist(k, dist, p, o);
            u = o[0]; v = o[1];
            return;
        }
        const double iz = 1. / p[2];
        const double x = (double)(float)(p[0] * iz), y = (double)(float)(p[1] * iz);
        u = (float)(x * fx + cx); v = (float)(y * fy + cy);
    }
    bool inImage(float u, float v) const { return u >= 0 && v >= 0 && u < w && v < h; }
};

inline float norm2f(float ax, float ay, float bx, float by) {   // (float) cv::norm(Point2f a - b): the sum is formed in double
    const float dx = ax - bx, dy = ay - by;
    return (float)sqrt((double)dx * dx + (double)dy * dy);
}
inline double norm2d(float ax, float ay, float bx, float by) {
    const float dx = ax - bx, dy = ay - by;
    return sqrt((double)dx * dx + (double)dy * dy);
}

// ------------------------------------------------------------------------------------------------ Keypoint / Frame / MapPoint
struct Keypoint {
    int id = -1;
    float px = 0, py = 0, ux = 0, uy = 0;
    double bv[3] = {0, 0, 0};
    bool is3d = false, has_desc = false;
    uint8_t desc[32] = {0};
};

struct Frame {
    int id = -1, kfid = 0;
    double ts = 0;
    std::unordered_map<int, Keypoint> kps;          // Frame::mapKeypoints_
    std::vector<std::vector<int>> grid;             // Frame::gridKeypointsIds_
    int ncw = 0, nch = 0, cell = 40, nocc = 0, n = 0, n2d = 0, n3d = 0;
    Se3 Twc, Tcw;
    const Camera* cam = nullptr;
    std::map<int, int> covis;                       // covisibleKeyframeIds_
    std::unordered_set<int> localmap;               // localMapPointIds_

    void init(const Camera* c, int cellsize) {
        cam = c; cell = cellsize;
        ncw = (int)ceilf((float)c->w / cellsize); nch = (int)ceilf((float)c->h / cellsize);
        grid.assign((size_t)ncw * nch, {});
        nocc = 0;
    }
    void reset() {
        id = -1; kfid = 0; ts = 0; kps.clear(); grid.assign((size_t)ncw * nch, {}); n = n2d = n3d = nocc = 0;
        Twc = Se3(); Tcw = Se3(); covis.clear(); localmap.clear();
    }
    void setTwc(const Se3& T) { Twc = T; Tcw = T.inverse(); }
    int cellIdx(float x, float y) const { return (int)floor(y / (float)cell) * ncw + (int)floor(x / (float)cell); }
    // un: the undistorted position when the backend computed it (the same model on the device), else NULL
    void compute(float x, float y, Keypoint& k, const float* un = nullptr) const {
        k.px = x; k.py = y;
        if (un) { k.ux = un[0]; k.uy = un[1]; }
        else cam->undistort(x, y, k.ux, k.uy);
        cam->bearing(k.ux, k.uy, k.bv);
    }
    void gridAdd(const Keypoint& k) {
        const int i = cellIdx(k.px, k.py);
        if (i < 0 || i >= (int)grid.size()) return;   // the reference's .at() would throw; cannot happen for in-image points
        if (grid[i].empty()) nocc++;
        grid[i].push_back(k.id);
    }
    void gridRemove(const Keypoint& k) {
        const int i = cellIdx(k.px, k.py);
        if (i < 0 || i >= (int)grid.size()) return;
        auto& v = grid[i];
        for (size_t j = 0; j < v.size(); j++)
            if (v[j] == k.id) { v.erase(v.begin() + j); if (v.empty()) nocc--; break; }
    }
    void add(const Keypoint& k) {
        if (kps.count(k.id)) return;
        kps.emplace(k.id, k);
        gridAdd(k);
        n++;
        if (k.is3d) n3d++; else n2d++;
    }
    void add(float x, float y, int id, const uint8_t* desc, const float* un = nullptr) {
        Keypoint k;
        k.id = id;
        compute(x, y, k, un);
        if (desc) { k.has_desc = true; memcpy(k.desc, desc, 32); }
        add(k);
    }
    void update(int id, float x, float y, const float* un = nullptr) {
        auto it = kps.find(id);
        if (it == kps.end()) return;
        Keypoint& k = it->second;   // same effect as the reference's copy / recompute / updateKeypointInGrid / assign
        if (cellIdx(k.px, k.py) != cellIdx(x, y)) { gridRemove(k); compute(x, y, k, un); gridAdd(k); }
        else compute(x, y, k, un);
    }
    void remove(int id) {
        auto it = kps.find(id);
        if (it == kps.end()) return;
        gridRemove(it->second);
        if (it->second.is3d) n3d--; else n2d--;
        n--;
        kps.erase(id);
    }
    void turn3d(int id) {
        auto it = kps.find(id);
        if (it == kps.end()) return;
        if (!it->second.is3d) { it->second.is3d = true; n3d++; n2d--; }
    }
    bool updateId(int prev, int next, bool is3d) {   // Frame::updateKeypointId
        if (kps.count(next)) return false;
        auto it = kps.find(prev);
        if (it == kps.end()) return false;
        Keypoint k = it->second;
        k.id = next; k.is3d = is3d;
        remove(prev);
        add(k);
        return true;
    }
    const Keypoint* find(int id) const { auto it = kps.find(id); return it == kps.end() ? nullptr : &it->second; }
    std::vector<Keypoint> all() const { std::vector<Keypoint> v; v.reserve(n); for (auto& kv : kps) v.push_back(kv.second); return v; }
    std::vector<Keypoint> all2d() const { std::vector<Keypoint> v; for (auto& kv : kps) if (!kv.second.is3d) v.push_back(kv.second); return v; }
    std::vector<Keypoint> all3d() const { std::vector<Keypoint> v; for (auto& kv : kps) if (kv.second.is3d) v.push_back(kv.second); return v; }
    void covisDecrease(int k) {
        if (k == kfid) return;
        auto it = covis.find(k);
        if (it != covis.end() && it->second != 0) { it->second -= 1; if (it->second == 0) covis.erase(it); }
    }
    void covisAdd(int k) {
        if (k == kfid) return;
        auto it = covis.find(k);
        if (it != covis.end()) it->second += 1; else covis.emplace(k, 1);
    }
};

struct Desc { uint8_t b[32]; };
inline int hamming256(const uint8_t* a, const uint8_t* b) {
    int d = 0;
    for (int i = 0; i < 32; i++) d += __builtin_popcount((unsigned)(a[i] ^ b[i]));
    return d;
}

struct MapPoint {
    int id = -1, kfid = 0;        // kfid: anchor keyframe
    bool observed = true, is3d = false;
    double invd = -1., p[3] = {0, 0, 0};
    std::set<int> obs;                               // observedKeyframeIds_
    std::unordered_map<int, Desc> kfdesc;            // mapKeyframeDescriptors_
    std::unordered_map<int, float> descdist;         // mapDescriptorsDist_
    bool has_desc = false;
    Desc desc;                                       // desc_

    bool isBad() {   // map_point.cpp:183-202 (it demotes the point as a side effect)
        if (obs.size() < 2 && !observed && is3d) { is3d = false; return true; }
        if (obs.size() == 0 && !observed) { is3d = false; return true; }
        return false;
    }
    // MapPoint::addDesc (map_point.cpp:129-180): keeps every keyframe's descriptor and the running distance sums; desc_ ends up
    // equal to the most recently added one (SURVEY App. C)
    void addDesc(int kf, const uint8_t* d) {
        if (kfdesc.count(kf)) return;
        Desc nd;
        memcpy(nd.b, d, 32);
        if (kfdesc.empty()) { kfdesc.emplace(kf, nd); descdist.emplace(kf, 0.f); desc = nd; has_desc = true; return; }
        kfdesc.emplace(kf, nd);
        descdist.emplace(kf, 0.f);
        float newsum = 0.f;
        for (auto& kv : kfdesc) {
            const float dist = (float)hamming256(nd.b, kv.second.b);
            descdist[kv.first] += dist;
            newsum += dist;
        }
        descdist[kf] = newsum;
        desc = nd; has_desc = true;
    }
    // MapPoint::removeObservedKeyframeId (map_point.cpp:70-127)
    void removeObs(int kf) {
        if (!obs.count(kf)) return;
        obs.erase(kf);
        if (obs.empty()) { has_desc = false; kfdesc.clear(); descdist.clear(); return; }
        if (kf == kfid) kfid = *obs.begin();
        auto itd = kfdesc.find(kf);
        if (itd != kfdesc.end()) {
            float minDist = has_desc ? 32 * 8.f : 0.f;
            int minId = -1;
            for (auto& kv : kfdesc) {
                if (kv.first == kf) continue;
                const float dist = (float)hamming256(itd->second.b, kv.second.b);
                float& s = descdist[kv.first];
                s -= dist;
                if (s < minDist) { minDist = s; minId = kv.first; }
            }
            kfdesc.erase(kf);
            descdist.erase(kf);
            if (minId > 0) { desc = kfdesc.at(minId); has_desc = true; }
        }
    }
};

struct MotionModel {   // visual_frontend.hpp:17-56
    double prevTime = -1.;
    Se3 prevTwc;
    double logRel[6] = {0, 0, 0, 0, 0, 0};
    void apply(Se3& Twc, double time) {
        if (prevTime > 0) {
            double xi[6];
            (Twc * prevTwc.inverse()).log(xi);
            bool zero = true;
            for (int i = 0; i < 6; i++) zero = zero && fabs(xi[i]) <= 1e-5;
            if (!zero) prevTwc = Twc;
            const double dt = time - prevTime;
            double s[6];
            for (int i = 0; i < 6; i++) s[i] = logRel[i] * dt;
            Twc = Twc * Se3::exp(s);
        }
    }
    void update(const Se3& Twc, double time) {
        if (prevTime < 0.) { prevTime = time; prevTwc = Twc; return; }
        const double dt = time - prevTime;
        prevTime = time;
        // dt == 0 (two frames inside one millisecond of the wall clock: a tracked frame takes well under 1 ms here) would turn the
        // reference's division (visual_frontend.hpp:42-53) into inf / NaN velocities that survive until the next P3P success:
        // keep the previous velocity instead.  dt > 0 is the reference's arithmetic unchanged.
        if (dt > 0.) {
            (prevTwc.inverse() * Twc).log(logRel);
            for (int i = 0; i < 6; i++) logRel[i] /= dt;
        }
        prevTwc = Twc;
    }
    void reset() { prevTime = -1.; for (int i = 0; i < 6; i++) logRel[i] = 0; }
};

// a Backend may offer the fused per-frame pose sequence (pose_chain); backends without it (the CPU oracle backend of the test
// suite) go through p3p() and pnp() one after the other -- both paths take the same decisions on the same numbers
template <class B, class = void> struct BackendHasPoseChain : std::false_type {};
template <class B> struct BackendHasPoseChain<B, std::void_t<decltype(std::declval<B&>().has_pose_chain())>> : std::true_type {};

// a Backend may undistort the points its klt() and detect() return (the CUDA backend does it on the device, in the same
// download): unpx() then gives their undistorted positions [n][2] until its next call, or NULL when it did not compute them.
// Backends without it (the CPU oracle backend) leave it to Camera::undistort -- the same arithmetic (camera_model.h).
template <class B, class = void> struct BackendHasUnpx : std::false_type {};
template <class B> struct BackendHasUnpx<B, std::void_t<decltype(std::declval<B&>().unpx())>> : std::true_type {};

// ------------------------------------------------------------------------------------------------ flat problems handed to a Backend
struct BaProblem {   // the layout of alva_k_ba_local
    int nkf = 0, nlm = 0, nobs = 0;
    double calib[4] = {0, 0, 0, 0};
    std::vector<double> poses;          // [nkf][7] in/out
    std::vector<uint8_t> pose_const;    // [nkf]
    std::vector<double> invd;           // [nlm] in/out
    std::vector<int32_t> anch_kf;       // [nlm] keyframe index
    std::vector<double> anch_uv;        // [nlm][2]
    std::vector<int32_t> obs_kf, obs_lm;
    std::vector<double> obs_uv;         // [nobs][2]
};
struct MatchProblem {   // Mapper::matchToMap on flat arrays (the contract of alva_k_match_to_map)
    double Twc_cur[7];
    int nkp3d = 0;
    std::vector<int32_t> kp_id, kp_mp;  // keypoints cell by cell; kp_mp = index of the keypoint's own map point in the table
    std::vector<float> kp_px;
    std::vector<int32_t> kf_id;         // keyframes referenced by the observations
    std::vector<double> kf_Twc;
    std::vector<int32_t> mp_id;         // map point table
    std::vector<double> mp_wpt;
    std::vector<uint8_t> mp_is3d;
    std::vector<int32_t> obs_start, obs_kfid;   // CSR; obs_kfid = keyframe ID, ascending per point
    std::vector<float> obs_px;
    std::vector<int32_t> desc_start, desc_kfid;
    std::vector<uint8_t> desc;
    std::vector<int32_t> local_mp;      // table indices of the local map, in the set's iteration order
    bool has_dist = false;              // lens distortion of the projections (Camera::dist)
    double dist[4] = {0, 0, 0, 0};
};

// ------------------------------------------------------------------------------------------------ the state machine
// Backend concept (host pointers in, host pointers out; < 0 = ALVA_E_* error):
//   int pyramid(const uint8_t* rgba)                       gray + pyramid + Scharr levels of the new frame; previous <- current
//                                                          (with CLAHE on, a backend matter: the pyramid is built on the equalised
//                                                          gray frame, visual_frontend.cpp:672-698)
//   int detect(const float* cur, int ncur, std::vector<float>& fresh)    grid detector on the current (equalised) image (adaptive quality kept)
//   int describe(const float* pts, int n, uint8_t* desc, uint8_t* kept)  ORB at the given points of the current RAW gray image
//                                                                        (map_manager.cpp:204, 218)
//   int klt(const float* pts, float* priors, int n, int levels, uint8_t* good)   forward-backward KLT previous -> current
//   int essential(const double* bv1, const double* bv2, int n, float fx, float fy, double* Rt12, uint8_t* outlier)  -> 1 / 0
//   int p3p(const double* bv, const double* X, int n, float fx, float fy, double* T12, uint8_t* outlier)            -> 1 / 0
//   int pnp(const double* uv, const double* X, int n, const double* K4, double* pose7, uint8_t* outlier)            -> 1 / 0
//   int triangulate(const double* Tlr7, const double* bvl, const double* bvr, int n, double* out)
//   bool has_ba_local(); int ba_local(BaProblem& io, int32_t* flags)         Optimizer::localBA's numerical body (two solves + flags)
//   bool has_match_to_map(); int match_to_map(const MatchProblem&, std::vector<int>& kp_match)   Mapper::matchToMap
//   optional: const float* unpx()                          see BackendHasUnpx
template <class Backend>
class SystemCore {
public:
    explicit SystemCore(Backend& b) : B(b) {}

    void configure(int w, int h, double fx, double fy, double cx, double cy) {
        cam.w = w; cam.h = h; cam.fx = fx; cam.fy = fy; cam.cx = cx; cam.cy = cy;
        cam.prepare();
        const double zero[4] = {0, 0, 0, 0};
        cam.setDistortion(zero);
        setPreset(40, 0.95f, true);   // State(w, h, 40), mapKeyframeFilteringRatio_ 0.95, p3pEnabled_ (system.cpp:15-19)
    }

    // The fields of the reference's preset table (state.hpp:9-17) the state machine reads: State(w, h, cell) and its
    // frameMaxNumKeypoints_ (state.cpp:3-12), the current Frame's grid (Frame(calibration, cell), frame.cpp:9-15), the keyframe
    // filtering ratio (mapper.cpp:75, 136) and p3pEnabled_ (visual_frontend.cpp:272).  The map and the tracked keypoints were
    // made on the old grid: reset.  (CLAHE, the table's fourth field, is the backend's pre-processing.)
    void setPreset(int cellsize, float filter_ratio, bool p3p) {
        cell = cellsize;
        max_kps = (int)(ceil((double)cam.w / cell) * ceil((double)cam.h / cell));
        kf_filter_ratio = filter_ratio;
        p3p_enabled = p3p;
        cur.init(&cam, cell);
        reset();
    }

    // the lens model of every later frame; the map and the tracked keypoints were made under the previous one: reset
    void setDistortion(const double* d) {
        cam.setDistortion(d);
        reset();
    }

    void reset() {   // System::reset (system.cpp:42-55)
        cur.reset();
        keyframes.clear(); mappoints.clear();
        n_mp_ids = n_kf_ids = n_kf = 0;
        ready_for_init = reset_requested = false;
        pose_failed = 0;
        // VisualFrontend::reset leaves the motion model and p3pReq_ alone (visual_frontend.cpp:718-728); so does this
    }

    // System::processCameraPose: returns 1 tracking / 2 reset / 3 not initialised, or a negative backend error
    int process(const uint8_t* rgba, double timestamp) {
        cur.id++;
        cur.ts = timestamp;
        err = 0;
        const bool kf = frontend(rgba, timestamp);
        if (err) return err;
        if (kf) {
            createKeyframe();
            if (err) return err;
            if (!reset_requested && ready_for_init) processNewKeyframe(cur.kfid);
            if (err) return err;
        }
        if (reset_requested) { reset(); return 2; }
        if (!ready_for_init) return 3;
        return 1;
    }

    // System::findPlane -> processPlane (system.cpp:123-137, 177-342) AS INTENDED.  The reference's own code cannot be matched
    // and does not do what it says: it seeds from std::random_device; `A.row(i).colRange(0, 3) = points[i].t()` re-allocates
    // the temporary row header (its points are CV_64F after cv::eigen2cv, A is CV_32F) so neither the 3-point sample planes
    // nor the final fit ever see the coordinates; `distances = dists` is taken after std::nth_element has permuted dists, so
    // inlier flags no longer belong to their points; and a normal parallel to (1, 0, 0) yields NaNs.  What it returns in
    // practice is the centroid of a haphazard subset of the observed map points with an axis-aligned rotation.  Here: the
    // same steps with those defects removed -- RANSAC over 3-point planes of the current frame's observed 3-D map points
    // (planes within 5 degrees of facing the world z axis only, score = the max(0.2 N, 20)-th smallest point-plane residual),
    // inliers below 1.4 x the best score, homogeneous least-squares refit, normal turned away from the camera, pose =
    // [Rodrigues(up x n, angle(up, n)) * Rodrigues((1, 0, 0)) | inlier centroid], written as Utils::toPoseArray(Mat) does
    // (column-major 4x4).  Sampling uses std::mt19937 seeded per call from a counter: repeatable.  Returns 1 / 0.
    int findPlane(float* out16, int iterations) {
        std::vector<double> pts;
        for (auto& kv : mappoints)
            if (kv.second.observed && kv.second.is3d) { pts.push_back(kv.second.p[0]); pts.push_back(kv.second.p[1]); pts.push_back(kv.second.p[2]); }
        const int n = (int)pts.size() / 3;
        if (n < 32) return 0;
        std::vector<int> indices(n), pick(3);
        for (int i = 0; i < n; i++) indices[i] = i;
        std::vector<float> dists(n), best_d(n, 0.f), tmp(n);
        float best = 1e10f;
        std::mt19937 rng(0x9e3779b9u + plane_calls++);
        const int kth = std::max((int)(0.2 * n), 20);
        for (int it = 0; it < iterations; it++) {
            std::sample(indices.begin(), indices.end(), pick.begin(), 3, rng);
            const double* p0 = &pts[3 * pick[0]];
            const double* p1 = &pts[3 * pick[1]];
            const double* p2 = &pts[3 * pick[2]];
            const double u[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]}, v[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
            double pl[4] = {u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0], 0};
            pl[3] = -(pl[0] * p0[0] + pl[1] * p0[1] + pl[2] * p0[2]);
            const double nn = sqrt(pl[0] * pl[0] + pl[1] * pl[1] + pl[2] * pl[2] + pl[3] * pl[3]);   // the SVD's null vector has unit 4-norm
            if (!(nn > 0)) continue;
            const float a = (float)(pl[0] / nn), b = (float)(pl[1] / nn), c = (float)(pl[2] / nn), d = (float)(pl[3] / nn);
            if (sqrt((double)a * a + (double)b * b) > sin(5.0f * 3.14159265358979323846 / 180.0f)) continue;   // |normal x z| > sin(5 deg)
            const float f = 1.0f / sqrtf(a * a + b * b + c * c + d * d);
            for (int i = 0; i < n; i++) dists[i] = fabsf((float)pts[3 * i] * a + (float)pts[3 * i + 1] * b + (float)pts[3 * i + 2] * c + d) * f;
            tmp = dists;
            std::nth_element(tmp.begin(), tmp.begin() + kth, tmp.end());
            if (tmp[kth] < best) { best = tmp[kth]; best_d = dists; }
        }
        const float thr = 1.4f * best;
        std::vector<int> inl;
        for (int i = 0; i < n; i++) if (best_d[i] < thr) inl.push_back(i);
        if ((int)inl.size() < 32 || !(best < 1e10f)) return 0;
        // homogeneous refit: the eigenvector of sum [p 1]^T [p 1] with the smallest eigenvalue (cyclic Jacobi, 4x4)
        double M[16] = {0}, origin[3] = {0, 0, 0};
        for (int i : inl) {
            const double q[4] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], 1.0};
            for (int r = 0; r < 4; r++) for (int cc = 0; cc < 4; cc++) M[4 * r + cc] += q[r] * q[cc];
            for (int r = 0; r < 3; r++) origin[r] += q[r];
        }
        for (int r = 0; r < 3; r++) origin[r] /= (double)inl.size();
        double V[16];
        for (int i = 0; i < 16; i++) V[i] = (i % 5 == 0);
        for (int sweep = 0; sweep < 60; sweep++) {
            double off = 0;
            for (int r = 0; r < 4; r++) for (int cc = r + 1; cc < 4; cc++) off += M[4 * r + cc] * M[4 * r + cc];
            if (off < 1e-300) break;
            for (int pI = 0; pI < 3; pI++)
                for (int qI = pI + 1; qI < 4; qI++) {
                    const double apq = M[4 * pI + qI];
                    if (apq == 0.0) continue;
                    const double theta = (M[5 * qI] - M[5 * pI]) / (2 * apq);
                    const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1));
                    const double cs = 1 / sqrt(t * t + 1), sn = t * cs;
                    for (int k = 0; k < 4; k++) { const double x = M[4 * k + pI], y = M[4 * k + qI]; M[4 * k + pI] = cs * x - sn * y; M[4 * k + qI] = sn * x + cs * y; }
                    for (int k = 0; k < 4; k++) { const double x = M[4 * pI + k], y = M[4 * qI + k]; M[4 * pI + k] = cs * x - sn * y; M[4 * qI + k] = sn * x + cs * y; }
                    for (int k = 0; k < 4; k++) { const double x = V[4 * k + pI], y = V[4 * k + qI]; V[4 * k + pI] = cs * x - sn * y; V[4 * k + qI] = sn * x + cs * y; }
                }
        }
        int m = 0;
        for (int i = 1; i < 4; i++) if (M[5 * i] < M[5 * m]) m = i;
        double a = V[m], b = V[4 + m], c = V[8 + m];
        const double fn = 1.0 / sqrt(a * a + b * b + c * c);
        // camera centre as the reference computes it from its transposed pose matrix (utils.cpp:51-75): Oc = -R t
        double Rm[9], Oc[3];
        cur.Twc.R(Rm);
        for (int r = 0; r < 3; r++) Oc[r] = -(Rm[3 * r] * cur.Twc.t[0] + Rm[3 * r + 1] * cur.Twc.t[1] + Rm[3 * r + 2] * cur.Twc.t[2]);
        if ((Oc[0] - origin[0]) * a + (Oc[1] - origin[1]) * b + (Oc[2] - origin[2]) * c > 0) { a = -a; b = -b; c = -c; }
        const double nx = a * fn, ny = b * fn, nz = c * fn;
        // R1 = Rodrigues((up x n) * angle / |up x n|), up = (1, 0, 0); R2 = Rodrigues(up) = 1 rad about x (as written in the reference)
        const double vx = 0, vy = -nz, vz = ny, sa = sqrt(vy * vy + vz * vz), ca = nx, ang = atan2(sa, ca);
        double R1[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        if (sa > 1e-12) {
            const double kx = vx / sa, ky = vy / sa, kz = vz / sa, cA = cos(ang), sA = sin(ang), C1 = 1 - cA;
            const double Rr[9] = {cA + kx * kx * C1, kx * ky * C1 - kz * sA, kx * kz * C1 + ky * sA,
                                  ky * kx * C1 + kz * sA, cA + ky * ky * C1, ky * kz * C1 - kx * sA,
                                  kz * kx * C1 - ky * sA, kz * ky * C1 + kx * sA, cA + kz * kz * C1};
            for (int i = 0; i < 9; i++) R1[i] = Rr[i];
        } else if (ca < 0) { R1[0] = -1; R1[4] = -1; }   // normal = -up: half a turn about z (the reference produces NaNs here)
        const double c1 = cos(1.0), s1 = sin(1.0);
        const double R2[9] = {1, 0, 0, 0, c1, -s1, 0, s1, c1};
        double Rp[9];
        for (int r = 0; r < 3; r++)
            for (int cc = 0; cc < 3; cc++) Rp[3 * r + cc] = R1[3 * r] * R2[cc] + R1[3 * r + 1] * R2[3 + cc] + R1[3 * r + 2] * R2[6 + cc];
        for (int cc = 0; cc < 3; cc++) { for (int r = 0; r < 3; r++) out16[4 * cc + r] = (float)Rp[3 * r + cc]; out16[4 * cc + 3] = 0.f; }
        out16[12] = (float)origin[0]; out16[13] = (float)origin[1]; out16[14] = (float)origin[2]; out16[15] = 1.f;
        return 1;
    }
    unsigned plane_calls = 0;
    std::vector<float> parallax_scratch;

    // ---- state the facade reads
    Camera cam;
    Frame cur;
    std::unordered_map<int, std::shared_ptr<Frame>> keyframes;   // MapManager::mapKeyframes_
    std::unordered_map<int, MapPoint> mappoints;                 // MapManager::mapMapPoints_
    int n_mp_ids = 0, n_kf_ids = 0, n_kf = 0;
    bool ready_for_init = false, reset_requested = false;
    int cell = 40, max_kps = 0;
    float kf_filter_ratio = 0.95f;   // State::mapKeyframeFilteringRatio_
    bool p3p_enabled = true;         // State::p3pEnabled_
    // what a run exercised, since construction (read by the tests and the golden generators): frames posed by PnP from the
    // motion prior, failures of that PnP (p3pReq_ set for the next frame), local BA solves, and solves in which the 21-free-pose
    // limit below held keyframes fixed
    int n_pnp_prior = 0, n_p3p_fallback = 0, n_local_ba = 0, n_free_pose_clamp = 0;

private:
    Backend& B;
    MotionModel motion;
    bool p3p_req = false;
    int pose_failed = 0, err = 0;

    // ------------------------------------------------------------------ MapManager pieces
    void removeObsFromCurr(int id) {
        cur.remove(id);
        auto it = mappoints.find(id);
        if (it != mappoints.end()) it->second.observed = false;
    }
    void removeMapPointObs(int mpid, int kfid) {   // map_manager.cpp:600-631
        auto kf = keyframes.find(kfid);
        if (kf != keyframes.end()) kf->second->remove(mpid);
        auto mp = mappoints.find(mpid);
        if (mp == mappoints.end()) return;
        mp->second.removeObs(kfid);
        if (kf != keyframes.end())
            for (int co : std::set<int>(mp->second.obs)) {
                auto ckf = keyframes.find(co);
                if (ckf != keyframes.end()) { kf->second->covisDecrease(co); ckf->second->covisDecrease(kfid); }
            }
    }
    void updateMapPoint(int id, const double* wpt, double invd) {   // map_manager.cpp:352-405
        auto it = mappoints.find(id);
        if (it == mappoints.end()) return;
        MapPoint& mp = it->second;
        if (!mp.is3d) {
            for (int k : std::set<int>(mp.obs)) {
                auto kf = keyframes.find(k);
                if (kf != keyframes.end()) kf->second->turn3d(id); else mp.removeObs(k);
            }
            if (mp.observed) cur.turn3d(id);
        }
        mp.p[0] = wpt[0]; mp.p[1] = wpt[1]; mp.p[2] = wpt[2];
        mp.is3d = true;
        if (invd >= 0.) mp.invd = invd;
    }

    void createKeyframe() {
        // prepareFrame (map_manager.cpp:24-66)
        cur.kfid = n_kf_ids;
        if (cur.n > max_kps) {
            for (size_t c = 0; c < cur.grid.size(); c++) {
                const std::vector<int> ids = cur.grid[c];
                if (ids.size() > 2) {
                    int victim = -1;
                    size_t min_obs = (size_t)-1;
                    for (int lm : ids) {   // the cell's keypoint seen by the fewest keyframes goes (a keypoint without map point first)
                        auto it = mappoints.find(lm);
                        if (it != mappoints.end()) { if (it->second.obs.size() < min_obs) { victim = lm; min_obs = it->second.obs.size(); } }
                        else { removeObsFromCurr(lm); break; }
                    }
                    if (victim >= 0) removeObsFromCurr(victim);
                }
            }
        }
        for (const Keypoint& k : cur.all()) {
            auto it = mappoints.find(k.id);
            if (it == mappoints.end()) { removeObsFromCurr(k.id); continue; }
            it->second.obs.insert(n_kf_ids);
        }
        // extractKeypoints (map_manager.cpp:193-222): describe the tracked keypoints, detect in the empty cells, describe those
        const std::vector<Keypoint> kps = cur.all();
        std::vector<float> pts(2 * kps.size() + 2);
        for (size_t i = 0; i < kps.size(); i++) { pts[2 * i] = kps[i].px; pts[2 * i + 1] = kps[i].py; }
        if (!kps.empty()) {
            std::vector<uint8_t> desc(32 * kps.size()), kept(kps.size());
            if ((err = B.describe(pts.data(), (int)kps.size(), desc.data(), kept.data())) < 0) return;
            err = 0;
            for (size_t i = 0; i < kps.size(); i++)
                if (kept[i]) {
                    auto it = cur.kps.find(kps[i].id);
                    if (it != cur.kps.end()) { it->second.has_desc = true; memcpy(it->second.desc, &desc[32 * i], 32); }
                    mappoints.at(kps[i].id).addDesc(cur.kfid, &desc[32 * i]);
                }
        }
        const int to_detect = max_kps - cur.nocc;
        if (to_detect > 0) {
            std::vector<float> fresh;
            if ((err = B.detect(pts.data(), (int)kps.size(), fresh)) < 0) return;
            err = 0;
            const float* un = backendUnpx();
            std::vector<float> fresh_un;
            if (un) fresh_un.assign(un, un + fresh.size());   // describe() below may reuse the backend's buffer
            const int nn = (int)fresh.size() / 2;
            if (nn > 0) {
                std::vector<uint8_t> desc(32 * (size_t)nn), kept(nn);
                if ((err = B.describe(fresh.data(), nn, desc.data(), kept.data())) < 0) return;
                err = 0;
                for (int i = 0; i < nn; i++) {   // addKeypointsToFrame + addMapPoint (map_manager.cpp:152-191, 255-330)
                    const uint8_t* d = kept[i] ? &desc[32 * (size_t)i] : nullptr;
                    cur.add(fresh[2 * i], fresh[2 * i + 1], n_mp_ids, d, un ? &fresh_un[2 * (size_t)i] : nullptr);
                    MapPoint mp;
                    mp.id = n_mp_ids; mp.kfid = n_kf_ids; mp.observed = true;
                    mp.obs.insert(n_kf_ids);
                    if (d) { mp.kfdesc.emplace(n_kf_ids, *(const Desc*)d); mp.descdist.emplace(n_kf_ids, 0.f); memcpy(mp.desc.b, d, 32); mp.has_desc = true; }
                    mappoints.emplace(n_mp_ids, mp);
                    n_mp_ids++;
                }
            }
        }
        // addKeyframe: an independent copy of the frame (map_manager.cpp:243-253)
        keyframes.emplace(n_kf_ids, std::make_shared<Frame>(cur));
        n_kf++;
        n_kf_ids++;
    }

    void updateFrameCovisibility(Frame& frame) {   // map_manager.cpp:68-150
        std::map<int, int> cov;
        std::unordered_set<int> local;
        for (const Keypoint& k : frame.all()) {
            auto it = mappoints.find(k.id);
            if (it == mappoints.end()) { removeMapPointObs(k.id, frame.kfid); removeObsFromCurr(k.id); continue; }
            for (int kf : it->second.obs)
                if (kf != frame.kfid) { auto c = cov.find(kf); if (c != cov.end()) c->second += 1; else cov.emplace(kf, 1); }
        }
        std::set<int> bad;
        for (auto& kv : cov) {
            auto it = keyframes.find(kv.first);
            if (it != keyframes.end()) {
                it->second->covis[frame.kfid] = kv.second;
                for (const Keypoint& k : it->second->all3d())
                    if (!frame.kps.count(k.id)) local.insert(k.id);
            } else bad.insert(kv.first);
        }
        for (int k : bad) cov.erase(k);
        frame.covis.swap(cov);
        if (local.size() > 0.5 * frame.localmap.size()) frame.localmap.swap(local);
        else frame.localmap.insert(local.begin(), local.end());
    }

    // ------------------------------------------------------------------ Mapper pieces
    void processNewKeyframe(int kfid) {   // mapper.cpp:9-64
        auto kfit = keyframes.find(kfid);
        if (kfit == keyframes.end()) return;
        std::shared_ptr<Frame> kf = kfit->second;
        if (kfid > 30) removeKeyframe(kfid - 30);
        if (kf->kfid > 0 && kf->n2d > 0) triangulateTemporal(*kf);
        if (err) return;
        if (ready_for_init) {
            if (kfid == 1 && kf->n3d < 30) { reset_requested = true; return; }
            if (kfid < 10 && kf->n3d < 3) { reset_requested = true; return; }
        }
        updateFrameCovisibility(*kf);
        cur.covis = kf->covis;
        if (kfid > 0) matchingToLocalMap(*kf);
        if (err) return;
        // Mapper::optimize (mapper.cpp:66-155)
        if (kf->kfid >= 2 && kf->n3d != 0) localBA(*kf);
        if (err) return;
        if (kf_filter_ratio < 1.0 && kf->kfid >= 20) filterKeyframes(*kf);   // State::mapKeyframeFilteringRatio_ < 1
    }

    // Mapper::matchingToLocalMap (mapper.cpp:293-352) + MapManager::mergeMapPoints (map_manager.cpp:407-495)
    void matchingToLocalMap(Frame& frame) {
        const size_t max_local = (size_t)max_kps * 10;
        const std::map<int, int> cov = frame.covis;
        if (!cov.empty() && frame.localmap.size() < max_local) {
            int kfid = cov.begin()->first;
            auto kf = keyframes.find(kfid);
            while (kf == keyframes.end() && kfid > 0) { kfid--; kf = keyframes.find(kfid); }
            if (kf != keyframes.end()) {
                const std::unordered_set<int> add = kf->second->localmap;
                frame.localmap.insert(add.begin(), add.end());
                // "another round" looks the same keyframe up again (mapper.cpp:318-331): its set is already merged
            }
        }
        if (frame.localmap.empty() || !B.has_match_to_map()) return;
        MatchProblem mp;
        buildMatchProblem(frame, mp);
        std::vector<int> kp_match(mp.kp_id.size(), -1);
        if ((err = B.match_to_map(mp, kp_match)) < 0) return;
        err = 0;
        std::map<int, int> prev_new;   // keypoint (= its own map point) id -> matched local map point id, ascending
        for (size_t i = 0; i < kp_match.size(); i++)
            if (kp_match[i] >= 0) prev_new.emplace(mp.kp_id[i], mp.mp_id[kp_match[i]]);
        for (auto& kv : prev_new) mergeMapPoints(kv.first, kv.second);
    }

    void mergeMapPoints(int prev, int next) {
        auto pit = mappoints.find(prev), nit = mappoints.find(next);
        if (pit == mappoints.end() || nit == mappoints.end() || !nit->second.is3d) return;
        const std::set<int> next_kfs = nit->second.obs, prev_kfs = pit->second.obs;
        const std::unordered_map<int, Desc> prev_desc = pit->second.kfdesc;
        for (int pk : prev_kfs) {
            auto kf = keyframes.find(pk);
            if (kf == keyframes.end()) continue;
            if (kf->second->updateId(prev, next, nit->second.is3d)) {
                nit->second.obs.insert(pk);
                for (int nk : next_kfs) {
                    auto co = keyframes.find(nk);
                    if (co != keyframes.end()) { kf->second->covisAdd(nk); co->second->covisAdd(pk); }
                }
            }
        }
        for (auto& kv : prev_desc) nit->second.addDesc(kv.first, kv.second.b);
        if (cur.kps.count(prev) && cur.updateId(prev, next, nit->second.is3d)) nit->second.observed = true;
        mappoints.erase(prev);
    }

    void buildMatchProblem(const Frame& frame, MatchProblem& m) {
        frame.Twc.to7(m.Twc_cur);
        m.nkp3d = frame.n3d;
        m.has_dist = cam.has_dist;
        for (int i = 0; i < 4; i++) m.dist[i] = cam.dist[i];
        // the frame's keypoints cell by cell, each cell in its insertion order (what Frame::getSurroundingKeypoints walks)
        std::unordered_map<int, int> mp_index;
        auto add_mp = [&](int id) -> int {
            auto it = mp_index.find(id);
            if (it != mp_index.end()) return it->second;
            auto mp = mappoints.find(id);
            if (mp == mappoints.end()) return -1;
            const int idx = (int)m.mp_id.size();
            mp_index.emplace(id, idx);
            m.mp_id.push_back(id);
            m.mp_is3d.push_back(mp->second.is3d ? 1 : 0);
            for (int i = 0; i < 3; i++) m.mp_wpt.push_back(mp->second.p[i]);
            for (int k : mp->second.obs) {   // ascending keyframe id
                auto kf = keyframes.find(k);
                if (kf == keyframes.end()) continue;
                const Keypoint* kk = kf->second->find(id);
                if (!kk) continue;
                int ki = -1;
                for (size_t j = 0; j < m.kf_id.size(); j++) if (m.kf_id[j] == k) ki = (int)j;
                if (ki < 0) { ki = (int)m.kf_id.size(); m.kf_id.push_back(k); double T[7]; kf->second->Twc.to7(T); m.kf_Twc.insert(m.kf_Twc.end(), T, T + 7); }
                m.obs_kfid.push_back(k); m.obs_px.push_back(kk->px); m.obs_px.push_back(kk->py);
            }
            m.obs_start.push_back((int)m.obs_kfid.size());
            for (auto& kv : mp->second.kfdesc) { m.desc_kfid.push_back(kv.first); m.desc.insert(m.desc.end(), kv.second.b, kv.second.b + 32); }
            m.desc_start.push_back((int)m.desc_kfid.size());
            return idx;
        };
        m.obs_start.push_back(0); m.desc_start.push_back(0);
        for (const auto& cellv : frame.grid)
            for (int id : cellv) {
                const Keypoint* k = frame.find(id);
                if (!k) continue;
                m.kp_id.push_back(id); m.kp_px.push_back(k->px); m.kp_px.push_back(k->py);
                m.kp_mp.push_back(add_mp(id));
            }
        for (int id : frame.localmap) { const int idx = add_mp(id); if (idx >= 0) m.local_mp.push_back(idx); }   // the set's iteration order
    }

    void removeMapPoint(int id) {   // map_manager.cpp:532-575
        auto it = mappoints.find(id);
        if (it == mappoints.end()) return;
        const std::set<int> obs = it->second.obs;
        for (int k : obs) {
            auto kf = keyframes.find(k);
            if (kf == keyframes.end()) continue;
            kf->second->remove(id);
            for (int co : obs)
                if (co != k) kf->second->covisDecrease(co);
        }
        if (it->second.observed) cur.remove(id);
        mappoints.erase(it);
    }

    void filterKeyframes(Frame& keyframe) {   // mapper.cpp:73-155
        const std::map<int, int> cov = keyframe.covis;
        for (auto it = cov.rbegin(); it != cov.rend(); ++it) {
            const int kfid = it->first;
            if (kfid == 0) break;
            if (kfid >= keyframe.kfid) continue;
            auto kfit = keyframes.find(kfid);
            if (kfit == keyframes.end()) continue;   // (the reference dereferences a null pointer here)
            std::shared_ptr<Frame> kf = kfit->second;
            if (kf->n3d < 25 / 2) { removeKeyframe(kfid); continue; }
            size_t good = 0, total = 0;
            for (const Keypoint& k : kf->all3d()) {
                auto mp = mappoints.find(k.id);
                if (mp == mappoints.end()) { removeMapPointObs(k.id, kfid); continue; }
                if (mp->second.isBad()) continue;
                if (mp->second.obs.size() > 4) good++;
                total++;
            }
            if ((float)good / (float)total > kf_filter_ratio) removeKeyframe(kfid);
        }
    }

    // Optimizer::localBA (optimizer.cpp:4-531): assembly in the reference's order, the numerical body on the device
    // (Backend::ba_local = alva_k_ba_local: two solves + both outlier passes), write-back and culling
    void localBA(Frame& nf) {
        const int min_cov = 25;   // State::baMinNumCommonKeypointsObservations_
        if (nf.n3d < min_cov || !B.has_ba_local()) return;
        std::map<int, int> cov = nf.covis;
        cov.emplace(nf.kfid, nf.n3d);
        std::unordered_map<int, std::shared_ptr<Frame>> local_kfs;   // map_local_pkfs (its iteration order fixes the gauge)
        std::unordered_set<int> bad_lms, lms2opt, cst_kfs;
        std::vector<int> kf_ids;                      // pose blocks in creation order
        std::unordered_map<int, int> kf_index;
        std::vector<double> poses;
        auto add_pose = [&](int kfid, const std::shared_ptr<Frame>& kf) {
            kf_index.emplace(kfid, (int)kf_ids.size());
            kf_ids.push_back(kfid);
            double T[7];
            kf->Twc.to7(T);
            poses.insert(poses.end(), T, T + 7);
        };
        bool all_cst = false;
        const int nmaxkfid = cov.rbegin()->first;
        for (auto it = cov.rbegin(); it != cov.rend(); ++it) {
            const int kfid = it->first;
            int score = it->second;
            if (kfid > nf.kfid) score = nf.n;
            auto kfit = keyframes.find(kfid);
            if (kfit == keyframes.end()) { if (kfid != nf.kfid) nf.covis.erase(kfid); continue; }
            add_pose(kfid, kfit->second);
            if (score >= min_cov && !all_cst && kfid > 0) {
                for (const Keypoint& k : kfit->second->all3d()) lms2opt.insert(k.id);
            } else { cst_kfs.insert(kfid); all_cst = true; }
            local_kfs.emplace(kfid, kfit->second);
        }
        struct Lm { int id, anch_kf; double au, av, invd; };
        std::vector<Lm> lms;
        std::unordered_map<int, int> lm_index;
        std::unordered_map<int, bool> local_lms;      // map_local_plms (keys; iterated in this container's order below)
        std::vector<int> obs_kf, obs_lm;
        std::vector<double> obs_uv;
        for (int lmid : lms2opt) {
            auto mpit = mappoints.find(lmid);
            if (mpit == mappoints.end()) continue;
            MapPoint& mp = mpit->second;
            if (mp.isBad()) { bad_lms.insert(lmid); continue; }
            local_lms.emplace(lmid, true);
            int anch = -1;
            for (int kfid : std::set<int>(mp.obs)) {
                if (kfid > nmaxkfid) continue;
                auto lk = local_kfs.find(kfid);
                std::shared_ptr<Frame> kf;
                if (lk == local_kfs.end()) {
                    auto kfit = keyframes.find(kfid);
                    if (kfit == keyframes.end()) { removeMapPointObs(kfid, mp.id); continue; }   // (argument order as in the reference)
                    kf = kfit->second;
                    local_kfs.emplace(kfid, kf);
                    add_pose(kfid, kf);
                    cst_kfs.insert(kfid);
                } else kf = lk->second;
                const Keypoint* kp = kf->find(lmid);
                if (!kp) { removeMapPointObs(lmid, kfid); continue; }
                if (anch < 0) {
                    anch = kfid;
                    double c[3];
                    kf->Tcw.apply(mp.p, c);
                    lm_index.emplace(lmid, (int)lms.size());
                    lms.push_back({lmid, kf_index.at(kfid), (double)kp->ux, (double)kp->uy, 1. / c[2]});
                    continue;
                }
                obs_kf.push_back(kf_index.at(kfid)); obs_lm.push_back(lm_index.at(lmid));
                obs_uv.push_back(kp->ux); obs_uv.push_back(kp->uy);
            }
        }
        size_t ncst = cst_kfs.size();
        if (ncst < 2)
            for (auto it = local_kfs.begin(); ncst < 2 && it != local_kfs.end(); ++it) { cst_kfs.insert(it->first); ncst++; }   // optimizer.cpp:240-248 (counts even a repeat)
        // the device solver factors a reduced camera system of at most 21 free poses (126 columns, one CTA's shared memory):
        // beyond that the OLDEST free keyframes are held fixed for this solve -- a deviation from the reference that its
        // 30-keyframe window can only reach when more than 21 covisible keyframes each share >= 25 points with the new one
        {
            std::vector<int> free_ids;
            for (int id : kf_ids) if (!cst_kfs.count(id)) free_ids.push_back(id);
            std::sort(free_ids.begin(), free_ids.end());
            if (free_ids.size() > 21) n_free_pose_clamp++;
            for (size_t i = 0; i + 21 < free_ids.size(); i++) cst_kfs.insert(free_ids[i]);
        }
        // ---- numerical body.  Landmarks without a residual are not part of Ceres' reduced program: leave them out
        const int nkf = (int)kf_ids.size(), nobs = (int)obs_lm.size();
        std::vector<int> used(lms.size(), -1), lm_of;
        for (int o = 0; o < nobs; o++) if (used[obs_lm[o]] < 0) { used[obs_lm[o]] = (int)lm_of.size(); lm_of.push_back(obs_lm[o]); }
        std::vector<int32_t> flags(nobs + 1, 0);
        if (nobs > 0) {
            BaProblem bp;
            bp.nkf = nkf; bp.nlm = (int)lm_of.size(); bp.nobs = nobs;
            bp.calib[0] = cam.fx; bp.calib[1] = cam.fy; bp.calib[2] = cam.cx; bp.calib[3] = cam.cy;
            bp.poses = poses;
            bp.pose_const.resize(nkf);
            for (int i = 0; i < nkf; i++) bp.pose_const[i] = cst_kfs.count(kf_ids[i]) ? 1 : 0;
            for (int l : lm_of) { bp.invd.push_back(lms[l].invd); bp.anch_kf.push_back(lms[l].anch_kf); bp.anch_uv.push_back(lms[l].au); bp.anch_uv.push_back(lms[l].av); }
            bp.obs_kf.assign(obs_kf.begin(), obs_kf.end());
            for (int o = 0; o < nobs; o++) bp.obs_lm.push_back(used[obs_lm[o]]);
            bp.obs_uv = obs_uv;
            n_local_ba++;
            if ((err = B.ba_local(bp, flags.data())) < 0) return;
            err = 0;
            poses = bp.poses;
            for (size_t i = 0; i < lm_of.size(); i++) lms[lm_of[i]].invd = bp.invd[i];
        }
        // ---- 5. update state (optimizer.cpp:361-531): pass-1 outliers first, then pass-2, as badKeyframeLandmarkIds is filled
        std::vector<std::pair<int, int>> bad;
        for (int pass = 1; pass <= 2; pass++)
            for (int o = 0; o < nobs; o++)
                if (flags[o] == pass) { bad.emplace_back(kf_ids[obs_kf[o]], lms[obs_lm[o]].id); bad_lms.insert(lms[obs_lm[o]].id); }
        for (auto& pr : bad) {
            if (local_kfs.count(pr.first)) removeMapPointObs(pr.second, pr.first);
            if (pr.first == cur.kfid) removeObsFromCurr(pr.second);
            bad_lms.insert(pr.second);
        }
        for (auto& kv : local_kfs) {
            if (cst_kfs.count(kv.first)) continue;
            kv.second->setTwc(Se3::from7(&poses[7 * (size_t)kf_index.at(kv.first)]));
        }
        for (auto& kv : local_lms) {
            const int lmid = kv.first;
            auto mpit = mappoints.find(lmid);
            if (mpit == mappoints.end()) { bad_lms.erase(lmid); continue; }
            MapPoint& mp = mpit->second;
            if (mp.isBad()) { removeMapPoint(lmid); bad_lms.erase(lmid); continue; }
            if (mp.obs.size() < 3 && mp.kfid < nf.kfid - 3 && !mp.observed) { removeMapPoint(lmid); bad_lms.erase(lmid); continue; }
            auto li = lm_index.find(lmid);
            if (li == lm_index.end()) { bad_lms.insert(lmid); continue; }
            const double invd = lms[li->second].invd, zanch = 1. / invd;
            if (zanch <= 0.) { removeMapPoint(lmid); bad_lms.erase(lmid); continue; }
            auto ak = local_kfs.find(mp.kfid);
            if (ak == local_kfs.end()) { bad_lms.insert(lmid); continue; }
            const Keypoint* kp = ak->second->find(lmid);
            float ux = 0.f, uy = 0.f;   // a missing keypoint yields the reference's default Keypoint (unpx = 0, 0)
            if (kp) { ux = kp->ux; uy = kp->uy; }
            double b[3], c[3], wpt[3];
            cam.inverseK(ux, uy, b);
            for (int i = 0; i < 3; i++) c[i] = zanch * b[i];
            ak->second->Twc.apply(c, wpt);
            updateMapPoint(lmid, wpt, invd);
        }
        for (int lmid : std::unordered_set<int>(bad_lms)) {
            auto mpit = mappoints.find(lmid);
            if (mpit == mappoints.end()) continue;
            if (mpit->second.isBad()) removeMapPoint(lmid);
            else if (mpit->second.obs.size() < 3 && mpit->second.kfid < nf.kfid - 3 && !mpit->second.observed) removeMapPoint(lmid);
        }
    }

    void removeKeyframe(int kfid) {   // map_manager.cpp:497-530
        auto it = keyframes.find(kfid);
        if (it == keyframes.end()) return;
        for (const Keypoint& k : it->second->all()) {
            auto mp = mappoints.find(k.id);
            if (mp != mappoints.end()) mp->second.removeObs(kfid);
        }
        for (auto& kv : it->second->covis) {
            auto co = keyframes.find(kv.first);
            if (co != keyframes.end() && kfid != co->second->kfid) co->second->covis.erase(kfid);
        }
        keyframes.erase(it);
        n_kf--;
    }

    void triangulateTemporal(Frame& frame) {   // mapper.cpp:157-291
        const std::vector<Keypoint> kps = frame.all2d();
        if (kps.empty()) return;
        const Se3 Twcj = frame.Twc;
        // pass 1: the candidates and the keyframe each is triangulated against (the first observer)
        struct Cand { size_t i; int kf; Keypoint kfkp; };
        std::vector<Cand> cands;
        for (size_t i = 0; i < kps.size(); i++) {
            auto mp = mappoints.find(kps[i].id);
            if (mp == mappoints.end()) { removeMapPointObs(kps[i].id, frame.kfid); continue; }
            if (mp->second.is3d) continue;
            if (mp->second.obs.size() < 2) continue;
            const int kfid = *mp->second.obs.begin();
            if (frame.kfid == kfid) continue;
            auto kf = keyframes.find(kfid);
            if (kf == keyframes.end()) continue;
            const Keypoint* kk = kf->second->find(kps[i].id);
            if (!kk || kk->id != kps[i].id) continue;
            cands.push_back({i, kfid, *kk});
        }
        // the triangulations are independent: one launch per partner keyframe (consecutive candidates share it almost always)
        std::vector<double> pts(3 * cands.size() + 3);
        size_t s = 0;
        while (s < cands.size()) {
            size_t e = s;
            while (e < cands.size() && cands[e].kf == cands[s].kf) e++;
            const Se3 Tcicj = keyframes.at(cands[s].kf)->Tcw * Twcj;
            double T7[7];
            Tcicj.to7(T7);
            std::vector<double> bl(3 * (e - s)), br(3 * (e - s));
            for (size_t c = s; c < e; c++) { memcpy(&bl[3 * (c - s)], cands[c].kfkp.bv, 24); memcpy(&br[3 * (c - s)], kps[cands[c].i].bv, 24); }
            if ((err = B.triangulate(T7, bl.data(), br.data(), (int)(e - s), &pts[3 * s])) < 0) return;
            err = 0;
            s = e;
        }
        // pass 2: the reference's gates, in its order
        for (size_t c = 0; c < cands.size(); c++) {
            const Keypoint& kp = kps[cands[c].i];
            const Keypoint& kk = cands[c].kfkp;
            std::shared_ptr<Frame> kf = keyframes.at(cands[c].kf);
            const Se3 Tcicj = kf->Tcw * Twcj, Tcjci = Tcicj.inverse();
            double rb[3];
            Tcicj.rot(kp.bv, rb);
            float ru, rv;
            cam.projCamToImage(rb, ru, rv);
            const double parallax = norm2d(kk.ux, kk.uy, ru, rv);
            const double* lp = &pts[3 * c];
            double rp[3];
            Tcjci.apply(lp, rp);
            if (lp[2] < 0.1 || rp[2] < 0.1) { if (parallax > 20.) removeMapPointObs(kk.id, frame.kfid); continue; }
            float lu, lv, pu, pv;
            cam.projCamToImage(lp, lu, lv);
            cam.projCamToImage(rp, pu, pv);
            const float ldist = norm2f(lu, lv, kk.ux, kk.uy), rdist = norm2f(pu, pv, kp.ux, kp.uy);
            if (ldist > 3.0f || rdist > 3.0f) { if (parallax > 20.) removeMapPointObs(kk.id, frame.kfid); continue; }   // mapMaxReprojectionError_
            double wpt[3];
            kf->Twc.apply(lp, wpt);
            updateMapPoint(kp.id, wpt, 1. / lp[2]);
        }
    }

    // ------------------------------------------------------------------ VisualFrontend pieces
    bool frontend(const uint8_t* rgba, double timestamp) {   // VisualFrontend::process
        if ((err = B.pyramid(rgba)) < 0) return false;
        err = 0;
        if (cur.id == 0) return true;
        Se3 Twc = cur.Twc;
        motion.apply(Twc, timestamp);
        cur.setTwc(Twc);
        kltTracking();
        if (err) return false;
        if (!ready_for_init) {
            if (cur.n2d < 50) { reset_requested = true; return false; }
            if (checkReadyForInit()) { ready_for_init = true; return true; }
            return false;
        }
        const bool ok = computePose();
        if (err) return false;
        if (!ok) {
            pose_failed++;
            if (pose_failed > 3) { reset_requested = true; return false; }
        }
        motion.update(cur.Twc, timestamp);
        return checkNewKeyframeRequired();
    }

    void kltTracking() {   // kltTrackingFromMotionPrior (kltUsePrior_ = true)
        std::vector<int> ids3, ids;
        std::vector<float> kps3, pri3, kps, pri;
        ids3.reserve(cur.n3d); kps3.reserve(2 * (size_t)cur.n3d); pri3.reserve(2 * (size_t)cur.n3d);
        ids.reserve(cur.n); kps.reserve(2 * (size_t)cur.n); pri.reserve(2 * (size_t)cur.n);
        double Rcw[9];
        cur.Tcw.R(Rcw);
        const double* tcw = cur.Tcw.t;
        for (auto& kv : cur.kps) {
            const Keypoint& k = kv.second;
            if (k.is3d) {
                double c[3];
                const double* X = mappoints.at(k.id).p;
                for (int i = 0; i < 3; i++) c[i] = (Rcw[3 * i] * X[0] + Rcw[3 * i + 1] * X[1] + Rcw[3 * i + 2] * X[2]) + tcw[i];
                float u, v;
                cam.projCamToImageDist(c, u, v);
                if (cam.inImage(u, v)) {
                    kps3.push_back(k.px); kps3.push_back(k.py); pri3.push_back(u); pri3.push_back(v); ids3.push_back(k.id);
                    continue;
                }
            }
            ids.push_back(k.id); kps.push_back(k.px); kps.push_back(k.py); pri.push_back(k.px); pri.push_back(k.py);
        }
        if (!ids3.empty()) {
            const size_t n3 = ids3.size();
            std::vector<uint8_t> good(n3);
            if ((err = B.klt(kps3.data(), pri3.data(), (int)n3, 1, good.data())) < 0) return;
            err = 0;
            const float* un = backendUnpx();
            size_t ngood = 0;
            for (size_t i = 0; i < n3; i++) {
                if (good[i]) { cur.update(ids3[i], pri3[2 * i], pri3[2 * i + 1], un ? un + 2 * i : nullptr); ngood++; }
                else { ids.push_back(ids3[i]); kps.push_back(kps3[2 * i]); kps.push_back(kps3[2 * i + 1]); pri.push_back(pri3[2 * i]); pri.push_back(pri3[2 * i + 1]); }
            }
            if (ngood < 0.33 * n3) { p3p_req = true; pri = kps; }
        }
        if (!ids.empty()) {
            const size_t n = ids.size();
            std::vector<uint8_t> good(n);
            if ((err = B.klt(kps.data(), pri.data(), (int)n, 3, good.data())) < 0) return;   // State::kltPyramidLevels_
            err = 0;
            const float* un = backendUnpx();
            for (size_t i = 0; i < n; i++) {
                if (good[i]) cur.update(ids[i], pri[2 * i], pri[2 * i + 1], un ? un + 2 * i : nullptr);
                else removeObsFromCurr(ids[i]);
            }
        }
    }

    // the undistorted positions of the points the last klt() / detect() returned, when the backend computed them
    const float* backendUnpx() {
        if constexpr (BackendHasUnpx<Backend>::value) if (cam.has_dist) return B.unpx();
        return nullptr;
    }

    void resetFrame() {   // visual_frontend.cpp:700-716
        const auto copy = cur.kps;
        for (auto& kv : copy) removeObsFromCurr(kv.first);
        cur.kps.clear();
        cur.grid.assign(cur.grid.size(), {});
        cur.n = cur.n2d = cur.n3d = cur.nocc = 0;
    }

    static bool finite3(const double* t) { return std::isfinite(t[0]) && std::isfinite(t[1]) && std::isfinite(t[2]); }

    bool computePose() {   // visual_frontend.cpp:245-417
        if (cur.n3d < 4) return false;
        std::vector<double> bvs, wpts, uv;
        std::vector<int> ids;
        bvs.reserve(3 * (size_t)cur.n3d); wpts.reserve(3 * (size_t)cur.n3d); uv.reserve(2 * (size_t)cur.n3d); ids.reserve(cur.n3d);
        const bool do_p3p = p3p_req || p3p_enabled;   // without P3P: PnP from the motion prior, P3P on the next frame if it fails
        for (auto& kv : cur.kps) {
            const Keypoint& k = kv.second;
            if (!k.is3d) continue;
            auto mp = mappoints.find(k.id);
            if (mp == mappoints.end()) continue;
            if (do_p3p) { bvs.push_back(k.bv[0]); bvs.push_back(k.bv[1]); bvs.push_back(k.bv[2]); }
            uv.push_back(k.ux); uv.push_back(k.uy);
            wpts.push_back(mp->second.p[0]); wpts.push_back(mp->second.p[1]); wpts.push_back(mp->second.p[2]);
            ids.push_back(k.id);
        }
        Se3 Twc = cur.Twc;
        std::vector<uint8_t> outl(ids.size() + 1);
        if constexpr (BackendHasPoseChain<Backend>::value) if (do_p3p && B.has_pose_chain()) {
            // Same decisions as below, replayed on the results of ONE device sequence (P3P-LMedS -> outliers dropped, P3P pose as the
            // PnP start -> PnP): the backend needs no host round trip between the two solvers.
            const int n = (int)ids.size();
            const double K4[4] = {(double)(float)cam.fx, (double)(float)cam.fy, (double)(float)cam.cx, (double)(float)cam.cy};
            double T12[12], pose7[7];
            std::vector<uint8_t> o2(n + 1);
            int ok1 = 0, ok2 = 0;
            const int rc = B.pose_chain(bvs.data(), wpts.data(), uv.data(), n, K4, (float)cam.fx, (float)cam.fy, T12, outl.data(), ok1, pose7, o2.data(), ok2);
            if (rc < 0) { err = rc; return false; }
            int nout = 0;
            for (int i = 0; i < n; i++) nout += outl[i] != 0;
            const double tt[3] = {T12[3], T12[7], T12[11]};
            if (!ok1 || n - nout < 5 || !finite3(tt)) { resetFrame(); return false; }
            const double Rm[9] = {T12[0], T12[1], T12[2], T12[4], T12[5], T12[6], T12[8], T12[9], T12[10]};
            Twc.setR(Rm);
            Twc.t[0] = tt[0]; Twc.t[1] = tt[1]; Twc.t[2] = tt[2];
            cur.setTwc(Twc);
            std::vector<int> ids2;
            ids2.reserve(n);
            for (int i = 0; i < n; i++) {
                if (outl[i]) { removeObsFromCurr(ids[i]); continue; }
                ids2.push_back(ids[i]);
            }
            const int n2 = (int)ids2.size();
            int nout2 = 0;
            for (int i = 0; i < n2; i++) nout2 += o2[i] != 0;
            if (!ok2 || n2 - nout2 < 5 || nout2 > 0.5 * n2 || !finite3(pose7)) { resetFrame(); return false; }
            cur.setTwc(Se3::from7(pose7));
            p3p_req = false;
            for (int i = 0; i < n2; i++)
                if (o2[i]) removeObsFromCurr(ids2[i]);
            return true;
        }
        if (do_p3p) {
            double T12[12];
            const int n = (int)ids.size();
            const int ok = B.p3p(bvs.data(), wpts.data(), n, (float)cam.fx, (float)cam.fy, T12, outl.data());
            if (ok < 0) { err = ok; return false; }
            int nout = 0;
            for (int i = 0; i < n; i++) nout += outl[i] != 0;
            const double tt[3] = {T12[3], T12[7], T12[11]};
            if (!ok || n - nout < 5 || !finite3(tt)) { resetFrame(); return false; }
            const double Rm[9] = {T12[0], T12[1], T12[2], T12[4], T12[5], T12[6], T12[8], T12[9], T12[10]};
            Twc.setR(Rm);
            Twc.t[0] = tt[0]; Twc.t[1] = tt[1]; Twc.t[2] = tt[2];
            cur.setTwc(Twc);
            std::vector<double> uv2, w2;
            std::vector<int> ids2;
            for (int i = 0; i < n; i++) {
                if (outl[i]) { removeObsFromCurr(ids[i]); continue; }
                uv2.push_back(uv[2 * i]); uv2.push_back(uv[2 * i + 1]);
                w2.push_back(wpts[3 * i]); w2.push_back(wpts[3 * i + 1]); w2.push_back(wpts[3 * i + 2]);
                ids2.push_back(ids[i]);
            }
            uv.swap(uv2); wpts.swap(w2); ids.swap(ids2);
        }
        const int n = (int)ids.size();
        double pose7[7];
        Twc.to7(pose7);
        const double K4[4] = {(double)(float)cam.fx, (double)(float)cam.fy, (double)(float)cam.cx, (double)(float)cam.cy};   // ceresPnP takes floats
        const int ok = B.pnp(uv.data(), wpts.data(), n, K4, pose7, outl.data());
        if (ok < 0) { err = ok; return false; }
        int nout = 0;
        for (int i = 0; i < n; i++) nout += outl[i] != 0;
        if (!ok || n - nout < 5 || nout > 0.5 * n || !finite3(pose7)) {
            if (!do_p3p) { p3p_req = true; n_p3p_fallback++; }
            resetFrame();
            return false;
        }
        if (!do_p3p) n_pnp_prior++;
        cur.setTwc(Se3::from7(pose7));
        p3p_req = false;
        for (int i = 0; i < n; i++)
            if (outl[i]) removeObsFromCurr(ids[i]);
        return true;
    }

    float computeParallax(int kfid, bool unrotate, bool median) {   // visual_frontend.cpp:596-670
        auto kfit = keyframes.find(kfid);
        if (kfit == keyframes.end()) return 0.f;
        const Frame& kf = *kfit->second;
        double Rk[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        if (unrotate) {
            double A[9], Bm[9];
            kf.Tcw.R(A); cur.Twc.R(Bm);
            for (int i = 0; i < 3; i++)
                for (int j = 0; j < 3; j++) Rk[3 * i + j] = A[3 * i] * Bm[j] + A[3 * i + 1] * Bm[3 + j] + A[3 * i + 2] * Bm[6 + j];
        }
        float avg = 0.f;
        int np = 0;
        std::vector<float>& s = parallax_scratch;   // the reference collects into a std::set<float>: DISTINCT values, ascending
        s.clear();
        for (auto& kv : cur.kps) {
            const Keypoint& k = kv.second;
            const Keypoint* kk = kf.find(k.id);
            if (!kk) continue;
            float ux = k.ux, uy = k.uy;
            if (unrotate) {
                double b[3];
                for (int i = 0; i < 3; i++) b[i] = Rk[3 * i] * k.bv[0] + Rk[3 * i + 1] * k.bv[1] + Rk[3 * i + 2] * k.bv[2];
                cam.projCamToImage(b, ux, uy);
            }
            const float parallax = norm2f(ux, uy, kk->ux, kk->uy);
            avg += parallax;
            np++;
            if (median) s.push_back(parallax);
        }
        if (np == 0) return 0.f;
        avg /= (float)np;
        if (median) {   // element size/2 of the set == of the sorted distinct values (no per-value node allocation here)
            std::sort(s.begin(), s.end());
            s.erase(std::unique(s.begin(), s.end()), s.end());
            avg = s[s.size() / 2];
        }
        return avg;
    }

    bool checkReadyForInit() {   // visual_frontend.cpp:419-552
        const double med = computeParallax(cur.kfid, false, true);
        if (med <= 40.0f) return false;   // State::minAvgRotationParallax_
        auto kfit = keyframes.find(cur.kfid);
        if (kfit == keyframes.end()) return false;
        const Frame& kf = *kfit->second;
        if (cur.n < 8) return false;
        std::vector<int> ids;
        std::vector<double> b1, b2;
        double Rm[9], A[9], Bm[9];
        kf.Tcw.R(A); cur.Twc.R(Bm);
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) Rm[3 * i + j] = A[3 * i] * Bm[j] + A[3 * i + 1] * Bm[3 + j] + A[3 * i + 2] * Bm[6 + j];
        int np = 0;
        float avg = 0.f;
        for (auto& kv : cur.kps) {
            const Keypoint& k = kv.second;
            const Keypoint* kk = kf.find(k.id);
            if (!kk) continue;
            for (int i = 0; i < 3; i++) { b1.push_back(kk->bv[i]); b2.push_back(k.bv[i]); }
            ids.push_back(k.id);
            double rb[3], un[3];
            for (int i = 0; i < 3; i++) rb[i] = Rm[3 * i] * k.bv[0] + Rm[3 * i + 1] * k.bv[1] + Rm[3 * i + 2] * k.bv[2];
            un[0] = cam.fx * rb[0] + cam.cx * rb[2]; un[1] = cam.fy * rb[1] + cam.cy * rb[2]; un[2] = rb[2];   // K_ * rotBv
            const float rx = (float)(un[0] / un[2]), ry = (float)(un[1] / un[2]);
            avg += norm2d(rx, ry, kk->ux, kk->uy);
            np++;
        }
        if (np < 8) return false;
        avg /= (float)np;
        if (avg < 40.0f) return false;
        double Rt[12];
        std::vector<uint8_t> outl(ids.size());
        const int ok = B.essential(b1.data(), b2.data(), (int)ids.size(), (float)cam.fx, (float)cam.fy, Rt, outl.data());
        if (ok < 0) { err = ok; return false; }
        if (!ok) return false;
        for (size_t i = 0; i < ids.size(); i++)
            if (outl[i]) removeObsFromCurr(ids[i]);
        double t[3] = {Rt[3], Rt[7], Rt[11]};
        const double nt = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
        const double Rw[9] = {Rt[0], Rt[1], Rt[2], Rt[4], Rt[5], Rt[6], Rt[8], Rt[9], Rt[10]};
        Se3 T;
        T.setR(Rw);
        T.t[0] = t[0] / nt; T.t[1] = t[1] / nt; T.t[2] = t[2] / nt;
        cur.setTwc(T);
        return true;
    }

    bool checkNewKeyframeRequired() {   // visual_frontend.cpp:554-594
        auto kfit = keyframes.find(cur.kfid);
        if (kfit == keyframes.end()) return false;
        const Frame& kf = *kfit->second;
        const double med = computeParallax(kf.kfid, true, true);
        const int id_diff = cur.id - kf.id;
        if (id_diff >= 5 && cur.nocc < 0.33 * max_kps) return true;
        if (id_diff >= 2 && cur.n3d < 20) return true;
        if (id_diff < 2 && cur.n3d > 0.5 * max_kps) return false;
        const bool cx = med >= 40.0f / 2.;
        const bool c0 = med >= 40.0f;
        const bool c1 = cur.n3d < 0.75 * kf.n3d;
        const bool c2 = cur.nocc < 0.5 * max_kps && cur.n3d < 0.85 * kf.n3d;
        return (c0 || c1 || c2) && cx;
    }
};

}  // namespace alva_sys
