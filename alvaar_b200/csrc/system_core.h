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
    // The lens model, explicit: the pinhole, OpenCV's radial-tangential model (k1 k2 p1 p2, CameraCalibration::D_) or OpenCV's
    // equidistant fisheye model (k1 k2 k3 k4 on theta).  has_dist = a model other than the pinhole is applied.  The
    // radial-tangential model with all coefficients zero is the pinhole: the two functions that apply it below then take their
    // pinhole forms, which give the same bits.  A fisheye lens with zero coefficients is the equidistant projection, not the
    // pinhole, so the model is never inferred from the coefficients.
    enum Lens { PINHOLE = 0, RADTAN = 1, FISHEYE = 2 };
    int lens = PINHOLE;
    double dist[4] = {0, 0, 0, 0};
    bool has_dist = false;
    void setDistortion(const double* d) {
        has_dist = false;
        for (int i = 0; i < 4; i++) { dist[i] = d[i]; has_dist = has_dist || d[i] != 0.0; }
        lens = has_dist ? RADTAN : PINHOLE;
    }
    void setFisheye(bool on, const double* k) {
        for (int i = 0; i < 4; i++) dist[i] = on ? k[i] : 0.0;
        lens = on ? FISHEYE : PINHOLE;
        has_dist = on;
    }
    // the value cv::fisheye::undistortPoints returns for a pixel it cannot undistort (Newton did not converge, or theta flipped):
    // 1e6 px outside any image, never the result of the radial-tangential model or of a converged fisheye point in practice
    static bool lensFailure(float ux, float uy) { return ux == -1000000.0f && uy == -1000000.0f; }
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
        if (lens == FISHEYE) {
            double k[4];
            float o[2];
            K4(k);
            alva_cam::undistort_point_fisheye(k, dist, u, v, o);
            ux = o[0]; uy = o[1];
            return;
        }
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
        if (lens == FISHEYE) {
            double k[4];
            float o[2];
            K4(k);
            alva_cam::project_dist_fisheye(k, dist, p, o);
            u = o[0]; v = o[1];
            return;
        }
        if (has_dist) {
            double k[4];
            float o[2];
            K4(k);
            alva_cam::project_dist(k, dist, p, o);
            u = o[0]; v = o[1];
            return;
        }
        double k[4];
        float o[2];
        K4(k);
        alva_cam::project_pinhole(k, p, o);
        u = o[0]; v = o[1];
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

// a Backend may relocalise a lost frame against the map (detect_lost + relocalise); with one that cannot, the relocalisation
// mode has no effect (the test suite's older CPU backends)
template <class B, class = void> struct BackendHasReloc : std::false_type {};
template <class B> struct BackendHasReloc<B, std::void_t<decltype(std::declval<B&>().detect_lost(std::declval<std::vector<float>&>()))>> : std::true_type {};

// a Backend may match fresh detections against the frozen map (reacquire); without it the localisation-only mode is refused
template <class B, class = void> struct BackendHasReacquire : std::false_type {};
template <class B> struct BackendHasReacquire<B, std::void_t<decltype(&B::reacquire)>> : std::true_type {};

// a Backend may rotate the 2-D KLT priors by the gyroscope's rotation (klt_rotated); without it the gyro mode is refused
template <class B, class = void> struct BackendHasRotatedKlt : std::false_type {};
template <class B> struct BackendHasRotatedKlt<B, std::void_t<decltype(&B::klt_rotated)>> : std::true_type {};

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
    bool fisheye = false;               // ... through the equidistant fisheye model instead of the radial-tangential one
    double dist[4] = {0, 0, 0, 0};
};
// the map a lost frame is matched against: every map point that is 3-D and has a descriptor, in ascending id order; its
// keyframe descriptors (MapPoint::kfdesc) in ascending keyframe id order, CSR.  The map is frozen while lost: built once, when
// the core enters LOST; `version` tells a backend that keeps a device copy when to upload it again.
struct RelocTable {
    std::vector<int32_t> mp_id;         // [n]
    std::vector<double> wpt;            // [n][3]
    std::vector<int32_t> desc_start;    // [n + 1]
    std::vector<uint8_t> desc;          // [rows][32]
    unsigned version = 0;
    void clear() { mp_id.clear(); wpt.clear(); desc_start.clear(); desc.clear(); version++; }
};
// what Backend::relocalise returns: the kept matches (query, table row) in ascending query order; P3P-RANSAC on them (T12, ok1,
// o1 [n_match]); PnP from the RANSAC pose on its inliers (pose7, ok2, o2 [n_match - #o1], in the inliers' order)
struct RelocResult {
    int n_match = 0, ok1 = 0, ok2 = 0;
    std::vector<int32_t> mq, mg;
    double T12[12] = {0}, pose7[7] = {0};
    std::vector<uint8_t> o1, o2;
};

// ------------------------------------------------------------------------------------------------ map blob byte order
// fixed-width little-endian fields, no padding (a little-endian host is assumed: x86-64 and aarch64 Linux)
static_assert(sizeof(float) == 4 && sizeof(double) == 8, "the map blob stores IEEE binary32 / binary64");
struct MapWriter {
    std::vector<uint8_t>& o;
    explicit MapWriter(std::vector<uint8_t>& out) : o(out) { o.clear(); }
    void raw(const void* p, size_t n) { const uint8_t* b = (const uint8_t*)p; o.insert(o.end(), b, b + n); }
    void u8(uint8_t v) { o.push_back(v); }
    void i32(int32_t v) { raw(&v, 4); }
    void u32(uint32_t v) { raw(&v, 4); }
    void u64(uint64_t v) { raw(&v, 8); }
    void f32(float v) { raw(&v, 4); }
    void f64(double v) { raw(&v, 8); }
    void se3(const Se3& T) { for (int i = 0; i < 3; i++) f64(T.t[i]); for (int i = 0; i < 4; i++) f64(T.q[i]); }
};
// every read is bounds-checked: false (and nothing read) past the end
struct MapReader {
    const uint8_t* p;
    size_t n, off = 0;
    MapReader(const uint8_t* d, size_t bytes) : p(d), n(bytes) {}
    size_t left() const { return n - off; }
    bool raw(void* dst, size_t k) { if (k > left()) return false; memcpy(dst, p + off, k); off += k; return true; }
    bool u8(uint8_t& v) { return raw(&v, 1); }
    bool flag(bool& v) { uint8_t b; if (!u8(b) || b > 1) return false; v = b != 0; return true; }   // 0 or 1 only
    bool i32(int32_t& v) { return raw(&v, 4); }
    bool u32(uint32_t& v) { return raw(&v, 4); }
    bool u64(uint64_t& v) { return raw(&v, 8); }
    bool f32(float& v) { return raw(&v, 4) && std::isfinite(v); }   // finite values only
    bool f64(double& v) { return raw(&v, 8) && std::isfinite(v); }
    bool se3(Se3& T) { for (int i = 0; i < 3; i++) if (!f64(T.t[i])) return false; for (int i = 0; i < 4; i++) if (!f64(T.q[i])) return false; return true; }
    // a count of records of at least `min_bytes` each that the rest of the blob can hold
    bool count(uint32_t& c, size_t min_bytes) { return u32(c) && (uint64_t)c * min_bytes <= left(); }
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
//   int detect_lost(std::vector<float>& fresh)             grid detector on the whole current image with its own adaptive quality
//                                                          (the tracker's is left as it was); unpx() as after detect()
//   int relocalise(const RelocTable&, const uint8_t* qdesc, const double* qbv, const double* quv, int nq, const double* K4,
//                  float fx, float fy, RelocResult&)       grouped Hamming 2-NN, match rules, P3P-RANSAC (512) and PnP (relocaliseFrame)
//   int reacquire(const RelocTable&, const uint8_t* skip, const double* Twc7, const float* qpx, const uint8_t* qdesc,
//                 const uint8_t* qkept, int nq, float radius, int32_t* row, int32_t* dist)
//                                                          alva_k_match_frame_to_map: per query the matched table row or -1
//                                                          (localisation-only mode, reacquireFrame)
//   int klt_rotated(const float* pts, float* priors, int n, int levels, uint8_t* good, const double* bv, const uint8_t* flag,
//                   const double* dR9, uint8_t* rotated)   klt() after the prior of every flagged point is replaced by
//                                                          alva_cam::rotate_prior of its bearing bv [n][3] under dR9 where that
//                                                          is valid (rotated [n] = 1; the lens is the backend's) -- gyro mode
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
        n_lens_drops = 0;
        setPreset(40, 0.95f, true);   // State(w, h, 40), mapKeyframeFilteringRatio_ 0.95, p3pEnabled_ (system.cpp:15-19)
        reloc_max = 0;
        setGyro(false, nullptr, nullptr);
        n_gyro_pred = n_gyro_fallback = n_gyro_carried = n_gyro_rot = n_gyro_kept = 0;
        gyro_have_prev = false;
    }

    // ------------------------------------------------------------------ gyro-aided tracking (not in the reference)
    // The gyroscope's rotation between two frames predicts the camera's rotation, so a fast pan does not outrun the tracker.
    //
    // Samples {t_ms, gx, gy, gz (rad/s, IMU axes), ax, ay, az (ignored)} arrive with the frames (addGyroSamples) and are kept in
    // time order.  After a frame at time t_k is integrated, every sample before the last one at or before t_k is discarded;
    // samples later than t_k wait for the next frame.
    //
    // Integration over [A, B] = [t_{k-1}, t_k] (the previous and the current frame's time stamps, whatever their status):
    //   omega(tau) at an end: with L the last sample at or before tau and H the first one after it, L + (H - L) (tau - t_L) /
    //     (t_H - t_L) when both exist and t_H - t_L <= 50 ms; else L held when tau - t_L <= 50 ms; else H held when
    //     t_H - tau <= 50 ms; else undefined.
    //   breakpoints: A, the samples with A < t < B in order (each with its own omega: equal time stamps make zero-length
    //     pieces), B.
    //   covered: B >= A, a previous frame exists, omega is defined at both ends, and no two consecutive samples inside (A, B)
    //     are more than 50 ms apart.
    //   dR = I; per piece [a, b] in time order: dR <- dR Exp(((omega(a) + omega(b)) / 2 - bias) (b - a) / 1000), double
    //     precision, Exp = Rodrigues (I + a K + b K^2, K = [phi]x; a = 1 - th^2 / 6, b = 1/2 - th^2 / 24 below th = 1e-6).
    //   dR_c = R_ci dR R_ci^T: the rotation of the current camera in the previous one's axes (R_wc,k = R_wc,k-1 dR_c).
    // A frame whose interval is not covered takes the camera-only path unchanged (counted in n_gyro_fallback).
    //
    // A covered frame:
    //   - tracked (after the initialisation): the motion model's prediction keeps its translation, its rotation becomes
    //     R_wc,k-1 dR_c; 3-D keypoints are projected with that pose as before (n_gyro_pred also counts covered frames before
    //     the initialisation, whose pose is not predicted);
    //   - KLT's second pass: every keypoint whose prior would be its previous position -- 2-D keypoints, 3-D keypoints whose
    //     projection leaves the image, and all of them after a failed first pass -- starts from alva_cam::rotate_prior(dR_c,
    //     bv) instead where that ray is in front of the camera and projects inside the image (n_gyro_rot), else from its
    //     previous position (n_gyro_kept).  3-D keypoints that fail the first pass keep their projected prior;
    //   - lost (relocalisation on, including the frame that loses the track): the pose keeps its translation and its rotation
    //     advances by dR_c (n_gyro_carried); relocalisation itself uses no prior.
    // setGyro needs a backend with klt_rotated (MAP_STATE otherwise).  R_ci (NULL: identity) takes IMU-axis vectors to camera
    // axes; bias (NULL: zero) is a constant gyro bias in rad/s on the IMU axes.  A non-finite value, or an R_ci with an entry
    // of R^T R - I above 1e-9 or a negative determinant, is refused (MAP_INVALID).  Disabling drops the samples.  configure
    // ends the mode; reset, setPreset, setDistortion, setFisheye, setRelocalisation, setLocalisationOnly and loadMap keep it.
    int setGyro(bool on, const double* Rci, const double* bias) {
        if (!on) { gyro_on = gyro_ok = false; gyro_buf.clear(); gyroIdentity(gyro_dRc); return 0; }
        double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, b[3] = {0, 0, 0};
        if (Rci) for (int i = 0; i < 9; i++) R[i] = Rci[i];
        if (bias) for (int i = 0; i < 3; i++) b[i] = bias[i];
        for (int i = 0; i < 9; i++) if (!std::isfinite(R[i])) { map_error = "non-finite R_ci"; return MAP_INVALID; }
        for (int i = 0; i < 3; i++) if (!std::isfinite(b[i])) { map_error = "non-finite bias"; return MAP_INVALID; }
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                const double d = R[i] * R[j] + R[3 + i] * R[3 + j] + R[6 + i] * R[6 + j] - (i == j ? 1.0 : 0.0);
                if (!(fabs(d) <= 1e-9)) { map_error = "R_ci is not orthonormal"; return MAP_INVALID; }
            }
        const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
        if (det < 0) { map_error = "R_ci is a reflection (negative determinant)"; return MAP_INVALID; }
        if (!BackendHasRotatedKlt<Backend>::value) { map_error = "the backend cannot rotate KLT priors"; return MAP_STATE; }
        memcpy(gyro_Rci, R, sizeof R);
        memcpy(gyro_bias, b, sizeof b);
        gyro_on = true;
        return 0;
    }

    // samples [n][7] = {t_ms, gx, gy, gz, ax, ay, az} for the next frame.  Refused (MAP_INVALID, nothing kept) for n < 0, NULL
    // with n > 0, a non-finite value, time stamps that decrease within the call or a sample older than the newest one held.
    // Checked with the mode off too; kept only with it on.
    int addGyroSamples(const double* s, int n) {
        if (n < 0 || (!s && n > 0)) { map_error = "bad sample array"; return MAP_INVALID; }
        double last = gyro_buf.empty() ? -INFINITY : gyro_buf.back().t;
        for (int i = 0; i < n; i++) {
            for (int c = 0; c < 7; c++) if (!std::isfinite(s[7 * (size_t)i + c])) { map_error = "non-finite sample"; return MAP_INVALID; }
            if (s[7 * (size_t)i] < last) { map_error = "sample time stamps decrease"; return MAP_INVALID; }
            last = s[7 * (size_t)i];
        }
        if (!gyro_on) return 0;
        for (int i = 0; i < n; i++) {
            const double* p = s + 7 * (size_t)i;
            gyro_buf.push_back({p[0], {p[1], p[2], p[3]}});
        }
        return 0;
    }
    size_t gyroSamplesHeld() const { return gyro_buf.size(); }

    // relocalisation after a tracking loss (0 = off: the reference's reset on the fourth failed pose); kept by reset().  The
    // localisation-only mode needs it: turning it off then is refused (MAP_STATE).
    int setRelocalisation(int max_lost_frames) {
        if (frozen && max_lost_frames <= 0) { map_error = "the localisation-only mode needs relocalisation"; return MAP_STATE; }
        reloc_max = max_lost_frames;
        return 0;
    }

    // ------------------------------------------------------------------ localisation only (not in the reference)
    // Track against a frozen map: no keyframe, no triangulation, no local BA, no keyframe removal; keyframes and map points
    // never change except the per-frame `observed` flag, and no id counter moves.  Points KLT loses come back through
    // reacquireFrame.  A loss runs the relocalisation as usual but never resets the map.  Enabling needs relocalisation on
    // and a map (MAP_STATE otherwise); it drops the frame's 2-D keypoints (only a keyframe could triangulate them) and keeps
    // the relocalisation table loadMap or the loss built, or builds it for a tracking session.  The table is then neither
    // rebuilt nor re-versioned until the mode ends.  Disabling is always allowed: mapping resumes on the next keyframe
    // decision, ids continue from the counters, and a frame still lost gets max_lost_frames frames from then on.
    // configure, reset, setPreset, setDistortion and setFisheye end the mode; loadMap keeps it (the loaded map is frozen).
    int setLocalisationOnly(bool on) {
        if (!on) {
            if (frozen && lost) lost_frames = 0;
            frozen = false;
            reacq_pending = false;
            return 0;
        }
        if (reloc_max <= 0 || !BackendHasReloc<Backend>::value || !BackendHasReacquire<Backend>::value) {
            map_error = "relocalisation is off";
            return MAP_STATE;
        }
        if (!ready_for_init) { map_error = "no map: not initialised"; return MAP_STATE; }
        if (frozen) return 0;
        for (const Keypoint& k : cur.all2d()) removeObsFromCurr(k.id);
        if (!lost) buildRelocTable();
        frozen = true;
        reacq_pending = true;
        return 0;
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
        n_lens_drops = 0;
        reset();
    }
    // the equidistant fisheye model (on = false: the pinhole); replaces the radial-tangential model and is replaced by it
    void setFisheye(bool on, const double* k) {
        cam.setFisheye(on, k);
        n_lens_drops = 0;
        reset();
    }

    void reset() {   // System::reset (system.cpp:42-55)
        cur.reset();
        keyframes.clear(); mappoints.clear();
        n_mp_ids = n_kf_ids = n_kf = 0;
        ready_for_init = reset_requested = false;
        pose_failed = 0;
        lost = false; lost_frames = 0;
        reloc_table.clear();
        frozen = reacq_pending = false;
        reacq_nocc = 0;
        // VisualFrontend::reset leaves the motion model and p3pReq_ alone (visual_frontend.cpp:718-728); so does this
    }

    // ------------------------------------------------------------------ the map blob (not in the reference)
    // The layout is documented in include/alva_b200.h (alva_system_save_map) and INTEGRATION.md.  Return codes: 0, MAP_STATE
    // (= ALVA_E_STATE) or MAP_INVALID (= ALVA_E_INVALID); map_error names the failed check.
    enum { MAP_INVALID = -1, MAP_STATE = -4 };
    static constexpr uint32_t MAP_VERSION = 1;
    mutable const char* map_error = "";

    // the blob of the current map; allowed once initialised (also while lost).  Reads the containers only.
    int saveMap(std::vector<uint8_t>& out) const {
        if (!ready_for_init) { map_error = "not initialised"; return MAP_STATE; }
        MapWriter w(out);
        std::vector<int> kf_ids, mp_ids;
        for (auto& kv : keyframes) kf_ids.push_back(kv.first);
        for (auto& kv : mappoints) mp_ids.push_back(kv.first);
        std::sort(kf_ids.begin(), kf_ids.end());
        std::sort(mp_ids.begin(), mp_ids.end());
        w.raw("ALMP", 4); w.u32(MAP_VERSION); w.u64(0); w.u32((uint32_t)kf_ids.size()); w.u32((uint32_t)mp_ids.size());
        w.i32(cam.w); w.i32(cam.h); w.f64(cam.fx); w.f64(cam.fy); w.f64(cam.cx); w.f64(cam.cy); w.i32(cam.lens);
        for (int i = 0; i < 4; i++) w.f64(cam.dist[i]);
        w.i32(cell);
        w.i32(n_kf_ids); w.i32(n_mp_ids); w.i32(n_kf);
        w.se3(cur.Twc);
        for (int id : kf_ids) {
            const Frame& f = *keyframes.at(id);
            w.i32(id); w.i32(cur.id - f.id); w.se3(f.Twc);
            std::vector<int> kp;
            for (auto& kv : f.kps) kp.push_back(kv.first);
            std::sort(kp.begin(), kp.end());
            w.u32((uint32_t)kp.size());
            for (int k : kp) {
                const Keypoint& p = f.kps.at(k);
                w.i32(p.id); w.f32(p.px); w.f32(p.py); w.f32(p.ux); w.f32(p.uy);
                for (int i = 0; i < 3; i++) w.f64(p.bv[i]);
                w.u8(p.is3d); w.u8(p.has_desc); w.raw(p.desc, 32);
            }
            w.u32((uint32_t)f.covis.size());
            for (auto& kv : f.covis) { w.i32(kv.first); w.i32(kv.second); }
            std::vector<int> lm(f.localmap.begin(), f.localmap.end());
            std::sort(lm.begin(), lm.end());
            w.u32((uint32_t)lm.size());
            for (int k : lm) w.i32(k);
        }
        for (int id : mp_ids) {
            const MapPoint& m = mappoints.at(id);
            // `observed` as the lost state holds it: entering LOST clears the flag of every point of the current frame
            w.i32(m.id); w.i32(m.kfid); w.u8(m.observed && !cur.kps.count(m.id)); w.u8(m.is3d); w.f64(m.invd);
            for (int i = 0; i < 3; i++) w.f64(m.p[i]);
            w.u32((uint32_t)m.obs.size());
            for (int k : m.obs) w.i32(k);
            std::vector<int> dk;
            for (auto& kv : m.kfdesc) dk.push_back(kv.first);
            std::sort(dk.begin(), dk.end());
            w.u32((uint32_t)dk.size());
            for (int k : dk) { w.i32(k); w.raw(m.kfdesc.at(k).b, 32); w.f32(m.descdist.at(k)); }
            // desc_ of a point that never had a descriptor is uninitialised (and never read): zeros then
            static const uint8_t zero[32] = {0};
            w.u8(m.has_desc); w.raw(m.has_desc ? m.desc.b : zero, 32);
        }
        const uint64_t total = out.size();
        memcpy(&out[8], &total, 8);
        return 0;
    }

    // Replace the map with a blob's and enter the lost state: the next frames relocalise into it (status 4 while lost, 1 once
    // relocalised, 2 after reloc_max failures).  The whole blob is parsed and checked before anything changes; a refused blob
    // leaves the system as it was.
    int loadMap(const uint8_t* data, size_t bytes) {
        if (reloc_max <= 0 || !BackendHasReloc<Backend>::value) { map_error = "relocalisation is off"; return MAP_STATE; }
        if (!data) { map_error = "null buffer"; return MAP_INVALID; }
        LoadedMap L;
        if (!parseMap(data, bytes, L)) return MAP_INVALID;
        const bool keep_frozen = frozen;   // the localisation-only mode survives a load: the loaded map is frozen
        reset();
        frozen = keep_frozen;
        // fresh containers: bucket counts, and so the iteration order of what is inserted next, depend on the blob alone
        keyframes = std::unordered_map<int, std::shared_ptr<Frame>>();
        mappoints = std::unordered_map<int, MapPoint>();
        cur.kps = std::unordered_map<int, Keypoint>();
        cur.covis.clear(); cur.localmap = std::unordered_set<int>();
        for (auto& f : L.kfs) keyframes.emplace(f->kfid, f);
        for (auto& m : L.mps) mappoints.emplace(m.id, std::move(m));
        n_kf_ids = L.n_kf_ids; n_mp_ids = L.n_mp_ids; n_kf = L.n_kf;
        ready_for_init = true;
        motion.reset();
        p3p_req = true;
        cur.kfid = n_kf_ids > 0 ? n_kf_ids - 1 : 0;   // createKeyframe's; the newest keyframe is never filtered out
        cur.setTwc(L.pose);
        buildRelocTable();
        lost = true;
        lost_frames = 0;
        return 0;
    }

    // System::processCameraPose: returns 1 tracking / 2 reset / 3 not initialised / 4 lost (relocalisation on), or a negative
    // backend error
    int process(const uint8_t* rgba, double timestamp) {
        cur.id++;
        cur.ts = timestamp;
        err = 0;
        if (gyro_on) gyroFrame(timestamp);
        gyro_prev_t = timestamp;
        gyro_have_prev = true;
        bool kf = false;
        if (lost) {
            if constexpr (BackendHasReloc<Backend>::value) {
                const int st = relocaliseFrame(rgba, timestamp, kf);
                if (st != 1) return st;
            }
        } else {
            kf = frontend(rgba, timestamp);
            if (err) return err;
            if (lost) return 4;
        }
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
    int reloc_max = 0;               // frames a lost track may relocalise for (0: off)
    bool frozen = false;             // localisation only (setLocalisationOnly)
    // re-acquisition in that mode: frames it ran on and points it supplied since construction, and the last run's points
    int n_reacq_runs = 0, n_reacq_points = 0, reacq_last_points = 0;
    bool lost = false;
    int lost_frames = 0;             // consecutive frames returned as lost
    RelocTable reloc_table;
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
    // relocalisation: times the track was lost, frames relocalised, and the matches / PnP inliers of the last attempt
    int n_lost = 0, n_relocalised = 0, reloc_last_matches = 0, reloc_last_inliers = 0;
    // keypoints dropped because the fisheye model could not undistort them (tracked, detected or relocalisation queries), since
    // configure or the last lens change
    int n_lens_drops = 0;
    // the gyro mode (setGyro): on, R_ci and bias; dR_c of the last frame integrated (identity when it was not covered); since
    // configure: frames predicted from the gyro, frames that fell back to the motion model, lost frames whose rotation the
    // gyro carried, 2-D priors rotated and 2-D priors kept at the previous position
    bool gyro_on = false;
    double gyro_Rci[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, gyro_bias[3] = {0, 0, 0};
    double gyro_dRc[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    int n_gyro_pred = 0, n_gyro_fallback = 0, n_gyro_carried = 0, n_gyro_rot = 0, n_gyro_kept = 0;

private:
    Backend& B;
    struct GyroSample { double t, w[3]; };
    std::vector<GyroSample> gyro_buf;   // ascending t
    bool gyro_ok = false;               // this frame's interval is covered: gyro_dRc holds its rotation
    bool gyro_have_prev = false;
    double gyro_prev_t = 0;             // the previous frame's time stamp

    // ------------------------------------------------------------------ gyro integration (the rule: setGyro's comment)
    static void gyroIdentity(double* R) { for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.0 : 0.0; }
    static void mul3(const double* A, const double* Bm, double* C) {
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) C[3 * i + j] = (A[3 * i] * Bm[j] + A[3 * i + 1] * Bm[3 + j]) + A[3 * i + 2] * Bm[6 + j];
    }
    static void expSO3(const double* p, double* R) {
        const double th2 = (p[0] * p[0] + p[1] * p[1]) + p[2] * p[2], th = sqrt(th2);
        double a, b;
        if (th < 1e-6) { a = 1.0 - th2 / 6.0; b = 0.5 - th2 / 24.0; }
        else { a = sin(th) / th; b = (1.0 - cos(th)) / th2; }
        // I + a [p]x + b [p]x^2, [p]x^2 = p p^T - th2 I
        R[0] = 1.0 + b * (p[0] * p[0] - th2); R[1] = -a * p[2] + b * (p[0] * p[1]); R[2] = a * p[1] + b * (p[0] * p[2]);
        R[3] = a * p[2] + b * (p[1] * p[0]); R[4] = 1.0 + b * (p[1] * p[1] - th2); R[5] = -a * p[0] + b * (p[1] * p[2]);
        R[6] = -a * p[1] + b * (p[2] * p[0]); R[7] = a * p[0] + b * (p[2] * p[1]); R[8] = 1.0 + b * (p[2] * p[2] - th2);
    }
    size_t gyroUpper(double t) const {   // the first sample after t
        return (size_t)(std::upper_bound(gyro_buf.begin(), gyro_buf.end(), t, [](double v, const GyroSample& s) { return v < s.t; }) - gyro_buf.begin());
    }
    bool gyroAt(double tau, double* w) const {
        const size_t hi = gyroUpper(tau);
        const GyroSample* L = hi > 0 ? &gyro_buf[hi - 1] : nullptr;
        const GyroSample* H = hi < gyro_buf.size() ? &gyro_buf[hi] : nullptr;
        if (L && H && H->t - L->t <= 50.0) {
            const double f = (tau - L->t) / (H->t - L->t);
            for (int c = 0; c < 3; c++) w[c] = L->w[c] + (H->w[c] - L->w[c]) * f;
            return true;
        }
        if (L && tau - L->t <= 50.0) { for (int c = 0; c < 3; c++) w[c] = L->w[c]; return true; }
        if (H && H->t - tau <= 50.0) { for (int c = 0; c < 3; c++) w[c] = H->w[c]; return true; }
        return false;
    }
    bool gyroIntegrate(double A, double Bt, double* dR) const {
        double wa[3], wb[3];
        if (!(Bt >= A) || !gyroAt(A, wa) || !gyroAt(Bt, wb)) return false;
        const size_t i0 = gyroUpper(A);
        size_t i1 = i0;
        while (i1 < gyro_buf.size() && gyro_buf[i1].t < Bt) i1++;
        for (size_t i = i0 + 1; i < i1; i++) if (gyro_buf[i].t - gyro_buf[i - 1].t > 50.0) return false;
        gyroIdentity(dR);
        double ta = A;
        const double* w0 = wa;
        for (size_t i = i0; i <= i1; i++) {
            const double tb = i < i1 ? gyro_buf[i].t : Bt;
            const double* w1 = i < i1 ? gyro_buf[i].w : wb;
            double phi[3], E[9], T[9];
            for (int c = 0; c < 3; c++) phi[c] = ((w0[c] + w1[c]) / 2.0 - gyro_bias[c]) * ((tb - ta) / 1000.0);
            expSO3(phi, E);
            mul3(dR, E, T);
            memcpy(dR, T, sizeof T);
            ta = tb;
            w0 = w1;
        }
        return true;
    }
    // the current frame: dR_c over [previous frame, this frame], the counters of the frames that fall back, and the samples
    // no later frame needs
    void gyroFrame(double t) {
        double dR[9], T[9], Rt[9];
        gyroIdentity(gyro_dRc);
        gyro_ok = gyro_have_prev && gyroIntegrate(gyro_prev_t, t, dR);
        if (gyro_ok) {
            for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Rt[3 * i + j] = gyro_Rci[3 * j + i];
            mul3(gyro_Rci, dR, T);
            mul3(T, Rt, gyro_dRc);
        }
        const bool tracking_path = lost || cur.id > 0;   // (a frame 0 starts the track: nothing to predict)
        if (tracking_path && !gyro_ok) n_gyro_fallback++;
        if (!lost && cur.id > 0 && gyro_ok) n_gyro_pred++;
        const size_t hi = gyroUpper(t);
        if (hi > 1) gyro_buf.erase(gyro_buf.begin(), gyro_buf.begin() + (hi - 1));
    }
    bool gyroUse() const { return gyro_on && gyro_ok; }
    // prev with its rotation advanced by this frame's dR_c and the translation t
    Se3 gyroRotated(const Se3& prev, const double* t) const {
        Se3 D;
        D.setR(gyro_dRc);
        Se3 r = prev * D;
        for (int i = 0; i < 3; i++) r.t[i] = t[i];
        return r;
    }
    MotionModel motion;
    bool p3p_req = false;
    bool reacq_pending = false;      // re-acquire on the next tracked frame (after freezing or a relocalisation)
    int reacq_nocc = 0;              // the frame's occupied cells right after the last re-acquisition
    int pose_failed = 0, err = 0;

    // ------------------------------------------------------------------ map blob parsing: nothing of the system is touched
    struct LoadedMap {
        std::vector<std::shared_ptr<Frame>> kfs;    // ascending id
        std::vector<MapPoint> mps;                  // ascending id
        int n_kf_ids = 0, n_mp_ids = 0, n_kf = 0;
        Se3 pose;
    };
    // every rotation the state machine stores went through Se3::normalize (or exp's sin / cos): unit up to rounding
    static bool unitQuat(const Se3& T) {
        const double n2 = T.q[0] * T.q[0] + T.q[1] * T.q[1] + T.q[2] * T.q[2] + T.q[3] * T.q[3];
        return fabs(n2 - 1.0) <= 1e-9;
    }
    bool parseMap(const uint8_t* data, size_t bytes, LoadedMap& L) {
        auto fail = [this](const char* why) { map_error = why; return false; };
        MapReader r(data, bytes);
        char magic[4];
        uint32_t version = 0, nkf = 0, nmp = 0;
        uint64_t total = 0;
        if (!r.raw(magic, 4) || memcmp(magic, "ALMP", 4) != 0) return fail("bad magic");
        if (!r.u32(version) || version != MAP_VERSION) return fail("unsupported version");
        if (!r.u64(total) || total != (uint64_t)bytes) return fail("byte count differs from the blob's length");
        if (!r.u32(nkf) || !r.u32(nmp)) return fail("truncated header");
        int32_t w = 0, h = 0, lens = 0, cs = 0;
        double K[4], D[4];
        bool ok = r.i32(w) && r.i32(h);
        for (int i = 0; i < 4; i++) ok = ok && r.f64(K[i]);
        ok = ok && r.i32(lens);
        for (int i = 0; i < 4; i++) ok = ok && r.f64(D[i]);
        if (!ok) return fail("truncated or non-finite camera section");
        bool same = w == cam.w && h == cam.h && K[0] == cam.fx && K[1] == cam.fy && K[2] == cam.cx && K[3] == cam.cy && lens == cam.lens;
        for (int i = 0; i < 4; i++) same = same && D[i] == cam.dist[i];
        if (!same) return fail("camera or lens differs from the configured one");
        if (!r.i32(cs)) return fail("truncated grid section");
        if (cs != cell) return fail("grid cell size differs from the preset's");
        if (!r.i32(L.n_kf_ids) || !r.i32(L.n_mp_ids) || !r.i32(L.n_kf)) return fail("truncated counters");
        // below 2^30: the counters keep growing after the load and must not overflow
        auto counter_ok = [](int v) { return v >= 0 && v <= (1 << 30); };
        if (!counter_ok(L.n_kf_ids) || !counter_ok(L.n_mp_ids) || L.n_kf != (int64_t)nkf)
            return fail("counters out of range or inconsistent with the section counts");
        if (!r.se3(L.pose)) return fail("truncated or non-finite pose");
        if (!unitQuat(L.pose)) return fail("pose rotation is not a unit quaternion");
        // keyframes: id, age, Twc [7], keypoints, covis, localmap
        if ((uint64_t)nkf * 76 > r.left()) return fail("keyframe count exceeds the blob");
        int prev = -1;
        for (uint32_t k = 0; k < nkf; k++) {
            int32_t id, age;
            Se3 T;
            if (!r.i32(id) || !r.i32(age) || !r.se3(T)) return fail("truncated or non-finite keyframe");
            if (!unitQuat(T)) return fail("keyframe rotation is not a unit quaternion");
            if (id <= prev || id >= L.n_kf_ids) return fail("keyframe ids not ascending, or not below n_kf_ids");
            if (age < 0 || age > (1 << 30)) return fail("keyframe age out of range");
            prev = id;
            auto f = std::make_shared<Frame>();
            f->init(&cam, cell);
            f->id = -1 - age;   // the frame that saved the map is frame -1 of this session
            f->kfid = id;
            f->setTwc(T);
            uint32_t nkp;
            if (!r.count(nkp, 78)) return fail("keypoint count exceeds the blob");
            int pk = -1;
            for (uint32_t i = 0; i < nkp; i++) {
                Keypoint p;
                ok = r.i32(p.id) && r.f32(p.px) && r.f32(p.py) && r.f32(p.ux) && r.f32(p.uy);
                for (int c = 0; c < 3; c++) ok = ok && r.f64(p.bv[c]);
                ok = ok && r.flag(p.is3d) && r.flag(p.has_desc) && r.raw(p.desc, 32);
                if (!ok) return fail("truncated, non-finite or non-boolean keypoint");
                if (p.id <= pk || p.id >= L.n_mp_ids) return fail("keypoint ids not ascending, or not below n_mp_ids");
                if (!(fabsf(p.px) <= 16777216.f && fabsf(p.py) <= 16777216.f)) return fail("keypoint position out of range");
                pk = p.id;
                f->add(p);
            }
            uint32_t nc;
            if (!r.count(nc, 8)) return fail("covisibility count exceeds the blob");
            int pc = -1;
            for (uint32_t i = 0; i < nc; i++) {
                int32_t kf, cnt;
                if (!r.i32(kf) || !r.i32(cnt)) return fail("truncated covisibility");
                if (kf <= pc) return fail("covisibility ids not ascending");
                pc = kf;
                f->covis.emplace(kf, cnt);
            }
            uint32_t nl;
            if (!r.count(nl, 4)) return fail("local map count exceeds the blob");
            int pl = -1;
            for (uint32_t i = 0; i < nl; i++) {
                int32_t m;
                if (!r.i32(m)) return fail("truncated local map");
                // a local map lists candidates and outlives the map points culled since (buildMatchProblem skips those): an
                // entry must be an id the counter has issued, not necessarily a map point of the blob
                if (m <= pl || m >= L.n_mp_ids) return fail("local map ids not ascending, or not below n_mp_ids");
                pl = m;
                f->localmap.insert(m);
            }
            L.kfs.push_back(f);
        }
        // map points: id, anchor, observed, is3d, invd, p [3], obs, (kfid, desc, descdist), has_desc, desc
        if ((uint64_t)nmp * 83 > r.left()) return fail("map point count exceeds the blob");
        L.mps.reserve(nmp);
        prev = -1;
        for (uint32_t k = 0; k < nmp; k++) {
            MapPoint m;
            ok = r.i32(m.id) && r.i32(m.kfid) && r.flag(m.observed) && r.flag(m.is3d) && r.f64(m.invd);
            for (int c = 0; c < 3; c++) ok = ok && r.f64(m.p[c]);
            if (!ok) return fail("truncated, non-finite or non-boolean map point");
            if (m.id <= prev || m.id >= L.n_mp_ids) return fail("map point ids not ascending, or not below n_mp_ids");
            prev = m.id;
            uint32_t no;
            if (!r.count(no, 4)) return fail("observation count exceeds the blob");
            int po = -1;
            for (uint32_t i = 0; i < no; i++) {
                int32_t o;
                if (!r.i32(o)) return fail("truncated observations");
                if (o <= po) return fail("observations not ascending");
                po = o;
                m.obs.insert(m.obs.end(), o);
            }
            uint32_t nd;
            if (!r.count(nd, 40)) return fail("descriptor count exceeds the blob");
            int pd = -1;
            for (uint32_t i = 0; i < nd; i++) {
                int32_t kf;
                Desc d;
                float dist;
                if (!r.i32(kf) || !r.raw(d.b, 32) || !r.f32(dist)) return fail("truncated or non-finite keyframe descriptor");
                if (kf <= pd) return fail("keyframe descriptors not ascending");
                pd = kf;
                m.kfdesc.emplace(kf, d);
                m.descdist.emplace(kf, dist);
            }
            if (!r.flag(m.has_desc) || !r.raw(m.desc.b, 32)) return fail("truncated map point descriptor");
            if (!m.has_desc)
                for (int i = 0; i < 32; i++) if (m.desc.b[i]) return fail("a descriptor on a map point without one");
            L.mps.push_back(std::move(m));
        }
        if (r.left() != 0) return fail("bytes after the last map point");
        // Every reference names an issued id (0 <= id < its counter): a record of the blob, or a keyframe or map point removed
        // since.  A live map holds the latter once keyframes leave it (filterKeyframes, the 30-keyframe window): removeObs
        // leaves the anchor of a point whose last observation went, localBA erases covisibility entries lazily, a culled
        // point stays in local maps.  The state machine looks every such id up with find() and skips a missing record, so
        // keeping them makes the loaded map the saved one.
        auto kf_ok = [&](int id) { return id >= 0 && id < L.n_kf_ids; };
        auto mp_ok = [&](int id) { return id >= 0 && id < L.n_mp_ids; };
        for (auto& f : L.kfs) {
            for (auto& kv : f->kps) if (kv.second.is3d && !mp_ok(kv.first)) return fail("a 3-D keypoint names no issued map point");
            for (auto& kv : f->covis) if (!kf_ok(kv.first)) return fail("a covisibility entry names no issued keyframe");
        }
        for (auto& m : L.mps) {
            if (!kf_ok(m.kfid)) return fail("a map point's anchor names no issued keyframe");
            for (int o : m.obs) if (!kf_ok(o)) return fail("an observation names no issued keyframe");
            for (auto& kv : m.kfdesc) if (!kf_ok(kv.first)) return fail("a keyframe descriptor names no issued keyframe");
        }
        return true;
    }

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
                    if (lensDrop(fresh[2 * i], fresh[2 * i + 1], un ? &fresh_un[2 * (size_t)i] : nullptr)) continue;
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
        m.fisheye = cam.lens == Camera::FISHEYE;
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
        const Se3 tracked = cur.Twc;
        motion.apply(Twc, timestamp);
        if (gyroUse() && ready_for_init) Twc = gyroRotated(tracked, Twc.t);   // the gyro's rotation, the motion model's translation
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
        if (!ok && reloc_max > 0 && BackendHasReloc<Backend>::value) {
            if (gyroUse()) { enterLost(gyroRotated(tracked, tracked.t)); n_gyro_carried++; }
            else enterLost(tracked);
            return false;
        }
        if (!ok) {
            pose_failed++;
            if (pose_failed > 3) { reset_requested = true; return false; }
        }
        motion.update(cur.Twc, timestamp);
        if (frozen) { reacquireFrame(); return false; }
        return checkNewKeyframeRequired();
    }

    // ------------------------------------------------------------------ relocalisation (not in the reference)
    // the first failed pose after the initialisation: the frame is emptied, the last tracked pose kept, the map frozen and
    // its descriptor table built for the lost frames that follow
    void enterLost(const Se3& tracked) {
        resetFrame();
        cur.setTwc(tracked);
        lost = true;
        lost_frames = 1;
        n_lost++;
        if (!frozen) buildRelocTable();   // a frozen map keeps its table (and its device copy)
    }
    void buildRelocTable() {
        RelocTable& t = reloc_table;
        t.clear();
        std::vector<int> ids;
        for (auto& kv : mappoints)
            if (kv.second.is3d && !kv.second.kfdesc.empty()) ids.push_back(kv.first);
        std::sort(ids.begin(), ids.end());
        t.desc_start.push_back(0);
        for (int id : ids) {
            const MapPoint& mp = mappoints.at(id);
            std::vector<int> kfs;
            for (auto& kv : mp.kfdesc) kfs.push_back(kv.first);
            std::sort(kfs.begin(), kfs.end());
            t.mp_id.push_back(id);
            t.wpt.insert(t.wpt.end(), mp.p, mp.p + 3);
            for (int k : kfs) { const Desc& d = mp.kfdesc.at(k); t.desc.insert(t.desc.end(), d.b, d.b + 32); }
            t.desc_start.push_back((int32_t)(t.desc.size() / 32));
        }
    }

    // one lost frame: pyramid (KLT's previous level once tracking resumes), grid detector over the whole frame, ORB on the raw
    // image, then Backend::relocalise against the frozen map.  Returns 1 relocalised (kf: the reference's keyframe decision
    // for this frame), 4 still lost, 2 gave up (reset, as the reference), or a negative backend error.
    int relocaliseFrame(const uint8_t* rgba, double timestamp, bool& kf) {
        kf = false;
        if ((err = B.pyramid(rgba)) < 0) return err;
        err = 0;
        std::vector<float> fresh;
        if ((err = B.detect_lost(fresh)) < 0) return err;
        err = 0;
        const float* un = backendUnpx();
        std::vector<float> fresh_un;
        if (un) fresh_un.assign(un, un + fresh.size());
        const int nn = (int)fresh.size() / 2;
        std::vector<uint8_t> desc(32 * (size_t)nn + 32), kept(nn + 1);
        if (nn > 0 && (err = B.describe(fresh.data(), nn, desc.data(), kept.data())) < 0) return err;
        err = 0;
        std::vector<Keypoint> qk;                    // the queries: points ORB kept, in detector order
        std::vector<uint8_t> qdesc;
        std::vector<double> qbv, quv;
        for (int i = 0; i < nn; i++) {
            if (!kept[i]) continue;
            if (lensDrop(fresh[2 * i], fresh[2 * i + 1], un ? &fresh_un[2 * (size_t)i] : nullptr)) continue;
            Keypoint k;
            cur.compute(fresh[2 * i], fresh[2 * i + 1], k, un ? &fresh_un[2 * (size_t)i] : nullptr);
            memcpy(k.desc, &desc[32 * (size_t)i], 32);
            k.has_desc = true;
            qdesc.insert(qdesc.end(), k.desc, k.desc + 32);
            qbv.insert(qbv.end(), k.bv, k.bv + 3);
            quv.push_back(k.ux); quv.push_back(k.uy);
            qk.push_back(k);
        }
        const double K4[4] = {(double)(float)cam.fx, (double)(float)cam.fy, (double)(float)cam.cx, (double)(float)cam.cy};
        RelocResult R;
        if ((err = B.relocalise(reloc_table, qdesc.data(), qbv.data(), quv.data(), (int)qk.size(), K4, (float)cam.fx, (float)cam.fy, R)) < 0)
            return err;
        err = 0;
        // the decisions: >= 30 matches, a RANSAC model, PnP with >= 30 inliers that flags at most half of its input
        const double tt[3] = {R.T12[3], R.T12[7], R.T12[11]};
        bool ok = R.n_match >= 30 && R.ok1 && finite3(tt) && R.ok2 && finite3(R.pose7);
        std::vector<int> surv;                       // RANSAC inliers: indices into the matches
        for (int i = 0; ok && i < R.n_match; i++) if (!R.o1[i]) surv.push_back(i);
        int nout2 = 0;
        for (size_t i = 0; ok && i < surv.size(); i++) nout2 += R.o2[i] != 0;
        const int n2 = (int)surv.size();
        ok = ok && n2 - nout2 >= 30 && nout2 <= 0.5 * n2;
        reloc_last_matches = R.n_match;
        reloc_last_inliers = ok ? n2 - nout2 : 0;
        if (!ok) {
            if (frozen) { if (lost_frames < INT32_MAX) lost_frames++; gyroCarry(); return 4; }   // a frozen map is never reset
            if (++lost_frames > reloc_max) { reset(); return 2; }
            gyroCarry();
            return 4;
        }
        // the PnP inliers become the frame's keypoints, observing their map points
        for (int s2 = 0; s2 < n2; s2++) {
            if (R.o2[s2]) continue;
            const int m = surv[s2];
            Keypoint k = qk[R.mq[m]];
            k.id = reloc_table.mp_id[R.mg[m]];
            k.is3d = true;
            auto mp = mappoints.find(k.id);
            if (mp == mappoints.end()) continue;
            mp->second.observed = true;
            cur.add(k);
        }
        cur.setTwc(Se3::from7(R.pose7));
        motion.reset();                              // the gap makes the last velocity meaningless
        motion.update(cur.Twc, timestamp);
        lost = false;
        lost_frames = 0;
        n_relocalised++;
        if (frozen) { reacq_pending = true; return 1; }   // no keyframe; the next tracked frame re-acquires
        kf = checkNewKeyframeRequired();
        return 1;
    }

    // a lost frame with the gyro: the reported pose turns with the camera, its translation held
    void gyroCarry() {
        if (!gyroUse()) return;
        cur.setTwc(gyroRotated(cur.Twc, cur.Twc.t));
        n_gyro_carried++;
    }

    // ------------------------------------------------------------------ re-acquisition (localisation only)
    // A tracked frame of a frozen map gets map points back without a keyframe.  It runs when (a) it is the first tracked frame
    // after freezing or after a relocalisation, (b) the frame's occupied cells fell below 0.85 x their count right after the
    // last re-acquisition, or (c) the frame has fewer than 30 3-D keypoints.  Then: the grid detector in the cells the
    // frame's keypoints leave empty (the tracker's adaptive quality, as at a keyframe), ORB on the raw image, the lens drops of
    // createKeyframe, and Backend::reacquire against the frozen table with the frame's map points masked out (radius 2 px, 4
    // px below 30 3-D keypoints, as matchToMap's maxProjPxDist).  Each matched detection joins the frame as a 3-D keypoint of
    // its map point, in detector order, while the frame holds fewer than twice the grid's cell count (the bound the
    // keyframe's pruning keeps otherwise); the rest are discarded.  This frame's pose is not re-solved: the points enter PnP
    // on the next frame.
    void reacquireFrame() {
        if (!(reacq_pending || cur.nocc < 0.85 * reacq_nocc || cur.n3d < 30)) return;
        reacq_pending = false;
        n_reacq_runs++;
        reacq_last_points = 0;
        if (max_kps - cur.nocc > 0) {
            const std::vector<Keypoint> kps = cur.all();
            std::vector<float> pts(2 * kps.size() + 2);
            for (size_t i = 0; i < kps.size(); i++) { pts[2 * i] = kps[i].px; pts[2 * i + 1] = kps[i].py; }
            std::vector<float> fresh;
            if ((err = B.detect(pts.data(), (int)kps.size(), fresh)) < 0) return;
            err = 0;
            const float* un = backendUnpx();
            std::vector<float> fresh_un;
            if (un) fresh_un.assign(un, un + fresh.size());
            const int nn = (int)fresh.size() / 2;
            if (nn > 0) {
                std::vector<uint8_t> desc(32 * (size_t)nn), kept(nn);
                if ((err = B.describe(fresh.data(), nn, desc.data(), kept.data())) < 0) return;
                err = 0;
                for (int i = 0; i < nn; i++)
                    if (lensDrop(fresh[2 * i], fresh[2 * i + 1], un ? &fresh_un[2 * (size_t)i] : nullptr)) kept[i] = 0;
                const std::vector<int32_t>& ids = reloc_table.mp_id;   // ascending
                std::vector<uint8_t> skip(ids.size() + 1, 0);
                for (auto& kv : cur.kps) {
                    auto it = std::lower_bound(ids.begin(), ids.end(), kv.first);
                    if (it != ids.end() && *it == kv.first) skip[it - ids.begin()] = 1;
                }
                double T7[7];
                cur.Twc.to7(T7);
                std::vector<int32_t> row(nn, -1), dist(nn, -1);
                if constexpr (BackendHasReacquire<Backend>::value)   // (the mode is refused without it)
                    if ((err = B.reacquire(reloc_table, skip.data(), T7, fresh.data(), desc.data(), kept.data(), nn, cur.n3d < 30 ? 4.0f : 2.0f,
                                           row.data(), dist.data())) < 0)
                        return;
                err = 0;
                for (int i = 0; i < nn && cur.n < 2 * max_kps; i++) {
                    if (row[i] < 0 || row[i] >= (int)ids.size()) continue;
                    auto mp = mappoints.find(ids[row[i]]);
                    if (mp == mappoints.end()) continue;
                    Keypoint k;
                    cur.compute(fresh[2 * i], fresh[2 * i + 1], k, un ? &fresh_un[2 * (size_t)i] : nullptr);
                    k.id = ids[row[i]];
                    k.is3d = true;
                    k.has_desc = true;
                    memcpy(k.desc, &desc[32 * (size_t)i], 32);
                    mp->second.observed = true;
                    cur.add(k);
                    reacq_last_points++;
                }
                n_reacq_points += reacq_last_points;
            }
        }
        reacq_nocc = cur.nocc;
    }

    void kltTracking() {   // kltTrackingFromMotionPrior (kltUsePrior_ = true)
        std::vector<int> ids3, ids;
        std::vector<float> kps3, pri3, kps, pri;
        // gyro mode: per second-pass point its bearing and whether its prior is the previous position (then rotated)
        const bool rot = gyroUse();
        std::vector<double> bvs;
        std::vector<uint8_t> rflag;
        auto second = [&](const Keypoint& k, bool prev_prior) {
            if (!rot) return;
            bvs.insert(bvs.end(), k.bv, k.bv + 3);
            rflag.push_back(prev_prior ? 1 : 0);
        };
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
            second(k, true);
        }
        if (!ids3.empty()) {
            const size_t n3 = ids3.size();
            std::vector<uint8_t> good(n3);
            if ((err = B.klt(kps3.data(), pri3.data(), (int)n3, 1, good.data())) < 0) return;
            err = 0;
            const float* un = backendUnpx();
            size_t ngood = 0;
            for (size_t i = 0; i < n3; i++) {
                if (good[i] && lensDrop(pri3[2 * i], pri3[2 * i + 1], un ? un + 2 * i : nullptr)) { removeObsFromCurr(ids3[i]); continue; }
                if (good[i]) { cur.update(ids3[i], pri3[2 * i], pri3[2 * i + 1], un ? un + 2 * i : nullptr); ngood++; }
                else {
                    ids.push_back(ids3[i]); kps.push_back(kps3[2 * i]); kps.push_back(kps3[2 * i + 1]); pri.push_back(pri3[2 * i]); pri.push_back(pri3[2 * i + 1]);
                    if (rot) second(*cur.find(ids3[i]), false);   // (not updated: still the previous frame's keypoint)
                }
            }
            if (ngood < 0.33 * n3) { p3p_req = true; pri = kps; rflag.assign(rflag.size(), 1); }   // the rotation is trusted still
        }
        if (!ids.empty()) {
            const size_t n = ids.size();
            std::vector<uint8_t> good(n);
            if (rot) {
                std::vector<uint8_t> rotated(n);
                if constexpr (BackendHasRotatedKlt<Backend>::value)   // (the mode is refused without it)
                    if ((err = B.klt_rotated(kps.data(), pri.data(), (int)n, 3, good.data(), bvs.data(), rflag.data(), gyro_dRc, rotated.data())) < 0)
                        return;
                for (size_t i = 0; i < n; i++)
                    if (rflag[i]) { if (rotated[i]) n_gyro_rot++; else n_gyro_kept++; }
            } else if ((err = B.klt(kps.data(), pri.data(), (int)n, 3, good.data())) < 0) {   // State::kltPyramidLevels_
                return;
            }
            err = 0;
            const float* un = backendUnpx();
            for (size_t i = 0; i < n; i++) {
                if (good[i] && !lensDrop(pri[2 * i], pri[2 * i + 1], un ? un + 2 * i : nullptr)) cur.update(ids[i], pri[2 * i], pri[2 * i + 1], un ? un + 2 * i : nullptr);
                else removeObsFromCurr(ids[i]);
            }
        }
    }

    // A keypoint at (x, y) whose fisheye undistortion fails is dropped, the same way whichever side undistorted it (un: the
    // backend's result, else Camera::undistort): a tracked point is removed as a KLT failure, a detected point or a
    // relocalisation query is never added.  Counted in n_lens_drops.  Never true for the pinhole or radial-tangential lens.
    bool lensDrop(float x, float y, const float* un) {
        if (cam.lens != Camera::FISHEYE) return false;
        float ux, uy;
        if (un) { ux = un[0]; uy = un[1]; }
        else cam.undistort(x, y, ux, uy);
        if (!Camera::lensFailure(ux, uy)) return false;
        n_lens_drops++;
        return true;
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
