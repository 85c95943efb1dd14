// alva_system.hpp -- the reference's `class System` (src/slam/src/system.hpp:19-56) as a header-only shim over the C ABI of
// libalva_b200.so, so that the reference's own binding (src/slam/src/embind.cpp:9-18) and its JavaScript driver
// (src/system.js) compile against it unchanged:
//
//     #include "alva_system.hpp"      // instead of "./system.hpp"
//     class_<System>("System").constructor().function("configure", &System::configure) ...   (embind.cpp as it is)
//
// Method names, argument order and return conventions are the reference's (system.cpp:13-175): findCameraPose returns
// 1 tracking / 2 the tracker was reset during this call / 3 not initialised yet; the pose buffer receives 16 floats laid out as
// Utils::toPoseArray does (R rows in [0..2], [4..6], [8..10], t in [12..14], [15] = 1); buffers are caller-owned and the image
// is only read.  The `int` overloads are the reference's wasm32 signatures (embind passes heap offsets as ints, system.cpp:59-61,
// 108-109, 132, 141): usable wherever a pointer fits an int (wasm32, or buffers mapped below 2 GiB); native 64-bit hosts call the
// pointer overloads.  Deviations, both deliberate: getFramePoints writes at most 2048 pairs and returns the true count (the
// reference overruns its 4096-int buffer, system.cpp:143-153); configure with non-zero lens distortion is rejected (lastError()):
// configure with zeros, then call alva_system_set_distortion(handle, k1, k2, p1, p2) (alva_b200.h).
#pragma once
#include <cstdint>
#include <vector>
#include "alva_b200.h"

class System {
public:
    System() : h_(alva_system_create(/*device=*/0)) {}
    ~System() { alva_system_destroy(h_); }
    System(const System&) = delete;
    System& operator=(const System&) = delete;

    void configure(int imageWidth, int imageHeight, double fx, double fy, double cx, double cy, double k1, double k2, double p1,
                   double p2) {
        status_ = alva_system_configure(h_, imageWidth, imageHeight, fx, fy, cx, cy, k1, k2, p1, p2);
    }
    void reset() { alva_system_reset(h_); }
    // not in the reference's class: its FAST / AVERAGE / ACCURATE presets (ALVA_PRESET_*, alva_b200.h); 0 or an ALVA_E_* code
    int setPreset(int preset) { return alva_system_set_preset(h_, preset); }
    // not in the reference's class: relocalise for up to maxLostFrames frames after a tracking loss instead of resetting
    // (findCameraPose then returns ALVA_STATUS_LOST while lost; 0 = the reference's reset); 0 or an ALVA_E_* code
    int setRelocalisation(int maxLostFrames) { return alva_system_set_relocalisation(h_, maxLostFrames); }
    // not in the reference's class: OpenCV's equidistant fisheye lens (k1..k4 on theta; enabled = 0: the pinhole), for
    // wide-angle cameras; resets the tracker and the map; 0 or an ALVA_E_* code
    int setFisheye(int enabled, double k1, double k2, double k3, double k4) { return alva_system_set_fisheye(h_, enabled, k1, k2, k3, k4); }
    int setDistortionCoeffs(const double* coeffs, int n) { return alva_system_set_distortion_coeffs(h_, coeffs, n); }
    // not in the reference's class: the map as bytes (alva_system_save_map / alva_system_load_map, alva_b200.h).  saveMap
    // replaces `out` with the blob; loadMap needs setRelocalisation > 0 and enters the lost state.  0 or an ALVA_E_* code
    // (one serialisation when `out`'s capacity already holds the map, e.g. when it is reused from call to call)
    int saveMap(std::vector<uint8_t>& out) {
        size_t n = 0;
        out.resize(out.capacity() > 65536 ? out.capacity() : 65536);
        int e = alva_system_save_map(h_, out.data(), out.size(), &n);
        if (e == ALVA_E_CAPACITY) {
            out.resize(n);
            e = alva_system_save_map(h_, out.data(), out.size(), &n);
        }
        out.resize(e == 0 ? n : 0);
        return e;
    }
    int loadMap(const std::vector<uint8_t>& blob) { return alva_system_load_map(h_, blob.data(), blob.size()); }
    // not in the reference's class: track against the map without changing it (alva_system_set_localisation_only); needs
    // setRelocalisation > 0 and a map (loaded or initialised); loadMap keeps it on.  0 or an ALVA_E_* code
    int setLocalisationOnly(bool enabled) { return alva_system_set_localisation_only(h_, enabled ? 1 : 0); }
    // not in the reference's class: gyro-aided tracking (alva_system_set_gyro); R_ci9 (row-major IMU -> camera axes, NULL:
    // identity; diag(1, -1, -1) for devicemotion and a rear camera) and bias3 (rad/s, NULL: zero).  0 or an ALVA_E_* code
    int setGyro(int enabled, const double* R_ci9 = nullptr, const double* bias3 = nullptr) { return alva_system_set_gyro(h_, enabled, R_ci9, bias3); }

    // ---- the reference's wasm32 signatures
    int findCameraPose(int imageRGBADataPtr, int posePtr) { return findCameraPose(ptr<const uint8_t>(imageRGBADataPtr), ptr<float>(posePtr)); }
    int findCameraPoseWithIMU(int imageRGBADataPtr, int imuDataPtr, int posePtr) {
        return findCameraPoseWithIMU(ptr<const uint8_t>(imageRGBADataPtr), ptr<const double>(imuDataPtr), ptr<float>(posePtr));
    }
    int findPlane(int locationPtr, int numIterations) { return findPlane(ptr<float>(locationPtr), numIterations); }
    int getFramePoints(int pointsPtr) { return getFramePoints(ptr<int32_t>(pointsPtr)); }

    // ---- the same operations with real pointers (native hosts)
    int findCameraPose(const uint8_t* imageRGBA, float* pose16) { return alva_system_find_camera_pose(h_, imageRGBA, pose16); }
    int findCameraPose(const uint8_t* imageRGBA, double timestampMs, float* pose16) {   // caller-supplied time stamp
        return alva_system_find_camera_pose_ts(h_, imageRGBA, timestampMs, pose16);
    }
    int findCameraPoseWithIMU(const uint8_t* imageRGBA, const double* imuData, float* pose16) {
        return alva_system_find_camera_pose_imu(h_, imageRGBA, imuData, pose16);
    }
    // not in the reference's class: findCameraPose with n gyro samples [n][7] = {t_ms, gx, gy, gz, ax, ay, az} (the JS shim's
    // IMU buffer layout) for setGyro's mode; with the mode off it equals findCameraPose(imageRGBA, timestampMs, pose16)
    int findCameraPoseWithGyro(const uint8_t* imageRGBA, double timestampMs, const double* samples, int n, float* pose16) {
        return alva_system_find_camera_pose_gyro(h_, imageRGBA, timestampMs, samples, n, pose16);
    }
    int findPlane(float* location16, int numIterations) { return alva_system_find_plane(h_, location16, numIterations); }
    int getFramePoints(int32_t* pointsXY) { return alva_system_get_frame_points(h_, pointsXY, 2048); }

    int configureStatus() const { return status_; }            // 0, or the ALVA_E_* code configure() could not return
    const char* lastError() const { return alva_last_error(); }

private:
    template <class T> static T* ptr(int p) { return reinterpret_cast<T*>(static_cast<uintptr_t>(static_cast<uint32_t>(p))); }
    alva_system* h_;
    int status_ = 0;
};
