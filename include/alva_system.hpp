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
    int findPlane(float* location16, int numIterations) { return alva_system_find_plane(h_, location16, numIterations); }
    int getFramePoints(int32_t* pointsXY) { return alva_system_get_frame_points(h_, pointsXY, 2048); }

    int configureStatus() const { return status_; }            // 0, or the ALVA_E_* code configure() could not return
    const char* lastError() const { return alva_last_error(); }

private:
    template <class T> static T* ptr(int p) { return reinterpret_cast<T*>(static_cast<uintptr_t>(static_cast<uint32_t>(p))); }
    alva_system* h_;
    int status_ = 0;
};
