// oracle/ref_clahe.cpp -- TEST INFRASTRUCTURE ONLY (never on the product path).
//
// The reference's CLAHE behind a C ABI, built by oracle/build_ref_clahe.sh into oracle/_ref/libalva_ref_clahe.so beside
// libalva_ref.so (and only where that one can be built):
//   ref_clahe             cv::createCLAHE(clip_limit, Size(tiles_x, tiles_y))->apply on one frame, the reference's own OpenCV
//                         4.5.5 sources built by the same recipe (oracle/build_ref.sh), linked statically;
//   ref_system_set_clahe  the three State fields of the CLAHE pre-processing (state.hpp:43-45) of a System created by
//                         libalva_ref.so's ref_system_create, and its VisualFrontend's CLAHE object set to what the constructor
//                         would create from them (visual_frontend.cpp:16-18).  The reference has no setter; its preset table
//                         (state.hpp:9-17) is what changes them.  The object is re-parametrised through its own virtual
//                         setters, so all CLAHE code that runs in the System is the reference library's own.
// Private members are reached as in ref_system.cpp: every std / third-party header first, then `private` redefined for the
// reference's own headers only.
#include <opencv2/core.hpp>
#include <opencv2/core/utility.hpp>
#include <opencv2/imgproc.hpp>
#include <opencv2/highgui.hpp>
#include <opencv2/features2d.hpp>
#include <opencv2/video/tracking.hpp>
#include <opencv2/calib3d.hpp>
#include <Eigen/Core>
#include <Eigen/Geometry>
#include <Eigen/LU>
#include <opencv2/core/eigen.hpp>
#include <sophus/se3.hpp>
#include <ceres/ceres.h>
#include <chrono>
#include <iostream>
#include <memory>
#include <map>
#include <set>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include <string>
#include <cstring>
#define private public
#define protected public
#include "system.hpp"
#undef private
#undef protected

extern "C" {

// VisualFrontend::preprocessImage's clahe_->apply(image, currImage_) (visual_frontend.cpp:678-681) on one frame
void ref_clahe(const uint8_t* src, int w, int h, double clip_limit, int tiles_x, int tiles_y, uint8_t* dst) {
    cv::Mat s(h, w, CV_8UC1, (void*)src), d;
    cv::createCLAHE(clip_limit, cv::Size(tiles_x, tiles_y))->apply(s, d);
    memcpy(dst, d.data, (size_t)w * h);
}

void ref_system_set_clahe(void* h, int enabled, double clip_limit, int tile_size) {
    System* s = (System*)h;
    s->state_->claheEnabled_ = enabled != 0;
    s->state_->claheContrastLimit_ = (float)clip_limit;   // a float in State
    s->state_->claheTileSize_ = tile_size;
    cv::Size gridSize(s->state_->imgWidth_ / s->state_->claheTileSize_, s->state_->imgHeight_ / s->state_->claheTileSize_);
    s->visualFrontend_->clahe_->setClipLimit(s->state_->claheContrastLimit_);
    s->visualFrontend_->clahe_->setTilesGridSize(gridSize);
}

}  // extern "C"
