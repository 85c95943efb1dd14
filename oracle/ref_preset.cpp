// oracle/ref_preset.cpp -- TEST INFRASTRUCTURE ONLY (never on the product path).
//
// The reference's preset table (state.hpp:9-17) applied to a System created by libalva_ref.so's ref_system_create, built by
// oracle/build_ref_preset.sh into oracle/_ref/libalva_ref_preset.so (linked against libalva_ref.so, so every constructor and
// method that runs is the reference library's own):
//   ref_system_set_preset  rebuilds, IN PLACE, the two objects that hold the grid cell size, through the reference's own
//                          constructors -- State(w, h, cell) (state.cpp:3-12: frameMaxCellSize_, frameMaxNumKeypoints_) with the
//                          preset's mapKeyframeFilteringRatio_ / p3pEnabled_ and the pins ref_system_create sets, and
//                          Frame(calibration, cell) (frame.cpp:9-20: cellSize_, numCellsW_ / H_, the empty grid) -- then runs
//                          System::reset().  In place, because State and the current Frame are shared: MapManager, Mapper,
//                          VisualFrontend and Optimizer hold the same shared_ptr<State>, MapManager / Mapper / VisualFrontend the
//                          same shared_ptr<Frame>, and they must all see the new values.
//   CLAHE, the table's fourth field, goes through ref_system_set_clahe (oracle/ref_clahe.cpp) with State's clip 3 / tile 50.
// No other reference object caches the cell size (checked in the sources): FeatureExtractor::detectFeaturePoints takes it per
// call from state_->frameMaxCellSize_ (map_manager.cpp:213); MapManager (map_manager.cpp:30, 206), Mapper (mapper.cpp:75, 136,
// 296) and VisualFrontend (visual_frontend.cpp:272, 571-589) read frameMaxNumKeypoints_, the filtering ratio and p3pEnabled_
// from the shared State on every use; keyframes copy the current Frame's grid when they are created (frame.cpp:22-30), and
// System::reset() clears them; VisualFrontend's CLAHE object depends on the CLAHE tile size only.
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

// cell: frameMaxCellSize_; filter_ratio: mapKeyframeFilteringRatio_; p3p: p3pEnabled_
void ref_system_set_preset(void* h, int cell, double filter_ratio, int p3p) {
    System* s = (System*)h;
    const double w = s->state_->imgWidth_, hh = s->state_->imgHeight_;
    *s->state_ = State(w, hh, cell);
    s->state_->debug_ = false;                        // as System::configure (system.cpp:16)
    s->state_->multiViewRandomEnabled_ = false;       // ref_system_create's determinism pin
    s->state_->mapKeyframeFilteringRatio_ = (float)filter_ratio;
    s->state_->p3pEnabled_ = p3p != 0;
    *s->currFrame_ = Frame(s->cameraCalibration_, s->state_->frameMaxCellSize_);
    s->reset();
}

// State::frameMaxCellSize_, frameMaxNumKeypoints_, the current Frame's cellSize_ / numCellsW_ / numCellsH_: what the preset set
void ref_system_grid(void* h, int32_t* out5) {
    System* s = (System*)h;
    out5[0] = s->state_->frameMaxCellSize_; out5[1] = s->state_->frameMaxNumKeypoints_;
    out5[2] = (int)s->currFrame_->cellSize_; out5[3] = (int)s->currFrame_->numCellsW_; out5[4] = (int)s->currFrame_->numCellsH_;
}

// VisualFrontend::p3pReq_: set when PnP from the motion prior failed, so that the next frame runs P3P (visual_frontend.cpp:384-389)
int ref_system_p3p_req(void* h) { return ((System*)h)->visualFrontend_->p3pReq_ ? 1 : 0; }

}  // extern "C"
