/* include/alva_b200.h -- C ABI of libalva_b200.so: the H100-native per-frame visual-SLAM hot path
 * behind AlvaAR's `System` API.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference exposes its C++ `System` class to JavaScript
 * through embind (reference: src/slam/src/embind.cpp:9-18, src/slam/src/system.hpp:19-56); pointers
 * cross as 32-bit ints because the host there is wasm32.  This header is what a native host binds
 * instead: opaque handles, real pointers, explicit sizes, no C++/torch types.
 *
 *   alva_system_*   : one-to-one with System::{configure,reset,findCameraPose,findCameraPoseWithIMU,
 *                     findPlane,getFramePoints}  (system.hpp:28-38)
 *   alva_k_*        : kernel-level entry points for each stage of the hot path (device pointers),
 *                     the units the parity tests address
 *   alva_h_*        : the same stages on HOST buffers (H2D + kernel + D2H inside the call) -- the
 *                     "e2e" leg of bench.py and what a non-CUDA host would call
 *
 * All functions return 0 on success or a negative ALVA_E_* code; alva_last_error() gives the text.
 * A context is bound to one CUDA device and one stream; it is not thread-safe (the reference System
 * is single-threaded and non-re-entrant too, SURVEY 8b "Threading").
 */
#ifndef ALVA_B200_H
#define ALVA_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALVA_OK            0
#define ALVA_E_INVALID    -1   /* bad argument */
#define ALVA_E_CUDA       -2   /* CUDA runtime/driver error (see alva_last_error) */
#define ALVA_E_CAPACITY   -3   /* an output list overflowed its capacity */
#define ALVA_E_STATE      -4   /* call out of order (e.g. not configured) */

/* Packed corner key: (y << 20) | (x << 8) | score.  Sorting keys ascending == cv::FAST's row-major
 * output order (reference: opencv/modules/features2d/src/fast.cpp:283-288). */
#define ALVA_KEY_X(k)     (((k) >> 8) & 0xFFFu)
#define ALVA_KEY_Y(k)     (((k) >> 20) & 0xFFFu)
#define ALVA_KEY_SCORE(k) ((k) & 0xFFu)
#define ALVA_MAX_DIM      4095

#define ALVA_ORB_FMA        1   /* blur with fused multiply-add (native AVX2 OpenCV dispatch); default = unfused
                                   (SSE baseline == the shipped WASM simd128 arithmetic) */
#define ALVA_ORB_HARRIS     4   /* alva_pipeline only: select the features as ORB::detectAndCompute does (HARRIS_SCORE,
                                   orb.cpp:849-925): retainBest(2n) on the FAST score, then retainBest(n) on the Harris
                                   response -- instead of retainBest(n) on the FAST score alone */
#define ALVA_ORB_IC_ANGLE   2   /* steer rBRIEF by the intensity-centroid angle (ORB::detect mode) instead of
                                   AlvaAR's constant -1 degree (feature_extractor.cpp:179-182) */

typedef struct alva_ctx alva_ctx;
typedef struct alva_system alva_system;

int         alva_version(void);
const char* alva_last_error(void);

/* ---- context ------------------------------------------------------------------------------- */
/* device: CUDA ordinal.  stream: a cudaStream_t to run on; NULL = the context creates its own non-blocking stream
 * (to run on the legacy default stream pass cudaStreamLegacy, i.e. (void*)0x1). */
alva_ctx* alva_ctx_create(int device, void* stream);
void      alva_ctx_destroy(alva_ctx* ctx);
int       alva_ctx_sync(alva_ctx* ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
long long alva_ctx_launches(const alva_ctx* ctx);

/* ---- kernel-level stages (DEVICE pointers; batches of nframes tightly packed frames) --------- */

/* cv::cvtColor(RGBA2GRAY)  -- reference call site src/slam/src/system.cpp:111-112 */
int alva_k_gray(alva_ctx*, const uint8_t* rgba, uint8_t* gray, int w, int h, int nframes);

/* cv::pyrDown, one level   -- level step of cv::buildOpticalFlowPyramid,
 * reference call site src/slam/src/visual_frontend.cpp:696 (opencv video/src/lkpyramid.cpp:726-822) */
int alva_k_pyrdown(alva_ctx*, const uint8_t* src, uint8_t* dst, int w, int h, int nframes);

/* Scharr derivative image of one pyramid level, as cv::buildOpticalFlowPyramid(withDerivatives = true) builds it for the KLT
 * tracker (visual_frontend.cpp:696 -> video/src/lkpyramid.cpp:57-150, 800-808): deriv [nframes][h][w][2] int16 = (dx, dy),
 * dx = [3 10 3]^T x [-1 0 1], dy = [-1 0 1]^T x [3 10 3], reflect-101 neighbours.  (The reference then pads the derivative
 * image with a CONSTANT 0 border of the window size; that padding is a view concern of its Mat, not stored here.) */
int alva_k_scharr(alva_ctx*, const uint8_t* gray, int16_t* deriv, int w, int h, int nframes);

/* CLAHE: cv::createCLAHE(clip_limit, Size(tiles_x, tiles_y))->apply(src, dst), 8-bit, bit-exact (the reference's optional
 * pre-processing before the KLT pyramid, visual_frontend.cpp:672-698 -> opencv imgproc/src/clahe.cpp:142-313, 349-429).
 * src / dst: [nframes][h][w] u8 device buffers; dst may equal src.  clip_limit 0 = no clipping.  ALVA_E_INVALID for
 * tiles < 1, tiles > the image size on either axis, or a negative / NaN clip_limit. */
int alva_k_clahe(alva_ctx*, const uint8_t* src, uint8_t* dst, int w, int h, int nframes, double clip_limit, int tiles_x, int tiles_y);

/* Lens distortion: OpenCV's radial-tangential model with D4 = {k1, k2, p1, p2}, as the reference's CameraCalibration applies it
 * (camera_calibration.cpp:34-72), bit-exact.  K4 = {fx, fy, cx, cy} and D4 are HOST arrays (read at the call); the points are
 * DEVICE buffers.  ALVA_E_INVALID for null pointers, non-finite K4 / D4, fx or fy == 0, or misaligned point buffers.
 *
 * alva_k_undistort_points: cv::undistortPoints(px, unpx, K, D, K) -- 5 fixed-point iterations, the pinhole fallback where the
 * model folds back, the result in pixels -- for every keypoint px [nframes][cap][2] float (8-byte aligned); counts [nframes]
 * (DEVICE, optional: NULL = cap points per frame) limits each frame.  unpx [nframes][cap][2] float; entries past a frame's count
 * are not written.
 * alva_k_project_points: CameraCalibration::projectCamToImageDist for n camera-frame points Xc [n][3] double: the normalised
 * point is rounded to a cv::Point3f and projected with cv::projectPoints; uv [n][2] float (8-byte aligned). */
int alva_k_undistort_points(alva_ctx*, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                            const double* D4, float* unpx);
int alva_k_project_points(alva_ctx*, const double* Xc, int n, const double* K4, const double* D4, float* uv);

/* cv::FAST(gray, thr, nms=true, TYPE_9_16) on each frame (opencv features2d/src/fast.cpp:496).
 * keys[f*cap + i]: packed corner keys; counts[f] = true number found (may exceed cap: then only cap
 * are stored and the call returns ALVA_E_CAPACITY after completing).  sorted != 0: row-major order. */
int alva_k_fast9(alva_ctx*, const uint8_t* gray, int w, int h, int nframes, int thr,
                 uint32_t* keys, int32_t* counts, int cap, int sorted);

/* Fused front end: RGBA -> gray L0 (+ L1..L3 Gaussian pyramid) + FAST-9 corners of L0 in one pass over
 * the input (system.cpp:112 + visual_frontend.cpp:672-698 + orb.cpp:849-850).  L1/L2/L3 may be NULL
 * (then the pyramid stops at the first NULL level).  Level k is ((w_{k-1}+1)/2) x ((h_{k-1}+1)/2). */
int alva_k_frontend(alva_ctx*, const uint8_t* rgba, int w, int h, int nframes,
                    uint8_t* l0, uint8_t* l1, uint8_t* l2, uint8_t* l3,
                    int thr, uint32_t* keys, int32_t* counts, int cap, int sorted);

/* KeyPointsFilter::retainBest(n) on FAST keys (features2d/src/keypoint.cpp:69-90): keeps every corner
 * whose score >= the n-th best score (ties can make it more than n), border-filtered like ORB
 * (edge = 31: orb.cpp:1130) when edge > 0; result sorted row-major.  out_counts[f] <= out_cap. */
int alva_k_retain_best(alva_ctx*, const uint32_t* keys, const int32_t* counts, int cap, int nframes,
                       int w, int h, int n, int edge, uint32_t* out_keys, int32_t* out_counts, int out_cap);

/* ORB pre-blur: GaussianBlur(7x7, sigma 2, REFLECT_101) as ORB applies it (orb.cpp:1188). */
int alva_k_orb_blur(alva_ctx*, const uint8_t* gray, uint8_t* blurred, int w, int h, int nframes, int flags);

/* rBRIEF-256 at given points (FeatureExtractor::describeFeaturePoints, feature_extractor.cpp:160-214 ->
 * ORB::compute, orb.cpp:219-350).  pts: [nframes][npts][2] float (x, y); npts_per_frame may be NULL
 * (= npts for every frame).  desc: [nframes][npts][32]; kept: [nframes][npts] (0 = dropped by the 31-px
 * border rule).  angles_out (optional, [nframes][npts]): the angle used, in degrees.
 * `gray` is needed only with ALVA_ORB_IC_ANGLE (moments are taken on the un-blurred image). */
int alva_k_orb_describe(alva_ctx*, const uint8_t* gray, const uint8_t* blurred, int w, int h, int nframes,
                        const float* pts, const int32_t* npts_per_frame, int npts, int flags,
                        uint8_t* desc, uint8_t* kept, float* angles_out);

/* HarrisResponses (features2d/src/orb.cpp:130-177; blockSize 7, k 0.04) at the given points: resp [nframes][npts] float
 * (0 for unused slots and for points closer than 4 px to the border).  pts / npts_per_frame as alva_k_orb_describe. */
int alva_k_harris(alva_ctx*, const uint8_t* gray, int w, int h, int nframes, const float* pts,
                  const int32_t* npts_per_frame, int npts, float* resp);

/* ORB::detectAndCompute with nlevels = 1, HARRIS_SCORE, edgeThreshold = patchSize = 31 (orb.cpp:970-1218, computeKeyPoints
 * :785-958): FAST(fast_thr, nms) -> border 31 -> retainBest(2*nfeatures) on the FAST score -> Harris -> retainBest(nfeatures)
 * on the Harris response (ties kept, so counts can exceed nfeatures) -> IC angle -> blur -> steered rBRIEF.
 * kp_out [nframes][out_cap][4] float = {x, y, Harris response, angle in degrees}; desc [nframes][out_cap][32];
 * counts[f] = keypoints found (only the first out_cap are stored).  Order: row-major (y, x) -- the reference's order is
 * whatever std::nth_element leaves, so compare as sets.  flags: ALVA_ORB_FMA selects the blur arithmetic. */
int alva_k_orb_detect(alva_ctx*, const uint8_t* gray, int w, int h, int nframes, int nfeatures, int fast_thr, int flags,
                      float* kp_out, uint8_t* desc, int32_t* counts, int out_cap);

/* Brute-force Hamming 2-NN (BFMatcher(NORM_HAMMING).knnMatch(k=2), features2d/src/matchers.cpp:757;
 * tie rule core/src/batch_distance.cpp:235-248).  q: [nq][32], t: [nt][32] bytes;
 * out[4*i] = {idx0, dist0, idx1, dist1} (int32; -1 when nt < 2). */
int alva_k_hamming_knn2(alva_ctx*, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out);

/* Batched variant: q is [nbatch][qcap][32] of which only the first counts[b] slots of batch b are live (qcap a
 * multiple of 8); dead slots come back as -1. */
int alva_k_hamming_knn2_batch(alva_ctx*, const uint8_t* q, const int32_t* counts, int nbatch, int qcap,
                              const uint8_t* t, int nt, int32_t* out);

/* The reference's keyframe corner detector, FeatureExtractor::detectFeaturePoints(image, cell, currKeypoints, roi)
 * (src/slam/src/feature_extractor.cpp:11-158; caller MapManager::extractKeypoints, map_manager.cpp:193-222), batched over frames:
 * per empty grid cell, GaussianBlur 3x3 -> cornerMinEigenVal(block 3, Sobel 3) -> best and second-best maximum under a shared
 * suppression mask (discs of radius cell/4 around the frame's current keypoints and around accepted maxima, in the
 * reference's serial cell order), ROI and quality gates, primaries in cell order followed by secondaries, the quality
 * adaptation x0.5 / x1.5, and cv::cornerSubPix(3x3 half-window, 30 it, 0.01).  DEVICE pointers.
 *   gray [nframes][h][w]; cur [nframes][cur_cap][2] float pixel positions of the current keypoints, ncur [nframes] (both may
 *   be NULL); roi (HOST) = {x, y, width, height} (CameraCalibration's border rect, 20 px); quality [nframes] double IN/OUT =
 *   maxQuality_ (0.001 at start, system.cpp:29); out [nframes][out_cap][2] float sub-pixel corners; out_int (optional)
 *   [nframes][out_cap][2] int32 the integer maxima before refinement; counts [nframes] (true count; only out_cap are stored).
 * 8 <= cell <= 64 (the reference uses 40).  Bit-identical to the reference run with cv::setNumThreads(1). */
int alva_k_detect_grid(alva_ctx*, const uint8_t* gray, int w, int h, int nframes, int cell, const float* cur,
                       const int32_t* ncur, int cur_cap, const int32_t* roi, double* quality, float* out, int32_t* out_int,
                       int32_t* counts, int out_cap);

/* cv::cornerSubPix(image, pts, Size(3, 3), Size(-1, -1), TermCriteria(EPS + MAX_ITER, 30, 0.01)) alone
 * (imgproc/src/cornersubpix.cpp:44-160; feature_extractor.cpp:148-155): pts [nframes][cap][2] IN/OUT, counts [nframes]. */
int alva_k_corner_subpix(alva_ctx*, const uint8_t* gray, int w, int h, int nframes, float* pts, const int32_t* counts, int cap);

/* Pyramidal Lucas-Kanade on prebuilt pyramids: cv::calcOpticalFlowPyrLK(prevPyr, nextPyr, prevPts, nextPts, status, err,
 * Size(win, win), levels, TermCriteria(COUNT+EPS, max_count, epsilon), [USE_INITIAL_FLOW] | LK_GET_MIN_EIGENVALS, 1e-4)
 * (opencv video/src/lkpyramid.cpp:1238-1398, LKTrackerInvoker :183-722) -- the call FeatureTracker::fbKltTracking makes
 * (src/slam/src/feature_tracker.cpp:35-38).  prev_img / prev_der / cur_img: HOST arrays of pyr_levels + 1 DEVICE pointers,
 * level k = [nframes][h_k][w_k] u8 (alva_k_frontend / alva_k_pyrdown) resp. [nframes][h_k][w_k][2] int16 (alva_k_scharr),
 * w_k = (w_{k-1} + 1) / 2; the reference's padded borders (REFLECT_101 image, constant-0 derivative) are implied.
 * pts / next: [nframes][npts][2] float (next: initial flow in, tracked position out); npts_per_frame may be NULL;
 * status [nframes][npts] u8, err (optional) [nframes][npts] float = min eigenvalue at level 0.  win must be 9
 * (State::kltWinSizeWH_, src/slam/src/state.hpp:52).  Results are bit-identical to the reference's SSE float path. */
int alva_k_klt_lk(alva_ctx*, const uint8_t* const* prev_img, const int16_t* const* prev_der, const uint8_t* const* cur_img,
                  int w, int h, int nframes, int pyr_levels, int levels, int win, int max_count, double epsilon,
                  int use_initial, const float* pts, float* next, const int32_t* npts_per_frame, int npts,
                  uint8_t* status, float* err);

/* FeatureTracker::fbKltTracking (src/slam/src/feature_tracker.cpp:5-111; caller VisualFrontend::kltTrackingFromMotionPrior,
 * visual_frontend.cpp:103-243) in ONE launch: forward LK from the priors on `levels` levels (criteria 30 it / 0.01 px,
 * system.cpp:31), the reference's gates (status, min-eig err > error_value, 1-px inBorder), backward LK on level 0 from
 * the tracked position towards the original one, and the |p - back| > max_fb_dist gate.  priors [nframes][npts][2] in/out
 * (written for every live point, like the reference's priorKeypoints); good [nframes][npts] u8 = keypointStatus. */
int alva_k_klt_fb(alva_ctx*, const uint8_t* const* prev_img, const int16_t* const* prev_der, const uint8_t* const* cur_img,
                  const int16_t* const* cur_der, int w, int h, int nframes, int pyr_levels, int levels, int win,
                  float error_value, float max_fb_dist, const float* pts, float* priors, const int32_t* npts_per_frame,
                  int npts, uint8_t* good);

/* Per-frame pose, step 1: MultiViewGeometry::p3pRansac(observations, wPoints, max_iter, err_px, optimize = false, doRandom,
 * fx, fy, Twc, outliers) (src/slam/src/multi_view_geometry.cpp:24-127; caller VisualFrontend::computePose,
 * visual_frontend.cpp:299-312) = Kneip P3P inside OpenGV's Least-Median-of-Squares loop (always max_iter successful draws,
 * sample size 4, score = median of squared bearing distances, inliers: distance <= 1 - cos(atan(err_px / focal))), batched
 * over nprob independent problems.  DEVICE pointers, FP64: bvs / wpts [nprob][cap][3] (unit bearing vectors / world points;
 * only the first counts[p] are live, counts may be NULL, cap <= 4096).  seed: the sampler's std::mt19937 seed -- the
 * reference uses 12345 when State::multiViewRandomEnabled_ is false and the clock otherwise (state.hpp:67).
 * Twc_out [nprob][12]: camera-to-world [R | t], 3x4 row-major (unspecified when the problem fails); outlier [nprob][cap]
 * (1 = outlier / dead slot); info (optional) [nprob][4] = {success (>= 5 inliers and R orthogonal: what p3pRansac returns),
 * #inliers, best median, #draws}. */
int alva_k_p3p_lmeds(alva_ctx*, int nprob, int cap, const double* bvs, const double* wpts, const int32_t* counts,
                     int max_iter, float err_px, float fx, float fy, uint32_t seed, double* Twc_out, uint8_t* outlier,
                     double* info);

/* Per-frame pose, step 2: MultiViewGeometry::ceresPnP (src/slam/src/multi_view_geometry.cpp:129-223; functor
 * DirectSE3::ReprojectionErrorSE3, ceres_parametrization.cpp:96-155): Levenberg-Marquardt on the 6-dof pose with
 * Huber(huber_delta) (use_robust), residuals with chi2 > chi2_thr or non-positive depth at their last evaluation flagged as
 * outliers, and (apply_l2) a second, non-robust solve without them.  Solved the way ceres::Solve does with the reference's
 * options (<= max_iter iterations, function_tolerance 1e-3, Jacobi scaling; the 5 ms wall-clock cap is lifted), batched
 * over nprob problems, every decision on the device.  K [nprob][4] = fx fy cx cy; uv [nprob][cap][2] undistorted pixels;
 * X [nprob][cap][3]; poses [nprob][7] = [t, q(x,y,z,w)] camera-to-world IN/OUT (left untouched when every point is an
 * outlier, as in the reference); outlier [nprob][cap]; summary [nprob][12] = {initial cost, final cost, #successful,
 * #iterations, termination} of solve 1, the same of solve 2 (zeros if skipped), return value of ceresPnP (0/1), #outliers. */
int alva_k_pnp(alva_ctx*, int nprob, int cap, const double* K, const double* uv, const double* X, const int32_t* counts,
               double* poses, double huber_delta, double chi2_thr, int max_iter, int use_robust, int apply_l2,
               uint8_t* outlier, double* summary);

/* Map initialisation: MultiViewGeometry::compute5ptEssentialMatrix(observations1, observations2, max_iter, err_px, optimize,
 * doRandom, fx, fy, Rwc, twc, outliers) (src/slam/src/multi_view_geometry.cpp:225-318; caller
 * VisualFrontend::checkReadyForInit, visual_frontend.cpp:517-528) = OpenGV's Ransac over CentralRelativePoseSacProblem (Nister's
 * five-point solver on the first 5 of 8 drawn correspondences, the 8 disambiguate the <= 40 (R, t) candidates; inliers:
 * mid-point triangulation error e1 + e2 < 2 (1 - cos(atan(err_px / focal))); adaptive iteration bound, probability 0.99;
 * >= 10 inliers required) followed by relative_pose::optimize_nonlinear over the inliers when optimize != 0, batched over
 * nprob independent problems.  DEVICE pointers, FP64: bv1 / bv2 [nprob][cap][3] = unit bearing vectors of the keyframe and of
 * the current frame (only the first counts[p] are live; counts may be NULL; cap <= 8192).  seed as in alva_k_p3p_lmeds.
 * Rt_out [nprob][12]: [Rwc | twc] 3x4 row-major, twc NOT normalised (the caller normalises it, visual_frontend.cpp:547);
 * written only on success.  outlier [nprob][cap] (1 = outlier / dead slot).  info (optional) [nprob][4] = {success, #inliers,
 * #RANSAC iterations, #draws}.
 * optimize: 0 = RANSAC model only; 1 = refinement by Levenberg-Marquardt on central differences (block-parallel; the default
 * of `System`: it converges to the cost's minimum and is insensitive to rounding noise); 2 = the reference's own minimiser
 * restated -- MINPACK LM on a forward-difference Jacobian, ftol = xtol = 10 eps (csrc/lmdif_core.h; one thread).  The
 * reference's end point is noise-limited (its Jacobian carries ~10 % rounding noise): modes 1 and 2 both end as far from it as
 * the reference ends from itself when it is rebuilt with other compiler flags (DESIGN.md section 4.11). */
int alva_k_essential_5pt(alva_ctx*, int nprob, int cap, const double* bv1, const double* bv2, const int32_t* counts,
                         int max_iter, float err_px, int optimize, float fx, float fy, uint32_t seed, double* Rt_out,
                         uint8_t* outlier, double* info);

/* MultiViewGeometry::triangulate (src/slam/src/multi_view_geometry.cpp:12-22 -> opengv::triangulation::triangulate2, the
 * mid-point of the two rays; caller Mapper::triangulateTemporal, mapper.cpp:157-291) for n bearing-vector pairs.  DEVICE
 * pointers, FP64: Tlr [7] = [t, q(x,y,z,w)] (pose of the right camera in the left one); bvl / bvr [n][3]; out [n][3] = points
 * in the left camera frame. */
int alva_k_triangulate(alva_ctx*, const double* Tlr, const double* bvl, const double* bvr, int n, double* out);

/* Mapper::matchToMap (src/slam/src/mapper.cpp:354-587; caller matchingToLocalMap :293-352): every local-map point the
 * keyframe does not observe yet is projected into it (depth >= 0.1, view angle, in image), compared with the keypoints of
 * the 2x2 grid cells around the projection (pixel gate max_proj_err, doubled below 30 3-D keypoints; the two map points never
 * observed in one keyframe; mean co-projection error of the keypoint's own observations; minimum Hamming distance over all
 * per-keyframe descriptor pairs, MapPoint::computeMinDescDist), best / second best with the 0.9 ratio test, and per keypoint
 * the map point with the smallest distance (the last one in processing order on ties).  The map is flat SoA, DEVICE pointers:
 *   Twc_cur [7] = [t, q(x,y,z,w)]; keypoints in grid insertion order: kp_mp [n_kp] = index of the keypoint's own map point in
 *   the table (-1: none), kp_px [n_kp][2]; nkp3d (HOST int) = Frame::numKeypoints3d_; kf_Twc [n_kf][7], n_kf <= 64;
 *   map point table: mp_wpt [n_mp][3], mp_is3d [n_mp], observations CSR obs_start [n_mp + 1] -> obs_kf (keyframe INDEX,
 *   ascending keyframe id) / obs_px [..][2], descriptors CSR desc_start [n_mp + 1] -> desc [..][32] (16-byte aligned);
 *   local_mp [n_local] = table indices of the local map in the host's iteration order (that order decides ties, as the
 *   reference's unordered_set order does).  Zero lens distortion (what the JS shim passes; see alva_k_match_to_map_dist).
 * Out: kp_match [n_kp] = table index of the matched local map point or -1, kp_dist (optional) its Hamming distance,
 * n_match [1] the number of matched keypoints. */
int alva_k_match_to_map(alva_ctx*, int w, int h, int cell, double fx, double fy, double cx, double cy, const double* Twc_cur,
                        int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf, const double* kf_Twc, int n_mp,
                        const double* mp_wpt, const uint8_t* mp_is3d, const int32_t* obs_start, const int32_t* obs_kf,
                        const float* obs_px, const int32_t* desc_start, const uint8_t* desc, int n_local, const int32_t* local_mp,
                        float max_proj_err, float dist_ratio, int32_t* kp_match, float* kp_dist, int32_t* n_match);
/* The same with lens distortion: dist4 = {k1, k2, p1, p2} (HOST array; NULL or all zero = alva_k_match_to_map) is applied to
 * the map point's projection and to the co-projection errors, as the reference's Frame::projCamToImageDist /
 * projWorldToImageDist do (mapper.cpp:425, 504).  ALVA_E_INVALID for a non-finite coefficient. */
int alva_k_match_to_map_dist(alva_ctx*, int w, int h, int cell, double fx, double fy, double cx, double cy, const double* Twc_cur,
                             int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf, const double* kf_Twc, int n_mp,
                             const double* mp_wpt, const uint8_t* mp_is3d, const int32_t* obs_start, const int32_t* obs_kf,
                             const float* obs_px, const int32_t* desc_start, const uint8_t* desc, int n_local, const int32_t* local_mp,
                             float max_proj_err, float dist_ratio, int32_t* kp_match, float* kp_dist, int32_t* n_match,
                             const double* dist4);

/* Local bundle adjustment, batched over nprob independent problems of identical dimensions
 * (Optimizer::localBA, src/slam/src/optimizer.cpp:4-531, solved the way ceres::Solve does with the reference's
 * options: SPARSE_SCHUR elimination of the inverse depths, Levenberg-Marquardt, Huber(huber_delta), Jacobi scaling,
 * function_tolerance 1e-3, at most max_iter iterations, no wall-clock cap).  All pointers are DEVICE pointers, FP64.
 *   calib [nprob][4] (fx fy cx cy)                poses [nprob][nkf][7] = [t, q(x,y,z,w)] camera-to-world, IN/OUT
 *   pose_const [nprob][nkf] (1 = fixed)           invd [nprob][nlm] inverse depth in the anchor keyframe, IN/OUT
 *   anch_kf [nprob][nlm], anch_uv [nprob][nlm][2]  anchor keyframe index and (undistorted) pixel of each landmark
 *   obs_kf/obs_lm [nprob][nobs], obs_uv [nprob][nobs][2]   the non-anchor observations; obs_lm = -1 marks an unused slot
 *   summary [nprob][8] (optional): initial cost, final cost, #successful steps, #iterations, termination
 *   (0 convergence, 1 iteration limit, 2 failure), reduced-system width, final radius, last iteration index. */
int alva_k_ba_solve(alva_ctx*, int nprob, int nkf, int nlm, int nobs, const double* calib, double* poses,
                    const uint8_t* pose_const, double* invd, const int32_t* anch_kf, const double* anch_uv,
                    const int32_t* obs_kf, const int32_t* obs_lm, const double* obs_uv, double huber_delta, int max_iter,
                    double* summary);

/* The numerical body of Optimizer::localBA after problem assembly (src/slam/src/optimizer.cpp:251-359), batched like
 * alva_k_ba_solve and entirely on the device (no host decision between the steps):
 *   1. solve (as alva_k_ba_solve, <= max_iter iterations)                                 optimizer.cpp:251-271
 *   2. an observation is an outlier if, at the point its cost functor was evaluated LAST (the last candidate the
 *      minimiser evaluated, accepted or not), chi2 = |r|^2 > chi2_thr or the depth is not positive; outliers are removed
 *      (flags = 1)                                                                        optimizer.cpp:273-299
 *   3. per problem, only if it lost observations and huber_delta > 0: solve again, <= 5 iterations, same loss
 *                                                                                         optimizer.cpp:305-327
 *   4. flag (flags = 2, not removed) the observations that are outliers after that solve   optimizer.cpp:330-356
 * obs_lm is not modified; flags [nprob][nobs] int32 (0 = inlier / unused slot); summary (optional) [nprob][10]:
 * {initial cost, final cost, #successful, #iterations, termination} of solve 1, then of solve 2 (zeros if skipped).
 * The reference's 1 ms wall-clock cap on step 3 (and 5 ms on step 1) is lifted, as everywhere in this library.
 * Size limits (alva_k_ba_solve too): 1 <= nkf <= 256 (else ALVA_E_INVALID), and at most 21 free (non-constant, referenced)
 * poses per problem -- the reduced camera system is factored in one CTA's shared memory.  A problem with more free poses is
 * refused, alone (the rest of the batch is solved): its parameters are untouched and its summary reads initial and final
 * cost 0, 0 successful steps, 0 iterations, termination 2 (alva_k_ba_solve: width 0, radius 1e4, last iteration 0).
 * alva_k_ba_local still tests the outliers, at the untouched input, and removes them (flags 1); if it removed any and
 * huber_delta > 0, the second solve runs on the residuals left, and is refused the same way (summary[5..9] = 0, 0, 0, 0, 2)
 * while they still reference more than 21 free poses. */
int alva_k_ba_local(alva_ctx*, int nprob, int nkf, int nlm, int nobs, const double* calib, double* poses,
                    const uint8_t* pose_const, double* invd, const int32_t* anch_kf, const double* anch_uv,
                    const int32_t* obs_kf, const int32_t* obs_lm, const double* obs_uv, double huber_delta, double chi2_thr,
                    int max_iter, int32_t* flags, double* summary);

/* Library-wide switches.  "ba_dense_schur" = 1: compute the -(E'F)'(E'E)^-1(E'F) part of the Schur complement as a dense
 * FP64 tensor-core SYRK (S -= Wt'Wt, DMMA) instead of per-landmark atomics (default 0).
 * "frontend_antipodal" = 1: EXPERIMENTAL variant of the fused front end's FAST-9 pre-test (antipodal flag sharing, csrc/fast_swar.h;
 * same results by construction, checked by host emulation, not yet validated on a GPU) -- default 0.
 * "pipeline_ba_overlap" = 0: alva_pipeline runs the local BA after the per-frame stages instead of beside them on its own
 * stream (default 1; results are identical, only the schedule changes).
 * "pipeline_ba_lag" = 1: the BA chain of step s is joined at the end of step s + 1 instead of step s (default 0; per-step results
 * are the same numbers, delivered one step later; see alva_pipeline_drain).
 * "ba_ctl_threads" = 256 | 512 | 1024: CTA size of the BA control kernels (default 1024; results differ at rounding level: the
 * block reductions partition differently).
 * "pipeline_graphs" = 0: alva_pipeline launches kernel by kernel instead of replaying CUDA graphs (default 1; results identical).
 * "knn_qpw" = 4 | 8: queries a warp of the Hamming matcher keeps in registers (8: 128 registers / 16 warps per SM;
 * 4: 80 registers / 24 warps per SM).  Results are identical.
 * "knn_mma" = 0 | 1 | 2: the tensor-core formulation of the Hamming matcher (hamming_mma.cu: descriptors expanded to +-1
 * int8, wgmma s8 x s8 -> s32, dot = 256 - 2 * distance): 0 never, 1 for large query sets (default), 2 always.  Results
 * are identical.  "knn_mma_kind" = 0 | 1: operand kind of that kernel (0: +-1 as int8, int32 accumulators -- default;
 * 1: +-1.0 as E4M3, fp32 accumulators).  "knn_mma_mode" = 0 | 1 | 2: its
 * shared-memory operand layout (0 no swizzle, 1 128-byte swizzle, 2 debugging variant).
 * "frontend_variant" = 2 | 0: the fused front-end kernel (2: frontend_tile_kernel_v2, default; 0: the round-1 kernel, which
 * also serves geometries a TMA tensor map cannot express).  Results are identical.
 * "frontend_prefetch" = 0 | 1: variant 2 also pulls the tile at the same position a few frames ahead into L2 (TMA prefetch)
 * while it works on its own (default 0).  Results are identical. */
int alva_set_option(const char* name, int value);
/* Debugging aid: the tensor-core matcher unconditionally on q [nq][32] x t [nt][32] (device pointers, 16-byte aligned);
 * dbg_dev (optional, 16384 int32 of device memory) receives the raw dot products of the first 128 x 128 tile. */
int alva_debug_knn2_mma(alva_ctx*, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out, int32_t* dbg_dev);

/* Residual / Jacobian build alone (DirectSE3::ReprojectionErrorKSE3AnchInvDepth::Evaluate,
 * src/slam/src/ceres_parametrization.cpp:157-269, + Huber corrector): res [nobs][2], Ja/Jp [nobs][2][6] (local
 * Jacobians wrt anchor / observing pose), Jd [nobs][2] (wrt inverse depth), cost_per_obs [nobs]. */
int alva_k_ba_linearize(alva_ctx*, int nkf, int nlm, int nobs, const double* calib, const double* poses, const double* invd,
                        const int32_t* anch_kf, const double* anch_uv, const int32_t* obs_kf, const int32_t* obs_lm,
                        const double* obs_uv, double huber_delta, double* res, double* Ja, double* Jp, double* Jd,
                        double* cost_per_obs);

/* Test hook: the reduced camera system of alva_k_ba_solve's first Levenberg-Marquardt iteration (the input point's
 * linearisation, Jacobi scaling and LM diagonal; inputs as alva_k_ba_solve, not modified), assembled by the path the solve takes
 * (atomic = 0) or by the atomic per-landmark path (atomic = 1).  S_out [nprob][128][128] (rows / columns past the width are 0),
 * rhs_out [nprob][128], info [nprob][2] = {reduced-system width, 1 if the gather path assembled it}.  Needs ba_dense_schur off. */
int alva_k_ba_schur_dump(alva_ctx*, int nprob, int nkf, int nlm, int nobs, const double* calib, const double* poses,
                         const uint8_t* pose_const, const double* invd, const int32_t* anch_kf, const double* anch_uv,
                         const int32_t* obs_kf, const int32_t* obs_lm, const double* obs_uv, double huber_delta, int atomic,
                         double* S_out, double* rhs_out, double* info);

/* ---- the whole per-frame hot path as one object ------------------------------------------------
 * A batch of frames goes gray + pyramid + FAST -> retainBest -> ORB -> Hamming 2-NN vs the local map -> local BA on
 * the step's keyframes, every intermediate resident in HBM, no host synchronisation inside a step
 * (reference per-frame / per-keyframe sequence: System::findCameraPose system.cpp:106-121 -> VisualFrontend::track
 * visual_frontend.cpp:21-35 -> MapManager::createKeyframe map_manager.cpp:24,193 -> Mapper::matchingToLocalMap
 * mapper.cpp:293 -> Optimizer::localBA optimizer.cpp:4). */
typedef struct alva_pipeline alva_pipeline;
typedef struct alva_pipeline_config {
    int w, h, batch;        /* frame geometry and frames per step */
    int fast_thr;           /* FAST threshold (ORB default 20) */
    int nfeatures;          /* retainBest target per frame */
    int orb_flags;          /* ALVA_ORB_* */
    int map_size;           /* descriptors in the local map (0 = no matching) */
    int kf_interval;        /* one local BA per kf_interval frames (0 = no BA) */
    int ba_nkf, ba_nlm, ba_nobs, ba_max_iter;
    double ba_huber;
    int derivatives;        /* != 0: also build the Scharr derivative image of every pyramid level, as the reference's
                               buildOpticalFlowPyramid(..., withDerivatives = true) does each frame (visual_frontend.cpp:696) */
    int reserved;
} alva_pipeline_config;

alva_pipeline* alva_pipeline_create(alva_ctx*, const alva_pipeline_config*);
void alva_pipeline_destroy(alva_pipeline*);
int  alva_pipeline_set_map(alva_pipeline*, const uint8_t* desc_host, int n);
int  alva_pipeline_set_ba(alva_pipeline*, int slot, const double* calib, const double* poses, const uint8_t* pose_const,
                          const double* invd, const int32_t* anch_kf, const double* anch_uv, const int32_t* obs_kf,
                          const int32_t* obs_lm, const double* obs_uv);
int  alva_pipeline_step_dev(alva_pipeline*, const uint8_t* rgba_dev);
int  alva_pipeline_step_host(alva_pipeline*, const uint8_t* rgba_host, int32_t* nfeat_host, int32_t* matches_host,
                             double* ba_poses_host, double* ba_summary_host);
/* Asynchronous form of step_host for throughput hosts: submit enqueues a batch (upload in chunks, compute, results back to the
 * given host buffers) and returns at once; at most two submissions may be outstanding, so the upload of one overlaps the
 * compute of the other.  wait blocks until the OLDEST outstanding submission has delivered its results.  The host buffers must
 * stay valid (and the result buffers distinct per outstanding submission) until the matching wait returns.
 * step_host == submit + wait. */
int  alva_pipeline_submit_host(alva_pipeline*, const uint8_t* rgba_host, int32_t* nfeat_host, int32_t* matches_host,
                               double* ba_poses_host, double* ba_summary_host);
int  alva_pipeline_wait(alva_pipeline*);
int  alva_pipeline_profile(alva_pipeline*, int enable);
int  alva_pipeline_frontend_ms(alva_pipeline*, float* ms, int n);   /* CUDA-event durations of the fused front-end launch */
int  alva_pipeline_info(const alva_pipeline*, int32_t* out4);
/* {CUDA graphs captured so far, graph launches so far, 1 if a capture failed and the pipeline fell back to direct launches} */
int  alva_pipeline_graph_stats(alva_pipeline*, int32_t* out3);
/* With alva_set_option("pipeline_ba_lag", 1) a step's local-BA chain is joined at the end of the NEXT step (two chains in
 * flight on two streams; a step then delivers the BA poses / summary of the step before it, as the reference's mapper thread
 * delivers its results asynchronously).  alva_pipeline_drain makes the context stream wait for every chain still in flight;
 * afterwards the BA buffers hold the newest step's result.  A no-op in the default (same-step) mode. */
int  alva_pipeline_drain(alva_pipeline*);
void* alva_pipeline_buffer(alva_pipeline*, int which);

/* ---- System: the reference's public class, one handle per camera stream ------------------------
 * One-to-one with System::{configure, reset, findCameraPose, findCameraPoseWithIMU, findPlane, getFramePoints}
 * (reference src/slam/src/system.hpp:28-38; JS caller src/system.js:58-237).  Host pointers, caller-owned buffers:
 * rgba = W*H*4 bytes (read only), pose16 = 16 floats (R rows in [0..2],[4..6],[8..10], t in [12..14], [15] = 1;
 * src/slam/src/utils.cpp:3-27).  findCameraPose returns 1 tracking / 2 tracker was reset / 3 not initialised
 * (system.cpp:163-174) or a negative ALVA_E_* code. */
alva_system* alva_system_create(int device);
void alva_system_destroy(alva_system*);
int  alva_system_configure(alva_system*, int w, int h, double fx, double fy, double cx, double cy,
                           double k1, double k2, double p1, double p2);
int  alva_system_reset(alva_system*);
/* CLAHE on the gray frame before the KLT pyramid and the detector: State::claheEnabled_ / claheContrastLimit_ / claheTileSize_
 * (state.hpp:43-45) with VisualFrontend's grid, Size(w / tile_size, h / tile_size) (visual_frontend.cpp:16-18).  ORB descriptors
 * stay on the raw gray frame (map_manager.cpp:204, 218).  Off by default; configure turns it off again (system.cpp:17), reset keeps
 * it; it applies from the next frame.  ALVA_E_STATE before configure; ALVA_E_INVALID for an empty grid (tile_size > w or h, or
 * < 1) or, when enabling, a negative / NaN clip_limit. */
int  alva_system_set_clahe(alva_system*, int enabled, double clip_limit, int tile_size);
/* Lens distortion of a configured System: the reference's configure(..., k1, k2, p1, p2) coefficients (OpenCV's radial-tangential
 * model), applied where its CameraCalibration applies them -- every tracked and detected keypoint is undistorted (on the device),
 * the KLT priors of 3-D keypoints and the local-map matcher's projections are distorted.  It resets the tracker and the map as
 * reset() does; the next frame starts under the new model.  All zero = the pinhole camera.  configure clears it, reset keeps it.
 * ALVA_E_STATE before configure; ALVA_E_INVALID for a null handle or a non-finite coefficient. */
int  alva_system_set_distortion(alva_system*, double k1, double k2, double p1, double p2);
/* The reference's three tuned configurations (state.hpp:9-17), and DEFAULT = what configure sets (system.cpp:15-19):
 *              grid cell  CLAHE (clip 3, tile 50)  keyframe filtering ratio  P3P on every tracked frame
 *   DEFAULT    40 px      off                      0.95                      yes
 *   FAST       50 px      off                      0.9                       yes
 *   AVERAGE    45 px      off                      0.9                       no: PnP from the motion prior, P3P on the next frame if it fails
 *   ACCURATE   35 px      on                       0.95                      no
 * The cell size sets the detector grid, the keypoint budget ceil(w / cell) * ceil(h / cell), the local-map size, the keyframe
 * rules and the grid the local-map matcher searches.  It resets the tracker and the map as reset() does (the frame grid
 * changes); the next frame starts under the new preset.  It sets the CLAHE switch from the table: a later
 * alva_system_set_clahe overrides it.  configure returns the handle to DEFAULT, reset keeps the preset, the lens model is left
 * alone.  ALVA_E_STATE before configure; ALVA_E_INVALID for a null handle or an unknown preset. */
#define ALVA_PRESET_DEFAULT  0
#define ALVA_PRESET_FAST     1
#define ALVA_PRESET_AVERAGE  2
#define ALVA_PRESET_ACCURATE 3
int  alva_system_set_preset(alva_system*, int preset);
int  alva_system_find_camera_pose(alva_system*, const uint8_t* rgba, float* pose16);
/* the same with the frame's time stamp (milliseconds) supplied by the caller instead of read from the system clock
 * (system.cpp:114): deterministic replays, and hosts that deliver frames faster than real time (two frames inside one
 * millisecond give the reference's motion model dt = 0) */
int  alva_system_find_camera_pose_ts(alva_system*, const uint8_t* rgba, double t_ms, float* pose16);
int  alva_system_find_camera_pose_imu(alva_system*, const uint8_t* rgba, const double* imu, float* pose16);
/* System::findPlane (system.cpp:123-137, 177-342): RANSAC plane through the current frame's observed 3-D map points; out16 =
 * plane pose, column-major 4x4 as Utils::toPoseArray(cv::Mat) writes it; returns 1 / 0 (fewer than 32 points or inliers).  The
 * procedure is the reference's as intended -- its own code never fits a plane to the coordinates (DESIGN.md section 6). */
int  alva_system_find_plane(alva_system*, float* out16, int iterations);
int  alva_system_get_frame_points(alva_system*, int32_t* xy, int cap_pairs);   /* returns the true count */
int  alva_system_num_matched(alva_system*);   /* keypoints of the current frame (Frame::numKeypoints_) */
/* every keypoint of the current frame in the frame's own order: track ids (keypoint id == map point id,
 * src/slam/src/map_manager.cpp:166-191), pixel positions px [cap][2], and optionally is3d [cap] and the map points' world
 * positions wpt [cap][3] (zeros for 2-D keypoints); returns the true count */
int  alva_system_get_tracks(alva_system*, int32_t* ids, float* px, uint8_t* is3d, double* wpt, int cap);
/* their 256-bit ORB descriptors (Keypoint::desc_, feature_extractor.cpp:160-214), same order: desc [cap][32], has [cap] (0 = the
 * reference keeps an empty Mat: point within 31 px of the border) */
int  alva_system_get_descriptors(alva_system*, uint8_t* desc, uint8_t* has, int cap);
/* Page-lock (cudaHostRegister) a caller-owned frame buffer that is reused from call to call -- the reference's shim allocates its
 * image buffer once (system.js:63-67) -- so that alva_system_find_camera_pose uploads it at the host link's rate; unpin before
 * freeing it (alva_system_destroy unpins what is left).  Optional: un-pinned buffers work, through the driver's pageable staging. */
int  alva_system_pin_buffer(alva_system*, void* host_ptr, size_t bytes);
int  alva_system_unpin_buffer(alva_system*, void* host_ptr);
/* TEST HOOK: the result ([Rwc | twc] 3x4 row-major, outlier flags of the n correspondences) the NEXT 5-point initialisation
 * returns instead of running alva_k_essential_5pt -- used by the parity tests to plug in the reference's own initialisation
 * result (whose refinement is noise-limited, DESIGN.md) and check everything downstream of it at 1e-7; ignored when n does not
 * match the number of correspondences of that initialisation. */
/* ---- cross-stream loop closure (SURVEY 8e / 8f.4; the reference has none: parity unpinned, validated by determinism and
 * planted revisits).  KEYFRAME BLOCK wire format (what one rank contributes per new keyframe to the NCCL all-gather;
 * little-endian, fixed size so that the exchange has static shapes):
 *     offset 0    int32 magic = ALVA_LC_MAGIC ('ALKF'), int32 version = ALVA_LC_VERSION, int32 stream id (rank), int32 keyframe
 *                 sequence number, int32 count (live entries, <= n_max; a reader clamps it to [0, n_max]), int32 n_max,
 *                 float32 fx, fy, cx, cy, 6 x int32 reserved (0)
 *     offset 64   float32 px[n_max][2]      pixel position of keypoint i (entries >= count are 0)
 *     then        uint8   desc[n_max][32]   its 256-bit ORB descriptor
 * alva_lc_block_bytes(n_max) = 64 + 40 * n_max.  A step's exchange is [world][kf_per_step] such blocks.
 * alva_lc_pack      : this rank's kf_per_step new keyframes (frames kf_frames[e] of a frame-major batch: desc [nframes][cap][32],
 *                     pts [nframes][cap][2] float, counts [nframes]; all DEVICE pointers) -> send (device, kf_per_step blocks).
 *                     K4 (host): fx, fy, cx, cy.  kf_seq0: sequence number of the first of them.
 * alva_lc_detect    : on the gathered blocks (device, [world][kf_per_step] blocks): Hamming 2-NN of keyframe e of this rank against
 *                     keyframe e of every other rank, ratio test; five-point RANSAC (32 hypotheses) on the putative matches of the
 *                     step's NEWEST keyframe against every remote stream with >= min_matches of them; enqueues only.
 * alva_lc_poll      : finished steps are consumed in order; a loop with remote stream r is reported on the newest keyframe of a
 *                     step when the last min_consecutive keyframe events against r all had >= min_matches putative matches and
 *                     that keyframe passed RANSAC with >= min_inliers inliers.  Returns the number of events. */
#define ALVA_LC_MAGIC        0x464B4C41   /* "ALKF" */
#define ALVA_LC_VERSION      1
#define ALVA_LC_HEADER_BYTES 64
#define ALVA_LC_PAIR_CAP     512          /* putative matches kept per keyframe pair (the first ones in local-index order) */
typedef struct alva_lc alva_lc;
typedef struct {
    int32_t n_max, kf_per_step, world, rank;
    int32_t min_matches;       /* putative matches a keyframe event needs to count / before the geometric check runs: at least this
                                * (default 30) and at least 1/8 of the local keyframe's descriptors */
    int32_t max_dist;          /* absolute Hamming gate on the best match (default 64) */
    int32_t ratio_num, ratio_den;   /* ratio test: best * ratio_den < second * ratio_num (default 4 / 5) */
    int32_t min_consecutive;   /* keyframe events in a row that must have enough matches (default 3) */
    int32_t min_inliers;       /* RANSAC inliers needed (default 20) */
    float err_px, fx_hint, fy_hint;   /* RANSAC threshold in pixels (default 3) at this focal length (default 500) */
} alva_lc_config;
typedef struct {
    int32_t local_kf, remote_rank, remote_kf, n_matches, n_inliers, consecutive;
    double Rt[12];             /* relative pose [R | t] (3 x 4 row-major, t up to scale) of the remote keyframe in the local one */
} alva_lc_event;
size_t   alva_lc_block_bytes(int n_max);
alva_lc* alva_lc_create(alva_ctx*, const alva_lc_config*);
void     alva_lc_destroy(alva_lc*);
int      alva_lc_pack(alva_lc*, const uint8_t* desc, const float* pts, const int32_t* counts, int cap, const int32_t* kf_frames,
                      int kf_seq0, const float* K4, uint8_t* send);
/* The same with the pack kernel enqueued on `on`'s stream (NULL: the detector's): pass the context that produced desc / pts so that
 * packing never waits behind a detection still running on the detector's stream. */
int alva_lc_pack_on(alva_lc*, alva_ctx* on, const uint8_t* desc, const float* pts, const int32_t* counts, int cap,
                    const int32_t* kf_frames, int kf_seq0, const float* K4, uint8_t* send);
int      alva_lc_detect(alva_lc*, const uint8_t* gathered);
int      alva_lc_poll(alva_lc*, alva_lc_event* out, int cap, int wait);
/* steps enqueued by alva_lc_detect whose results alva_lc_poll has not consumed yet (at most 4 may be in flight) */
int      alva_lc_inflight(const alva_lc*);
/* diagnostics: per keyframe pair of the last step, out [kf_per_step][world][4] = {matches, RANSAC success, inliers, remote keyframe} */
int      alva_lc_last_scores(alva_lc*, double* out);
/* tests / diagnostics: the internal state of the last step.  nn [kf_per_step][world][n_max][4] = {idx0, dist0, idx1, dist1} of the
 * Hamming 2-NN (-1 where there is none; only rows below the local keyframe's live count are defined), npair [kf_per_step][world] =
 * correspondences handed to the geometric check, bv_local / bv_remote [kf_per_step][world][ALVA_LC_PAIR_CAP][3] = the bearing
 * vectors of the putative matches in local-index order (rows below min(matches, ALVA_LC_PAIR_CAP) are defined).  Any output
 * may be NULL. */
int      alva_lc_last_matches(alva_lc*, int32_t* nn, int32_t* npair, double* bv_local, double* bv_remote);

/* N independent camera streams in one call (SURVEY 8e: streams are independent, System holds all state): handles[i]
 * processes the frame rgba[i] with time stamp t_ms[i] (t_ms NULL = the system clock).  poses16 [n][16], status [n] (the value
 * alva_system_find_camera_pose_ts would return for that stream).  The streams run concurrently on the device (every System
 * owns a CUDA stream).  Returns 0, or the first negative status. */
int  alva_system_find_camera_pose_batch(alva_system* const* handles, const uint8_t* const* rgba, const double* t_ms, int n,
                                        float* poses16, int* status);
int  alva_system_debug_set_initialisation(alva_system*, const double* Rt12, const uint8_t* outlier, int n);
/* the current frame's camera-to-world pose in double: [t, q(x,y,z,w)] */
int  alva_system_get_pose(alva_system*, double* Twc7);
/* {frame id, keyframe id, #keypoints, #3-D keypoints, initialised, #keyframes, #occupied grid cells, #map point ids} */
int  alva_system_get_info(alva_system*, int32_t* out8);

/* ---- host-buffer variants (copies inside; used for e2e timing and by non-CUDA hosts) ---------- */
int alva_h_frontend(alva_ctx*, const uint8_t* rgba_host, int w, int h, int nframes, int thr,
                    uint32_t* keys_host, int32_t* counts_host, int cap);

#ifdef __cplusplus
}
#endif
#endif /* ALVA_B200_H */
