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
/* The same two calls through OpenCV's equidistant fisheye model (cv::fisheye, "Kannala-Brandt"), D4 = {k1, k2, k3, k4} on the
 * incidence angle theta: theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8).  Same shapes, layout, counts
 * and argument checks as above; zero coefficients are the equidistant projection, not the pinhole.
 * alva_k_undistort_points_fisheye: cv::fisheye::undistortPoints(px, unpx, K, D, noArray(), K) -- theta_d clamped to
 * [-pi/2, pi/2], at most 10 Newton steps (stop at |step| < 1e-8), the result in pixels of the same K; (-1e6, -1e6) where the
 * iteration does not converge or theta changes sign.
 * alva_k_project_points_fisheye: cv::fisheye::projectPoints of the float point (x/z, y/z, 1), zero rvec / tvec, alpha 0.
 * Bit-exact with the library up to atan / tan, which here are one deterministic double version on host and device (a float
 * result can differ from a glibc build only where its double lies within a few ulps of a float rounding boundary). */
int alva_k_undistort_points_fisheye(alva_ctx*, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                    const double* D4, float* unpx);
int alva_k_project_points_fisheye(alva_ctx*, const double* Xc, int n, const double* K4, const double* D4, float* uv);
/* The same two calls with OpenCV's whole distortion vector: coeffs (HOST) holds ncoeffs = 4, 5, 8, 12 or 14 entries of
 * {k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4, tau_x, tau_y} (what cv::calibrateCamera returns by default and with
 * CALIB_RATIONAL_MODEL, CALIB_THIN_PRISM_MODEL or CALIB_TILTED_MODEL), zero-padded to 14.  The tilt matrices of a non-zero
 * tau_x / tau_y are built once on the host, as OpenCV builds them.  Same shapes, layout, counts and checks as
 * alva_k_undistort_points / alva_k_project_points, and bit-exact with cv::undistortPoints / cv::projectPoints of the vector;
 * (k1, k2, p1, p2) padded with zeros gives exactly their bits.  ALVA_E_INVALID also for another ncoeffs, a non-finite
 * coefficient, or |tau_x| or |tau_y| >= pi/2. */
int alva_k_undistort_points_full(alva_ctx*, const float* px, const int32_t* counts, int nframes, int cap, const double* K4,
                                 const double* coeffs, int ncoeffs, float* unpx);
int alva_k_project_points_full(alva_ctx*, const double* Xc, int n, const double* K4, const double* coeffs, int ncoeffs, float* uv);
/* The rotation-compensated KLT priors of System's gyro mode (alva_system_set_gyro; not in the reference).  For every point i with
 * flag[i] != 0: c = R^T bv[i] (bv [n][3] double, the keypoint's bearing in the previous camera; R9 row-major, the camera's
 * rotation from the previous frame to the current one, HOST array), projected through the lens -- 0 the pinhole, 1 the
 * radial-tangential model (alva_k_project_points), 2 the fisheye model (alva_k_project_points_fisheye), 3 the full vector
 * (alva_k_project_points_full; D4 then holds all 14 coefficients) -- and written to
 * prior [n][2] float (8-byte aligned) with rotated[i] = 1 only when c.z > 0 and the projection lies inside the w x h image
 * (0 <= u < w, 0 <= v < h).  Every other point keeps its prior, with rotated[i] = 0.  K4 / D4 / R9 are host arrays (D4 NULL:
 * zeros); bv, flag, prior, rotated are device arrays; n = 0 is a no-op.  Bit-exact with the host build of the same arithmetic
 * (camera_model.h).  ALVA_E_INVALID for a bad pointer, size or lens, a zero focal length or a non-finite coefficient. */
int alva_k_rotate_priors(alva_ctx*, const double* bv, const uint8_t* flag, int n, int w, int h, const double* K4, const double* D4,
                         int lens, const double* R9, float* prior, uint8_t* rotated);

/* cv::FAST(gray, thr, nms=true, TYPE_9_16) on each frame (opencv features2d/src/fast.cpp:496); thr is clamped to 0..255 as
 * cv::FAST does.  Asynchronous on the context's stream.  keys[f*cap + i]: packed corner keys; counts[f] = the true number found.
 * It may exceed cap: then cap of the corners are stored, and which ones is unspecified (the caller compares counts[f] with cap;
 * a cap of ceil(w/2) * ceil(h/2), the bound of the strict 3x3 NMS, never overflows).  sorted != 0: the stored keys in
 * row-major order. */
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
 * (edge = 31: orb.cpp:1130) when edge > 0, of the first min(counts[f], cap) keys; result sorted row-major.  When more than
 * out_cap are kept, the first out_cap in row-major order are stored (the same on every call): out_counts[f] =
 * min(kept, out_cap).  n < 0 keeps every key inside the border; n = 0 none. */
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
 * counts[f] = keypoints found (the first out_cap in row-major order are stored).  Order: row-major (y, x) -- the reference's order is
 * whatever std::nth_element leaves, so compare as sets.  flags: ALVA_ORB_FMA selects the blur arithmetic. */
int alva_k_orb_detect(alva_ctx*, const uint8_t* gray, int w, int h, int nframes, int nfeatures, int fast_thr, int flags,
                      float* kp_out, uint8_t* desc, int32_t* counts, int out_cap);

/* Brute-force Hamming 2-NN (BFMatcher(NORM_HAMMING).knnMatch(k=2), features2d/src/matchers.cpp:757;
 * tie rule core/src/batch_distance.cpp:235-248).  q: [nq][32], t: [nt][32] bytes;
 * out[4*i] = {idx0, dist0, idx1, dist1} (int32; -1 when nt < 2).  DEVICE pointers, each 16-byte aligned; nq >= 1 and
 * 1 <= nt < 2^22 (a key holds a 22-bit train index), else ALVA_E_INVALID before anything runs. */
int alva_k_hamming_knn2(alva_ctx*, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out);

/* Batched variant: q is [nbatch][qcap][32] of which only the first counts[b] slots of batch b are live (nbatch >= 1, qcap a
 * positive multiple of 8); out is [nbatch][qcap][4].  counts (device memory) are clamped to [0, qcap]: a count above qcap makes
 * every slot of its batch live, a negative one none.  Every dead slot comes back as four -1s.  Pointers and the limits on nt as
 * alva_k_hamming_knn2. */
int alva_k_hamming_knn2_batch(alva_ctx*, const uint8_t* q, const int32_t* counts, int nbatch, int qcap,
                              const uint8_t* t, int nt, int32_t* out);

/* Hamming 2-NN over GROUPS of descriptors (System's relocalisation: a map point is a group of the descriptors its keyframes
 * gave it).  q [nq][32]; the table is CSR: desc_start [n_grp + 1] (ascending, desc_start[0] = 0, desc_start[n_grp] = n_rows)
 * row offsets into desc [n_rows][32].  A group's distance to a query is the minimum over its rows; groups without rows are never
 * candidates.  out [nq][4] = {grp0, d0, grp1, d1} (int32, 16-byte aligned): the nearest and second-nearest groups, ties to the
 * lower group index, -1 / -1 where there are fewer than 1 / 2 candidates.  DEVICE pointers (q, desc 16-byte aligned);
 * nq <= 65535. */
int alva_k_hamming_knn2_grouped(alva_ctx*, const uint8_t* q, int nq, const int32_t* desc_start, int n_grp, const uint8_t* desc,
                                int n_rows, int32_t* out);

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
 * 8 <= cell <= 64 (the reference uses 40), any grid the frame size allows.  A current keypoint in (-cell, 0) marks row /
 * column 0 occupied, as the reference's truncating cell index does.  Bit-identical to the reference run with
 * cv::setNumThreads(1). */
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

/* P3P-RANSAC with the arguments and outputs of alva_k_p3p_lmeds: the same sampler and Kneip hypotheses (the same seed draws the
 * same hypotheses), each scored by its number of inliers (bearing distance <= 1 - cos(atan(err_px / focal))); the first
 * hypothesis with the strictly largest count is the model (none without inliers).  Survives outlier shares where LMedS
 * breaks down (> 50 %): System's relocalisation, whose matches carry no pose prior.  cap <= 8192, max_iter <= 1024.
 * info (optional) [nprob][4] = {success (>= 5 inliers and R orthogonal), #inliers, index of the selected hypothesis (-1: none),
 * #draws}. */
int alva_k_p3p_ransac(alva_ctx*, int nprob, int cap, const double* bvs, const double* wpts, const int32_t* counts,
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
/* The same through the equidistant fisheye model: fisheye4 = {k1, k2, k3, k4} (HOST array, required; zeros are a valid lens)
 * projects the map point and the co-projection errors as alva_k_project_points_fisheye does.  ALVA_E_INVALID for a NULL or
 * non-finite fisheye4. */
int alva_k_match_to_map_fisheye(alva_ctx*, int w, int h, int cell, double fx, double fy, double cx, double cy, const double* Twc_cur,
                                int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf, const double* kf_Twc, int n_mp,
                                const double* mp_wpt, const uint8_t* mp_is3d, const int32_t* obs_start, const int32_t* obs_kf,
                                const float* obs_px, const int32_t* desc_start, const uint8_t* desc, int n_local, const int32_t* local_mp,
                                float max_proj_err, float dist_ratio, int32_t* kp_match, float* kp_dist, int32_t* n_match,
                                const double* fisheye4);
/* The same through OpenCV's whole distortion vector (coeffs / ncoeffs as alva_k_undistort_points_full, HOST): the map point and
 * the co-projection errors are projected as alva_k_project_points_full does.  ALVA_E_INVALID for a vector it refuses. */
int alva_k_match_to_map_full(alva_ctx*, int w, int h, int cell, double fx, double fy, double cx, double cy, const double* Twc_cur,
                             int n_kp, const int32_t* kp_mp, const float* kp_px, int nkp3d, int n_kf, const double* kf_Twc, int n_mp,
                             const double* mp_wpt, const uint8_t* mp_is3d, const int32_t* obs_start, const int32_t* obs_kf,
                             const float* obs_px, const int32_t* desc_start, const uint8_t* desc, int n_local, const int32_t* local_mp,
                             float max_proj_err, float dist_ratio, int32_t* kp_match, float* kp_dist, int32_t* n_match,
                             const double* coeffs, int ncoeffs);
/* Projection-gated matching of a tracked frame's fresh detections against a frozen map table (the re-acquisition of
 * alva_system_set_localisation_only; not in the reference).  The gates of Mapper::matchToMap (mapper.cpp:354-587) for queries
 * without a map point of their own.  Device pointers except coef4 (HOST, required for lens 1 / 2 / 3):
 *   camera w, h, fx, fy, cx, cy; lens 0 pinhole, 1 radial-tangential (k1 k2 p1 p2), 2 fisheye (k1..k4), 3 OpenCV's whole
 *   vector (coef4 then holds 14 coefficients, as alva_k_undistort_points_full's); cell: the grid cell
 *   Twc [7] = [t, q(x,y,z,w)] of the frame
 *   table (the relocalisation table's layout, ascending map point id): wpt [n_mp][3] FP64, CSR desc_start [n_mp + 1] ->
 *   desc [rows][32] (16-byte aligned); skip [n_mp] (optional): 1 = leave the row out (map points the frame already tracks)
 *   queries: q_px [nq][2] FP32 distorted pixels as the detector returns them, q_desc [nq][32] (16-byte aligned), q_kept [nq]
 *   (0 = never a candidate: no ORB descriptor, or a lens drop); radius: candidate distance in px (2, or 4 below 30 3-D
 *   keypoints).
 * Per row: skip, c = Tcw X with c_z >= 0.1 and |c_z| / |c| >= cos(atan(max(w / 2fx, h / 2fy))), the lens projection inside
 * the image; candidates: the kept queries within radius, found through every grid cell the radius disc touches (the
 * reference's getSurroundingKeypoints scans only the projection's cell and its upper-left neighbours); distance: the minimum
 * Hamming distance over the row's descriptors; best / second best with `<=` from 51.2 in ascending query order, the best
 * rejected if a second exists and 0.9 * second < best.  Per query: the row with the smallest distance, the highest row among
 * equal ones.  Out: q_row [nq] the matched row or -1, q_dist [nq] its distance or -1.  One-to-one and deterministic; the
 * CPU restatement is oracle/reacquire_oracle.c.  Three launches, no synchronisation. */
int alva_k_match_frame_to_map(alva_ctx*, int w, int h, int cell, double fx, double fy, double cx, double cy, int lens,
                              const double* coef4, const double* Twc, int n_mp, const double* wpt, const int32_t* desc_start,
                              const uint8_t* desc, const uint8_t* skip, int nq, const float* q_px, const uint8_t* q_desc,
                              const uint8_t* q_kept, float radius, int32_t* q_row, int32_t* q_dist);

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
 * Setting any option to a new value makes alva_pipeline capture its graphs again, so the kernels an option selects take
 * effect at the next step (see alva_pipeline_graph_stats).
 * "knn_qpw" = 4 | 8: queries a warp of the Hamming matcher keeps in registers (8: 128 registers / 16 warps per SM;
 * 4: 80 registers / 24 warps per SM).  Results are identical.
 * "knn_mma" = 0 | 1 | 2: the tensor-core formulation of the Hamming matcher (hamming_mma.cu: descriptors expanded to +-1
 * int8, wgmma s8 x s8 -> s32, dot = 256 - 2 * distance): 0 never, 1 for large query sets (default), 2 always.  Results
 * are identical.  "knn_mma_kind" = 0 | 1 | 2: operand kind of that kernel (2: 1-bit rows [a | ~a] x [~b | b], wgmma
 * .b1.and.popc, the int32 accumulator is the distance -- default; 0: +-1 as int8, int32 accumulators; 1: +-1.0 as E4M3, fp32
 * accumulators).  "knn_mma_mode" = 0 | 1 | 2: the shared-memory operand layout of kinds 0 and 1 (0 no swizzle, 1 128-byte
 * swizzle, 2 a debugging variant of 0 for the wgmma descriptor convention, whose results are not guaranteed); kind 2 always
 * uses the unswizzled layout.
 * "frontend_variant" = 2 | 0: the fused front-end kernel (2: frontend_tile_kernel_v2, default; 0: the round-1 kernel, which
 * also serves geometries a TMA tensor map cannot express).  Results are identical.
 * "frontend_prefetch" = 0 | 1: variant 2 also pulls the tile at the same position a few frames ahead into L2 (TMA prefetch)
 * while it works on its own (default 0).  Results are identical. */
int alva_set_option(const char* name, int value);
/* Debugging aid: the tensor-core matcher unconditionally on q [nq][32] x t [nt][32] (device pointers, 16-byte aligned);
 * dbg_dev (optional, 16384 int32 of device memory) receives the raw accumulators of the first 128 x 128 tile: Hamming
 * distances under "knn_mma_kind" 2, dot products 256 - 2 * distance under kinds 0 and 1. */
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
    int nfeatures;          /* retainBest target per frame.  Ties at the n-th best can keep more; a frame has
                               fcap = 1.5 * nfeatures rounded up to 64 feature slots (alva_pipeline_info), and a selection
                               larger than that keeps its first fcap in row-major order.  Every FAST corner of a frame is a
                               candidate (the key capacity is the NMS bound, ceil(w/2) * ceil(h/2)). */
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
/* {CUDA graphs captured so far, graph launches so far, 1 if a capture failed and the pipeline fell back to direct launches}.
 * A graph is replayed only while the context workspaces it baked in and the alva_set_option values are those it was captured
 * under; after a change (a call on the pipeline's context that grew a workspace, another pipeline on that context, an option
 * set to a new value) it is dropped, its frame range runs directly once and is captured again -- the first count includes
 * such re-captures. */
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
 * (system.cpp:163-174), ALVA_STATUS_LOST (4, only with alva_system_set_relocalisation on) or a negative ALVA_E_* code. */
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
/* The equidistant fisheye lens of a configured System (OpenCV's cv::fisheye, k1..k4 on theta): the wide-angle cameras the
 * radial-tangential model cannot describe.  enabled = 1 selects it, with any finite coefficients (zeros are the equidistant
 * projection); enabled = 0 returns to the pinhole.  It is applied where set_distortion's model is -- tracked and detected
 * keypoints are undistorted on the device with cv::fisheye::undistortPoints, the KLT priors of 3-D keypoints and the local-map
 * matcher project with cv::fisheye::projectPoints -- and everything downstream works on undistorted pixels.  A keypoint the
 * model cannot undistort (OpenCV's (-1e6, -1e6)) is dropped: a tracked one as a KLT failure, a detected one is never added;
 * alva_system_lens_drops counts them.  set_distortion and set_fisheye each replace the other's model.  It resets the tracker and
 * the map as reset() does; configure clears it; reset, set_preset, set_clahe and set_relocalisation keep it.  ALVA_E_STATE
 * before configure; ALVA_E_INVALID for a null handle or a non-finite coefficient.  Fields of view of 180 degrees or more are
 * out of its range (OpenCV clamps theta_d to pi/2). */
int  alva_system_set_fisheye(alva_system*, int enabled, double k1, double k2, double k3, double k4);
/* OpenCV's whole distortion vector for a configured System: coeffs (HOST) holds n = 4, 5, 8, 12 or 14 entries of
 * {k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4, tau_x, tau_y}, as cv::calibrateCamera returns them (5 by default; 8, 12, 14
 * with CALIB_RATIONAL_MODEL, CALIB_THIN_PRISM_MODEL, CALIB_TILTED_MODEL).  All zero selects the pinhole; only k1 k2 p1 p2
 * non-zero is exactly set_distortion(k1, k2, p1, p2), in every bit of the trace and the map blob; anything else applies
 * cv::undistortPoints / cv::projectPoints with the whole vector wherever set_distortion's model is applied, bit-exact on the
 * device (alva_k_undistort_points_full).  Like the radial-tangential model it never fails (where it folds back, the pinhole
 * point), so alva_system_lens_drops stays 0.  set_distortion, set_fisheye and set_distortion_coeffs each replace the others'
 * model; it resets the tracker and the map (ending localisation-only); configure clears it; reset, set_preset, set_clahe,
 * set_relocalisation and set_gyro keep it.  ALVA_E_STATE before configure; ALVA_E_INVALID for a null handle, another n, a
 * non-finite coefficient or |tau_x| or |tau_y| >= pi/2.  A refusal changes nothing. */
int  alva_system_set_distortion_coeffs(alva_system*, const double* coeffs, int n);
/* keypoints dropped because the fisheye model could not undistort them, since configure or the last set_distortion /
 * set_fisheye / set_distortion_coeffs (always 0 for the pinhole, the radial-tangential lens and OpenCV's whole vector, lens 3) */
int  alva_system_lens_drops(alva_system*);
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
/* Relocalisation instead of a reset after a tracking loss.  max_lost_frames = 0 (the default): the reference's behaviour -- a
 * failed pose empties the frame and the fourth failure since the last reset discards the map (status 2).  n > 0: the first
 * failed pose after the initialisation freezes the map, the keyframes and the motion model and returns ALVA_STATUS_LOST; every
 * following frame is matched against the whole map (grid detector + ORB, Hamming 2-NN over each map point's keyframe
 * descriptors, distance <= 51 and ratio 0.8, P3P-RANSAC with 512 hypotheses, PnP) and tracking resumes with status 1 once >= 30
 * PnP inliers agree.  After n lost frames in a row the map is discarded as the reference would (status 2).  While lost, pose16
 * holds the last tracked pose and the frame has no keypoints.  configure turns it off; reset, set_preset, set_distortion and
 * set_clahe keep the setting (those that reset the map also end the lost state).  ALVA_E_STATE before configure;
 * ALVA_E_INVALID for a null handle or a negative value. */
#define ALVA_STATUS_LOST 4
int  alva_system_set_relocalisation(alva_system*, int max_lost_frames);
/* Localisation only: track against the current map without ever changing it -- a venue or site map built once, a map shared
 * between devices, AR content that must stay where it was placed.  enabled = 1 freezes the map: no keyframe, no
 * triangulation, no local BA and no keyframe removal; keyframes, map points and the id counters stay as they are.  Map points
 * the tracker loses come back without a keyframe: on the first tracked frame after freezing or after a relocalisation, when
 * the frame's occupied grid cells fall below 0.85 x their count after the last re-acquisition, or when it has fewer than 30
 * 3-D keypoints, the grid detector runs in the empty cells and its ORB-described points are matched against the whole map
 * (alva_k_match_frame_to_map); matched points join the frame as 3-D keypoints and enter the pose on the next frame.  A loss
 * relocalises as usual (status 4, then 1) but the map is never reset, whatever max_lost_frames says; statuses are 1 and 4, never
 * 2.  The usual flow is set_relocalisation(n) -> load_map(blob) -> set_localisation_only(1); a live, initialised session can
 * also freeze its own map (the frame's 2-D keypoints are dropped: only a keyframe could triangulate them).  enabled = 0
 * resumes mapping on the next keyframe decision, with ids continuing from the counters; a frame still lost then gets
 * max_lost_frames frames.  load_map and set_clahe keep the mode (a loaded map stays frozen); configure, reset, set_preset,
 * set_distortion and set_fisheye discard the map and end it.  A refusal changes nothing: ALVA_E_INVALID for a null handle or
 * enabled other than 0 / 1; ALVA_E_STATE before configure, or when enabling with relocalisation off or before the
 * initialisation; alva_system_set_relocalisation(0) returns ALVA_E_STATE while the mode is on.  Disabling is always allowed. */
int  alva_system_set_localisation_only(alva_system*, int enabled);
/* out4 = {mode on, frames re-acquisition ran on, map points it returned to the frame, those of its last run}, since the
 * handle was created */
int  alva_system_localisation_stats(alva_system*, int32_t* out4);
/* Gyro-aided tracking: the gyroscope's rotation between two frames predicts the camera's, so a fast pan (which a 9x9 KLT
 * without a rotation prior loses within a few frames) keeps tracking.  enabled = 1 turns it on; samples then come with the
 * frames through alva_system_find_camera_pose_gyro.
 *   R_ci9: row-major rotation taking IMU-axis vectors to camera axes (omega_c = R_ci omega_i); NULL = identity.  For the W3C
 *          `devicemotion` rotationRate axes (x right, y up, z out of the screen) and a rear camera (x right, y down, z forward)
 *          it is diag(1, -1, -1).
 *   bias3: a constant gyro bias in rad/s on the IMU axes, subtracted from every sample; NULL = zero.
 * Between the previous and the current frame's time stamps omega is taken piecewise linear between samples and integrated
 * piece by piece in double precision (the exact rule is in alvaar_b200/csrc/system_core.h, SystemCore::setGyro).  An interval
 * is covered when omega is known at both ends (interpolated, or held from a sample at most 50 ms away) and no two samples
 * inside it are more than 50 ms apart; a frame whose interval is not covered is tracked exactly as without the mode.  On a
 * covered frame: the motion model's predicted rotation is replaced by the gyro's (its translation kept); every KLT prior that
 * would start at the keypoint's previous position starts at the projection of its bearing turned by that rotation (on the
 * device, alva_k_rotate_priors), where that lies in front of the camera and inside the image; and a lost frame (relocalisation
 * on) reports its last pose turned by the rotation, its translation held -- pose16 and a map saved while lost carry it.
 * enabled = 0 turns it off and drops the samples held.  configure clears it; reset, set_preset, set_clahe, set_distortion,
 * set_fisheye, set_relocalisation, set_localisation_only and load_map keep it.  ALVA_E_STATE before configure;
 * ALVA_E_INVALID for a null handle, enabled other than 0 / 1, a non-finite value, or an R_ci that is not a rotation (an
 * entry of R^T R - I above 1e-9 in magnitude, or a negative determinant).  A refusal changes nothing. */
int  alva_system_set_gyro(alva_system*, int enabled, const double* R_ci9, const double* bias3);
/* alva_system_find_camera_pose_ts with gyro samples.  samples [n][7] in the reference's per-sample layout {t_ms, gx, gy, gz
 * (rad/s), ax, ay, az}: the tail of its JS shim's IMU buffer can be passed unchanged; the accelerometer fields are ignored.
 * Samples may run ahead of t_ms: they are kept for the next frame.  With the mode off the samples are checked and ignored and
 * the call equals alva_system_find_camera_pose_ts bit for bit.  Refused with ALVA_E_INVALID -- no frame processed, nothing
 * changed -- for n < 0, samples NULL with n > 0, a non-finite value, time stamps that decrease within the call, or a sample
 * older than the newest one the handle holds (equal time stamps are allowed: Date.now() has a 1 ms resolution). */
int  alva_system_find_camera_pose_gyro(alva_system*, const uint8_t* rgba, double t_ms, const double* samples, int n, float* pose16);
/* out5 = {frames whose rotation was predicted from the gyro, frames that fell back to the motion model (interval not
 * covered), lost frames whose rotation the gyro carried, KLT priors rotated, KLT priors kept at the previous position
 * (rotated ray behind the camera or outside the image)}, since configure; dR9 (may be NULL) = the last frame's rotation
 * dR_c = R_ci dR R_ci^T, row-major (identity when its interval was not covered). */
int  alva_system_gyro_stats(alva_system*, int32_t* out5, double* dR9);
/* The map as a self-contained byte string, to resume a session in a new handle or to start another stream in this one's map and
 * coordinate frame.
 *
 * alva_system_save_map writes the map into buf (cap bytes) and its length into *bytes.  buf = NULL only queries the length; a
 * short buffer returns ALVA_E_CAPACITY with *bytes set.  It is allowed once the system is initialised, also while lost (else
 * ALVA_E_STATE), and changes nothing.
 *
 * alva_system_load_map replaces the map with a blob's and enters the lost state: the next frames return ALVA_STATUS_LOST with
 * the saved pose until one relocalises into the map (status 1; new keyframe and map point ids continue from the saved
 * counters), and after max_lost_frames failures the map is discarded (status 2).  It needs relocalisation on
 * (alva_system_set_relocalisation > 0), else ALVA_E_STATE.  The whole blob is checked before anything changes; a blob that
 * fails a check returns ALVA_E_INVALID and leaves the system as it was: bad magic / version, a byte count other than `bytes`,
 * a camera, lens or grid cell size other than the configured ones, truncated or trailing data, ids not strictly ascending,
 * counters above 2^30 or not above every stored id, a reference to an id never issued, a non-finite number, a rotation that
 * is not a unit quaternion (|q|^2 off 1 by more than 1e-9) or a flag other than 0 / 1.
 * configure, reset, set_preset, set_distortion and set_fisheye discard a loaded map as they discard any map.
 *
 * Format, version 1: little-endian, fixed-width fields, no padding (i32 / u32 / u64 / f32 / f64, u8 flags 0 or 1).
 *   header     "ALMP", u32 version = 1, u64 total bytes, u32 keyframe count, u32 map point count
 *   camera     i32 w, h; f64 fx, fy, cx, cy; i32 lens (0 pinhole, 1 radial-tangential, 2 fisheye, 3 OpenCV's whole vector);
 *              f64 coefficients [4] for lenses 0..2, [14] for lens 3
 *   grid       i32 cell size of the preset
 *   counters   i32 n_kf_ids, n_mp_ids (the next ids), n_kf (= the keyframe count)
 *   pose       f64 t [3], q [4] (x y z w): the pose the lost frames report
 *   keyframes, ascending id:
 *              i32 id; i32 age (frames from the keyframe's frame to the saving frame); f64 Twc t [3], q [4];
 *              u32 n, then n keypoints, ascending id: i32 id; f32 px, py, ux, uy; f64 bv [3]; u8 is3d, has_desc; u8 desc [32]
 *              u32 n, then n covisibility pairs, ascending keyframe id: i32 keyframe id, i32 count
 *              u32 n, then n local map point ids, ascending
 *   map points, ascending id:
 *              i32 id, anchor keyframe id; u8 observed, is3d; f64 inverse depth; f64 p [3]
 *              u32 n, then n observing keyframe ids, ascending
 *              u32 n, then n (i32 keyframe id, u8 desc [32], f32 descriptor distance sum), ascending keyframe id
 *              u8 has_desc; u8 desc [32]
 * References (3-D keypoints' map points, anchors, observations, keyframe descriptors, covisibility, local maps) name issued
 * ids, 0 <= id < the counter: a record of the blob, or a keyframe or map point removed since.  A live map names removed ones
 * once keyframes leave it (keyframe filtering, the 30-keyframe window); the tracker looks every id up and skips missing
 * records, so they are kept and the loaded map equals the saved one.  Rebuilt on load, not stored: a
 * keyframe's grid, cell counts and keypoint counts (from its keypoints, inserted in ascending id order, and the cell size); Tcw
 * (the inverse of Twc); the current frame (empty, as a lost frame; its keyframe is the newest, n_kf_ids - 1).  `observed` is
 * saved as the lost state holds it (cleared for the current frame's points).  Frame ids restart at 0 in the loading session:
 * a keyframe's frame id becomes -1 - age.  Time stamps are not stored (the motion model restarts after a relocalisation). */
int  alva_system_save_map(alva_system*, uint8_t* buf, size_t cap, size_t* bytes);
int  alva_system_load_map(alva_system*, const uint8_t* buf, size_t bytes);
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
