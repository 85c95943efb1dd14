"""ctypes binding of libalva_b200.so (include/alva_b200.h).  Device buffers are torch CUDA tensors;
only their data pointers cross the boundary."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
ORB_FMA = 1
ORB_IC_ANGLE = 2
ORB_HARRIS = 4


class AlvaError(RuntimeError):
    pass


def lib_path():
    return os.path.join(_HERE, "libalva_b200.so")


_lib = None


def lib():
    """Load libalva_b200.so (built in-tree by __graft_entry__.build()).  Fails loudly if it is absent."""
    global _lib
    if _lib is None:
        p = lib_path()
        if not os.path.exists(p):
            raise AlvaError(f"{p} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(there is no CPU fallback)")
        L = C.CDLL(p)
        vp, i32, i64 = C.c_void_p, C.c_int, C.c_longlong
        L.alva_version.restype = i32
        L.alva_last_error.restype = C.c_char_p
        L.alva_ctx_create.restype = vp
        L.alva_ctx_create.argtypes = [i32, vp]
        L.alva_ctx_destroy.argtypes = [vp]
        L.alva_ctx_sync.argtypes = [vp]
        L.alva_ctx_launches.restype = i64
        L.alva_ctx_launches.argtypes = [vp]
        L.alva_k_gray.argtypes = [vp, vp, vp, i32, i32, i32]
        L.alva_k_pyrdown.argtypes = [vp, vp, vp, i32, i32, i32]
        L.alva_k_fast9.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, i32, i32]
        L.alva_k_frontend.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp, i32, vp, vp, i32, i32]
        L.alva_set_option.argtypes = [C.c_char_p, i32]
        L.alva_k_retain_best.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, i32]
        for name, args in _OPTIONAL.items():
            if hasattr(L, name):
                getattr(L, name).argtypes = args
        _lib = L
    return _lib


_vp, _i32 = C.c_void_p, C.c_int
_OPTIONAL = {
    "alva_k_orb_blur": [_vp, _vp, _vp, _i32, _i32, _i32, _i32],
    "alva_k_orb_describe": [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _i32, _i32, _vp, _vp, _vp],
    "alva_k_hamming_knn2": [_vp, _vp, _i32, _vp, _i32, _vp],
    "alva_k_hamming_knn2_batch": [_vp, _vp, _vp, _i32, _i32, _vp, _i32, _vp],
    "alva_h_frontend": [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _i32],
    "alva_k_scharr": [_vp, _vp, _vp, _i32, _i32, _i32],
    "alva_k_clahe": [_vp, _vp, _vp, _i32, _i32, _i32, C.c_double, _i32, _i32],
    "alva_k_detect_grid": [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _i32],
    "alva_k_corner_subpix": [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _i32],
    "alva_k_match_to_map": [_vp, _i32, _i32, _i32, C.c_double, C.c_double, C.c_double, C.c_double, _vp, _i32, _vp, _vp, _i32, _i32, _vp,
                            _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, C.c_float, C.c_float, _vp, _vp, _vp],
    "alva_k_match_to_map_dist": [_vp, _i32, _i32, _i32, C.c_double, C.c_double, C.c_double, C.c_double, _vp, _i32, _vp, _vp, _i32, _i32,
                                 _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, C.c_float, C.c_float, _vp, _vp, _vp, _vp],
    "alva_k_undistort_points": [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp],
    "alva_k_project_points": [_vp, _vp, _i32, _vp, _vp, _vp],
    "alva_k_match_to_map_fisheye": [_vp, _i32, _i32, _i32, C.c_double, C.c_double, C.c_double, C.c_double, _vp, _i32, _vp, _vp, _i32, _i32,
                                    _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, C.c_float, C.c_float, _vp, _vp, _vp, _vp],
    "alva_k_match_frame_to_map": [_vp, _i32, _i32, _i32, C.c_double, C.c_double, C.c_double, C.c_double, _i32, _vp, _vp, _i32, _vp, _vp,
                                  _vp, _vp, _i32, _vp, _vp, _vp, C.c_float, _vp, _vp],
    "alva_k_undistort_points_fisheye": [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp],
    "alva_k_project_points_fisheye": [_vp, _vp, _i32, _vp, _vp, _vp],
    "alva_k_rotate_priors": [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _vp, _vp],
    "alva_k_p3p_lmeds": [_vp, _i32, _i32, _vp, _vp, _vp, _i32, C.c_float, C.c_float, C.c_float, C.c_uint32, _vp, _vp, _vp],
    "alva_k_p3p_ransac": [_vp, _i32, _i32, _vp, _vp, _vp, _i32, C.c_float, C.c_float, C.c_float, C.c_uint32, _vp, _vp, _vp],
    "alva_k_hamming_knn2_grouped": [_vp, _vp, _i32, _vp, _i32, _vp, _i32, _vp],
    "alva_k_pnp": [_vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, C.c_double, C.c_double, _i32, _i32, _i32, _vp, _vp],
    "alva_k_essential_5pt": [_vp, _i32, _i32, _vp, _vp, _vp, _i32, C.c_float, _i32, C.c_float, C.c_float, C.c_uint32, _vp, _vp, _vp],
    "alva_k_triangulate": [_vp, _vp, _vp, _vp, _i32, _vp],
    "alva_k_klt_lk": [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, C.c_double, _i32, _vp, _vp, _vp, _i32, _vp, _vp],
    "alva_k_klt_fb": [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.c_float, C.c_float, _vp, _vp, _vp, _i32, _vp],
    "alva_k_harris": [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _i32, _vp],
    "alva_k_orb_detect": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _i32],
    "alva_k_ba_solve": [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_double, _i32, _vp],
    "alva_k_ba_local": [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_double, C.c_double,
                        _i32, _vp, _vp],
    "alva_k_ba_linearize": [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_double, _vp, _vp, _vp, _vp, _vp],
    "alva_k_ba_schur_dump": [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_double, _i32, _vp, _vp,
                             _vp],
}


def key_x(k):
    return (k >> 8) & 0xFFF


def key_y(k):
    return (k >> 20) & 0xFFF


def key_score(k):
    return k & 0xFF


def unpack_keys(keys):
    """packed uint32/int64 numpy array -> (n, 3) int32 array of (x, y, score)."""
    import numpy as np
    k = np.asarray(keys).astype(np.int64) & 0xFFFFFFFF
    return np.stack([(k >> 8) & 0xFFF, (k >> 20) & 0xFFF, k & 0xFF], -1).astype(np.int32)


def _ptr(t):
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def _f64x4(v):
    """four host doubles (intrinsics or distortion coefficients)"""
    return (C.c_double * 4)(*[float(x) for x in v])


class Context:
    """One CUDA device + stream (alva_ctx).  Methods mirror the alva_k_* entry points on torch tensors."""

    def __init__(self, device=0, stream=None):
        """stream: None -> the context creates its own non-blocking stream; an integer cudaStream_t handle otherwise.
        Handle 0 (torch's default stream) is passed as cudaStreamLegacy (0x1): in the C ABI a NULL stream means
        "create one", so the legacy default stream has to be named explicitly."""
        self.L = lib()
        if stream is not None and int(stream) == 0:
            stream = 1   # cudaStreamLegacy
        h = self.L.alva_ctx_create(int(device), C.c_void_p(int(stream)) if stream is not None else None)
        if not h:
            raise AlvaError(self.L.alva_last_error().decode())
        self.h = C.c_void_p(h)
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.L.alva_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc, allow_capacity=False):
        if rc != 0 and not (allow_capacity and rc == -3):
            raise AlvaError(f"rc={rc}: {self.L.alva_last_error().decode()}")
        return rc

    def sync(self):
        self._chk(self.L.alva_ctx_sync(self.h))

    @property
    def launches(self):
        return int(self.L.alva_ctx_launches(self.h))

    # ---- stages -------------------------------------------------------------------------------
    def gray(self, rgba, gray, w, h, n):
        self._chk(self.L.alva_k_gray(self.h, _ptr(rgba), _ptr(gray), w, h, n))

    def pyrdown(self, src, dst, w, h, n):
        self._chk(self.L.alva_k_pyrdown(self.h, _ptr(src), _ptr(dst), w, h, n))

    def fast9(self, gray, w, h, n, thr, keys, counts, cap, sorted_=True):
        self._chk(self.L.alva_k_fast9(self.h, _ptr(gray), w, h, n, thr, _ptr(keys), _ptr(counts), cap,
                                      1 if sorted_ else 0))

    def frontend(self, rgba, w, h, n, l0, l1, l2, l3, thr, keys, counts, cap, sorted_=False):
        self._chk(self.L.alva_k_frontend(self.h, _ptr(rgba), w, h, n, _ptr(l0), _ptr(l1), _ptr(l2), _ptr(l3),
                                         thr, _ptr(keys), _ptr(counts), cap, 1 if sorted_ else 0))

    def retain_best(self, keys, counts, cap, n, w, h, nkeep, edge, out_keys, out_counts, out_cap):
        self._chk(self.L.alva_k_retain_best(self.h, _ptr(keys), _ptr(counts), cap, n, w, h, nkeep, edge,
                                            _ptr(out_keys), _ptr(out_counts), out_cap))

    def orb_blur(self, gray, blurred, w, h, n, flags=0):
        self._chk(self.L.alva_k_orb_blur(self.h, _ptr(gray), _ptr(blurred), w, h, n, flags))

    def orb_describe(self, gray, blurred, w, h, n, pts, npts_per_frame, npts, flags, desc, kept, angles=None):
        self._chk(self.L.alva_k_orb_describe(self.h, _ptr(gray), _ptr(blurred), w, h, n, _ptr(pts),
                                             _ptr(npts_per_frame), npts, flags, _ptr(desc), _ptr(kept),
                                             _ptr(angles)))

    def hamming_knn2(self, q, nq, t, nt, out):
        self._chk(self.L.alva_k_hamming_knn2(self.h, _ptr(q), nq, _ptr(t), nt, _ptr(out)))

    def scharr(self, gray, deriv, w, h, nframes=1):
        self._chk(self.L.alva_k_scharr(self.h, _ptr(gray), _ptr(deriv), w, h, nframes))

    def clahe(self, src, dst, w, h, nframes, clip_limit, tiles_x, tiles_y):
        """cv::createCLAHE(clip_limit, (tiles_x, tiles_y))->apply on [nframes][h][w] uint8 frames; dst may be src"""
        self._chk(self.L.alva_k_clahe(self.h, _ptr(src), _ptr(dst), w, h, nframes, float(clip_limit), tiles_x, tiles_y))

    @staticmethod
    def _ptr_table(levels):
        """host array of device pointers (one per pyramid level)"""
        return (C.c_void_p * len(levels))(*[t.data_ptr() for t in levels])

    def klt_lk(self, prev_img, prev_der, cur_img, w, h, nframes, levels, pts, nxt, npts, status, err=None, win=9,
               max_count=30, epsilon=0.01, use_initial=True, npts_per_frame=None):
        """cv::calcOpticalFlowPyrLK on prebuilt pyramids (lists of per-level tensors) -- see alva_k_klt_lk."""
        self._chk(self.L.alva_k_klt_lk(self.h, self._ptr_table(prev_img), self._ptr_table(prev_der), self._ptr_table(cur_img),
                                       w, h, nframes, len(prev_img) - 1, levels, win, max_count, epsilon,
                                       1 if use_initial else 0, _ptr(pts), _ptr(nxt), _ptr(npts_per_frame), npts,
                                       _ptr(status), _ptr(err)))

    def klt_fb(self, prev_img, prev_der, cur_img, cur_der, w, h, nframes, levels, pts, priors, npts, good, win=9,
               error_value=30.0, max_fb_dist=0.5, npts_per_frame=None):
        """FeatureTracker::fbKltTracking, fused -- see alva_k_klt_fb."""
        self._chk(self.L.alva_k_klt_fb(self.h, self._ptr_table(prev_img), self._ptr_table(prev_der), self._ptr_table(cur_img),
                                       self._ptr_table(cur_der), w, h, nframes, len(prev_img) - 1, levels, win, error_value,
                                       max_fb_dist, _ptr(pts), _ptr(priors), _ptr(npts_per_frame), npts, _ptr(good)))

    def detect_grid(self, gray, w, h, nframes, cell, cur, ncur, cur_cap, roi, quality, out, out_int, counts, out_cap):
        """FeatureExtractor::detectFeaturePoints, batched -- see alva_k_detect_grid.  roi: 4 python ints (host)."""
        r = (C.c_int32 * 4)(*[int(v) for v in roi])
        self._chk(self.L.alva_k_detect_grid(self.h, _ptr(gray), w, h, nframes, cell, _ptr(cur), _ptr(ncur), cur_cap, r,
                                            _ptr(quality), _ptr(out), _ptr(out_int), _ptr(counts), out_cap))

    def corner_subpix(self, gray, w, h, nframes, pts, counts, cap):
        self._chk(self.L.alva_k_corner_subpix(self.h, _ptr(gray), w, h, nframes, _ptr(pts), _ptr(counts), cap))

    def match_to_map(self, w, h, cell, K, Twc_cur, kp_mp, kp_px, nkp3d, kf_Twc, mp_wpt, mp_is3d, obs_start, obs_kf, obs_px,
                     desc_start, desc, local_mp, kp_match, kp_dist, n_match, max_proj_err=2.0, dist_ratio=0.2, dist=None, fisheye=None):
        """Mapper::matchToMap on flat device arrays -- see alva_k_match_to_map; dist = (k1, k2, p1, p2): the lens-distorted
        projections of alva_k_match_to_map_dist; fisheye = (k1, k2, k3, k4): those of the equidistant fisheye model
        (alva_k_match_to_map_fisheye)."""
        args = (self.h, w, h, cell, K[0], K[1], K[2], K[3], _ptr(Twc_cur), kp_mp.numel(), _ptr(kp_mp), _ptr(kp_px), nkp3d,
                kf_Twc.shape[0], _ptr(kf_Twc), mp_wpt.shape[0], _ptr(mp_wpt), _ptr(mp_is3d), _ptr(obs_start), _ptr(obs_kf),
                _ptr(obs_px), _ptr(desc_start), _ptr(desc), local_mp.numel(), _ptr(local_mp), max_proj_err, dist_ratio,
                _ptr(kp_match), _ptr(kp_dist), _ptr(n_match))
        if fisheye is not None:
            if dist is not None:
                raise ValueError("match_to_map: dist and fisheye are two lens models; give one")
            self._chk(self.L.alva_k_match_to_map_fisheye(*args, _f64x4(fisheye)))
        elif dist is None:
            self._chk(self.L.alva_k_match_to_map(*args))
        else:
            self._chk(self.L.alva_k_match_to_map_dist(*args, _f64x4(dist)))

    def match_frame_to_map(self, w, h, cell, K, Twc, wpt, desc_start, desc, q_px, q_desc, q_kept, q_row, q_dist, radius=2.0, skip=None,
                           lens=0, coef=None):
        """the frozen map's re-acquisition of fresh detections -- see alva_k_match_frame_to_map.  Device tensors: Twc [7] float64,
        wpt [n][3] float64, desc_start [n + 1] int32, desc [rows][32] uint8, skip [n] uint8 or None, q_px [nq][2] float32,
        q_desc [nq][32] uint8, q_kept [nq] uint8; out q_row / q_dist [nq] int32.  lens 0 pinhole, 1 radial-tangential, 2 fisheye
        with coef = its four coefficients."""
        self._chk(self.L.alva_k_match_frame_to_map(self.h, w, h, cell, K[0], K[1], K[2], K[3], lens, _f64x4(coef) if lens else None,
                                                   _ptr(Twc), wpt.shape[0], _ptr(wpt), _ptr(desc_start), _ptr(desc), _ptr(skip),
                                                   q_px.shape[0], _ptr(q_px), _ptr(q_desc), _ptr(q_kept), float(radius), _ptr(q_row),
                                                   _ptr(q_dist)))

    def undistort_points(self, px, counts, nframes, cap, K, dist, unpx):
        """cv::undistortPoints(px, unpx, K, D, K) for px [nframes][cap][2] float32 (counts: int32 [nframes] device tensor or None
        = cap points per frame) -- see alva_k_undistort_points.  K = (fx, fy, cx, cy), dist = (k1, k2, p1, p2)."""
        self._chk(self.L.alva_k_undistort_points(self.h, _ptr(px), _ptr(counts), nframes, cap, _f64x4(K), _f64x4(dist), _ptr(unpx)))

    def project_points(self, Xc, n, K, dist, uv):
        """CameraCalibration::projectCamToImageDist of n camera-frame points Xc [n][3] float64 into uv [n][2] float32 -- see
        alva_k_project_points."""
        self._chk(self.L.alva_k_project_points(self.h, _ptr(Xc), n, _f64x4(K), _f64x4(dist), _ptr(uv)))

    def undistort_points_fisheye(self, px, counts, nframes, cap, K, k4, unpx):
        """cv::fisheye::undistortPoints(px, unpx, K, D, noArray(), K) -- see alva_k_undistort_points_fisheye; k4 = (k1, k2, k3, k4).
        Points the model cannot undistort come back as (-1e6, -1e6)."""
        self._chk(self.L.alva_k_undistort_points_fisheye(self.h, _ptr(px), _ptr(counts), nframes, cap, _f64x4(K), _f64x4(k4), _ptr(unpx)))

    def project_points_fisheye(self, Xc, n, K, k4, uv):
        """cv::fisheye::projectPoints of the float points (x/z, y/z, 1) -- see alva_k_project_points_fisheye."""
        self._chk(self.L.alva_k_project_points_fisheye(self.h, _ptr(Xc), n, _f64x4(K), _f64x4(k4), _ptr(uv)))

    def rotate_priors(self, bv, flag, n, w, h, K, D4, lens, R9, prior, rotated):
        """System's gyro-rotated KLT priors -- see alva_k_rotate_priors; K / D4 (None: zeros) / R9 on the host, lens 0 pinhole,
        1 radial-tangential, 2 fisheye."""
        R = (C.c_double * 9)(*[float(v) for v in R9])
        self._chk(self.L.alva_k_rotate_priors(self.h, _ptr(bv), _ptr(flag), n, w, h, _f64x4(K), None if D4 is None else _f64x4(D4), lens, R,
                                              _ptr(prior), _ptr(rotated)))

    def p3p_lmeds(self, nprob, cap, bvs, wpts, counts, Twc_out, outlier, info=None, max_iter=100, err_px=3.0, fx=1.0, fy=1.0,
                  seed=12345):
        """MultiViewGeometry::p3pRansac (Kneip P3P + LMedS), batched -- see alva_k_p3p_lmeds."""
        self._chk(self.L.alva_k_p3p_lmeds(self.h, nprob, cap, _ptr(bvs), _ptr(wpts), _ptr(counts), max_iter, err_px, fx, fy,
                                          seed, _ptr(Twc_out), _ptr(outlier), _ptr(info)))

    def p3p_ransac(self, nprob, cap, bvs, wpts, counts, Twc_out, outlier, info=None, max_iter=512, err_px=3.0, fx=1.0, fy=1.0,
                   seed=12345):
        """P3P-RANSAC (the hypotheses of p3p_lmeds scored by inlier count), batched -- see alva_k_p3p_ransac."""
        self._chk(self.L.alva_k_p3p_ransac(self.h, nprob, cap, _ptr(bvs), _ptr(wpts), _ptr(counts), max_iter, err_px, fx, fy,
                                           seed, _ptr(Twc_out), _ptr(outlier), _ptr(info)))

    def hamming_knn2_grouped(self, q, nq, desc_start, n_grp, desc, n_rows, out):
        """Hamming 2-NN over CSR groups of descriptors (min over a group's rows) -- see alva_k_hamming_knn2_grouped."""
        self._chk(self.L.alva_k_hamming_knn2_grouped(self.h, _ptr(q), nq, _ptr(desc_start), n_grp, _ptr(desc), n_rows, _ptr(out)))

    def essential_5pt(self, nprob, cap, bv1, bv2, counts, Rt_out, outlier, info=None, max_iter=100, err_px=3.0, optimize=True,
                      fx=1.0, fy=1.0, seed=12345):
        """MultiViewGeometry::compute5ptEssentialMatrix (Nister 5-point RANSAC + refinement), batched -- see alva_k_essential_5pt."""
        self._chk(self.L.alva_k_essential_5pt(self.h, nprob, cap, _ptr(bv1), _ptr(bv2), _ptr(counts), max_iter, err_px,
                                              int(optimize), fx, fy, seed, _ptr(Rt_out), _ptr(outlier), _ptr(info)))

    def triangulate(self, Tlr, bvl, bvr, n, out):
        """MultiViewGeometry::triangulate (mid-point) for n bearing-vector pairs -- see alva_k_triangulate."""
        self._chk(self.L.alva_k_triangulate(self.h, _ptr(Tlr), _ptr(bvl), _ptr(bvr), n, _ptr(out)))

    def pnp(self, nprob, cap, K, uv, X, counts, poses, outlier, summary, huber_delta, chi2_thr, max_iter=5, use_robust=True,
            apply_l2=True):
        """MultiViewGeometry::ceresPnP, batched -- see alva_k_pnp."""
        self._chk(self.L.alva_k_pnp(self.h, nprob, cap, _ptr(K), _ptr(uv), _ptr(X), _ptr(counts), _ptr(poses), huber_delta,
                                    chi2_thr, max_iter, 1 if use_robust else 0, 1 if apply_l2 else 0, _ptr(outlier),
                                    _ptr(summary)))

    def hamming_knn2_batch(self, q, counts, nbatch, qcap, t, nt, out):
        self._chk(self.L.alva_k_hamming_knn2_batch(self.h, _ptr(q), _ptr(counts), nbatch, qcap, _ptr(t), nt, _ptr(out)))

    def harris(self, gray, w, h, nframes, pts, npts_per_frame, npts, resp):
        self._chk(self.L.alva_k_harris(self.h, _ptr(gray), w, h, nframes, _ptr(pts), _ptr(npts_per_frame), npts, _ptr(resp)))

    def orb_detect(self, gray, w, h, nframes, nfeatures, fast_thr, flags, kp_out, desc, counts, out_cap):
        """ORB::detectAndCompute (nlevels 1, HARRIS_SCORE) -- see alva_k_orb_detect."""
        self._chk(self.L.alva_k_orb_detect(self.h, _ptr(gray), w, h, nframes, nfeatures, fast_thr, flags, _ptr(kp_out),
                                           _ptr(desc), _ptr(counts), out_cap))

    def ba_solve(self, nprob, nkf, nlm, nobs, calib, poses, pose_const, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv,
                 huber, max_iter, summary=None):
        self._chk(self.L.alva_k_ba_solve(self.h, nprob, nkf, nlm, nobs, _ptr(calib), _ptr(poses), _ptr(pose_const), _ptr(invd),
                                         _ptr(anch_kf), _ptr(anch_uv), _ptr(obs_kf), _ptr(obs_lm), _ptr(obs_uv), huber,
                                         max_iter, _ptr(summary)))

    def ba_local(self, nprob, nkf, nlm, nobs, calib, poses, pose_const, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv,
                 huber, chi2_thr, max_iter, flags, summary=None):
        """Optimizer::localBA steps 2-4 (solve, remove outliers, conditional re-solve, flag) -- see alva_k_ba_local."""
        self._chk(self.L.alva_k_ba_local(self.h, nprob, nkf, nlm, nobs, _ptr(calib), _ptr(poses), _ptr(pose_const), _ptr(invd),
                                         _ptr(anch_kf), _ptr(anch_uv), _ptr(obs_kf), _ptr(obs_lm), _ptr(obs_uv), huber,
                                         chi2_thr, max_iter, _ptr(flags), _ptr(summary)))

    def ba_linearize(self, nkf, nlm, nobs, calib, poses, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv, huber, res, Ja, Jp,
                     Jd, cost):
        self._chk(self.L.alva_k_ba_linearize(self.h, nkf, nlm, nobs, _ptr(calib), _ptr(poses), _ptr(invd), _ptr(anch_kf),
                                             _ptr(anch_uv), _ptr(obs_kf), _ptr(obs_lm), _ptr(obs_uv), huber, _ptr(res),
                                             _ptr(Ja), _ptr(Jp), _ptr(Jd), _ptr(cost)))

    def ba_schur_dump(self, nprob, nkf, nlm, nobs, calib, poses, pose_const, invd, anch_kf, anch_uv, obs_kf, obs_lm, obs_uv,
                      huber, atomic, S, rhs, info):
        """test hook: the first LM iteration's reduced camera system -- see alva_k_ba_schur_dump"""
        self._chk(self.L.alva_k_ba_schur_dump(self.h, nprob, nkf, nlm, nobs, _ptr(calib), _ptr(poses), _ptr(pose_const),
                                              _ptr(invd), _ptr(anch_kf), _ptr(anch_uv), _ptr(obs_kf), _ptr(obs_lm), _ptr(obs_uv),
                                              huber, int(atomic), _ptr(S), _ptr(rhs), _ptr(info)))
