"""ctypes binding of the System facade (alva_system_*): the reference's public class -- configure / findCameraPose / findPlane /
getFramePoints / reset (src/slam/src/system.hpp:28-38) -- for Python hosts, tests and bench.py.  Thin: every call is one C call."""
import ctypes as C

import numpy as np

from .lib import AlvaError, lib

_vp, _i32, _f64 = C.c_void_p, C.c_int, C.c_double


def _bind():
    L = lib()
    if getattr(L, "_alva_system_bound", False):
        return L
    L.alva_system_create.restype = _vp
    L.alva_system_create.argtypes = [_i32]
    L.alva_system_destroy.argtypes = [_vp]
    L.alva_system_reset.argtypes = [_vp]
    L.alva_system_set_clahe.argtypes = [_vp, _i32, _f64, _i32]
    L.alva_system_set_distortion.argtypes = [_vp] + [_f64] * 4
    L.alva_system_set_fisheye.argtypes = [_vp, _i32] + [_f64] * 4
    L.alva_system_lens_drops.argtypes = [_vp]
    L.alva_system_set_preset.argtypes = [_vp, _i32]
    L.alva_system_set_relocalisation.argtypes = [_vp, _i32]
    L.alva_system_save_map.argtypes = [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]
    L.alva_system_load_map.argtypes = [_vp, C.c_char_p, C.c_size_t]
    L.alva_system_set_localisation_only.argtypes = [_vp, _i32]
    L.alva_system_localisation_stats.argtypes = [_vp, _vp]
    L.alva_system_set_gyro.argtypes = [_vp, _i32, _vp, _vp]
    L.alva_system_find_camera_pose_gyro.argtypes = [_vp, _vp, _f64, _vp, _i32, _vp]
    L.alva_system_gyro_stats.argtypes = [_vp, _vp, _vp]
    L.alva_system_num_matched.argtypes = [_vp]
    L.alva_system_configure.argtypes = [_vp, _i32, _i32] + [_f64] * 8
    L.alva_system_find_camera_pose.argtypes = [_vp, _vp, _vp]
    L.alva_system_find_camera_pose_ts.argtypes = [_vp, _vp, _f64, _vp]
    L.alva_system_find_camera_pose_imu.argtypes = [_vp, _vp, _vp, _vp]
    L.alva_system_find_plane.argtypes = [_vp, _vp, _i32]
    L.alva_system_get_frame_points.argtypes = [_vp, _vp, _i32]
    L.alva_system_get_tracks.argtypes = [_vp, _vp, _vp, _vp, _vp, _i32]
    L.alva_system_get_descriptors.argtypes = [_vp, _vp, _vp, _i32]
    L.alva_system_get_pose.argtypes = [_vp, _vp]
    L.alva_system_get_info.argtypes = [_vp, _vp]
    L.alva_system_pin_buffer.argtypes = [_vp, _vp, C.c_size_t]
    L.alva_system_unpin_buffer.argtypes = [_vp, _vp]
    L.alva_last_error.restype = C.c_char_p
    L._alva_system_bound = True
    return L


class System:
    """One camera stream.  Status codes of find_camera_pose: 1 tracking, 2 the tracker was reset during the call, 3 not
    initialised (the reference's), and 4 lost -- tracking lost, map kept, relocalising (only with set_relocalisation on)."""

    TRACKING, RESET, NOT_INITIALISED, LOST = 1, 2, 3, 4

    def __init__(self, width, height, fx, fy, cx, cy, k1=0.0, k2=0.0, p1=0.0, p2=0.0, device=0):
        self.L = _bind()
        self.h = C.c_void_p(self.L.alva_system_create(device))
        self.width, self.height = width, height
        rc = self.L.alva_system_configure(self.h, width, height, fx, fy, cx, cy, k1, k2, p1, p2)
        if rc != 0:
            msg = self.L.alva_last_error().decode()
            self.close()
            raise AlvaError(f"alva_system_configure -> {rc}: {msg}")

    def close(self):
        if self.h:
            self.L.alva_system_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rgba):
        if rgba.dtype != np.uint8 or rgba.shape != (self.height, self.width, 4) or not rgba.flags["C_CONTIGUOUS"]:
            raise ValueError(f"expected a C-contiguous uint8 array of shape ({self.height}, {self.width}, 4)")

    def find_camera_pose(self, rgba, t_ms=None):
        """-> (status, pose[16] float32 laid out as Utils::toPoseArray); t_ms: the frame's time stamp (default: the system clock)."""
        self._check(rgba)
        pose = np.zeros(16, np.float32)
        if t_ms is None:
            st = self.L.alva_system_find_camera_pose(self.h, rgba.ctypes.data_as(_vp), pose.ctypes.data_as(_vp))
        else:
            st = self.L.alva_system_find_camera_pose_ts(self.h, rgba.ctypes.data_as(_vp), float(t_ms), pose.ctypes.data_as(_vp))
        if st < 0:
            raise AlvaError(f"alva_system_find_camera_pose -> {st}: {self.L.alva_last_error().decode()}")
        return st, pose

    def find_plane(self, iterations=250):
        """-> plane pose[16] (column-major, as the reference writes it) or None"""
        out = np.zeros(16, np.float32)
        return out if self.L.alva_system_find_plane(self.h, out.ctypes.data_as(_vp), iterations) == 1 else None

    def frame_points(self, cap=2048):
        xy = np.zeros((cap, 2), np.int32)
        n = self.L.alva_system_get_frame_points(self.h, xy.ctypes.data_as(_vp), cap)
        return xy[:min(n, cap)]

    def tracks(self, cap=8192):
        """-> ids, px [n, 2], is3d, wpt [n, 3] of every keypoint of the current frame, in the frame's own order"""
        ids = np.zeros(cap, np.int32); px = np.zeros((cap, 2), np.float32); d3 = np.zeros(cap, np.uint8); wp = np.zeros((cap, 3))
        n = min(self.L.alva_system_get_tracks(self.h, ids.ctypes.data_as(_vp), px.ctypes.data_as(_vp), d3.ctypes.data_as(_vp), wp.ctypes.data_as(_vp), cap), cap)
        return ids[:n], px[:n], d3[:n], wp[:n]

    def pose(self):
        T = np.zeros(7)
        self.L.alva_system_get_pose(self.h, T.ctypes.data_as(_vp))
        return T

    def info(self):
        o = np.zeros(8, np.int32)
        self.L.alva_system_get_info(self.h, o.ctypes.data_as(_vp))
        return dict(zip(("frame", "keyframe", "keypoints", "keypoints_3d", "initialised", "keyframes", "occupied_cells", "map_point_ids"), o.tolist()))

    def pin(self, array):
        """page-lock a frame buffer that is reused from call to call (alva_system_pin_buffer).  The array is kept alive
        until unpin() / close(): a garbage-collected buffer would stay registered with the driver."""
        ok = self.L.alva_system_pin_buffer(self.h, array.ctypes.data_as(_vp), array.nbytes) == 0
        if ok:
            if not hasattr(self, "_pinned"):
                self._pinned = {}
            self._pinned[array.ctypes.data] = array
        return ok

    def unpin(self, array):
        """undo pin() (alva_system_unpin_buffer)"""
        ok = self.L.alva_system_unpin_buffer(self.h, array.ctypes.data_as(_vp)) == 0
        getattr(self, "_pinned", {}).pop(array.ctypes.data, None)
        return ok

    def reset(self):
        self.L.alva_system_reset(self.h)

    def set_clahe(self, enabled=True, clip_limit=3.0, tile_size=50):
        """CLAHE on the gray frame before the KLT pyramid and the detector (the reference's State::claheEnabled_,
        claheContrastLimit_, claheTileSize_; its ACCURATE preset turns it on with these defaults).  The grid is
        (width // tile_size) x (height // tile_size); ORB descriptors keep reading the raw gray frame.  Applies from the next
        frame, survives reset(); a new System starts with it off."""
        rc = self.L.alva_system_set_clahe(self.h, 1 if enabled else 0, float(clip_limit), int(tile_size))
        if rc != 0:
            raise AlvaError(f"alva_system_set_clahe -> {rc}: {self.L.alva_last_error().decode()}")

    PRESETS = {"default": 0, "fast": 1, "average": 2, "accurate": 3}   # ALVA_PRESET_* (include/alva_b200.h)

    def set_preset(self, name):
        """The reference's tuned configurations: "default" (what configuring sets: 40-px grid cells, P3P on every frame,
        keyframe filtering ratio 0.95, CLAHE off), "fast" (50 px, 0.9), "average" (45 px, 0.9, PnP from the motion prior
        instead of P3P) or "accurate" (35 px, PnP from the prior, CLAHE on with clip 3 and 50-px tiles).  Resets the tracker
        and the map; the next frame starts under the preset.  Survives reset(); set_clahe() afterwards overrides its CLAHE
        setting; the lens model is kept."""
        if name not in self.PRESETS:
            raise ValueError(f"unknown preset {name!r}: one of {sorted(self.PRESETS)}")
        rc = self.L.alva_system_set_preset(self.h, self.PRESETS[name])
        if rc != 0:
            raise AlvaError(f"alva_system_set_preset -> {rc}: {self.L.alva_last_error().decode()}")

    def set_distortion(self, k1, k2, p1, p2):
        """OpenCV's radial-tangential lens model (the reference's configure(..., k1, k2, p1, p2)): keypoints are undistorted,
        projections distorted, as the reference's CameraCalibration does.  Resets the tracker and the map; the next frame starts
        under the new model.  Survives reset(); all zero is the pinhole camera."""
        rc = self.L.alva_system_set_distortion(self.h, float(k1), float(k2), float(p1), float(p2))
        if rc != 0:
            raise AlvaError(f"alva_system_set_distortion -> {rc}: {self.L.alva_last_error().decode()}")

    def set_fisheye(self, enabled, k1=0.0, k2=0.0, k3=0.0, k4=0.0):
        """OpenCV's equidistant fisheye lens (cv::fisheye, k1..k4 on the incidence angle) for wide-angle cameras: keypoints are
        undistorted with cv::fisheye::undistortPoints, projections use cv::fisheye::projectPoints.  enabled=False returns to the
        pinhole; zero coefficients with enabled=True are the equidistant projection.  Replaces set_distortion's model (and is
        replaced by it); resets the tracker and the map; survives reset() and set_preset(); configuring clears it.  Keypoints
        the model cannot undistort are dropped (lens_drops())."""
        rc = self.L.alva_system_set_fisheye(self.h, 1 if enabled else 0, float(k1), float(k2), float(k3), float(k4))
        if rc != 0:
            raise AlvaError(f"alva_system_set_fisheye -> {rc}: {self.L.alva_last_error().decode()}")

    def lens_drops(self):
        """keypoints dropped because the fisheye model could not undistort them, since configuring or the last lens change"""
        return int(self.L.alva_system_lens_drops(self.h))

    def set_relocalisation(self, max_lost_frames):
        """Relocalise against the kept map after a tracking loss instead of discarding it.  0 (the default) is the reference's
        behaviour: a failed pose empties the frame and the fourth failure since the last reset resets the map (status 2).
        With n > 0 a failed pose returns status 4 (LOST) with the last tracked pose; the map, keyframes and motion model are
        frozen and every following frame is matched against the whole map (P3P-RANSAC + PnP).  Tracking resumes with status 1
        when that succeeds; after n lost frames in a row the map is reset as the reference would (status 2).  Status codes:
        1 tracking, 2 reset during the call, 3 not initialised, 4 lost.  A new System starts with it off; reset(),
        set_preset(), set_distortion() and set_clahe() keep it."""
        rc = self.L.alva_system_set_relocalisation(self.h, int(max_lost_frames))
        if rc != 0:
            raise AlvaError(f"alva_system_set_relocalisation -> {rc}: {self.L.alva_last_error().decode()}")

    def save_map(self):
        """-> the map as bytes (a versioned, self-contained blob; the format is in include/alva_b200.h), to resume the session
        in a new System or to start another stream in this one's map and coordinate frame.  Allowed once initialised, also
        while lost; it changes nothing.  AlvaError before the initialisation."""
        # one serialisation per call: a buffer with room for the last blob and a quarter more; only a map that outgrew it
        # (ALVA_E_CAPACITY, which reports the length) is serialised a second time
        cap = getattr(self, "_map_cap", 1 << 20)
        n = C.c_size_t(0)
        buf = C.create_string_buffer(cap)
        rc = self.L.alva_system_save_map(self.h, buf, cap, C.byref(n))
        if rc == -3:
            cap = n.value
            buf = C.create_string_buffer(cap)
            rc = self.L.alva_system_save_map(self.h, buf, cap, C.byref(n))
        if rc == 0:
            self._map_cap = max(1 << 16, n.value + n.value // 4)
        if rc != 0:
            raise AlvaError(f"alva_system_save_map -> {rc}: {self.L.alva_last_error().decode()}")
        return buf.raw[:n.value]

    def load_map(self, data):
        """Replace the map with a blob from save_map() and enter the lost state.  Needs set_relocalisation(n > 0), and a System
        configured with the same camera, lens and preset cell size as the one that saved it.  The next frames return status 4
        (LOST) with the saved pose until one relocalises into the map; tracking then resumes with status 1 in the saved
        coordinate frame, and new keyframe and map point ids continue from the saved map's.  After n lost frames the map is
        discarded (status 2), as after any loss.  The blob is checked whole before anything changes: AlvaError for a blob that
        fails a check or relocalisation off, and the System is left as it was.  configure, reset(), set_preset(),
        set_distortion() and set_fisheye() discard a loaded map like any other."""
        data = bytes(data)
        rc = self.L.alva_system_load_map(self.h, data, len(data))
        if rc != 0:
            raise AlvaError(f"alva_system_load_map -> {rc}: {self.L.alva_last_error().decode()}")

    def set_localisation_only(self, enabled=True):
        """Track against the current map without ever changing it: a venue or site map built once, a map shared between
        devices, AR content that must stay where it was placed.  With it on there is no keyframe, no triangulation, no local BA
        and no keyframe removal; keyframes, map points and ids stay as they are.  Map points the tracker loses are matched back
        from the map without a keyframe (re-acquisition, on the first tracked frame after freezing or after a relocalisation,
        when the frame's occupied grid cells fall below 0.85 x their count after the last re-acquisition, or below 30 3-D
        keypoints).  A loss relocalises as usual (status 4, then 1) and never resets the map.  Usual flow:
        set_relocalisation(n), load_map(blob), set_localisation_only(True); a live, initialised session can also freeze its own
        map.  enabled=False resumes mapping on the next keyframe decision.  load_map() and set_clahe() keep the mode;
        configuring, reset(), set_preset(), set_distortion() and set_fisheye() end it with the map.  AlvaError (nothing
        changed) when enabling with relocalisation off or before the initialisation; set_relocalisation(0) is refused while
        it is on."""
        rc = self.L.alva_system_set_localisation_only(self.h, 1 if enabled else 0)
        if rc != 0:
            raise AlvaError(f"alva_system_set_localisation_only -> {rc}: {self.L.alva_last_error().decode()}")

    def localisation_stats(self):
        """{"on", "runs": frames re-acquisition ran on, "points": map points it returned, "last": those of its last run}"""
        o = np.zeros(4, np.int32)
        self.L.alva_system_localisation_stats(self.h, o.ctypes.data_as(_vp))
        return dict(zip(("on", "runs", "points", "last"), o.tolist()))

    def set_gyro(self, enabled=True, R_ci=None, bias=None):
        """Gyro-aided tracking: the gyroscope's rotation between frames predicts the camera's, so fast pans keep tracking.
        Samples then come with the frames through find_camera_pose_gyro().  R_ci (3x3, default identity) takes IMU-axis
        vectors to camera axes -- diag(1, -1, -1) for the W3C devicemotion rotationRate axes and a rear camera; bias (3, rad/s
        on the IMU axes, default zero) is subtracted from every sample.  enabled=False turns it off and drops the samples
        held.  Survives reset(), set_preset(), set_clahe(), set_distortion(), set_fisheye(), set_relocalisation(),
        set_localisation_only() and load_map(); a new System starts with it off.  AlvaError (nothing changed) for a
        non-finite value or an R_ci that is not a rotation."""
        R = None if R_ci is None else np.ascontiguousarray(R_ci, np.float64).reshape(9)
        b = None if bias is None else np.ascontiguousarray(bias, np.float64).reshape(3)
        rc = self.L.alva_system_set_gyro(self.h, 1 if enabled else 0, None if R is None else R.ctypes.data_as(_vp),
                                         None if b is None else b.ctypes.data_as(_vp))
        if rc != 0:
            raise AlvaError(f"alva_system_set_gyro -> {rc}: {self.L.alva_last_error().decode()}")

    def find_camera_pose_gyro(self, rgba, t_ms, samples):
        """find_camera_pose with gyro samples -> (status, pose[16]).  samples: [n, 7] rows {t_ms, gx, gy, gz (rad/s), ax, ay,
        az} (the reference's IMU layout; the accelerometer columns are ignored), in time order, none older than the samples
        already given; samples later than t_ms are kept for the next frame.  With set_gyro off they are checked and ignored.
        AlvaError (no frame processed) for a refused sample array."""
        self._check(rgba)
        s = np.ascontiguousarray(samples, np.float64).reshape(-1, 7)
        pose = np.zeros(16, np.float32)
        st = self.L.alva_system_find_camera_pose_gyro(self.h, rgba.ctypes.data_as(_vp), float(t_ms), s.ctypes.data_as(_vp) if len(s) else None,
                                                      len(s), pose.ctypes.data_as(_vp))
        if st < 0:
            raise AlvaError(f"alva_system_find_camera_pose_gyro -> {st}: {self.L.alva_last_error().decode()}")
        return st, pose

    def gyro_stats(self):
        """-> ({"predicted": frames whose rotation came from the gyro, "fallback": frames whose interval the samples did not
        cover, "carried": lost frames whose rotation the gyro advanced, "rotated" / "kept": KLT priors rotated / kept at the
        previous position}, dR [3, 3]: the last frame's camera rotation from the gyro, identity when not covered)"""
        o = np.zeros(5, np.int32)
        dR = np.zeros(9)
        self.L.alva_system_gyro_stats(self.h, o.ctypes.data_as(_vp), dR.ctypes.data_as(_vp))
        return dict(zip(("predicted", "fallback", "carried", "rotated", "kept"), o.tolist())), dR.reshape(3, 3)
