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
    L.alva_system_set_preset.argtypes = [_vp, _i32]
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
    """One camera stream.  status codes as the reference: 1 tracking, 2 the tracker was reset during the call, 3 not initialised."""

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
