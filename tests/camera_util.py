"""Shared by the lens-distortion tests and tools/make_golden_distortion.py: the seeded point cases of tests/golden/camera.npz,
the distorted frames of tests/golden/system_dist.npz, the camera oracle (oracle/camera_oracle.c and oracle/match_dist_oracle.c,
built on demand into tests/_build/libcamera_oracle.so), the
reference's CameraCalibration harness (oracle/_ref/libalva_ref_camera.so, where it was built) and the CPU oracle build of the
System with the distortion switch (tests/host/system_cpu_dist.cpp), which also exports the host side of camera_model.h."""
import ctypes as C
import os
import subprocess

import numpy as np

from ref_golden import digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the System trace's lens: a moderate barrel with a little decentring
SYSTEM_DIST = (-0.25, 0.08, 1e-3, -5e-4)

# (name, w, h, (k1, k2, p1, p2))
CASES = [
    ("webcam_640x480", 640, 480, SYSTEM_DIST),
    ("strong_barrel_1280x720", 1280, 720, (-0.45, 0.22, 2e-3, -1.5e-3)),
    ("fold_back_640x480", 640, 480, (-1.5, 0.1, -2e-3, 1e-3)),       # 1 + k1 r2 + k2 r4 < 0 beyond r2 ~ 0.7: icdist < 0 fires
]


def case_K(k):
    from alvaar_b200 import synth
    name, w, h, d = CASES[k]
    return np.array(synth.intrinsics(w, h)), np.array(d, np.float64)


def case_pixels(k):
    """[n][2] float32 pixels: uniform inside the image, near its four corners, up to 100 px outside it, and the exact corners
    and border lines (about 8e4 points)"""
    name, w, h, d = CASES[k]
    rng = np.random.default_rng(2000 + k)
    inside = rng.uniform((0, 0), (w, h), (50000, 2))
    corners = np.concatenate([c + rng.uniform(-40, 40, (2500, 2)) for c in ((0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1))])
    outside = rng.uniform((-100, -100), (w + 100, h + 100), (20000, 2))
    exact = np.array([(x, y) for x in (-100, 0, w / 2, w - 1, w, w + 100) for y in (-100, 0, h / 2, h - 1, h, h + 100)])
    return np.ascontiguousarray(np.concatenate([inside, corners, outside, exact]).astype(np.float32))


def case_points(k):
    """[n][3] float64 camera-frame points: in front of the camera across and beyond the view, behind it (z < 0), and on its
    plane (z = 0, the origin included) (about 2.2e4 points)"""
    name, w, h, d = CASES[k]
    K, _ = case_K(k)
    rng = np.random.default_rng(3000 + k)
    uv = rng.uniform((-150, -150), (w + 150, h + 150), (15000, 2))
    z = rng.uniform(0.05, 20.0, 15000)
    front = np.stack([(uv[:, 0] - K[2]) / K[0] * z, (uv[:, 1] - K[3]) / K[1] * z, z], 1)
    behind = np.concatenate([rng.uniform(-5, 5, (6000, 2)), -rng.uniform(0.01, 10.0, (6000, 1))], 1)
    plane = np.concatenate([rng.uniform(-5, 5, (1000, 2)), np.zeros((1000, 1))], 1)
    plane[:3] = [[0, 0, 0], [1, 0, 0], [0, -1, 0]]
    return np.ascontiguousarray(np.concatenate([front, behind, plane]))


def canonical(a):
    """float32 results with every NaN replaced by one bit pattern: a NaN's payload is not part of the model's result
    (x86 and the GPU produce different ones for 0 * inf)"""
    a = np.array(a, np.float32, copy=True)
    a[np.isnan(a)] = np.float32(np.nan)
    return a.view(np.uint32)


def same_bits(a, b):
    return canonical(a).shape == canonical(b).shape and (canonical(a) == canonical(b)).all()


def cdigest(a):
    return digest(canonical(a))


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def oracle_lib():
    """orc_undistort_points / orc_project_points (oracle/camera_oracle.c) and orc_match_to_map_dist
    (oracle/match_dist_oracle.c), built on demand into tests/_build -- test infrastructure"""
    so = os.path.join(ROOT, "tests", "_build", "libcamera_oracle.so")
    srcs = [os.path.join(ROOT, "oracle", f) for f in ("camera_oracle.c", "match_dist_oracle.c")]
    if _stale(so, srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-std=gnu11",
                               "-shared", "-o", so] + srcs + ["-lm"])
    L = C.CDLL(so)
    L.orc_undistort_points.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_project_points.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def ref_camera_lib():
    """the reference's CameraCalibration (oracle/ref_camera.cpp) when it is built here, else None"""
    so = os.path.join(ROOT, "oracle", "_ref", "libalva_ref_camera.so")
    if not os.path.exists(so):
        return None
    L = C.CDLL(so)
    L.ref_undistort_points.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.ref_project_points.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    return L


def cpu_dist_system_lib():
    """alvaar_b200/csrc/system_core.h over the CPU oracle with the distortion switch (tests/host/system_cpu_dist.cpp) -- test
    infrastructure"""
    oracle_lib()
    so = os.path.join(ROOT, "tests", "_build", "libsystem_cpu_dist.so")
    orc = os.path.join(ROOT, "oracle", "_build", "libalva_oracle.so")
    corc = os.path.join(ROOT, "tests", "_build", "libcamera_oracle.so")
    if not os.path.exists(orc):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL)
    csrc = os.path.join(ROOT, "alvaar_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "host", "system_cpu_dist.cpp"), os.path.join(ROOT, "tests", "host", "system_cpu_backend.cpp"),
            os.path.join(csrc, "system_core.h"), os.path.join(csrc, "camera_model.h"), orc, corc]
    if _stale(so, srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc, corc,
                               "-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + os.path.dirname(corc)])
    S = C.CDLL(so)
    vp = C.c_void_p
    S.cpu_dist_system_create.restype = vp
    S.cpu_dist_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    S.cpu_system_set_distortion.argtypes = [vp] + [C.c_double] * 4
    S.cpu_dist_system_process.argtypes = [vp, vp, C.c_double, vp]
    S.cpu_dist_system_keypoints.argtypes = [vp] * 5 + [C.c_int]
    S.cpu_dist_system_frame_points.argtypes = [vp, vp, C.c_int]
    S.cpu_dist_system_info.argtypes = [vp, vp]
    S.cpu_dist_system_set_essential_hook.argtypes = [vp, vp]
    S.cpu_dist_system_destroy.argtypes = [vp]
    for f in ("cpu_cam_undistort_points", "cpu_radtan_undistort_points"):
        getattr(S, f).argtypes = [vp, C.c_int, vp, vp, vp]
    for f in ("cpu_cam_project_points", "cpu_radtan_project_points"):
        getattr(S, f).argtypes = [vp, C.c_int, vp, vp, vp]
    return S


def run_points(fn, pts, K, D, width=2):
    """fn(in, n, K4, D4, out) over a point array -> [n][2] float32"""
    out = np.zeros((len(pts), width), np.float32)
    P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    fn(P(pts), len(pts), P(np.ascontiguousarray(K, np.float64)), P(np.ascontiguousarray(D, np.float64)), P(out))
    return out


def run_ref(fn, pts, K, D, w, h):
    out = np.zeros((len(pts), 2), np.float32)
    P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    fn(P(pts), len(pts), P(np.ascontiguousarray(K, np.float64)), P(np.ascontiguousarray(D, np.float64)), w, h, P(out))
    return out
