"""Shared by the fisheye tests and tools/make_golden_fisheye.py: the seeded point cases of tests/golden/fisheye.npz, the
rounding-boundary exemption, the plain-C fisheye oracle (oracle/fisheye_oracle.c, and oracle/match_dist_oracle.c with its
projection taken through it), built on demand into tests/_build/libfisheye_oracle.so, OpenCV's cv::fisheye behind
oracle/_ref/libalva_ref_fisheye.so (where it was built), and the CPU oracle build of the System with the fisheye switch
(tests/host/system_cpu_fisheye.cpp), which also exports the host side of camera_model.h."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

from camera_util import canonical

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
vp = C.c_void_p

# the System sequences' lens, with synth.intrinsics(640, 480): a wide-angle equidistant lens (the corners are ~40 degrees
# off-axis, where the pinhole model misplaces them by ~80 px)
SYSTEM_FISHEYE = (0.03, -0.01, 0.002, 0.0)

# (name, w, h, (fx, fy, cx, cy), (k1, k2, k3, k4))
CASES = [
    ("wide_640x480", 640, 480, (400.0, 401.5, 321.3, 238.7), (0.012, -0.004, 0.0008, -0.0001)),
    # the image diagonal reaches theta_d = pi/2 (a ~180 degree lens); the pixels outside it are clamped
    ("fov180_1280x720", 1280, 720, (468.0, 468.0, 640.0, 360.0), (-0.02, 0.006, -0.001, 0.0002)),
    # theta_d(theta) peaks at 0.566: beyond it Newton does not converge or flips, and (-1e6, -1e6) is returned
    ("newton_fails_640x480", 640, 480, (400.0, 400.0, 320.0, 240.0), (-0.5, 0.05, 0.0, 0.0)),
]
NAMES = [c[0] for c in CASES]


def case_K(k):
    return np.array(CASES[k][3], np.float64), np.array(CASES[k][4], np.float64)


def case_pixels(k):
    """[n][2] float32 pixels: uniform inside the image, near its four corners, up to 100 px outside it, the exact corners and
    border lines, and the principal point and its neighbours (about 8e4 points)"""
    name, w, h, K, _ = CASES[k]
    rng = np.random.default_rng(5000 + k)
    inside = rng.uniform((0, 0), (w, h), (50000, 2))
    corners = np.concatenate([c + rng.uniform(-40, 40, (2500, 2)) for c in ((0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1))])
    outside = rng.uniform((-100, -100), (w + 100, h + 100), (20000, 2))
    exact = np.array([(x, y) for x in (-100, 0, w / 2, w - 1, w, w + 100) for y in (-100, 0, h / 2, h - 1, h, h + 100)])
    cx, cy = np.float32(K[2]), np.float32(K[3])
    centre = np.array([(cx, cy), (np.nextafter(cx, np.float32(1e9)), cy), (cx, np.nextafter(cy, np.float32(-1e9))), (K[2], K[3])])
    return np.ascontiguousarray(np.concatenate([inside, corners, outside, exact, centre]).astype(np.float32))


def case_points(k):
    """[n][3] float64 camera-frame points: rays up to 86 degrees off the axis at depths 0.05 - 20, rays past 90 degrees
    (z < 0), points on the camera plane (z = 0, the origin included) and on the optical axis in front and behind (about 2.4e4)"""
    rng = np.random.default_rng(6000 + k)
    th = rng.uniform(0, 1.5, 15000)
    ph = rng.uniform(0, 2 * np.pi, 15000)
    d = rng.uniform(0.05, 20.0, 15000)
    front = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], 1) * d[:, None]
    behind = np.concatenate([rng.uniform(-5, 5, (6000, 2)), -rng.uniform(0.01, 10.0, (6000, 1))], 1)
    plane = np.concatenate([rng.uniform(-5, 5, (1000, 2)), np.zeros((1000, 1))], 1)
    plane[:3] = [[0, 0, 0], [1, 0, 0], [0, -1, 0]]
    axis = np.stack([np.zeros(2000), np.zeros(2000), np.concatenate([rng.uniform(0.01, 20, 1000), -rng.uniform(0.01, 20, 1000)])], 1)
    axis[:2, 0] = [1e-12, -3e-9]   # r just below / around the 1e-8 guard
    return np.ascontiguousarray(np.concatenate([front, behind, plane, axis]))


def rounding_exempt(mine, ref32, ref64):
    """For float results `mine` and OpenCV's `ref32` (same shape) and the double `ref64` OpenCV rounded to ref32: the flat
    indices where the bits differ, and whether each such difference is the exemption -- the two floats are adjacent and the
    double lies within 4 double ulps of the rounding boundary between them, so that only how atan / tan round decides it"""
    a, b = canonical(mine).ravel(), canonical(ref32).ravel()
    idx = np.flatnonzero(a != b)
    ok = np.zeros(len(idx), bool)
    fa, fb, d = np.asarray(mine, np.float32).ravel()[idx], np.asarray(ref32, np.float32).ravel()[idx], np.asarray(ref64).ravel()[idx]
    adjacent = (np.nextafter(fa, fb) == fb) & np.isfinite(fa) & np.isfinite(fb)
    mid = (fa.astype(np.float64) + fb.astype(np.float64)) / 2
    ok = adjacent & (np.abs(d - mid) <= 4 * np.spacing(np.abs(d)))
    return idx, ok


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def _fisheye_match_source():
    """oracle/match_dist_oracle.c with its projection taken through the fisheye model (every coefficient set, zeros included, is a
    lens), exported as orc_match_to_map_fisheye"""
    src = open(os.path.join(ROOT, "oracle", "match_dist_oracle.c")).read()
    subs = [(r"\borc_project_cam_dist\b", "orc_fisheye_project_cam", 4),
            (r"if \(dist4 && \(dist4\[0\] != 0 \|\| dist4\[1\] != 0 \|\| dist4\[2\] != 0 \|\| dist4\[3\] != 0\)\) C\.dist = dist4;",
             "if (dist4) C.dist = dist4;", 1),
            (r"\borc_match_to_map_dist\b", "orc_match_to_map_fisheye", 2)]
    for pat, rep, n in subs:
        src, got = re.subn(pat, rep, src)
        assert got == n, (pat, got)
    return src


def oracle_lib():
    """orc_fisheye_* (oracle/fisheye_oracle.c) and orc_match_to_map_fisheye, built on demand into tests/_build"""
    so = os.path.join(BUILD, "libfisheye_oracle.so")
    srcs = [os.path.join(ROOT, "oracle", "fisheye_oracle.c"), os.path.join(ROOT, "oracle", "match_dist_oracle.c"), os.path.abspath(__file__)]
    if _stale(so, srcs):
        os.makedirs(BUILD, exist_ok=True)
        gen = os.path.join(BUILD, "match_fisheye_oracle.c")
        with open(gen, "w") as f:
            f.write(_fisheye_match_source())
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-std=gnu11",
                               "-shared", "-o", so, srcs[0], gen, "-lm"])
    L = C.CDLL(so)
    L.orc_fisheye_undistort_points.argtypes = [vp, C.c_int, vp, vp, vp]
    L.orc_fisheye_project_points.argtypes = [vp, C.c_int, vp, vp, vp]
    return L


def ref_lib():
    """OpenCV's cv::fisheye (oracle/ref_fisheye.cpp) when it is built here, else None"""
    so = os.path.join(ROOT, "oracle", "_ref", "libalva_ref_fisheye.so")
    if not os.path.exists(so):
        return None
    L = C.CDLL(so)
    L.ref_fisheye_undistort_points.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    L.ref_fisheye_project_points.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    return L


def run_ref(fn, pts, K, D):
    """-> OpenCV's float results and the doubles they were rounded from"""
    o32, o64 = np.zeros((len(pts), 2), np.float32), np.zeros((len(pts), 2))
    P = lambda a: a.ctypes.data_as(vp)  # noqa: E731
    fn(P(pts), len(pts), P(np.ascontiguousarray(K, np.float64)), P(np.ascontiguousarray(D, np.float64)), P(o32), P(o64))
    return o32, o64


def cpu_system_lib():
    """alvaar_b200/csrc/system_core.h over the CPU oracle with the fisheye switch (tests/host/system_cpu_fisheye.cpp)"""
    oracle_lib()
    so = os.path.join(BUILD, "libsystem_cpu_fisheye.so")
    orc = os.path.join(ROOT, "oracle", "_build", "libalva_oracle.so")
    forc = os.path.join(BUILD, "libfisheye_oracle.so")
    if not os.path.exists(orc):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL)
    csrc = os.path.join(ROOT, "alvaar_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "host", "system_cpu_fisheye.cpp"), os.path.join(ROOT, "tests", "host", "system_cpu_backend.cpp"),
            os.path.join(csrc, "system_core.h"), os.path.join(csrc, "camera_model.h"), orc, forc]
    if _stale(so, srcs):
        os.makedirs(BUILD, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc, forc,
                               "-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + os.path.dirname(forc)])
    S = C.CDLL(so)
    S.cpu_fish_system_create.restype = vp
    S.cpu_fish_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    S.cpu_fish_system_set_fisheye.argtypes = [vp, C.c_int] + [C.c_double] * 4
    S.cpu_fish_system_process.argtypes = [vp, vp, C.c_double, vp]
    S.cpu_fish_system_keypoints.argtypes = [vp] * 5 + [C.c_int]
    S.cpu_fish_system_frame_points.argtypes = [vp, vp, C.c_int]
    S.cpu_fish_system_info.argtypes = [vp, vp]
    S.cpu_fish_system_lens_drops.argtypes = [vp]
    S.cpu_fish_system_local_bas.argtypes = [vp]
    S.cpu_fish_system_destroy.argtypes = [vp]
    for f in ("cpu_fish_undistort_points", "cpu_fish_project_points", "cpu_fish_cam_undistort_points", "cpu_fish_cam_project_points"):
        getattr(S, f).argtypes = [vp, C.c_int, vp, vp, vp]
    for f in ("cpu_det_atan", "cpu_det_tan"):
        getattr(S, f).argtypes = [vp, C.c_int, vp]
    return S


def run_points(fn, pts, K, D):
    """fn(in, n, K4, D4, out) over a point array -> [n][2] float32"""
    out = np.zeros((len(pts), 2), np.float32)
    P = lambda a: a.ctypes.data_as(vp)  # noqa: E731
    fn(P(pts), len(pts), P(np.ascontiguousarray(K, np.float64)), P(np.ascontiguousarray(D, np.float64)), P(out))
    return out


def system_frames(n=100, w=640, h=480, seed=99, lens=SYSTEM_FISHEYE):
    """the rendered sequence the System tests run: synth.make_frames through the fisheye lens, and its true camera poses"""
    from alvaar_b200 import synth
    return synth.make_frames(n, w, h, seed=seed, rgba=True, fisheye=lens)


def run_cpu_system(S, frames, K, lens=SYSTEM_FISHEYE, cap=8192):
    """the CPU state machine over the frames (lens None: the pinhole); per frame (status, Twc [7], info [8], ids, px, is3d,
    frame points, lens drops so far)"""
    P = lambda a: a.ctypes.data_as(vp)  # noqa: E731
    s = S.cpu_fish_system_create(frames.shape[2], frames.shape[1], K[0], K[1], K[2], K[3])
    if lens is not None:
        S.cpu_fish_system_set_fisheye(s, 1, *lens)
    out = []
    for k in range(len(frames)):
        T = np.zeros(7)
        st = S.cpu_fish_system_process(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(T))
        ids = np.zeros(cap, np.int32); px = np.zeros((cap, 2), np.float32); d3 = np.zeros(cap, np.uint8); wp = np.zeros((cap, 3))
        info = np.zeros(8, np.int32); xy = np.zeros((cap, 2), np.int32)
        n = S.cpu_fish_system_keypoints(s, P(ids), P(px), P(d3), P(wp), cap)
        m = S.cpu_fish_system_frame_points(s, P(xy), cap)
        S.cpu_fish_system_info(s, P(info))
        out.append((st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy(), xy[:m].copy(), S.cpu_fish_system_lens_drops(s)))
    nba = S.cpu_fish_system_local_bas(s)
    S.cpu_fish_system_destroy(s)
    return out, nba


def true_Twc(poses):
    """synth's (R_wc, t_wc) poses as [t, q(x, y, z, w)]"""
    from alvaar_b200.synth import _quat_from_R
    return np.array([np.concatenate([t, _quat_from_R(R)]) for R, t in poses])


def trajectory_error(Twc, poses, frames):
    """camera positions of the given (tracked) frames against the rendered truth after the one similarity transform a
    monocular map leaves open (rotation, translation and scale, least squares, Umeyama): -> (max position error relative to
    the true path length over those frames, max rotation error in degrees)"""
    from alvaar_b200.synth import quat_to_R
    gt = true_Twc(poses)[frames]
    p, g = Twc[frames, :3], gt[:, :3]
    mp, mg = p.mean(0), g.mean(0)
    U, S, Vt = np.linalg.svd((g - mg).T @ (p - mp) / len(p))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    R = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / ((p - mp) ** 2).sum(1).mean()
    err = np.linalg.norm((s * (p - mp) @ R.T + mg) - g, axis=1)
    path = float(np.linalg.norm(np.diff(g, axis=0), axis=1).sum())
    rot = []
    for k in range(len(frames)):
        c = (np.trace((R @ quat_to_R(Twc[frames[k], 3:])).T @ quat_to_R(gt[k, 3:])) - 1) / 2
        rot.append(np.degrees(np.arccos(np.clip(c, -1, 1))))
    return float(err.max() / max(path, 1e-12)), float(max(rot))
