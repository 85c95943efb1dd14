"""Shared by the full-vector lens tests and tools/make_golden_distortion_full.py: the test lenses of tests/golden/camera_full.npz
(OpenCV distortion vectors of 5, 8, 12 and 14 entries, and one that folds back inside the image), their seeded points (the
generators of camera_util, seeded per lens), the plain-C oracle (oracle/camera_full_oracle.c), the host build of the product's
arithmetic (tests/host/camera_full_host.cpp over camera_model.h and system_core.h), both built on demand into tests/_build, and
OpenCV's own cv::undistortPoints / cv::projectPoints (oracle/_ref/libalva_ref_distortion_full.so, where it was built)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

from camera_util import canonical

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, w, h, coefficients as cv::calibrateCamera returns them)
CASES = [
    ("phone_k3_640x480", 640, 480, (0.12, -0.35, 1e-3, -6e-4, 0.25)),
    ("rational_wide_1280x720", 1280, 720, (2.1, 0.6, 5e-4, -3e-4, 0.02, 2.45, 1.3, 0.15)),
    ("thin_prism_640x480", 640, 480, (-0.25, 0.08, 1e-3, -5e-4, 0.01, 0.0, 0.0, 0.0, 2e-3, -1e-4, -1.5e-3, 2e-4)),
    ("tilted_640x480", 640, 480, (-0.2, 0.05, 5e-4, 2e-4, 0.01, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.02, -0.015)),
    ("fold_back_640x480", 640, 480, (-1.5, 0.1, -2e-3, 1e-3, 0.05)),   # 1 + k1 r2 + k2 r4 + k3 r6 < 0 beyond r2 ~ 0.7: icdist < 0
]
NAMES = [c[0] for c in CASES]


def case_K(k):
    from alvaar_b200 import synth
    name, w, h, d = CASES[k]
    return np.array(synth.intrinsics(w, h)), np.array(d, np.float64)


def case_pixels(k):
    """[n][2] float32 pixels: uniform inside the image, near its four corners, up to 100 px outside it, the exact corners and
    border lines (about 8e4 points)"""
    name, w, h, d = CASES[k]
    rng = np.random.default_rng(5000 + k)
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
    rng = np.random.default_rng(6000 + k)
    uv = rng.uniform((-150, -150), (w + 150, h + 150), (15000, 2))
    z = rng.uniform(0.05, 20.0, 15000)
    front = np.stack([(uv[:, 0] - K[2]) / K[0] * z, (uv[:, 1] - K[3]) / K[1] * z, z], 1)
    behind = np.concatenate([rng.uniform(-5, 5, (6000, 2)), -rng.uniform(0.01, 10.0, (6000, 1))], 1)
    plane = np.concatenate([rng.uniform(-5, 5, (1000, 2)), np.zeros((1000, 1))], 1)
    plane[:3] = [[0, 0, 0], [1, 0, 0], [0, -1, 0]]
    return np.ascontiguousarray(np.concatenate([front, behind, plane]))


def rounding_exempt(mine, ref32, ref64):
    """The flat indices where float results `mine` differ from OpenCV's `ref32`, and whether each difference is the
    rounding-boundary exemption: the two floats are adjacent and OpenCV's double `ref64` lies within 4 double ulps of the
    boundary between them"""
    a, b = canonical(mine).ravel(), canonical(ref32).ravel()
    idx = np.flatnonzero(a != b)
    fa, fb, d = np.asarray(mine, np.float32).ravel()[idx], np.asarray(ref32, np.float32).ravel()[idx], np.asarray(ref64).ravel()[idx]
    adjacent = (np.nextafter(fa, fb) == fb) & np.isfinite(fa) & np.isfinite(fb)
    mid = (fa.astype(np.float64) + fb.astype(np.float64)) / 2
    return idx, adjacent & (np.abs(d - mid) <= 4 * np.spacing(np.abs(d)))


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def _point_args(L, names):
    vp = C.c_void_p
    for f in names:
        getattr(L, f).argtypes = [vp, C.c_int, vp, vp, C.c_int, vp]


def _match_full_source():
    """oracle/match_dist_oracle.c with its projection taken through the 14-coefficient model (orc_full_project_cam), exported as
    orc_match_to_map_full"""
    src = open(os.path.join(ROOT, "oracle", "match_dist_oracle.c")).read()
    subs = [(r"\borc_project_cam_dist\b", "orc_full_project_cam", 4),
            (r"if \(dist4 && \(dist4\[0\] != 0 \|\| dist4\[1\] != 0 \|\| dist4\[2\] != 0 \|\| dist4\[3\] != 0\)\) C\.dist = dist4;",
             "if (dist4) C.dist = dist4;", 1),
            (r"\borc_match_to_map_dist\b", "orc_match_to_map_full", 2)]
    for pat, rep, n in subs:
        src, got = re.subn(pat, rep, src)
        assert got == n, (pat, got)
    return src


def _reacquire_full_source():
    """oracle/reacquire_oracle.c with lens 3 (coef: 14 coefficients, projected by orc_full_project_cam), exported as
    orc_match_frame_to_map_full"""
    src = open(os.path.join(ROOT, "oracle", "reacquire_oracle.c")).read()
    subs = [(r"(void orc_fisheye_project_cam\(const double\* K4, const double\* D4, const double\* p, float\* out\);)",
             r"\1\nvoid orc_full_project_cam(const double* K4, const double* k14, const double* p, float* out);", 1),
            (r"(    if \(lens == 2\) \{ orc_fisheye_project_cam\(K4, D4, c, px\); return; \})",
             r"\1\n    if (lens == 3) { orc_full_project_cam(K4, D4, c, px); return; }", 1),
            (r"lens < 0 \|\| lens > 2", "lens < 0 || lens > 3", 1),
            (r"double D4\[4\] = \{0, 0, 0, 0\};\n    if \(lens\) for \(int i = 0; i < 4; i\+\+\) D4\[i\] = coef4\[i\];",
             "double D4[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};\n    if (lens) for (int i = 0; i < (lens == 3 ? 14 : 4); i++) D4[i] = coef4[i];", 1),
            (r"\borc_match_frame_to_map\b", "orc_match_frame_to_map_full", 1)]
    for pat, rep, n in subs:
        src, got = re.subn(pat, rep, src)
        assert got == n, (pat, got)
    return src


def oracle_lib():
    """orc_full_* (oracle/camera_full_oracle.c), orc_match_to_map_full and orc_match_frame_to_map_full (the matcher and
    re-acquisition oracles with lens 3), built on demand into tests/_build -- test infrastructure"""
    build = os.path.join(ROOT, "tests", "_build")
    so = os.path.join(build, "libcamera_full_oracle.so")
    srcs = [os.path.join(ROOT, "oracle", f) for f in ("camera_full_oracle.c", "camera_oracle.c", "fisheye_oracle.c", "match_dist_oracle.c",
                                                      "reacquire_oracle.c")] + [os.path.abspath(__file__)]
    if _stale(so, srcs):
        os.makedirs(build, exist_ok=True)
        gm, gr = os.path.join(build, "match_full_oracle.c"), os.path.join(build, "reacquire_full_oracle.c")
        with open(gm, "w") as f:
            f.write(_match_full_source())
        with open(gr, "w") as f:
            f.write(_reacquire_full_source())
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-std=gnu11",
                               "-shared", "-o", so] + srcs[:3] + [gm, gr, "-lm"])
    L = C.CDLL(so)
    _point_args(L, ("orc_full_undistort_points", "orc_full_project_points"))
    vp = C.c_void_p
    L.orc_full14_project_points.argtypes = [vp, C.c_int, vp, vp, vp]
    L.orc_match_frame_to_map_full.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_double] * 4 + [C.c_int, vp, vp, C.c_int, vp, vp, vp, vp,
                                                                                                 C.c_int, vp, vp, vp, C.c_float, vp, vp]
    return L


def host_lib():
    """the product's arithmetic built for the host (tests/host/camera_full_host.cpp) -- test infrastructure"""
    so = os.path.join(ROOT, "tests", "_build", "libcamera_full_host.so")
    csrc = os.path.join(ROOT, "alvaar_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "host", "camera_full_host.cpp"), os.path.join(csrc, "camera_model.h"), os.path.join(csrc, "system_core.h")]
    if _stale(so, srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0]])
    L = C.CDLL(so)
    vp = C.c_void_p
    _point_args(L, ("cpu_full_undistort_points", "cpu_full_project_points"))
    L.cpu_full_tilt.argtypes = [vp, C.c_int, vp, vp]
    L.cpu_cam_full.argtypes = [vp, C.c_int, vp, vp, C.c_int, C.c_int, vp]
    return L


def ref_lib():
    """OpenCV's own calls (oracle/ref_distortion_full.cpp) when they are built here, else None"""
    so = os.path.join(ROOT, "oracle", "_ref", "libalva_ref_distortion_full.so")
    if not os.path.exists(so):
        return None
    L = C.CDLL(so)
    vp = C.c_void_p
    for f in ("ref_full_undistort_points", "ref_full_project_points"):
        getattr(L, f).argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def run_points(fn, pts, K, D):
    """fn(in, n, K4, coeffs, ncoeffs, out) -> [n][2] float32"""
    out = np.zeros((len(pts), 2), np.float32)
    D = np.ascontiguousarray(D, np.float64)
    rc = fn(_p(pts), len(pts), _p(np.ascontiguousarray(K, np.float64)), _p(D), len(D), _p(out))
    assert rc == 0, rc
    return out


def run_cam(L, pts, K, D, mode):
    """the state machine's Camera after setDistortionCoeffs(D): (its lens, [n][2] float32)"""
    out = np.zeros((len(pts), 2), np.float32)
    D = np.ascontiguousarray(D, np.float64)
    lens = L.cpu_cam_full(_p(pts), len(pts), _p(np.ascontiguousarray(K, np.float64)), _p(D), len(D), mode, _p(out))
    return lens, out


def run_ref(fn, pts, K, D):
    """OpenCV's float results and the doubles they were rounded from"""
    out, out64 = np.zeros((len(pts), 2), np.float32), np.zeros((len(pts), 2))
    D = np.ascontiguousarray(D, np.float64)
    fn(_p(pts), len(pts), _p(np.ascontiguousarray(K, np.float64)), _p(D), len(D), _p(out), _p(out64))
    return out, out64


def n_fold(px, K, D):
    """pixels whose first iteration already meets icdist < 0 (the pinhole fallback of cv::undistortPoints), in numpy double
    arithmetic on the untilted point -- a count for the case's coverage, not a bit-exact model"""
    k = np.zeros(14)
    k[:len(D)] = D
    x = (px[:, 0].astype(np.float64) - K[2]) / K[0]
    y = (px[:, 1].astype(np.float64) - K[3]) / K[1]
    r2 = x * x + y * y
    icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
    return int((icdist < 0).sum())


# the lenses of the System sequences (640x480): a rational lens and a tilted sensor with thin-prism terms; both invert over
# the whole frame (synth.undistort_normalised_full)
SYSTEM_RATIONAL = (-0.28, 0.09, 8e-4, -4e-4, 0.02, 0.06, 0.015, 0.004)
SYSTEM_TILTED = (-0.22, 0.07, 6e-4, 3e-4, 0.01, 0.0, 0.0, 0.0, 1.5e-3, -2e-4, -1e-3, 1e-4, 0.03, -0.02)


def system_frames(lens, n=100, w=640, h=480, seed=99):
    """the rendered sequence the System tests run: synth.make_frames through the lens, and its true camera poses"""
    from alvaar_b200 import synth
    return synth.make_frames(n, w, h, seed=seed, rgba=True, dist_full=lens)


def cpu_system_lib():
    """alvaar_b200/csrc/system_core.h over the CPU oracle with setDistortionCoeffs (tests/host/system_cpu_lens_full.cpp)"""
    oracle_lib()
    build = os.path.join(ROOT, "tests", "_build")
    so = os.path.join(build, "libsystem_cpu_lens_full.so")
    orc = os.path.join(ROOT, "oracle", "_build", "libalva_oracle.so")
    forc = os.path.join(build, "libcamera_full_oracle.so")
    if not os.path.exists(orc):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL)
    csrc = os.path.join(ROOT, "alvaar_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "host", "system_cpu_lens_full.cpp"), os.path.join(ROOT, "tests", "host", "system_cpu_backend.cpp"),
            os.path.join(csrc, "system_core.h"), os.path.join(csrc, "camera_model.h"), orc, forc]
    if _stale(so, srcs):
        os.makedirs(build, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc, forc,
                               "-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + os.path.dirname(forc)])
    S = C.CDLL(so)
    vp = C.c_void_p
    S.cpu_full_system_create.restype = vp
    S.cpu_full_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    S.cpu_full_system_set_coeffs.argtypes = [vp, vp, C.c_int]
    S.cpu_full_system_process.argtypes = [vp, vp, C.c_double, vp]
    S.cpu_full_system_keypoints.argtypes = [vp] * 5 + [C.c_int]
    S.cpu_full_system_frame_points.argtypes = [vp, vp, C.c_int]
    S.cpu_full_system_info.argtypes = [vp, vp]
    S.cpu_full_system_lens_drops.argtypes = [vp]
    S.cpu_full_system_local_bas.argtypes = [vp]
    S.cpu_full_system_destroy.argtypes = [vp]
    return S


def run_cpu_system(S, frames, K, lens, cap=8192):
    """the CPU state machine over the frames under setDistortionCoeffs(lens); per frame (status, Twc [7], info [8], ids, px, is3d,
    frame points, lens drops so far), and the number of local BAs"""
    s = S.cpu_full_system_create(frames.shape[2], frames.shape[1], K[0], K[1], K[2], K[3])
    D = np.ascontiguousarray(lens, np.float64)
    assert S.cpu_full_system_set_coeffs(s, _p(D), len(D)) == 3
    out = []
    for k in range(len(frames)):
        T = np.zeros(7)
        st = S.cpu_full_system_process(s, _p(np.ascontiguousarray(frames[k])), k * 33.333, _p(T))
        ids = np.zeros(cap, np.int32); px = np.zeros((cap, 2), np.float32); d3 = np.zeros(cap, np.uint8); wp = np.zeros((cap, 3))
        info = np.zeros(8, np.int32); xy = np.zeros((cap, 2), np.int32)
        n = S.cpu_full_system_keypoints(s, _p(ids), _p(px), _p(d3), _p(wp), cap)
        m = S.cpu_full_system_frame_points(s, _p(xy), cap)
        S.cpu_full_system_info(s, _p(info))
        out.append((st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy(), xy[:m].copy(), S.cpu_full_system_lens_drops(s)))
    nba = S.cpu_full_system_local_bas(s)
    S.cpu_full_system_destroy(s)
    return out, nba


def run_reacquire_oracle(p):
    """orc_match_frame_to_map_full on a localisation_util.Problem (lens 3: p.coef holds 14 coefficients) -> (row, dist)"""
    L = oracle_lib()
    nq = len(p.q_px)
    row, dist = np.full(max(nq, 1), -7, np.int32), np.full(max(nq, 1), -7, np.int32)
    coef = np.ascontiguousarray(p.coef if p.coef is not None else np.zeros(14), np.float64)
    skip = None if p.skip is None else _p(np.ascontiguousarray(p.skip, np.uint8))
    n = L.orc_match_frame_to_map_full(p.w, p.h, p.cell, *p.K, p.lens, _p(coef), _p(np.ascontiguousarray(p.Twc, np.float64)), p.n_mp,
                                      _p(np.ascontiguousarray(p.wpt, np.float64)), _p(np.ascontiguousarray(p.desc_start, np.int32)),
                                      _p(np.ascontiguousarray(p.desc, np.uint8)), skip, nq, _p(np.ascontiguousarray(p.q_px, np.float32)),
                                      _p(np.ascontiguousarray(p.q_desc, np.uint8)), _p(np.ascontiguousarray(p.q_kept, np.uint8)), p.radius,
                                      _p(row), _p(dist))
    assert n >= 0
    return row[:nq], dist[:nq]
