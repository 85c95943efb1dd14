"""Shared by the CLAHE tests and tools/make_golden_clahe.py: the seeded input cases of tests/golden/clahe.npz, the
contrast-compressed frames of tests/golden/system_clahe.npz, the CLAHE oracle (oracle/clahe_oracle.c), the reference's CLAHE
harness (oracle/_ref/libalva_ref_clahe.so, where it was built) and the CPU oracle build of the System with the CLAHE switch."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, w, h, nframes, clip_limit, tiles_x, tiles_y, image kind)
CASES = [
    ("system_640x480", 640, 480, 1, 3.0, 12, 9, "noise"),        # the System grids: Size(w / 50, h / 50)
    ("system_1280x720", 1280, 720, 1, 3.0, 25, 14, "noise"),
    ("system_1920x1080", 1920, 1080, 1, 3.0, 38, 21, "noise"),
    ("divisible", 640, 480, 1, 3.0, 8, 8, "noise"),
    ("x_only_divisible", 640, 479, 1, 3.0, 8, 8, "noise"),
    ("y_only_divisible", 641, 480, 1, 3.0, 8, 8, "noise"),
    ("neither_divisible", 333, 257, 1, 3.0, 7, 5, "noise"),
    ("tiles_eq_width", 40, 30, 1, 3.0, 40, 7, "noise"),            # x extended by a full 40 = w: reflect-101 reflects twice
    ("tiles_eq_height", 50, 9, 1, 3.0, 3, 9, "noise"),
    ("clip_0", 320, 240, 1, 0.0, 8, 8, "noise"),
    ("clip_40", 320, 240, 1, 40.0, 8, 8, "noise"),
    ("clip_1e9", 640, 480, 1, 1e9, 12, 9, "noise"),
    ("constant", 320, 240, 1, 3.0, 5, 5, "constant"),
    ("two_valued", 320, 240, 1, 3.0, 6, 4, "two_valued"),
    ("batch_4", 320, 240, 4, 2.5, 4, 3, "noise"),
]


def case_input(k):
    """[nframes][h][w] uint8 input of CASES[k]: a dim, low-contrast gradient with noise, a constant, or two values"""
    name, w, h, n, clip, tx, ty, kind = CASES[k]
    rng = np.random.default_rng(1000 + k)
    if kind == "constant":
        return np.full((n, h, w), 77, np.uint8)
    if kind == "two_valued":
        return np.where(rng.random((n, h, w)) < 0.3, 40, 200).astype(np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    base = 30 + 40 * xx / max(w - 1, 1) + 20 * yy / max(h - 1, 1)
    return np.clip(base[None] + rng.normal(0, 6, (n, h, w)), 0, 255).astype(np.uint8)


def compress_contrast(frames_rgba):
    """The fixed integer map of the system_clahe trace: every colour channel v -> 16 + v // 4 (a dim, low-contrast camera:
    values 16..79); alpha unchanged."""
    out = frames_rgba.copy()
    out[..., :3] = 16 + frames_rgba[..., :3] // 4
    return out


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def clahe_oracle_lib():
    """orc_clahe (oracle/clahe_oracle.c), built on demand into tests/_build -- test infrastructure"""
    so = os.path.join(ROOT, "tests", "_build", "libclahe_oracle.so")
    src = os.path.join(ROOT, "oracle", "clahe_oracle.c")
    if _stale(so, [src]):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-std=gnu11", "-shared", "-o", so, src, "-lm"])
    L = C.CDLL(so)
    L.orc_clahe.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int]
    return L


def ref_clahe_lib(ref):
    """the reference's CLAHE (oracle/ref_clahe.cpp) when the reference is built here, else None (the tests then read the digests)"""
    so = os.path.join(ROOT, "oracle", "_ref", "libalva_ref_clahe.so")
    if ref is None or not os.path.exists(so):
        return None
    L = C.CDLL(so)
    L.ref_clahe.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_void_p]
    L.ref_system_set_clahe.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int]
    return L


def cpu_clahe_system_lib():
    """alvaar_b200/csrc/system_core.h over the CPU oracle with the CLAHE switch (tests/host/system_cpu_clahe.cpp) -- test
    infrastructure"""
    so = os.path.join(ROOT, "tests", "_build", "libsystem_cpu_clahe.so")
    orc = os.path.join(ROOT, "oracle", "_build", "libalva_oracle.so")
    clahe_oracle_lib()
    corc = os.path.join(ROOT, "tests", "_build", "libclahe_oracle.so")
    srcs = [os.path.join(ROOT, "tests", "host", "system_cpu_clahe.cpp"), os.path.join(ROOT, "tests", "host", "system_cpu_backend.cpp"),
            os.path.join(ROOT, "alvaar_b200", "csrc", "system_core.h"), orc, corc]
    if not os.path.exists(orc):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL)
    if _stale(so, srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc, corc,
                               "-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + os.path.dirname(corc)])
    S = C.CDLL(so)
    S.cpu_clahe_system_create.restype = C.c_void_p
    S.cpu_clahe_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    S.cpu_system_set_clahe.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int]
    S.cpu_clahe_system_process.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    S.cpu_clahe_system_keypoints.argtypes = [C.c_void_p] * 5 + [C.c_int]
    S.cpu_clahe_system_info.argtypes = [C.c_void_p, C.c_void_p]
    S.cpu_clahe_system_set_essential_hook.argtypes = [C.c_void_p, C.c_void_p]
    S.cpu_clahe_system_destroy.argtypes = [C.c_void_p]
    return S
