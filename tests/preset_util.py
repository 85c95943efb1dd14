"""Shared by the preset tests and tools/make_golden_presets.py: the reference's preset table (state.hpp:9-17), the CPU oracle
build of the System with the preset switch (tests/host/system_cpu_preset.cpp), the local-map matching oracle on a grid of any
cell size, and the reference's preset harness (oracle/_ref/libalva_ref_preset.so, where it was built)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
CAP = 4096

# name -> (ALVA_PRESET_*, frameMaxCellSize_, mapKeyframeFilteringRatio_, p3pEnabled_, claheEnabled_)
PRESETS = {"default": (0, 40, 0.95, 1, 0), "fast": (1, 50, 0.9, 1, 0), "average": (2, 45, 0.9, 0, 0), "accurate": (3, 35, 0.95, 0, 1)}


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def match_cell_oracle_lib():
    """orc_match_to_map_cell: oracle/match_dist_oracle.c with its frame grid's 40-px cell read from the global orc_match_cell.
    The source is the committed oracle, rewritten at build time into tests/_build (two substitutions, both checked: the cell of
    its grid, and the function's name); with no coefficients it is orc_match_to_map's procedure.  Test infrastructure."""
    so = os.path.join(ROOT, "tests", "_build", "libmatch_cell_oracle.so")
    srcs = [os.path.join(ROOT, "oracle", "match_dist_oracle.c"), os.path.join(ROOT, "oracle", "camera_oracle.c")]
    if _stale(so, srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        src = open(srcs[0]).read()
        src, n1 = re.subn(r"m_cam C = \{w, h, 40,", "m_cam C = {w, h, orc_match_cell,", src)
        src, n2 = re.subn(r"\bint orc_match_to_map_dist\(", "int orc_match_to_map_cell(", src)
        assert n1 == 1 and n2 == 1, "oracle/match_dist_oracle.c changed: update the rewrite in tests/preset_util.py"
        gen = os.path.join(ROOT, "tests", "_build", "match_cell_oracle.c")
        with open(gen, "w") as f:
            f.write("/* generated from oracle/match_dist_oracle.c by tests/preset_util.py: the grid cell is a parameter */\n")
            f.write("int orc_match_cell = 40;\n" + src)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-std=gnu11", "-shared", "-o", so, gen, srcs[1], "-lm"])
    L = C.CDLL(so)
    L.orc_match_to_map_cell.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4 + [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int] + \
        [C.c_void_p] * 2 + [C.c_int] + [C.c_void_p] * 9 + [C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def cpu_preset_system_lib():
    """alvaar_b200/csrc/system_core.h over the CPU oracle with the preset switch (tests/host/system_cpu_preset.cpp) -- test
    infrastructure"""
    from clahe_util import clahe_oracle_lib
    so = os.path.join(ROOT, "tests", "_build", "libsystem_cpu_preset.so")
    orc = os.path.join(ROOT, "oracle", "_build", "libalva_oracle.so")
    clahe_oracle_lib()
    match_cell_oracle_lib()
    corc = os.path.join(ROOT, "tests", "_build", "libclahe_oracle.so")
    morc = os.path.join(ROOT, "tests", "_build", "libmatch_cell_oracle.so")
    host = os.path.join(ROOT, "tests", "host")
    srcs = [os.path.join(host, "system_cpu_preset.cpp"), os.path.join(host, "system_cpu_clahe.cpp"), os.path.join(host, "system_cpu_backend.cpp"),
            os.path.join(ROOT, "alvaar_b200", "csrc", "system_core.h"), orc, corc, morc]
    if not os.path.exists(orc):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL)
    if _stale(so, srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc, corc, morc,
                               "-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + os.path.dirname(corc)])
    S = C.CDLL(so)
    S.cpu_preset_system_create.restype = C.c_void_p
    S.cpu_preset_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    S.cpu_preset_system_set_preset.argtypes = [C.c_void_p, C.c_int]
    S.cpu_preset_system_set_clahe.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int]
    S.cpu_preset_system_process.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    S.cpu_preset_system_keypoints.argtypes = [C.c_void_p] * 5 + [C.c_int]
    S.cpu_preset_system_info.argtypes = [C.c_void_p, C.c_void_p]
    S.cpu_preset_system_counters.argtypes = [C.c_void_p, C.c_void_p]
    S.cpu_preset_system_set_essential_hook.argtypes = [C.c_void_p, C.c_void_p]
    S.cpu_preset_system_reset.argtypes = [C.c_void_p]
    S.cpu_preset_system_destroy.argtypes = [C.c_void_p]
    return S


def ref_preset_lib(ref):
    """the reference's preset harness (oracle/ref_preset.cpp) and its CLAHE harness, when the reference is built here, else None"""
    from clahe_util import ref_clahe_lib
    so = os.path.join(ROOT, "oracle", "_ref", "libalva_ref_preset.so")
    rc = ref_clahe_lib(ref)
    if ref is None or rc is None or not os.path.exists(so):
        return None
    L = C.CDLL(so)
    L.ref_system_set_preset.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int]
    L.ref_system_grid.argtypes = [C.c_void_p, C.c_void_p]
    L.ref_system_p3p_req.argtypes = [C.c_void_p]
    L.clahe = rc
    return L


def ref_system_create(R, RP, name, w, h, K):
    """a reference System configured as System::configure does, then turned into the preset `name` (ref_preset.cpp)"""
    R.ref_system_create.restype = C.c_void_p
    R.ref_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 8
    _, cell, ratio, p3p, clahe = PRESETS[name]
    s = R.ref_system_create(w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0)
    RP.ref_system_set_preset(s, cell, ratio, p3p)
    RP.clahe.ref_system_set_clahe(s, clahe, 3.0, 50)
    return s


def ref_frame(R, RP, s, rgba, t_ms):
    """one frame through the reference System: (status, Twc7, info8, ids, px, is3d, wpt, p3pReq_ afterwards)"""
    R.ref_system_find_camera_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    R.ref_system_keypoints.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    R.ref_system_info8.argtypes = [C.c_void_p, C.c_void_p]
    pose = np.zeros(16, np.float32)
    st = R.ref_system_find_camera_pose(s, P(np.ascontiguousarray(rgba)), t_ms, P(pose))
    ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); T = np.zeros(7)
    info = np.zeros(8, np.int32)
    n = R.ref_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP, P(T))
    R.ref_system_info8(s, P(info))
    return st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy(), wp[:n].copy(), RP.ref_system_p3p_req(s)


class CpuRun:
    """the CPU state machine under a preset, frame by frame"""

    def __init__(self, S, name, w, h, K, hook=None):
        self.S = S
        self.s = S.cpu_preset_system_create(w, h, K[0], K[1], K[2], K[3])
        assert S.cpu_preset_system_set_preset(self.s, PRESETS[name][0]) == 0
        if hook is not None:
            S.cpu_preset_system_set_essential_hook(self.s, hook)

    def frame(self, rgba, t_ms):
        S, s = self.S, self.s
        T = np.zeros(7)
        st = S.cpu_preset_system_process(s, P(np.ascontiguousarray(rgba)), t_ms, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); info = np.zeros(8, np.int32)
        n = S.cpu_preset_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP)
        S.cpu_preset_system_info(s, P(info))
        return st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy(), wp[:n].copy()

    def counters(self):
        """{pnp_prior, p3p_fallback, local_ba, free_pose_clamp, max_kps, cell}"""
        o = np.zeros(6, np.int32)
        self.S.cpu_preset_system_counters(self.s, P(o))
        return dict(zip(("pnp_prior", "p3p_fallback", "local_ba", "free_pose_clamp", "max_kps", "cell"), o.tolist()))

    def close(self):
        self.S.cpu_preset_system_destroy(self.s)
