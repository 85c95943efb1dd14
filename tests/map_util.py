"""Shared by the map blob tests: the CPU oracle build of the System state machine with the map blob
(tests/host/system_cpu_map.cpp), optionally under AddressSanitizer and UBSan, a frame-by-frame runner, and a parser of the blob's
section boundaries (include/alva_b200.h, alva_system_save_map) for the refusal tests."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np

import reloc_util as U
from alvaar_b200 import synth

ROOT = U.ROOT
BUILD = os.path.join(ROOT, "tests", "_build")
P = U.P
CAP = 8192
E_INVALID, E_CAPACITY, E_STATE = -1, -3, -4


def cpu_map_system_lib(sanitize=False):
    """alvaar_b200/csrc/system_core.h over the CPU oracle with relocalisation and the map blob; sanitize=True builds it with
    -fsanitize=address,undefined (load it only in a process started with libasan preloaded)"""
    import fisheye_util
    U.cpu_reloc_system_lib()      # builds the oracles it links
    fisheye_util.oracle_lib()
    name = "libsystem_cpu_map_san.so" if sanitize else "libsystem_cpu_map.so"
    so = os.path.join(BUILD, name)
    orc = U._oracle_so()
    libs = [os.path.join(BUILD, n) for n in ("libclahe_oracle.so", "libmatch_cell_oracle.so", "libreloc_oracle.so", "libfisheye_oracle.so")]
    host = os.path.join(ROOT, "tests", "host")
    srcs = [os.path.join(host, f) for f in ("system_cpu_map.cpp", "system_cpu_reloc.cpp", "system_cpu_preset.cpp", "system_cpu_clahe.cpp",
                                            "system_cpu_backend.cpp")]
    srcs += [os.path.join(ROOT, "alvaar_b200", "csrc", "system_core.h"), os.path.join(ROOT, "alvaar_b200", "csrc", "camera_model.h"), orc] + libs
    if U._stale(so, srcs):
        flags = ["-O1", "-g", "-fno-omit-frame-pointer", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"] if sanitize else ["-O2"]
        subprocess.check_call(["g++"] + flags + ["-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc] + libs +
                              ["-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + BUILD])
    return so


def bind(so):
    S = C.CDLL(so)
    vp = C.c_void_p
    S.cpu_map_system_create.restype = vp
    S.cpu_map_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    S.cpu_map_system_destroy.argtypes = [vp]
    S.cpu_map_system_reset.argtypes = [vp]
    S.cpu_map_system_set_relocalisation.argtypes = [vp, C.c_int]
    S.cpu_map_system_set_preset.argtypes = [vp, C.c_int]
    S.cpu_map_system_set_distortion.argtypes = [vp] + [C.c_double] * 4
    S.cpu_map_system_set_fisheye.argtypes = [vp, C.c_int] + [C.c_double] * 4
    S.cpu_map_system_process.argtypes = [vp, vp, C.c_double, vp]
    S.cpu_map_system_keypoints.argtypes = [vp, vp, vp, vp, C.c_int]
    S.cpu_map_system_info.argtypes = [vp, vp]
    S.cpu_map_system_counters.argtypes = [vp, vp]
    S.cpu_map_system_save.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    S.cpu_map_system_load.argtypes = [vp, C.c_char_p, C.c_size_t]
    S.cpu_map_system_error.argtypes = [vp]
    S.cpu_map_system_error.restype = C.c_char_p
    return S


class CpuMapRun:
    """the CPU state machine, frame by frame: frame() -> (status, Twc7, info8, ids, px, is3d); save() -> bytes; load(bytes) -> rc"""

    def __init__(self, S, max_lost=None, preset=None, dist=None, fisheye=None, w=U.W, h=U.H):
        K = synth.intrinsics(w, h)
        self.S, self.s = S, S.cpu_map_system_create(w, h, *K)
        if preset is not None:
            assert S.cpu_map_system_set_preset(self.s, preset) == 0
        if dist is not None:
            S.cpu_map_system_set_distortion(self.s, *dist)
        if fisheye is not None:
            S.cpu_map_system_set_fisheye(self.s, 1, *fisheye)
        if max_lost is not None:
            assert S.cpu_map_system_set_relocalisation(self.s, max_lost) == 0

    def frame(self, rgba, t_ms):
        S, s = self.S, self.s
        T = np.zeros(7)
        st = S.cpu_map_system_process(s, P(np.ascontiguousarray(rgba)), t_ms, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8)
        info = np.zeros(8, np.int32)
        n = S.cpu_map_system_keypoints(s, P(ids), P(px), P(d3), CAP)
        S.cpu_map_system_info(s, P(info))
        return st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy()

    def save(self):
        """-> bytes, or the negative error code"""
        n = C.c_size_t(0)
        rc = self.S.cpu_map_system_save(self.s, None, 0, C.byref(n))
        if rc:
            return rc
        buf = C.create_string_buffer(max(n.value, 1))
        rc = self.S.cpu_map_system_save(self.s, buf, n.value, C.byref(n))
        return rc if rc else buf.raw[:n.value]

    def load(self, blob):
        return self.S.cpu_map_system_load(self.s, blob, len(blob))

    def error(self):
        return self.S.cpu_map_system_error(self.s).decode()

    def counters(self):
        o = np.zeros(8, np.int32)
        self.S.cpu_map_system_counters(self.s, P(o))
        return dict(zip(("n_kf_ids", "n_mp_ids", "lost", "lost_frames", "table_points", "table_version", "keyframes", "mappoints"), o.tolist()))

    def close(self):
        self.S.cpu_map_system_destroy(self.s)


def same_frame(x, y):
    """status, pose, info, ids, pixels and 3-D flags bit for bit"""
    return (x[0] == y[0] and (x[1].view(np.uint64) == y[1].view(np.uint64)).all() and (x[2] == y[2]).all() and len(x[3]) == len(y[3])
            and (x[3] == y[3]).all() and (x[4].view(np.uint32) == y[4].view(np.uint32)).all() and (x[5] == y[5]).all())


# ------------------------------------------------------------------------------------------------ blob layout
def sections(blob):
    """the offsets where each section and record of a version-1 blob starts, by name, and the parsed counters.
    -> (list of (name, offset)), dict"""
    b = memoryview(blob)
    off = 0
    out = [("header", 0)]
    magic, ver, total, nkf, nmp = struct.unpack_from("<4sIQII", b, off); off += 24
    out.append(("camera", off)); off += 4 + 4 + 32 + 4 + 32
    out.append(("grid", off)); off += 4
    out.append(("counters", off))
    n_kf_ids, n_mp_ids, n_kf = struct.unpack_from("<iii", b, off); off += 12
    out.append(("pose", off)); off += 56
    for k in range(nkf):
        out.append(("keyframe%d" % k, off))
        off += 4 + 4 + 56
        (nkp,) = struct.unpack_from("<I", b, off); off += 4
        out.append(("keypoints%d" % k, off))
        off += 78 * nkp
        (nc,) = struct.unpack_from("<I", b, off); off += 4
        out.append(("covis%d" % k, off))
        off += 8 * nc
        (nl,) = struct.unpack_from("<I", b, off); off += 4
        out.append(("localmap%d" % k, off))
        off += 4 * nl
    first_mp = off
    for k in range(nmp):
        out.append(("mappoint%d" % k, off))
        off += 4 + 4 + 1 + 1 + 8 + 24
        (no,) = struct.unpack_from("<I", b, off); off += 4 + 4 * no
        (nd,) = struct.unpack_from("<I", b, off); off += 4 + 40 * nd
        off += 33
    assert off == len(blob) == total
    return out, dict(magic=magic, version=ver, total=total, nkf=nkf, nmp=nmp, n_kf_ids=n_kf_ids, n_mp_ids=n_mp_ids, n_kf=n_kf,
                     first_mp=first_mp)


def mappoint_records(blob):
    """[(offset, id, anchor, obs offsets)] of every map point record"""
    secs, info = sections(blob)
    b = memoryview(blob)
    recs = []
    for name, off in secs:
        if not name.startswith("mappoint"):
            continue
        mid, anchor = struct.unpack_from("<ii", b, off)
        (no,) = struct.unpack_from("<I", b, off + 42)
        recs.append((off, mid, anchor, [off + 46 + 4 * i for i in range(no)]))
    return recs
