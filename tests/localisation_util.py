"""Shared by the localisation-only tests: the oracle of the re-acquisition match (oracle/reacquire_oracle.c, with the lens
projections of camera_oracle.c and fisheye_oracle.c), a brute-force numpy model of it, random problems with planted boundary
cases, and the CPU oracle build of the System state machine with the mode (tests/host/system_cpu_localisation.cpp),
optionally under AddressSanitizer and UBSan."""
import ctypes as C
import os
import subprocess

import numpy as np

import map_util as M
import reloc_util as U
from alvaar_b200 import synth

ROOT = U.ROOT
BUILD = os.path.join(ROOT, "tests", "_build")
P = U.P
vp = C.c_void_p
CAP = 8192
LENSES = {"pinhole": (0, None), "radtan": (1, (-0.12, 0.03, 0.001, -0.0005)), "fisheye": (2, (0.05, -0.01, 0.004, -0.001))}


def oracle_lib():
    """orc_match_frame_to_map (oracle/reacquire_oracle.c) and the lens projections it calls, built on demand into tests/_build"""
    so = os.path.join(BUILD, "libreacquire_oracle.so")
    srcs = [os.path.join(ROOT, "oracle", n) for n in ("reacquire_oracle.c", "camera_oracle.c", "fisheye_oracle.c")]
    if U._stale(so, srcs):
        os.makedirs(BUILD, exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-std=gnu11",
                               "-shared", "-o", so] + srcs + ["-lm"])
    L = C.CDLL(so)
    L.orc_match_frame_to_map.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_double] * 4 + [C.c_int, vp, vp, C.c_int, vp, vp, vp, vp,
                                                                                            C.c_int, vp, vp, vp, C.c_float, vp, vp]
    L.orc_project_points.argtypes = [vp, C.c_int, vp, vp, vp]
    L.orc_fisheye_project_points.argtypes = [vp, C.c_int, vp, vp, vp]
    return L


class Problem:
    """one re-acquisition problem: camera, lens, pose, table (RelocTable layout) and queries"""

    def __init__(self, w, h, cell, K, lens, coef, Twc, wpt, desc_start, desc, skip, q_px, q_desc, q_kept, radius):
        self.__dict__.update(locals())
        del self.__dict__["self"]

    @property
    def n_mp(self):
        return len(self.wpt)


def run_oracle(L, p):
    nq = len(p.q_px)
    row, dist = np.full(max(nq, 1), -7, np.int32), np.full(max(nq, 1), -7, np.int32)
    coef = np.ascontiguousarray(p.coef if p.coef is not None else np.zeros(4), np.float64)
    ds = np.ascontiguousarray(p.desc_start, np.int32)
    desc = np.ascontiguousarray(p.desc if len(p.desc) else np.zeros((1, 32), np.uint8))
    wpt = np.ascontiguousarray(p.wpt if len(p.wpt) else np.zeros((1, 3)), np.float64)
    qpx = np.ascontiguousarray(p.q_px if nq else np.zeros((1, 2), np.float32), np.float32)
    qd = np.ascontiguousarray(p.q_desc if nq else np.zeros((1, 32), np.uint8))
    qk = np.ascontiguousarray(p.q_kept if nq else np.zeros(1, np.uint8))
    skip = None if p.skip is None else np.ascontiguousarray(p.skip, np.uint8)
    n = L.orc_match_frame_to_map(p.w, p.h, p.cell, *p.K, p.lens, P(coef), P(np.ascontiguousarray(p.Twc, np.float64)), p.n_mp, P(wpt), P(ds),
                                 P(desc), None if skip is None else P(skip), nq, P(qpx), P(qd), P(qk), p.radius, P(row), P(dist))
    assert n >= 0
    return row[:nq], dist[:nq]


# ------------------------------------------------------------------------------------------------ the numpy model
_libm = C.CDLL("libm.so.6")
_libm.atanf.restype = _libm.cosf.restype = C.c_float
_libm.atanf.argtypes = _libm.cosf.argtypes = [C.c_float]


def world_to_cam(Twc, X):
    """Tcw X as map_geom.cuh computes it: the rotation from the normalised quaternion, in its expression order (float64)"""
    t, q = np.asarray(Twc[:3], np.float64), np.asarray(Twc[3:], np.float64)
    n = np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    x, y, z, w = q[0] / n, q[1] / n, q[2] / n, q[3] / n
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    R = [1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)]
    ti = [-(R[i] * t[0] + R[3 + i] * t[1] + R[6 + i] * t[2]) for i in range(3)]
    return np.stack([(R[i] * X[:, 0] + R[3 + i] * X[:, 1] + R[6 + i] * X[:, 2]) + ti[i] for i in range(3)], 1)


def project(L, p, c):
    """the pinhole in numpy; the lens models through the C camera oracles (pinned to OpenCV by their own tests)"""
    out = np.zeros((len(c), 2), np.float32)
    if len(c) == 0:
        return out
    K = np.ascontiguousarray(p.K, np.float64)
    if p.lens == 0:
        with np.errstate(divide="ignore", invalid="ignore"):
            iz = 1.0 / c[:, 2]
            x = (c[:, 0] * iz).astype(np.float32).astype(np.float64)
            y = (c[:, 1] * iz).astype(np.float32).astype(np.float64)
        return np.stack([(x * K[0] + K[2]).astype(np.float32), (y * K[1] + K[3]).astype(np.float32)], 1)
    cc = np.ascontiguousarray(c, np.float64)
    fn = L.orc_project_points if p.lens == 1 else L.orc_fisheye_project_points
    fn(P(cc), len(cc), P(K), P(np.ascontiguousarray(p.coef, np.float64)), P(out))
    return out


def run_numpy(L, p):
    """every map point against every query, no grid: the definition of the match"""
    nq = len(p.q_px)
    row, dist = np.full(nq, -1, np.int32), np.full(nq, -1, np.int32)
    if nq == 0 or p.n_mp == 0:
        return row, dist
    fovV, fovH = np.float32(0.5 * p.h / p.K[1]), np.float32(0.5 * p.w / p.K[0])
    view_th = _libm.cosf(_libm.atanf(float(fovH)) if fovH > fovV else _libm.atanf(float(fovV)))
    c = world_to_cam(p.Twc, np.asarray(p.wpt, np.float64))
    ok = np.ones(p.n_mp, bool) if p.skip is None else np.asarray(p.skip) == 0
    ok &= np.diff(p.desc_start) > 0
    ok &= c[:, 2] >= 0.1
    with np.errstate(divide="ignore", invalid="ignore"):
        va = (c[:, 2] / np.sqrt(c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1] + c[:, 2] * c[:, 2])).astype(np.float32)
    ok &= ~(np.abs(va.astype(np.float64)) < np.float64(np.float32(view_th)))
    proj = np.zeros((p.n_mp, 2), np.float32)
    proj[ok] = project(L, p, c[ok])
    ok &= (proj[:, 0] >= 0) & (proj[:, 1] >= 0) & (proj[:, 0].astype(np.float64) < p.w) & (proj[:, 1].astype(np.float64) < p.h)
    qpx = np.asarray(p.q_px, np.float32)
    qok = (np.asarray(p.q_kept) != 0) & np.isfinite(qpx).all(1)
    qbits = np.unpackbits(np.asarray(p.q_desc, np.uint8), axis=1).astype(np.int16)
    tbits = np.unpackbits(np.asarray(p.desc, np.uint8), axis=1).astype(np.int16) if len(p.desc) else np.zeros((0, 256), np.int16)
    best_d = np.full(nq, 1024)
    for m in np.nonzero(ok)[0]:
        dx = (proj[m, 0] - qpx[:, 0]).astype(np.float32).astype(np.float64)
        dy = (proj[m, 1] - qpx[:, 1]).astype(np.float32).astype(np.float64)
        pxd = np.sqrt(dx * dx + dy * dy).astype(np.float32)
        cand = np.nonzero(qok & (pxd <= np.float32(p.radius)))[0]
        if len(cand) == 0:
            continue
        rows = tbits[p.desc_start[m]:p.desc_start[m + 1]]
        d = (qbits[cand][:, None, :] != rows[None, :, :]).sum(-1).min(1)
        inside = d <= 51
        if not inside.any():
            continue
        dd, cq = d[inside], cand[inside]
        b = dd.min()
        q = cq[dd == b].max()
        if len(dd) >= 2:
            sec = np.sort(dd)[1]
            if 0.9 * float(sec) < float(b):
                continue
        if b <= best_d[q]:
            best_d[q] = b
            row[q] = m
    dist[row >= 0] = best_d[row >= 0]
    return row, dist


# ------------------------------------------------------------------------------------------------ random problems
def random_problem(rng, w=640, h=480, cell=40, lens="pinhole", n_mp=400, nq=300, max_rows=6, radius=2.0, min_rows=1):
    """a table of points in front of a random camera, and queries of which a share sit within the radius of a projection with
    a descriptor a few bits from one of the point's rows (close competitors, ties and ratio cases included)"""
    code, coef = LENSES[lens]
    fx = fy = 0.8 * w
    K = (fx, fy, w / 2 + 3.25, h / 2 - 2.5)
    ang = rng.normal(size=3) * 0.2
    from scipy.spatial.transform import Rotation
    q = Rotation.from_rotvec(ang).as_quat()
    t = rng.normal(size=3)
    Twc = np.concatenate([t, q])
    Rwc = Rotation.from_quat(q).as_matrix()
    # camera-frame points spread over (and a little beyond) the view, some behind or too close
    z = rng.uniform(-0.5, 8.0, n_mp)
    xs = (rng.uniform(-0.1, 1.1, n_mp) * w - K[2]) / fx * np.abs(z)
    ys = (rng.uniform(-0.1, 1.1, n_mp) * h - K[3]) / fy * np.abs(z)
    Xc = np.stack([xs, ys, z], 1)
    wpt = Xc @ Rwc.T + t
    rows = rng.integers(min_rows, max_rows + 1, n_mp)
    desc_start = np.concatenate([[0], np.cumsum(rows)]).astype(np.int32)
    desc = rng.integers(0, 256, (int(desc_start[-1]), 32), dtype=np.uint8)
    skip = (rng.random(n_mp) < 0.1).astype(np.uint8)
    p = Problem(w, h, cell, K, code, coef, Twc, wpt, desc_start, desc, skip, None, None, None, radius)
    L = oracle_lib()
    c = world_to_cam(Twc, wpt)
    front = c[:, 2] > 0.1
    proj = np.zeros((n_mp, 2), np.float32)
    proj[front] = project(L, p, c[front])
    qpx = np.zeros((nq, 2), np.float32)
    qdesc = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    src = rng.choice(np.nonzero(front)[0], nq) if front.any() else np.zeros(nq, int)
    for i in range(nq):
        m = src[i]
        r = rng.uniform(0, radius * 1.3)
        a = rng.uniform(0, 2 * np.pi)
        qpx[i] = proj[m] + np.float32([r * np.cos(a), r * np.sin(a)])
        if rng.random() < 0.8:
            row = desc[desc_start[m] + rng.integers(0, rows[m])]
            flip = np.packbits(rng.random(256) < rng.choice([0.0, 0.02, 0.1, 0.2, 0.3]))
            qdesc[i] = row ^ flip
    # duplicates: the same descriptor at several nearby queries (ties between queries and between map points)
    for i in range(0, nq - 1, 17):
        qdesc[i + 1] = qdesc[i]
        qpx[i + 1] = qpx[i] + np.float32([0.5, -0.25])
    qkept = (rng.random(nq) > 0.05).astype(np.uint8)
    p.q_px, p.q_desc, p.q_kept = qpx, qdesc, qkept
    return p


# ------------------------------------------------------------------------------------------------ the CPU state machine
def cpu_loc_system_lib(sanitize=False):
    """alvaar_b200/csrc/system_core.h over the CPU oracle with relocalisation, the map blob and the localisation-only mode"""
    M.cpu_map_system_lib()        # builds the oracles it links
    oracle_lib()
    name = "libsystem_cpu_loc_san.so" if sanitize else "libsystem_cpu_loc.so"
    so = os.path.join(BUILD, name)
    orc = U._oracle_so()
    libs = [os.path.join(BUILD, n) for n in ("libclahe_oracle.so", "libmatch_cell_oracle.so", "libreloc_oracle.so", "libfisheye_oracle.so",
                                             "libreacquire_oracle.so")]
    host = os.path.join(ROOT, "tests", "host")
    srcs = [os.path.join(host, f) for f in ("system_cpu_localisation.cpp", "system_cpu_map.cpp", "system_cpu_reloc.cpp", "system_cpu_preset.cpp",
                                            "system_cpu_clahe.cpp", "system_cpu_backend.cpp")]
    srcs += [os.path.join(ROOT, "alvaar_b200", "csrc", "system_core.h"), os.path.join(ROOT, "alvaar_b200", "csrc", "camera_model.h"), orc] + libs
    if U._stale(so, srcs):
        flags = ["-O1", "-g", "-fno-omit-frame-pointer", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"] if sanitize else ["-O2"]
        subprocess.check_call(["g++"] + flags + ["-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc] + libs +
                              ["-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + BUILD])
    return so


def bind(so):
    S = C.CDLL(so)
    S.cpu_loc_system_create.restype = vp
    S.cpu_loc_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    for n in ("destroy", "reset"):
        getattr(S, "cpu_loc_system_" + n).argtypes = [vp]
    for n in ("set_relocalisation", "set_localisation_only", "set_preset", "set_clahe"):
        getattr(S, "cpu_loc_system_" + n).argtypes = [vp, C.c_int]
    S.cpu_loc_system_set_distortion.argtypes = [vp] + [C.c_double] * 4
    S.cpu_loc_system_set_fisheye.argtypes = [vp, C.c_int] + [C.c_double] * 4
    S.cpu_loc_system_process.argtypes = [vp, vp, C.c_double, vp]
    S.cpu_loc_system_keypoints.argtypes = [vp, vp, vp, vp, C.c_int]
    S.cpu_loc_system_info.argtypes = [vp, vp]
    S.cpu_loc_system_counters.argtypes = [vp, vp]
    S.cpu_loc_system_save.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    S.cpu_loc_system_load.argtypes = [vp, C.c_char_p, C.c_size_t]
    S.cpu_loc_system_error.argtypes = [vp]
    S.cpu_loc_system_error.restype = C.c_char_p
    return S


COUNTERS = ("n_kf_ids", "n_mp_ids", "lost", "lost_frames", "table_points", "table_version", "keyframes", "mappoints", "frozen",
            "reacq_runs", "reacq_points", "reacq_last", "relocalised", "times_lost")


class CpuLocRun:
    """the CPU state machine, frame by frame: frame() -> (status, Twc7, info8, ids, px, is3d)"""

    def __init__(self, S, max_lost=None, preset=None, dist=None, fisheye=None, w=U.W, h=U.H):
        K = synth.intrinsics(w, h)
        self.S, self.s = S, S.cpu_loc_system_create(w, h, *K)
        if preset is not None:
            assert S.cpu_loc_system_set_preset(self.s, preset) == 0
        if dist is not None:
            S.cpu_loc_system_set_distortion(self.s, *dist)
        if fisheye is not None:
            S.cpu_loc_system_set_fisheye(self.s, 1, *fisheye)
        if max_lost is not None:
            assert S.cpu_loc_system_set_relocalisation(self.s, max_lost) == 0

    def frame(self, rgba, t_ms):
        S, s = self.S, self.s
        T = np.zeros(7)
        st = S.cpu_loc_system_process(s, P(np.ascontiguousarray(rgba)), t_ms, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8)
        info = np.zeros(8, np.int32)
        n = S.cpu_loc_system_keypoints(s, P(ids), P(px), P(d3), CAP)
        S.cpu_loc_system_info(s, P(info))
        return st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy()

    def freeze(self, on=True):
        return self.S.cpu_loc_system_set_localisation_only(self.s, 1 if on is True else (0 if on is False else on))

    def relocalisation(self, n):
        return self.S.cpu_loc_system_set_relocalisation(self.s, n)

    def save(self):
        n = C.c_size_t(0)
        rc = self.S.cpu_loc_system_save(self.s, None, 0, C.byref(n))
        if rc:
            return rc
        buf = C.create_string_buffer(max(n.value, 1))
        rc = self.S.cpu_loc_system_save(self.s, buf, n.value, C.byref(n))
        return rc if rc else buf.raw[:n.value]

    def load(self, blob):
        return self.S.cpu_loc_system_load(self.s, blob, len(blob))

    def error(self):
        return self.S.cpu_loc_system_error(self.s).decode()

    def counters(self):
        o = np.zeros(14, np.int32)
        self.S.cpu_loc_system_counters(self.s, P(o))
        return dict(zip(COUNTERS, o.tolist()))

    def close(self):
        self.S.cpu_loc_system_destroy(self.s)


def map_records(blob):
    """the keyframe and map point records of a blob with the fields a frozen session may change masked: the keyframes' ages
    (frame ids restart in every session) -> bytes"""
    secs, info = M.sections(blob)
    b = bytearray(blob)
    first = dict(secs)["keyframe0"] if info["nkf"] else info["first_mp"]
    for name, off in secs:
        if name.startswith("keyframe") and not name.startswith("keypoints"):
            b[off + 4:off + 8] = b"\0\0\0\0"
    return bytes(b[first:])
