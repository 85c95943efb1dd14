"""Shared by the gyro tests: the CPU oracle build of the System state machine with the gyro mode
(tests/host/system_cpu_gyro.cpp), a numpy model of the mode's integration rule (system_core.h, SystemCore::setGyro), and the
synthetic data -- a camera panning over synth's textured plane, rendered with synth.render_gray, its gyro samples from the
path's analytic angular velocity (white noise, a constant bias, the W3C devicemotion axes of a rear camera) and 30 Hz frame
time stamps."""
import ctypes as C
import os
import subprocess

import numpy as np

import localisation_util as LU
import reloc_util as U
from alvaar_b200 import synth

ROOT = U.ROOT
BUILD = os.path.join(ROOT, "tests", "_build")
P = U.P
vp = C.c_void_p
CAP = 8192
W, H = U.W, U.H
R_CI = np.diag([1.0, -1.0, -1.0])   # devicemotion rotationRate axes -> rear camera axes
BIAS = np.array([0.012, -0.018, 0.009])
FISHEYE = (0.05, -0.01, 0.004, -0.001)
FRAME_MS = 1000.0 / 30.0


def cpu_gyro_system_lib(sanitize=False):
    """alvaar_b200/csrc/system_core.h over the CPU oracle with relocalisation, the localisation-only mode and the gyro mode"""
    LU.cpu_loc_system_lib()       # builds the oracles it links
    name = "libsystem_cpu_gyro_san.so" if sanitize else "libsystem_cpu_gyro.so"
    so = os.path.join(BUILD, name)
    orc = U._oracle_so()
    libs = [os.path.join(BUILD, n) for n in ("libclahe_oracle.so", "libmatch_cell_oracle.so", "libreloc_oracle.so", "libfisheye_oracle.so",
                                             "libreacquire_oracle.so")]
    host = os.path.join(ROOT, "tests", "host")
    srcs = [os.path.join(host, f) for f in ("system_cpu_gyro.cpp", "system_cpu_localisation.cpp", "system_cpu_map.cpp", "system_cpu_reloc.cpp",
                                            "system_cpu_preset.cpp", "system_cpu_clahe.cpp", "system_cpu_backend.cpp")]
    srcs += [os.path.join(ROOT, "alvaar_b200", "csrc", "system_core.h"), os.path.join(ROOT, "alvaar_b200", "csrc", "camera_model.h"), orc] + libs
    if U._stale(so, srcs):
        flags = ["-O1", "-g", "-fno-omit-frame-pointer", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"] if sanitize else ["-O2"]
        subprocess.check_call(["g++"] + flags + ["-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc] + libs +
                              ["-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + BUILD])
    return so


def bind(so):
    S = C.CDLL(so)
    S.cpu_gyro_system_create.restype = vp
    S.cpu_gyro_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    for n in ("destroy", "reset", "configure"):
        getattr(S, "cpu_gyro_system_" + n).argtypes = [vp]
    S.cpu_gyro_system_set_relocalisation.argtypes = [vp, C.c_int]
    S.cpu_gyro_system_set_distortion.argtypes = [vp] + [C.c_double] * 4
    S.cpu_gyro_system_set_fisheye.argtypes = [vp, C.c_int] + [C.c_double] * 4
    S.cpu_gyro_system_set_gyro.argtypes = [vp, C.c_int, vp, vp]
    S.cpu_gyro_system_process.argtypes = [vp, vp, C.c_double, vp, C.c_int, vp]
    S.cpu_gyro_system_stats.argtypes = [vp, vp, vp]
    S.cpu_gyro_system_keypoints.argtypes = [vp, vp, vp, vp, C.c_int]
    S.cpu_gyro_system_info.argtypes = [vp, vp]
    S.cpu_gyro_system_counters.argtypes = [vp, vp]
    S.cpu_gyro_system_save.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    S.cpu_gyro_system_error.argtypes = [vp]
    S.cpu_gyro_system_error.restype = C.c_char_p
    S.cpu_gyro_rotate_priors.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp]
    return S


_LIB = {}


def lib(sanitize=False):
    if sanitize not in _LIB:
        _LIB[sanitize] = bind(cpu_gyro_system_lib(sanitize))
    return _LIB[sanitize]


def _arr(a, dtype=np.float64):
    return None if a is None else np.ascontiguousarray(a, dtype)


class CpuGyroRun:
    """the CPU state machine, frame by frame: frame() -> (status, Twc7, info8, ids, px, is3d)"""

    def __init__(self, S, max_lost=None, dist=None, fisheye=None, gyro=None, w=W, h=H):
        K = synth.intrinsics(w, h)
        self.S, self.s = S, S.cpu_gyro_system_create(w, h, *K)
        if dist is not None:
            S.cpu_gyro_system_set_distortion(self.s, *dist)
        if fisheye is not None:
            S.cpu_gyro_system_set_fisheye(self.s, 1, *fisheye)
        if max_lost is not None:
            assert S.cpu_gyro_system_set_relocalisation(self.s, max_lost) == 0
        if gyro is not None:
            assert self.set_gyro(1, *gyro) == 0, self.error()

    def set_gyro(self, enabled, R_ci=None, bias=None):
        self._keep = (_arr(R_ci), _arr(bias))
        return self.S.cpu_gyro_system_set_gyro(self.s, enabled, None if R_ci is None else P(self._keep[0]),
                                                None if bias is None else P(self._keep[1]))

    def process(self, rgba, t_ms, samples=None, n=None):
        """-> (status or refusal code, Twc7); samples [n][7] or None"""
        T = np.zeros(7)
        sm = None if samples is None else np.ascontiguousarray(samples, np.float64)
        if n is None:
            n = 0 if sm is None else len(sm)
        st = self.S.cpu_gyro_system_process(self.s, P(np.ascontiguousarray(rgba)), float(t_ms), None if sm is None or sm.size == 0 else P(sm),
                                            int(n), P(T))
        return st, T

    def frame(self, rgba, t_ms, samples=None):
        st, T = self.process(rgba, t_ms, samples)
        S, s = self.S, self.s
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8)
        info = np.zeros(8, np.int32)
        n = S.cpu_gyro_system_keypoints(s, P(ids), P(px), P(d3), CAP)
        S.cpu_gyro_system_info(s, P(info))
        return st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy()

    def stats(self):
        """-> ({predicted, fallback, carried, rotated, kept, held}, dR [3, 3])"""
        o = np.zeros(6, np.int32)
        dR = np.zeros(9)
        self.S.cpu_gyro_system_stats(self.s, P(o), P(dR))
        return dict(zip(("predicted", "fallback", "carried", "rotated", "kept", "held"), o.tolist())), dR.reshape(3, 3)

    def counters(self):
        o = np.zeros(3, np.int32)
        self.S.cpu_gyro_system_counters(self.s, P(o))
        return dict(zip(("times_lost", "relocalised", "lost"), o.tolist()))

    def save(self):
        n = C.c_size_t(0)
        rc = self.S.cpu_gyro_system_save(self.s, None, 0, C.byref(n))
        if rc:
            return rc
        buf = C.create_string_buffer(max(n.value, 1))
        rc = self.S.cpu_gyro_system_save(self.s, buf, n.value, C.byref(n))
        return rc if rc else buf.raw[:n.value]

    def error(self):
        return self.S.cpu_gyro_system_error(self.s).decode()

    def close(self):
        self.S.cpu_gyro_system_destroy(self.s)


def rotate_priors_host(S, bv, flag, w, h, K4, D4, lens, R9, prior):
    """cpu_gyro_rotate_priors: the host build of alva_k_rotate_priors -> (prior, rotated)"""
    n = len(flag)
    pr = np.ascontiguousarray(prior, np.float32).copy()
    rot = np.zeros(max(n, 1), np.uint8)
    S.cpu_gyro_rotate_priors(P(np.ascontiguousarray(bv, np.float64)), P(np.ascontiguousarray(flag, np.uint8)), n, w, h,
                             P(np.ascontiguousarray(K4, np.float64)), None if D4 is None else P(np.ascontiguousarray(D4, np.float64)), lens,
                             P(np.ascontiguousarray(R9, np.float64)), P(pr), P(rot))
    return pr, rot[:n]


# ------------------------------------------------------------------------------------------------ the numpy model
def _exp(p):
    th2 = (p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]
    th = np.sqrt(th2)
    if th < 1e-6:
        a, b = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0
    else:
        a, b = np.sin(th) / th, (1.0 - np.cos(th)) / th2
    K = np.array([[0, -p[2], p[1]], [p[2], 0, -p[0]], [-p[1], p[0], 0]])
    return np.eye(3) + a * K + b * (np.outer(p, p) - th2 * np.eye(3))


def _omega_at(buf, tau):
    hi = next((i for i, s in enumerate(buf) if s[0] > tau), len(buf))
    L = buf[hi - 1] if hi > 0 else None
    Hs = buf[hi] if hi < len(buf) else None
    if L is not None and Hs is not None and Hs[0] - L[0] <= 50.0:
        f = (tau - L[0]) / (Hs[0] - L[0])
        return L[1:4] + (Hs[1:4] - L[1:4]) * f
    if L is not None and tau - L[0] <= 50.0:
        return L[1:4].copy()
    if Hs is not None and Hs[0] - tau <= 50.0:
        return Hs[1:4].copy()
    return None


def integrate(buf, A, B, bias):
    """dR over [A, B] by the mode's rule, or None when the interval is not covered"""
    if not B >= A:
        return None
    wa, wb = _omega_at(buf, A), _omega_at(buf, B)
    if wa is None or wb is None:
        return None
    inner = [s for s in buf if A < s[0] < B]
    for s0, s1 in zip(inner, inner[1:]):
        if s1[0] - s0[0] > 50.0:
            return None
    dR = np.eye(3)
    pts = [(A, wa)] + [(s[0], s[1:4]) for s in inner] + [(B, wb)]
    for (ta, w0), (tb, w1) in zip(pts, pts[1:]):
        dR = dR @ _exp(((w0 + w1) / 2.0 - bias) * ((tb - ta) / 1000.0))
    return dR


class GyroModel:
    """the mode's sample buffer and integration, frame by frame: frame(t, samples) -> dR_c or None (a fallback)"""

    def __init__(self, R_ci=None, bias=None):
        self.R = np.eye(3) if R_ci is None else np.asarray(R_ci, np.float64)
        self.b = np.zeros(3) if bias is None else np.asarray(bias, np.float64)
        self.buf, self.prev = [], None

    def frame(self, t, samples):
        self.buf += [np.asarray(s, np.float64) for s in samples]
        dR = None if self.prev is None else integrate(self.buf, self.prev, t, self.b)
        self.prev = t
        hi = next((i for i, s in enumerate(self.buf) if s[0] > t), len(self.buf))
        if hi > 1:
            self.buf = self.buf[hi - 1:]
        return None if dR is None else self.R @ dR @ self.R.T


# ------------------------------------------------------------------------------------------------ the pan sequence
def _rx(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def _ry(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


class PanPath:
    """A camera over synth's textured plane: n_init frames of sideways drift (for the initialisation), then the drift goes on
    under yaw and pitch sweeps.  A sweep is a raised cosine, yaw(tau) = amp (1 - cos(2 pi tau / period)) / 2 from the pan
    start: it starts and ends at rest and peaks at pi amp / period.  R_wc(t) = Ry(yaw) Rx(pitch); the camera-frame angular
    velocity is Rx(pitch)^T e_y yaw' + e_x pitch'."""

    def __init__(self, peak_dps=180.0, amp_deg=24.0, n_init=28, drift_px=3.0, pitch_ratio=0.5, w=W, h=H):
        fx = synth.intrinsics(w, h)[0]
        self.v = drift_px * 4.0 / fx * 30.0 / 1000.0            # world units per ms (drift_px per 30 Hz frame at the plane)
        self.t0 = n_init * FRAME_MS
        self.amp_y = np.radians(amp_deg)
        self.per_y = np.pi * self.amp_y / np.radians(peak_dps) * 1000.0   # ms
        self.amp_p = self.amp_y * pitch_ratio
        self.per_p = self.per_y * 1.37

    def _ang(self, t):
        tau = max(t - self.t0, 0.0)
        wy, wp = 2 * np.pi / self.per_y, 2 * np.pi / self.per_p
        yaw = self.amp_y * (1 - np.cos(wy * tau)) / 2
        pitch = self.amp_p * (1 - np.cos(wp * tau)) / 2
        dyaw = self.amp_y * wy * np.sin(wy * tau) / 2 * 1000.0 if t > self.t0 else 0.0   # rad/s
        dpitch = self.amp_p * wp * np.sin(wp * tau) / 2 * 1000.0 if t > self.t0 else 0.0
        return yaw, pitch, dyaw, dpitch

    def pose(self, t):
        yaw, pitch, _, _ = self._ang(t)
        return _ry(yaw) @ _rx(pitch), np.array([self.v * t, 0.3 * self.v * t, 0.0])

    def omega_cam(self, t):
        _, pitch, dyaw, dpitch = self._ang(t)
        return _rx(pitch).T @ np.array([0.0, dyaw, 0.0]) + np.array([dpitch, 0.0, 0.0])


def pan_sequence(nframes=90, peak_dps=180.0, hz=200.0, noise=0.003, seed=5, dist=None, fisheye=None, texture_seed=1234, blackout=None,
                 w=W, h=H, **kw):
    """-> (frames RGBA, frame times ms, samples per frame ([m][7]: the samples after the previous frame up to this one),
    true poses).  blackout = (first, count): those frames are uniform noise (the pose stays the path's)."""
    path = PanPath(peak_dps=peak_dps, w=w, h=h, **kw)
    rng = np.random.default_rng(seed)
    tex = synth.make_texture(seed=texture_seed)
    times = [k * FRAME_MS for k in range(nframes)]
    dt = 1000.0 / hz
    st = np.arange(rng.uniform(0, dt) - 40.0, times[-1] + 1e-9, dt)
    om = np.array([R_CI.T @ path.omega_cam(t) for t in st]) + BIAS + rng.normal(0, noise, (len(st), 3))
    acc = np.tile([0.0, 9.81, 0.0], (len(st), 1))
    allsmp = np.concatenate([np.round(st, 3)[:, None], om, acc], 1)
    frames, smp, poses = [], [], []
    prev = -np.inf
    for k, t in enumerate(times):
        pose = path.pose(t)
        poses.append(pose)
        if blackout and blackout[0] <= k < blackout[0] + blackout[1]:
            frames.append(np.ascontiguousarray(rng.integers(0, 256, (h, w, 4), dtype=np.uint8)))
        else:
            frames.append(synth.gray_to_rgba(synth.render_gray(tex, pose, w, h, dist=dist, fisheye=fisheye)))
        smp.append(allsmp[(allsmp[:, 0] > prev) & (allsmp[:, 0] <= t)])
        prev = t
    return frames, times, smp, poses


def run_cpu(S, frames, times, smp, gyro=True, max_lost=None, dist=None, fisheye=None, R_ci=R_CI, bias=BIAS, stats_every=False):
    """the whole sequence on the CPU state machine -> list of (status, Twc7, info, ids, px, is3d) and the final stats"""
    r = CpuGyroRun(S, max_lost=max_lost, dist=dist, fisheye=fisheye, gyro=(R_ci, bias) if gyro else None)
    out = [r.frame(frames[k], times[k], smp[k]) for k in range(len(frames))]
    stats = r.stats()
    r.close()
    return out, stats
