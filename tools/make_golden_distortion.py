#!/usr/bin/env python3
"""Dump the lens-distortion golden vectors (committed) from the reference library (oracle/_ref/libalva_ref.so,
oracle/build_ref.sh) and its CameraCalibration harness (oracle/_ref/libalva_ref_camera.so, oracle/build_ref_camera.sh).

tests/golden/camera.npz: for every case of tests/camera_util.CASES (a webcam-like lens, a strong barrel at 1280x720, and a
lens whose model folds back inside the sampled range, so that cv::undistortPoints' icdist < 0 fallback fires) the SHA-256
digests (tests/ref_golden.digest; NaNs canonicalised, camera_util.canonical) of the seeded inputs and of the reference's
CameraCalibration::undistortImagePoint / projectCamToImageDist outputs: ~8e4 pixels inside, at the corners of and up to
100 px outside the image; ~2.2e4 camera points in front of, behind (z < 0) and on the plane of (z = 0) the camera.

tests/golden/system_dist.npz: the reference's own System configured with the lens camera_util.SYSTEM_DIST over 100 synthetic
640x480 frames rendered through that lens (synth.make_frames(..., dist=SYSTEM_DIST), seed 7; the frames' SHA-256 is stored).
The same `ref_*` fields as system.npz (status, ids in the reference's order, 3-D flags, counters, poses, world points,
getFramePoints `ref_xy*`, the API's pose16), the reference's initialisation result (`ref_init_Rt`, `ref_init_outlier`), every
call of its five-point stage (`ess_*`) for the CPU tests' initialisation hook, `cpu_*` (the CPU oracle state machine with the
lens, its own initialisation), and `ref_spread_*`: how far the reference moves from itself when one intrinsic changes by one
or two ulps (16 runs, as tools/make_golden_system.py; `ref_build_*` is zero: no FMA rebuild) -- the free-running pose band."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from alvaar_b200 import synth  # noqa: E402
from camera_util import (CASES, SYSTEM_DIST, case_K, case_pixels, case_points, cdigest, cpu_dist_system_lib,  # noqa: E402
                         ref_camera_lib, run_ref)
from ref_golden import digest  # noqa: E402

P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
CAP = 4096


def dump_cases(RC):
    d = {}
    for k, (name, w, h, dist) in enumerate(CASES):
        K, D = case_K(k)
        px, X = case_pixels(k), case_points(k)
        un = run_ref(RC.ref_undistort_points, px, K, D, w, h)
        uv = run_ref(RC.ref_project_points, X, K, D, w, h)
        d[f"{name}/K"], d[f"{name}/D"] = K, D
        d[f"{name}/px"], d[f"{name}/X"] = digest(px), digest(X)
        d[f"{name}/unpx"], d[f"{name}/uv"] = cdigest(un), cdigest(uv)
        # the fallback's own pixels: where the first iteration's icdist is negative (the result is the pinhole point)
        x, y = (px[:, 0] - K[2]) / K[0], (px[:, 1] - K[3]) / K[1]
        r2 = x * x + y * y
        fold = int((1 + (D[1] * r2 + D[0]) * r2 < 0).sum())
        d[f"{name}/n_fold"] = np.int32(fold)
        print(name, len(px), "pixels (max shift", float(np.abs(un - px).max()), "px,", fold, "fold back)", len(X), "points,",
              int(np.isnan(uv).any(1).sum()), "non-finite projections")
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "camera.npz"), **d)


class Trace:
    def __init__(self):
        self.status, self.T, self.info, self.start, self.ids, self.px, self.is3d, self.wpt = [], [], [], [0], [], [], [], []
        self.xy, self.xy_start = [], [0]

    def add(self, st, T, info, ids, px, is3d, wpt, xy=None):
        self.status.append(st); self.T.append(T.copy()); self.info.append(info.copy())
        self.ids.append(ids.copy()); self.px.append(px.copy()); self.is3d.append(is3d.copy()); self.wpt.append(wpt.copy())
        self.start.append(self.start[-1] + len(ids))
        if xy is not None:
            self.xy.append(xy.copy()); self.xy_start.append(self.xy_start[-1] + len(xy))

    def dump(self, pre):
        d = {pre + "status": np.array(self.status, np.int32), pre + "Twc": np.array(self.T), pre + "info": np.array(self.info, np.int32),
             pre + "start": np.array(self.start, np.int32), pre + "ids": np.concatenate(self.ids), pre + "px": np.concatenate(self.px),
             pre + "is3d": np.concatenate(self.is3d), pre + "wpt": np.concatenate(self.wpt)}
        if self.xy:
            d[pre + "xy"], d[pre + "xy_start"] = np.concatenate(self.xy), np.array(self.xy_start, np.int32)
        return d


def run_cpu(S, frames, K, hook=None):
    w, h = frames.shape[2], frames.shape[1]
    s = S.cpu_dist_system_create(w, h, K[0], K[1], K[2], K[3])
    S.cpu_system_set_distortion(s, *SYSTEM_DIST)
    if hook is not None:
        S.cpu_dist_system_set_essential_hook(s, hook)
    tr = Trace()
    for k in range(len(frames)):
        T = np.zeros(7)
        st = S.cpu_dist_system_process(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); info = np.zeros(8, np.int32)
        n = S.cpu_dist_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP)
        S.cpu_dist_system_info(s, P(info))
        tr.add(st, T, info, ids[:n], px[:n], d3[:n], wp[:n])
    S.cpu_dist_system_destroy(s)
    return tr


def ref_run(R, frames, K, keep=None):
    """the reference System with SYSTEM_DIST over the frames -> Trace (+ pose16 list)"""
    w, h, nf = frames.shape[2], frames.shape[1], len(frames)
    s = R.ref_system_create(w, h, K[0], K[1], K[2], K[3], *SYSTEM_DIST)
    tr, pose16 = Trace(), []
    for k in range(nf):
        pose = np.zeros(16, np.float32)
        st = R.ref_system_find_camera_pose(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(pose))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); T = np.zeros(7); info = np.zeros(8, np.int32)
        n = R.ref_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP, P(T))
        R.ref_system_info8(s, P(info))
        xy = np.zeros((CAP, 2), np.int32); i2 = np.zeros(CAP, np.int32); p2 = np.zeros((CAP, 2), np.float32)
        m = R.ref_system_get_frame_points(s, P(xy), P(i2), P(p2), CAP)
        tr.add(st, T, info, ids[:n], px[:n], d3[:n], wp[:n], xy[:m])
        pose16.append(pose)
        if keep is not None and not keep(k, st, ids[:n]):
            break
    R.ref_system_destroy(s)
    return tr, pose16


def dump_system(R):
    R.ref_system_create.restype = C.c_void_p
    R.ref_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 8
    R.ref_system_find_camera_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    R.ref_system_keypoints.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    R.ref_system_get_frame_points.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    R.ref_system_info8.argtypes = [C.c_void_p, C.c_void_p]
    R.ref_system_destroy.argtypes = [C.c_void_p]
    R.ref_config_time_caps(1)   # the Ceres solves' wall-clock caps lifted (oracle/build_ref.sh): the golden must not depend on host load
    w, h, nf, seed = 640, 480, 100, 7
    K = synth.intrinsics(w, h)
    frames = synth.make_frames(nf, w, h, seed=seed, rgba=True, dist=SYSTEM_DIST)[0]
    d = {"w": w, "h": h, "nframes": nf, "seed": seed, "K": np.array(K), "dist": np.array(SYSTEM_DIST),
         "sha256": hashlib.sha256(frames.tobytes()).hexdigest()}
    tr, pose16 = ref_run(R, frames, K)
    for k in range(nf):
        print(k, "status", tr.status[k], "keypoints", len(tr.ids[k]), "3-D", int(tr.is3d[k].sum()), "keyframe", tr.info[k][1])
    d.update(tr.dump("ref_"))
    d["ref_pose16"] = np.array(pose16)
    kfid = d["ref_info"][:, 1]
    d["first_ba_frame"] = int(np.argmax(kfid >= 2)) if (kfid >= 2).any() else nf   # Optimizer::localBA runs from keyframe id 2 on
    # the reference's own spread under a 1-2 ulp change of one intrinsic (tools/make_golden_system.py)
    base_T = np.array(tr.T)
    spread_t, spread_q, nruns = np.zeros(nf), np.zeros(nf), np.zeros(nf, np.int32)
    for which in range(4):
        for sgn in (+1, -1, +2, -2):
            Kp = list(K)
            for _ in range(abs(sgn)):
                Kp[which] = float(np.nextafter(Kp[which], Kp[which] + sgn))
            t2, _ = ref_run(R, frames, Kp, keep=lambda k, st, ids: st == tr.status[k] and len(ids) == len(tr.ids[k]) and (ids == tr.ids[k]).all())
            for k in range(len(t2.T)):
                if not (t2.status[k] == tr.status[k] and len(t2.ids[k]) == len(tr.ids[k]) and (t2.ids[k] == tr.ids[k]).all()):
                    break
                T = t2.T[k]
                spread_t[k] = max(spread_t[k], float(np.abs(T[:3] - base_T[k, :3]).max()))
                spread_q[k] = max(spread_q[k], float(np.sqrt(max(2.0 * (1.0 - abs(float(np.dot(T[3:], base_T[k, 3:])))), 0.0))))
                nruns[k] += 1
    d["ref_spread_t"], d["ref_spread_q"], d["ref_spread_runs"] = spread_t, spread_q, nruns
    d["ref_build_t"], d["ref_build_q"] = np.zeros(nf), np.zeros(nf)
    print("reference vs itself under a 1-ulp change of one intrinsic: max |dt|", float(spread_t.max()), "max |dq|", float(spread_q.max()))
    S = cpu_dist_system_lib()
    d.update(run_cpu(S, frames, K).dump("cpu_"))
    # the reference's five-point stage, call by call, as the initialisation hook of the CPU state machine
    calls = []
    HOOK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p)
    R.ref_essential_5pt.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p]

    def hook(b1, b2, n, it, err, opt, fx, fy, Rt, outl):
        ins = digest(np.concatenate([np.ctypeslib.as_array((C.c_double * (3 * n)).from_address(b1)),
                                     np.ctypeslib.as_array((C.c_double * (3 * n)).from_address(b2)),
                                     np.array([it, err, opt, fx, fy], np.float64)]))
        ok = R.ref_essential_5pt(b1, b2, n, it, err, opt, fx, fy, Rt, outl)
        calls.append({"in": ins, "ok": np.int32(ok), "Rt": np.ctypeslib.as_array((C.c_double * 12).from_address(Rt)).copy(),
                      "outl": np.ctypeslib.as_array((C.c_uint8 * n).from_address(outl)).copy()})
        return ok
    cb = HOOK(hook)
    hooked = run_cpu(S, frames, K, C.cast(cb, C.c_void_p))
    first = next(c for c in calls if c["ok"])
    d["ref_init_Rt"], d["ref_init_outlier"] = first["Rt"], first["outl"]
    d["ess_ncalls"] = len(calls)
    for i, c in enumerate(calls):
        d.update({f"ess_c{i}_{k}": v for k, v in c.items()})
    for k in range(nf):
        assert hooked.status[k] == tr.status[k] and (hooked.ids[k] == tr.ids[k]).all() and (hooked.px[k].view(np.uint32) == tr.px[k].view(np.uint32)).all(), k
        assert np.abs(hooked.T[k] - tr.T[k]).max() < 1e-9, k
    init = int(np.argmax(d["ref_status"] == 1))
    print("initialised at frame", init, "keyframes", int(kfid.max()), "first local BA at frame", d["first_ba_frame"],
          "; CPU state machine in lockstep given the reference's initialisation")
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "system_dist.npz"), **d)


def main():
    RC = ref_camera_lib()
    assert RC is not None, "oracle/_ref/libalva_ref_camera.so not built: bash oracle/build_ref_camera.sh"
    if "--system-only" not in sys.argv:
        dump_cases(RC)
    if "--cases-only" not in sys.argv:
        R = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libalva_ref.so"))
        R.ref_config(0, 1)
        dump_system(R)


if __name__ == "__main__":
    main()
