#!/usr/bin/env python3
"""Dump the CLAHE golden vectors (committed) from the reference library (oracle/_ref/libalva_ref.so, oracle/build_ref.sh) and
its CLAHE harness (oracle/_ref/libalva_ref_clahe.so, oracle/build_ref_clahe.sh).

tests/golden/clahe.npz: for every case of tests/clahe_util.CASES (the three System geometries with their grids; a divisible,
an x-only, a y-only and a non-divisible size; tiles == size on each axis; clip 0, 3, 40 and 1e9; constant, two-valued and
noise images; a 4-frame batch) the SHA-256 digests (tests/ref_golden.digest) of the input and of what
cv::createCLAHE(clip, Size(tx, ty))->apply returns, frame by frame.

tests/golden/system_clahe.npz: the reference's own System with CLAHE on -- ref_system_set_clahe(1, 3.0, 50), the ACCURATE
preset's setting (state.hpp:9-17) -- over the 100 synthetic frames of tests/golden/system.npz (same seed) after the fixed
contrast map of tests/clahe_util.compress_contrast (v -> 16 + v // 4 on the colour channels); the frames' SHA-256 is stored.
Same `ref_*` fields as system.npz, plus `cpu_*` (the CPU oracle state machine with CLAHE, its own initialisation), the
reference's initialisation result (`ref_init_Rt`, `ref_init_outlier`) and every call of its five-point stage (`ess_*`:
input digest, result) for the initialisation hook of the CPU tests."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from alvaar_b200 import synth  # noqa: E402
from clahe_util import CASES, case_input, compress_contrast, cpu_clahe_system_lib, ref_clahe_lib  # noqa: E402
from ref_golden import digest  # noqa: E402

P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
CAP = 4096


def dump_cases(RC):
    d = {}
    for k, (name, w, h, n, clip, tx, ty, kind) in enumerate(CASES):
        x = case_input(k)
        y = np.empty_like(x)
        for f in range(n):
            RC.ref_clahe(P(np.ascontiguousarray(x[f])), w, h, clip, tx, ty, P(y[f]))
        d[f"{name}/in"], d[f"{name}/out"] = digest(x), digest(y)
        print(name, "changed pixels", int((x != y).sum()), "of", x.size)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "clahe.npz"), **d)


class Trace:
    def __init__(self):
        self.status, self.T, self.info, self.start, self.ids, self.px, self.is3d, self.wpt = [], [], [], [0], [], [], [], []

    def add(self, st, T, info, ids, px, is3d, wpt):
        self.status.append(st); self.T.append(T.copy()); self.info.append(info.copy())
        self.ids.append(ids.copy()); self.px.append(px.copy()); self.is3d.append(is3d.copy()); self.wpt.append(wpt.copy())
        self.start.append(self.start[-1] + len(ids))

    def dump(self, pre):
        return {pre + "status": np.array(self.status, np.int32), pre + "Twc": np.array(self.T), pre + "info": np.array(self.info, np.int32),
                pre + "start": np.array(self.start, np.int32), pre + "ids": np.concatenate(self.ids), pre + "px": np.concatenate(self.px),
                pre + "is3d": np.concatenate(self.is3d), pre + "wpt": np.concatenate(self.wpt)}


def run_cpu(S, frames, K, hook=None):
    w, h = frames.shape[2], frames.shape[1]
    s = S.cpu_clahe_system_create(w, h, K[0], K[1], K[2], K[3])
    assert S.cpu_system_set_clahe(s, 1, 3.0, 50) == 0
    if hook is not None:
        S.cpu_clahe_system_set_essential_hook(s, hook)
    tr = Trace()
    for k in range(len(frames)):
        T = np.zeros(7)
        st = S.cpu_clahe_system_process(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); info = np.zeros(8, np.int32)
        n = S.cpu_clahe_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP)
        S.cpu_clahe_system_info(s, P(info))
        tr.add(st, T, info, ids[:n], px[:n], d3[:n], wp[:n])
    S.cpu_clahe_system_destroy(s)
    return tr


def dump_system(R, RC):
    R.ref_system_create.restype = C.c_void_p
    R.ref_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 8
    R.ref_system_find_camera_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    R.ref_system_keypoints.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    R.ref_system_info8.argtypes = [C.c_void_p, C.c_void_p]
    R.ref_system_destroy.argtypes = [C.c_void_p]
    R.ref_config_time_caps(1)   # the Ceres solves' wall-clock caps lifted (oracle/build_ref.sh): the golden must not depend on host load
    w, h, nf, seed = 640, 480, 100, 7
    K = synth.intrinsics(w, h)
    frames = compress_contrast(synth.make_frames(nf, w, h, seed=seed, rgba=True)[0])
    d = {"w": w, "h": h, "nframes": nf, "seed": seed, "K": np.array(K), "sha256": hashlib.sha256(frames.tobytes()).hexdigest(),
         "clip_limit": 3.0, "tile_size": 50}
    s = R.ref_system_create(w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0)
    RC.ref_system_set_clahe(s, 1, 3.0, 50)
    tr, pose16 = Trace(), []
    for k in range(nf):
        pose = np.zeros(16, np.float32)
        st = R.ref_system_find_camera_pose(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(pose))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); T = np.zeros(7); info = np.zeros(8, np.int32)
        n = R.ref_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP, P(T))
        R.ref_system_info8(s, P(info))
        tr.add(st, T, info, ids[:n], px[:n], d3[:n], wp[:n])
        pose16.append(pose)
        print(k, "status", st, "keypoints", n, "3-D", int(d3[:n].sum()), "keyframe", info[1])
    R.ref_system_destroy(s)
    d.update(tr.dump("ref_"))
    d["ref_pose16"] = np.array(pose16)
    kfid = d["ref_info"][:, 1]
    d["first_ba_frame"] = int(np.argmax(kfid >= 2)) if (kfid >= 2).any() else nf   # Optimizer::localBA runs from keyframe id 2 on
    S = cpu_clahe_system_lib()
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
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "system_clahe.npz"), **d)


def main():
    R = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libalva_ref.so"))
    R.ref_config(0, 1)
    RC = ref_clahe_lib(R)
    assert RC is not None, "oracle/_ref/libalva_ref_clahe.so not built: bash oracle/build_ref_clahe.sh"
    dump_cases(RC)
    dump_system(R, RC)


if __name__ == "__main__":
    main()
