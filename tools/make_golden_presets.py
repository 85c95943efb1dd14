#!/usr/bin/env python3
"""Dump the preset golden vectors (committed) from the reference library (oracle/_ref/libalva_ref.so, oracle/build_ref.sh), its
preset harness (oracle/_ref/libalva_ref_preset.so, oracle/build_ref_preset.sh) and its CLAHE harness (libalva_ref_clahe.so).

tests/golden/detect_presets.npz: FeatureExtractor::detectFeaturePoints at the preset cell sizes 35, 45 and 50 (the `cell & 3`
tails 3, 1 and 2 of OpenCV's 3x3 blur), in the format of tests/golden/detect.npz: image, cell, current points, roi, the
detected points and the float intermediate of one cell.

tests/golden/system_preset_{fast,average,accurate}.npz: the reference's own System under the preset (ref_system_set_preset +
ref_system_set_clahe: state.hpp:9-17) over the 100 synthetic frames of tests/golden/system.npz (same seed).  Same fields as
system_clahe.npz -- `ref_*` (with `ref_p3p_req`: VisualFrontend::p3pReq_ after each frame), `cpu_*` (the CPU oracle state
machine under the preset, its own initialisation), the reference's initialisation result (`ref_init_Rt`, `ref_init_outlier`)
and every call of its five-point stage (`ess_*`) -- plus what the trace exercised (`counters_*`).  The generator asserts that
the CPU state machine, given the reference's initialisation, follows the reference trace, and that the 21-free-pose limit of
the local BA (system_core.h) never engages."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from alvaar_b200 import synth  # noqa: E402
from preset_util import P, PRESETS, CpuRun, cpu_preset_system_lib, ref_frame, ref_preset_lib, ref_system_create  # noqa: E402
from ref_golden import digest  # noqa: E402

# tag -> (w, h, cell, seed, number of current points)
DETECT = {"c35": (320, 240, 35, 11, 0), "c45": (333, 251, 45, 12, 9), "c50": (640, 480, 50, 13, 40), "c35b": (480, 360, 35, 14, 60)}


def dump_detect(R):
    R.ref_detect_points.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_int]
    d = {}
    for tag, (w, h, cs, seed, ncur) in DETECT.items():
        fr, _ = synth.make_frames(1, w, h, seed=seed, rgba=False)
        img = np.ascontiguousarray(fr[0])
        rng = np.random.default_rng(seed)
        cur = np.stack([rng.uniform(0, w - 1, ncur), rng.uniform(0, h - 1, ncur)], 1).astype(np.float32) if ncur else np.zeros((0, 2), np.float32)
        roi = np.array([20, 20, w - 40, h - 40], np.int32)
        out = np.zeros((4096, 2), np.float32)
        n = R.ref_detect_points(P(img), w, h, cs, P(cur), ncur, P(roi), 0.001, P(out), 4096)
        hm = np.zeros((cs, cs), np.float32)
        bl = np.zeros((cs, cs), np.uint8)
        R.ref_min_eig_cell(P(img), w, h, cs, cs, cs, P(hm), P(bl))
        d.update({f"{tag}_img": img, f"{tag}_cell": cs, f"{tag}_cur": cur, f"{tag}_roi": roi, f"{tag}_pts": out[:n].copy(),
                  f"{tag}_hmap11": hm, f"{tag}_blur11": bl})
        print("detect", tag, f"{w}x{h} cell {cs}: points", n)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "detect_presets.npz"), **d)


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


def run_cpu(S, name, frames, K, hook=None):
    r = CpuRun(S, name, frames.shape[2], frames.shape[1], K, hook)
    tr = Trace()
    for k in range(len(frames)):
        tr.add(*r.frame(frames[k], k * 33.333))
    c = r.counters()
    r.close()
    return tr, c


def dump_system(R, RP, name):
    w, h, nf, seed = 640, 480, 100, 7
    K = synth.intrinsics(w, h)
    frames = synth.make_frames(nf, w, h, seed=seed, rgba=True)[0]
    preset, cell, ratio, p3p, clahe = PRESETS[name]
    d = {"w": w, "h": h, "nframes": nf, "seed": seed, "K": np.array(K), "sha256": hashlib.sha256(frames.tobytes()).hexdigest(),
         "preset": preset, "cell": cell, "filter_ratio": ratio, "p3p": p3p, "clahe": clahe}
    s = ref_system_create(R, RP, name, w, h, K)
    grid = np.zeros(5, np.int32)
    RP.ref_system_grid(s, P(grid))
    assert grid[0] == cell and grid[2] == cell and grid[1] == int(np.ceil(w / cell) * np.ceil(h / cell)), grid
    tr, pose16, p3p_req = Trace(), [], []
    for k in range(nf):
        st, T, info, ids, px, d3, wp, req = ref_frame(R, RP, s, frames[k], k * 33.333)
        tr.add(st, T, info, ids, px, d3, wp)
        p3p_req.append(req)
    R.ref_system_destroy.argtypes = [C.c_void_p]
    R.ref_system_destroy(s)
    d.update(tr.dump("ref_"))
    d["ref_p3p_req"] = np.array(p3p_req, np.int32)
    kfid = d["ref_info"][:, 1]
    d["first_ba_frame"] = int(np.argmax(kfid >= 2)) if (kfid >= 2).any() else nf
    S = cpu_preset_system_lib()
    own, c_own = run_cpu(S, name, frames, K)
    d.update(own.dump("cpu_"))
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
    hooked, c_hooked = run_cpu(S, name, frames, K, C.cast(cb, C.c_void_p))
    first = next(c for c in calls if c["ok"])
    d["ref_init_Rt"], d["ref_init_outlier"] = first["Rt"], first["outl"]
    d["ess_ncalls"] = len(calls)
    for i, c in enumerate(calls):
        d.update({f"ess_c{i}_{k}": v for k, v in c.items()})
    for k in range(nf):
        assert hooked.status[k] == tr.status[k] and (hooked.info[k] == tr.info[k]).all(), (k, hooked.status[k], tr.status[k])
        assert (hooked.ids[k] == tr.ids[k]).all() and (hooked.is3d[k] == tr.is3d[k]).all(), k
        assert np.abs(hooked.T[k] - tr.T[k]).max() < 1e-9, k
    for pre, c in (("own", c_own), ("lockstep", c_hooked)):
        d.update({f"counters_{pre}_{k}": np.int32(v) for k, v in c.items()})
    # the 21-free-pose limit (system_core.h, localBA) holds keyframes fixed where the reference would free them: a preset trace
    # that reaches it would no longer be the reference's behaviour
    assert c_own["free_pose_clamp"] == 0 and c_hooked["free_pose_clamp"] == 0, (c_own, c_hooked)
    init = int(np.argmax(d["ref_status"] == 1))
    print(f"{name}: cell {cell}, max keypoints {c_hooked['max_kps']}; initialised at frame {init}, keyframes {int(kfid.max())}, "
          f"first local BA at frame {d['first_ba_frame']}, local BAs {c_hooked['local_ba']}, frames posed by PnP from the prior "
          f"{c_hooked['pnp_prior']}, p3pReq_ fallbacks {c_hooked['p3p_fallback']} (reference: p3pReq_ set after "
          f"{int(d['ref_p3p_req'].sum())} frames), 21-free-pose limit engaged {c_hooked['free_pose_clamp']} times "
          f"(own initialisation: {c_own}); CPU state machine in lockstep given the reference's initialisation")
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", f"system_preset_{name}.npz"), **d)


def main():
    R = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libalva_ref.so"))
    R.ref_config(0, 1)
    R.ref_config_time_caps(1)   # the Ceres solves' wall-clock caps lifted (oracle/build_ref.sh): the golden must not depend on host load
    RP = ref_preset_lib(R)
    assert RP is not None, "oracle/_ref/libalva_ref_preset.so or libalva_ref_clahe.so not built: bash oracle/build_ref_preset.sh"
    dump_detect(R)
    for name in ("fast", "average", "accurate"):
        dump_system(R, RP, name)


if __name__ == "__main__":
    main()
