"""The fisheye lens on the H100, one run: (1) alva_k_undistort_points_fisheye on 64 frames x 2000 keypoints (the lens of
tests/fisheye_util.SYSTEM_FISHEYE at 1920x1080), CUDA events after a warm-up, and alva_k_project_points_fisheye on 128 000 camera
points, beside the radial-tangential kernels on the same points; (2) the per-tracked-frame latency of System.find_camera_pose at
640x480, 1280x720 and 1920x1080 on frames rendered through that lens, pinhole against fisheye, in two interleaved passes in the
same process on the same frames.  The card's name and power limit are read in the same run.  Prints one JSON object; --out FILE
also writes it there (profiles/fisheye_h100.json).
Usage: python tools/gpu_fisheye_bench.py [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import alvaar_b200  # noqa: E402
from alvaar_b200 import synth  # noqa: E402
from camera_util import SYSTEM_DIST  # noqa: E402
from fisheye_util import SYSTEM_FISHEYE  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def event_time(fn, iters=200, reps=5):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / iters * 1e-3)
    return float(np.median(times)), float(min(times))


def kernels(nframes=64, cap=2000, w=1920, h=1080):
    ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    K = synth.intrinsics(w, h)
    rng = np.random.default_rng(0)
    px = torch.from_numpy(rng.uniform((0, 0), (w, h), (nframes, cap, 2)).astype(np.float32)).cuda()
    counts = torch.full((nframes,), cap, dtype=torch.int32, device="cuda")
    un = torch.empty_like(px)
    n = nframes * cap
    z = rng.uniform(0.5, 10.0, n)
    Xc = torch.from_numpy(np.stack([rng.uniform(-0.8, 0.8, n) * z, rng.uniform(-0.45, 0.45, n) * z, z], 1)).cuda()
    uv = torch.empty((n, 2), dtype=torch.float32, device="cuda")
    out = {}
    for name, fn in (("alva_k_undistort_points_fisheye", lambda: ctx.undistort_points_fisheye(px, counts, nframes, cap, K, SYSTEM_FISHEYE, un)),
                     ("alva_k_undistort_points", lambda: ctx.undistort_points(px, counts, nframes, cap, K, SYSTEM_DIST, un)),
                     ("alva_k_project_points_fisheye", lambda: ctx.project_points_fisheye(Xc, n, K, SYSTEM_FISHEYE, uv)),
                     ("alva_k_project_points", lambda: ctx.project_points(Xc, n, K, SYSTEM_DIST, uv))):
        t, tmin = event_time(fn)
        out[name] = {"points": n, "time_us_median": t * 1e6, "time_us_min": tmin * 1e6, "ns_per_point": t * 1e9 / n}
    ctx.close()
    return out


def system_latency(w, h, nframes=60, passes=2):
    K = synth.intrinsics(w, h)
    frames, _ = synth.make_frames(nframes, w, h, seed=7, rgba=True, fisheye=SYSTEM_FISHEYE)
    out = {}
    for p in range(passes):   # pinhole / fisheye interleaved, so that both see the same host and device state
        for on in (False, True):
            s = alvaar_b200.System(w, h, *K)
            if on:
                s.set_fisheye(True, *SYSTEM_FISHEYE)
            lat = []
            for k in range(nframes):
                t0 = time.perf_counter()
                st, _ = s.find_camera_pose(frames[k], k * 33.333)   # returns after the device work of the frame is done
                dt = time.perf_counter() - t0
                if st == 1:
                    lat.append(dt)
            s.close()
            key = "fisheye" if on else "pinhole"
            out.setdefault(key, []).append({"tracked_frames": len(lat), "median_ms": float(np.median(lat)) * 1e3 if lat else None,
                                            "mean_ms": float(np.mean(lat)) * 1e3 if lat else None})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_fisheye_bench.py needs an H100")
    res = dict(card())
    res["lens"] = {"fisheye_k1_k4": list(SYSTEM_FISHEYE), "radial_tangential_k1_k2_p1_p2": list(SYSTEM_DIST)}
    res.update(kernels())
    res["system_per_tracked_frame"] = {f"{w}x{h}": system_latency(w, h) for w, h in ((640, 480), (1280, 720), (1920, 1080))}
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
