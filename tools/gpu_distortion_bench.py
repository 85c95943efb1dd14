"""Lens distortion on the H100, one run: (1) alva_k_undistort_points on 64 frames x 2000 keypoints (the lens of
tests/camera_util.SYSTEM_DIST at 1920x1080), CUDA events after a warm-up, and alva_k_project_points on as many camera points;
(2) for comparison, the host's own cost of the same model: camera_model.h's host side undistorting 1300 points (a 1080p
frame's keypoint budget) on this machine's CPU; (3) the per-tracked-frame latency of System.find_camera_pose at 640x480,
1280x720 and 1920x1080 on frames rendered through that lens, without and with set_distortion, interleaved in the same
process on the same frames.  The card's name and power limit are read in the same run.  Prints one JSON object; --out FILE
also writes it there.
Usage: python tools/gpu_distortion_bench.py [--out FILE]"""
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
from camera_util import SYSTEM_DIST, cpu_dist_system_lib, run_points  # noqa: E402


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
    t, tmin = event_time(lambda: ctx.undistort_points(px, counts, nframes, cap, K, SYSTEM_DIST, un))
    n = nframes * cap
    z = rng.uniform(0.5, 10.0, n)
    Xc = torch.from_numpy(np.stack([rng.uniform(-0.8, 0.8, n) * z, rng.uniform(-0.45, 0.45, n) * z, z], 1)).cuda()
    uv = torch.empty((n, 2), dtype=torch.float32, device="cuda")
    tp, tpmin = event_time(lambda: ctx.project_points(Xc, n, K, SYSTEM_DIST, uv))
    ctx.close()
    return {"alva_k_undistort_points": {"frames": nframes, "points_per_frame": cap, "time_us_median": t * 1e6, "time_us_min": tmin * 1e6,
                                        "ns_per_point": t * 1e9 / n},
            "alva_k_project_points": {"points": n, "time_us_median": tp * 1e6, "time_us_min": tpmin * 1e6, "ns_per_point": tp * 1e9 / n}}


def host_undistort(n=1300, w=1920, h=1080, reps=200):
    """camera_model.h on the host CPU, the work the device path takes off a 1080p frame (one call per frame's keypoints)"""
    S = cpu_dist_system_lib()
    K, D = np.array(synth.intrinsics(w, h)), np.array(SYSTEM_DIST)
    px = np.ascontiguousarray(np.random.default_rng(1).uniform((0, 0), (w, h), (n, 2)).astype(np.float32))
    for _ in range(10):
        run_points(S.cpu_cam_undistort_points, px, K, D)
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        run_points(S.cpu_cam_undistort_points, px, K, D)
        times.append(time.perf_counter() - t0)
    return {"points": n, "median_us": float(np.median(times)) * 1e6, "min_us": float(min(times)) * 1e6,
            "note": "host CPU of the GPU machine, one ctypes call per frame; includes the call overhead"}


def system_latency(w, h, nframes=60, passes=2):
    K = synth.intrinsics(w, h)
    frames, _ = synth.make_frames(nframes, w, h, seed=7, rgba=True, dist=SYSTEM_DIST)
    out = {}
    for p in range(passes):   # off / on interleaved, so that both see the same host and device state
        for on in (False, True):
            s = alvaar_b200.System(w, h, *K)
            if on:
                s.set_distortion(*SYSTEM_DIST)
            lat = []
            for k in range(nframes):
                t0 = time.perf_counter()
                st, _ = s.find_camera_pose(frames[k], k * 33.333)   # returns after the device work of the frame is done
                dt = time.perf_counter() - t0
                if st == 1:
                    lat.append(dt)
            s.close()
            key = "distortion_on" if on else "distortion_off"
            out.setdefault(key, []).append({"tracked_frames": len(lat), "median_ms": float(np.median(lat)) * 1e3 if lat else None,
                                            "mean_ms": float(np.mean(lat)) * 1e3 if lat else None})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_distortion_bench.py needs an H100")
    res = dict(card())
    res["lens"] = {"k1": SYSTEM_DIST[0], "k2": SYSTEM_DIST[1], "p1": SYSTEM_DIST[2], "p2": SYSTEM_DIST[3]}
    res.update(kernels())
    res["host_undistort_1080p_frame"] = host_undistort()
    res["system_per_tracked_frame"] = {f"{w}x{h}": system_latency(w, h) for w, h in ((640, 480), (1280, 720), (1920, 1080))}
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
