#!/usr/bin/env python3
"""H100 timing of OpenCV's whole distortion vector (alva_k_undistort_points_full / alva_k_project_points_full, and System with
alva_system_set_distortion_coeffs).  Writes one JSON file (default profiles/distortion_full_h100.json) with the card's name and
power limit read in the same run.
  points: 128 000 pixels undistorted and 128 000 camera points projected per lens of tests/camera_full_util.CASES, and the
          four-coefficient kernels on the same points; CUDA events around 200 launches after 20 warm-up launches
  system: per tracked frame (the median of the frames with status 1), lens 3 (SYSTEM_DIST plus k3 and a small tilt) against
          lens 1 (SYSTEM_DIST) on the same rendered sequence, at 640x480, 1280x720 and 1920x1080; the two are alternated in
          this one call, `rounds` times, and every median is reported, with the spread"""
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
from alvaar_b200 import Context, System, synth  # noqa: E402
from camera_full_util import CASES, case_K  # noqa: E402
from camera_util import SYSTEM_DIST  # noqa: E402

N = 128000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, reps=200, warm=20):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def points(ctx):
    rng = np.random.default_rng(0)
    out = {}
    for k, (name, w, h, d) in enumerate(CASES):
        K, D = case_K(k)
        px = torch.from_numpy(rng.uniform((0, 0), (w, h), (N, 2)).astype(np.float32)).cuda()
        z = rng.uniform(0.5, 10, N)
        X = torch.from_numpy(np.stack([(rng.uniform(0, w, N) - K[2]) / K[0] * z, (rng.uniform(0, h, N) - K[3]) / K[1] * z, z], 1)).cuda()
        un = torch.zeros((N, 2), dtype=torch.float32, device="cuda")
        uv = torch.zeros_like(un)
        out[name] = {"n_coeffs": len(d),
                     "undistort_full_us": timed(lambda: ctx.undistort_points_full(px, None, 1, N, K, D, un)),
                     "project_full_us": timed(lambda: ctx.project_points_full(X, N, K, D, uv)),
                     "undistort_4coef_us": timed(lambda: ctx.undistort_points(px, None, 1, N, K, D[:4], un)),
                     "project_4coef_us": timed(lambda: ctx.project_points(X, N, K, D[:4], uv))}
    return out


def system(w, h, nframes, rounds):
    fr, _ = synth.make_frames(nframes, w, h, seed=99, rgba=True, dist=SYSTEM_DIST)
    D3 = np.zeros(14)
    D3[:4] = SYSTEM_DIST
    D3[4], D3[12], D3[13] = 0.002, 1e-3, -1e-3
    res = {"lens1": [], "lens3": []}
    for _ in range(rounds):
        for key in ("lens1", "lens3"):
            s = System(w, h, *synth.intrinsics(w, h))
            if key == "lens1":
                s.set_distortion(*SYSTEM_DIST)
            else:
                s.set_distortion_coeffs(D3)
            ts = []
            for k in range(nframes):
                f = np.ascontiguousarray(fr[k])
                t0 = time.perf_counter()
                st, _ = s.find_camera_pose(f, k * 33.333)
                ts.append(((time.perf_counter() - t0) * 1e3, st))
            s.close()
            tracked = [t for t, st in ts if st == 1]
            res[key].append(float(np.median(tracked)) if tracked else None)
    return {k: {"ms_per_tracked_frame_medians": v, "spread_ms": (max(v) - min(v)) if None not in v else None} for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "distortion_full_h100.json"))
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    r = {"card": card(), "points": points(ctx), "n_points": N, "system": {}}
    ctx.close()
    for (w, h, n) in ((640, 480, 60), (1280, 720, 40), (1920, 1080, 30)):
        r["system"][f"{w}x{h}"] = system(w, h, n, a.rounds)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    json.dump(r, open(a.out, "w"), indent=1)
    print(json.dumps(r, indent=1))


if __name__ == "__main__":
    main()
