"""CLAHE on the H100, one run: (1) alva_k_clahe on 64 frames of 1280x720 (grid 25x14, clip 3: the System's 720p setting), CUDA
events after a warm-up, with its algorithmic bytes (read W*H for the histograms, read W*H + write W*H for the apply) and their
share of the H100 SXM's 3.35 TB/s; (2) the per-tracked-frame latency of System.find_camera_pose at 640x480 and 1280x720 with
CLAHE off and on, interleaved in the same process.  Prints one JSON object; --out FILE also writes it there.
Usage: python tools/gpu_clahe_bench.py [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alvaar_b200  # noqa: E402
from alvaar_b200 import synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def kernel(nframes=64, w=1280, h=720, tx=25, ty=14, iters=50):
    ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    rng = np.random.default_rng(0)
    yy, xx = np.mgrid[0:h, 0:w]
    x = np.clip(30 + 40 * xx / w + 20 * yy / h + rng.normal(0, 6, (nframes, h, w)), 0, 255).astype(np.uint8)
    src = torch.from_numpy(x).cuda()
    dst = torch.empty_like(src)
    for _ in range(10):
        ctx.clahe(src, dst, w, h, nframes, 3.0, tx, ty)
    torch.cuda.synchronize()
    times = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            ctx.clahe(src, dst, w, h, nframes, 3.0, tx, ty)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / iters * 1e-3)
    ctx.close()
    t = float(np.median(times))
    nbytes = 3 * w * h * nframes
    return {"frames": nframes, "w": w, "h": h, "tiles": [tx, ty], "clip_limit": 3.0, "time_us_median": t * 1e6,
            "time_us_min": min(times) * 1e6, "algorithmic_bytes": nbytes, "achieved_GBps": nbytes / t / 1e9,
            "fraction_of_3.35TBps": nbytes / t / HBM_BYTES_PER_S, "us_per_frame": t * 1e6 / nframes}


def system_latency(w, h, nframes=60, passes=2):
    K = synth.intrinsics(w, h)
    frames, _ = synth.make_frames(nframes, w, h, seed=7, rgba=True)
    out = {}
    for p in range(passes):   # off / on interleaved, so that both see the same host and device state
        for on in (False, True):
            s = alvaar_b200.System(w, h, *K)
            if on:
                s.set_clahe(True, 3.0, 50)
            lat = []
            for k in range(nframes):
                t0 = time.perf_counter()
                st, _ = s.find_camera_pose(frames[k], k * 33.333)   # returns after the device work of the frame is done
                dt = time.perf_counter() - t0
                if st == 1:
                    lat.append(dt)
            s.close()
            key = "clahe_on" if on else "clahe_off"
            out.setdefault(key, []).append({"tracked_frames": len(lat), "median_ms": float(np.median(lat)) * 1e3 if lat else None,
                                            "mean_ms": float(np.mean(lat)) * 1e3 if lat else None})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_clahe_bench.py needs an H100")
    res = dict(card())
    res["alva_k_clahe"] = kernel()
    res["system_per_tracked_frame"] = {f"{w}x{h}": system_latency(w, h) for w, h in ((640, 480), (1280, 720))}
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
