"""The presets on the H100, one run: the latency of System.find_camera_pose under DEFAULT, FAST, AVERAGE and ACCURATE at 640x480,
1280x720 and 1920x1080 over the synthetic sequence (seed 7), through the public call.  A tracked frame (status 1) that created a
keyframe (the keyframe id moved) is counted as a keyframe, every other tracked frame as a tracked frame; medians of each.  Two
passes, the presets interleaved within each, so that all see the same host and device state.  Records the card and its power
limit in the same run.  Prints one JSON object; --out FILE also writes it there.
Usage: python tools/gpu_preset_bench.py [--out FILE] [--frames N]"""
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

PRESETS = ("default", "fast", "average", "accurate")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def one(frames, w, h, K, preset):
    s = alvaar_b200.System(w, h, *K)
    s.set_preset(preset)
    tracked, keyframes, statuses = [], [], []
    kf_prev = 0
    for k in range(len(frames)):
        t0 = time.perf_counter()
        st, _ = s.find_camera_pose(frames[k], k * 33.333)   # returns after the device work of the frame is done
        dt = time.perf_counter() - t0
        kf = s.info()["keyframe"]
        statuses.append(st)
        if st == 1:
            (keyframes if kf != kf_prev else tracked).append(dt)
        kf_prev = kf
    s.close()
    med = lambda v: float(np.median(v)) * 1e3 if v else None  # noqa: E731
    return {"tracked_frames": len(tracked), "keyframes": len(keyframes), "tracked_median_ms": med(tracked),
            "keyframe_median_ms": med(keyframes), "status_counts": {str(c): statuses.count(c) for c in sorted(set(statuses))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--frames", type=int, default=100)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_preset_bench.py needs an H100")
    res = dict(card())
    res["frames"] = a.frames
    res["passes"] = 2
    res["system"] = {}
    for w, h in ((640, 480), (1280, 720), (1920, 1080)):
        K = synth.intrinsics(w, h)
        frames, _ = synth.make_frames(a.frames, w, h, seed=7, rgba=True)
        warm = alvaar_b200.System(w, h, *K)                  # first-use costs (module load, graph capture) outside the timings
        for k in range(3):
            warm.find_camera_pose(frames[k], k * 33.333)
        warm.close()
        r = {}
        for p in range(2):
            for preset in PRESETS:
                r.setdefault(preset, []).append(one(frames, w, h, K, preset))
        res["system"][f"{w}x{h}"] = r
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
