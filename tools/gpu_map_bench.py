"""The map blob on the H100, one run, at 640x480, 1280x720 and 1920x1080.  Session A tracks N frames of the synthetic sequence
(seed 7) with relocalisation on; then:
* blob size, and the median wall time of System.save_map (bytes returned to Python) over 20 calls;
* the median wall time of System.load_map into a fresh, configured System over 20 handles;
* from the load to the first status 1 in a new session: `lost` frames of another scene (texture seed 4321; each runs the whole
  device relocalisation chain and fails), then frame 20 of A's sequence (a revisited view).  The first lost frame after the
  load is reported apart (its table upload and first-use allocations), then the median of the others, and the relocalised
  frame.  Uniform noise is not used as the lost frames: it drives their adaptive detector quality so high that the revisited
  view then finds too few corners.
Records the card and its power limit in the same run.  Prints one JSON object; --out FILE also writes it there.
Usage: python tools/gpu_map_bench.py [--out FILE] [--frames N] [--lost N]"""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


med = lambda v: float(np.median(v)) * 1e3 if len(v) else None  # noqa: E731


def new_system(w, h, K):
    s = alvaar_b200.System(w, h, *K)
    s.set_relocalisation(100000)
    return s


def one_resolution(w, h, n_frames, n_lost):
    K = synth.intrinsics(w, h)
    frames, _ = synth.make_frames(n_frames, w, h, seed=7, rgba=True)
    other, _ = synth.make_frames(n_lost, w, h, seed=33, rgba=True, texture_seed=4321)
    a = new_system(w, h, K)
    for k in range(n_frames):
        a.find_camera_pose(frames[k], k * 33.333)
    info = a.info()
    a.save_map()
    t_save = []
    for _ in range(20):
        t0 = time.perf_counter()
        blob = a.save_map()
        t_save.append(time.perf_counter() - t0)
    a.close()
    t_load = []
    for _ in range(20):
        b = new_system(w, h, K)
        t0 = time.perf_counter()
        b.load_map(blob)
        t_load.append(time.perf_counter() - t0)
        b.close()
    b = new_system(w, h, K)
    b.load_map(blob)
    seq = list(other) + [frames[20]]
    times, sts = [], []
    for j, f in enumerate(seq):
        t0 = time.perf_counter()
        st, _ = b.find_camera_pose(np.ascontiguousarray(f), j * 33.333)
        times.append(time.perf_counter() - t0)
        sts.append(st)
    b.close()
    lost = [t for t, s in zip(times, sts) if s == 4]
    first_ok = sts.index(1) if 1 in sts else None
    return {"keyframes": info["keyframes"], "map_point_ids": info["map_point_ids"], "blob_bytes": len(blob),
            "save_median_ms": med(t_save), "load_median_ms": med(t_load),
            "first_lost_frame_ms": lost[0] * 1e3 if lost else None, "lost_median_ms": med(lost[1:]), "lost_frames": len(lost),
            "relocalised_frame_ms": times[first_ok] * 1e3 if first_ok is not None else None,
            "load_to_first_status1_ms": sum(times[:first_ok + 1]) * 1e3 if first_ok is not None else None,
            "statuses": sts}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--lost", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_map_bench.py needs an H100")
    res = dict(card())
    res.update(frames=a.frames, lost=a.lost, system={})
    for w, h in ((640, 480), (1280, 720), (1920, 1080)):
        K = synth.intrinsics(w, h)
        warm = alvaar_b200.System(w, h, *K)
        f, _ = synth.make_frames(3, w, h, seed=7, rgba=True)
        for k in range(3):
            warm.find_camera_pose(f[k], k * 33.333)
        warm.close()
        res["system"][f"{w}x{h}"] = one_resolution(w, h, a.frames, a.lost)
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
