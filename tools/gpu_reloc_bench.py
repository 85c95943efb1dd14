"""Relocalisation on the H100, one run, at 640x480, 1280x720 and 1920x1080:
* per lost frame: System.find_camera_pose on uniform-noise frames after N tracked frames of the synthetic sequence (seed 7),
  relocalisation on (max_lost_frames large enough never to reset), so that every lost frame runs the whole chain -- detector,
  ORB, grouped 2-NN against the map, match rules, P3P-RANSAC, PnP -- and fails; median wall time of the call;
* the kernels alone (CUDA events): alva_k_hamming_knn2_grouped with one query per grid cell against a map of 8 keyframes' worth
  of points (one group per cell and keyframe, 1-4 descriptors each), and alva_k_p3p_ransac (512 hypotheses) on 300
  correspondences with half of them outliers;
* per tracked frame with the mode on and off, two passes interleaved: median wall time of the status-1 frames that made no keyframe.
Records the card and its power limit in the same run.  Prints one JSON object; --out FILE also writes it there.
Usage: python tools/gpu_reloc_bench.py [--out FILE] [--frames N] [--lost N]"""
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


def tracked_run(frames, w, h, K, mode):
    s = alvaar_b200.System(w, h, *K)
    if mode:
        s.set_relocalisation(10)
    times, kf_prev = [], 0
    for k in range(len(frames)):
        t0 = time.perf_counter()
        st, _ = s.find_camera_pose(frames[k], k * 33.333)
        dt = time.perf_counter() - t0
        kf = s.info()["keyframe"]
        if st == 1 and kf == kf_prev:
            times.append(dt)
        kf_prev = kf
    s.close()
    return med(times)


def lost_run(frames, other, w, h, K):
    s = alvaar_b200.System(w, h, *K)
    s.set_relocalisation(100000)
    for k in range(len(frames)):
        s.find_camera_pose(frames[k], k * 33.333)
    info = s.info()
    times, statuses = [], []
    for j, f in enumerate(other):
        t0 = time.perf_counter()
        st, _ = s.find_camera_pose(f, (len(frames) + j) * 33.333)
        dt = time.perf_counter() - t0
        statuses.append(st)
        if st == 4:
            times.append(dt)
    s.close()
    return {"keyframes_in_map": info["keyframes"], "map_point_ids": info["map_point_ids"], "lost_frames": len(times),
            "lost_median_ms": med(times), "status_counts": {str(c): statuses.count(c) for c in sorted(set(statuses))}}


def kernel_ms(fn, reps=20):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def kernels(ctx, w, h):
    rng = np.random.default_rng(5)
    cells = ((w + 39) // 40) * ((h + 39) // 40)
    n_grp = 8 * cells
    rows = rng.integers(1, 5, n_grp)
    ds = np.concatenate([[0], np.cumsum(rows)]).astype(np.int32)
    d = rng.integers(0, 256, (int(ds[-1]), 32), dtype=np.uint8)
    q = rng.integers(0, 256, (cells, 32), dtype=np.uint8)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    qd, dsd, dd = dev(q), dev(ds), dev(d)
    out = torch.zeros((cells, 4), dtype=torch.int32, device="cuda")
    knn = kernel_ms(lambda: ctx.hamming_knn2_grouped(qd, cells, dsd, n_grp, dd, len(d), out))
    pr = synth.make_pose_problem(n=300, seed=4, w=w, h=h, outlier_frac=0.5)
    bv, X = dev(pr["bv"]), dev(pr["X"])
    T = torch.zeros(12, dtype=torch.float64, device="cuda"); o = torch.zeros(300, dtype=torch.uint8, device="cuda")
    fx = float(pr["K"][0])
    ransac = kernel_ms(lambda: ctx.p3p_ransac(1, 300, bv, X, None, T, o, None, max_iter=512, fx=fx, fy=fx))
    return {"knn2_grouped": {"queries": cells, "groups": n_grp, "rows": int(len(d)), "ms": knn},
            "p3p_ransac": {"points": 300, "hypotheses": 512, "ms": ransac}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--lost", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_reloc_bench.py needs an H100")
    res = dict(card())
    res.update(frames=a.frames, lost=a.lost, passes=2, system={})
    ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    for w, h in ((640, 480), (1280, 720), (1920, 1080)):
        K = synth.intrinsics(w, h)
        frames, _ = synth.make_frames(a.frames, w, h, seed=7, rgba=True)
        other = synth.random_rgba(w, h, a.lost, seed=3)
        other[..., 3] = 255
        warm = alvaar_b200.System(w, h, *K)
        for k in range(3):
            warm.find_camera_pose(frames[k], k * 33.333)
        warm.close()
        r = {"lost": lost_run(frames, other, w, h, K), "kernels": kernels(ctx, w, h), "tracked_median_ms": {"off": [], "on": []}}
        for p in range(2):
            for mode in ("off", "on"):
                r["tracked_median_ms"][mode].append(tracked_run(frames, w, h, K, mode == "on"))
        res["system"][f"{w}x{h}"] = r
    ctx.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
