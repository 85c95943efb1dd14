"""The localisation-only mode on the H100, one run, at 640x480, 1280x720 and 1920x1080.  Session A maps N frames of the synthetic
sequence (seed 99) with relocalisation on; its blob is loaded into a new System that is frozen (set_localisation_only) and
replays the same N frames.  Reported per resolution:
* per-frame wall time (median, p99, max) of the mapping session's tracked frames and of the frozen session's tracked frames,
  after the first 20 frames of each (initialisation and the relocalisation after the load are excluded);
* the share of the frozen session's tracked frames on which re-acquisition ran, and the points it returned;
* the kernel time of alva_k_match_frame_to_map by CUDA events (median over 200 calls, 20 warm-up calls) on a random problem the
  size of that session's map table and twice its grid's cell count of queries, and at 1920x1080 also on 100 000 points x 8 192
  queries.
Records the card and its power limit in the same run.  Prints one JSON object; --out FILE also writes it there.
Usage: python tools/gpu_localisation_bench.py [--out FILE] [--frames N]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import alvaar_b200  # noqa: E402
import localisation_util as LU  # noqa: E402
import map_util as M  # noqa: E402
from alvaar_b200 import synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def stats(v):
    v = np.asarray(v) * 1e3
    return {"median_ms": float(np.median(v)), "p99_ms": float(np.percentile(v, 99)), "max_ms": float(v.max()), "frames": int(len(v))} if len(v) else None


def kernel_ms(w, h, cell, n_mp, nq, max_rows=6, seed=1):
    p = LU.random_problem(np.random.default_rng(seed), w=w, h=h, cell=cell, n_mp=n_mp, nq=nq, max_rows=max_rows)
    want = LU.run_oracle(LU.oracle_lib(), p)
    ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()  # noqa: E731
    args = dict(Twc=d(p.Twc, np.float64), wpt=d(p.wpt, np.float64), desc_start=d(p.desc_start, np.int32), desc=d(p.desc, np.uint8),
                q_px=d(p.q_px, np.float32), q_desc=d(p.q_desc, np.uint8), q_kept=d(p.q_kept, np.uint8), skip=d(p.skip, np.uint8))
    row = torch.zeros(nq, dtype=torch.int32, device="cuda"); dist = torch.zeros_like(row)
    call = lambda: ctx.match_frame_to_map(w, h, cell, p.K, q_row=row, q_dist=dist, radius=p.radius, **args)  # noqa: E731
    for _ in range(20):
        call()
    torch.cuda.synchronize()
    assert (row.cpu().numpy() == want[0]).all() and (dist.cpu().numpy() == want[1]).all()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(200)]
    for a, b in ev:
        a.record(); call(); b.record()
    torch.cuda.synchronize()
    ctx.close()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def one_resolution(w, h, n):
    K = synth.intrinsics(w, h)
    frames, _ = synth.make_frames(n, w, h, seed=99, rgba=True)
    a = alvaar_b200.System(w, h, *K)
    a.set_relocalisation(10)
    t_map, st_map = [], []
    for k in range(n):
        f = np.ascontiguousarray(frames[k])
        t0 = time.perf_counter()
        st, _ = a.find_camera_pose(f, k * 33.333)
        t_map.append(time.perf_counter() - t0)
        st_map.append(st)
    info, blob = a.info(), a.save_map()
    a.close()
    b = alvaar_b200.System(w, h, *K)
    b.set_relocalisation(10)
    b.load_map(blob)
    b.set_localisation_only(True)
    t_loc, st_loc, ran = [], [], []
    for k in range(n):
        f = np.ascontiguousarray(frames[k])
        r0 = b.localisation_stats()["runs"]
        t0 = time.perf_counter()
        st, _ = b.find_camera_pose(f, k * 33.333)
        t_loc.append(time.perf_counter() - t0)
        st_loc.append(st)
        ran.append(b.localisation_stats()["runs"] > r0)
    ls = b.localisation_stats()
    b.close()
    _, sec = M.sections(blob)
    tracked = [k for k in range(20, n) if st_loc[k] == 1]
    cell = 40
    max_kps = -(-w // cell) * -(-h // cell)
    return {"keyframes": info["keyframes"], "map_point_ids": info["map_point_ids"], "blob_map_points": sec["nmp"],
            "mapping_tracked": stats([t_map[k] for k in range(20, n) if st_map[k] == 1]),
            "frozen_tracked": stats([t_loc[k] for k in tracked]),
            "frozen_reacquiring": stats([t_loc[k] for k in tracked if ran[k]]),
            "frozen_not_reacquiring": stats([t_loc[k] for k in tracked if not ran[k]]),
            "reacquire_share": float(np.mean([ran[k] for k in tracked])) if tracked else None,
            "reacquire_runs": ls["runs"], "reacquired_points": ls["points"],
            "frozen_statuses": {str(s): st_loc.count(s) for s in sorted(set(st_loc))},
            "kernel_ms_at_map_size": kernel_ms(w, h, cell, max(sec["nmp"], 1), 2 * max_kps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--frames", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_localisation_bench.py needs an H100")
    res = dict(card())
    res.update(frames=a.frames, system={})
    for w, h in ((640, 480), (1280, 720), (1920, 1080)):
        K = synth.intrinsics(w, h)
        warm = alvaar_b200.System(w, h, *K)
        f, _ = synth.make_frames(3, w, h, seed=99, rgba=True)
        for k in range(3):
            warm.find_camera_pose(f[k], k * 33.333)
        warm.close()
        res["system"][f"{w}x{h}"] = one_resolution(w, h, a.frames)
    res["kernel_ms_100k_points_8192_queries_1920x1080"] = kernel_ms(1920, 1080, 40, 100000, 8192, max_rows=12)
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
