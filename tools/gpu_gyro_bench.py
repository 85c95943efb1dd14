"""Gyro-aided tracking on the H100, one run, at 640x480, 1280x720 and 1920x1080.  The pan sequence of tests/gyro_util.py (90
frames at 30 Hz, 200 Hz gyro samples) at a 90 deg/s peak -- slow enough that the camera-only tracker follows it too, so both
modes time the same tracked frames -- runs four times per resolution, interleaved: gyro off, on, off, on.  Reported per
resolution and pass: per-frame wall time of alva_system_find_camera_pose_gyro (median, p99) over the frames tracked with status 1
after frame 20, and the statuses; per mode the spread between its two passes.  Then the kernel time of alva_k_rotate_priors by
CUDA events (median over 200 launches after 20 warm-up launches) at n = the grid's cell count and twice it, per lens.
Records the card and its power limit in the same run.  Prints one JSON object; --out FILE also writes it there.
Usage: python tools/gpu_gyro_bench.py [--out FILE]"""
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
import gyro_util as G  # noqa: E402
from alvaar_b200 import synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def stats(v):
    v = np.asarray(v) * 1e3
    return {"median_ms": float(np.median(v)), "p99_ms": float(np.percentile(v, 99)), "frames": int(len(v))} if len(v) else None


def one_pass(w, h, seq, gyro):
    frames, times, smp, _ = seq
    s = alvaar_b200.System(w, h, *synth.intrinsics(w, h))
    s.set_relocalisation(30)
    if gyro:
        s.set_gyro(True, G.R_CI, G.BIAS)
    t, st = [], []
    for k in range(len(frames)):
        f = np.ascontiguousarray(frames[k])
        t0 = time.perf_counter()
        a, _ = s.find_camera_pose_gyro(f, times[k], smp[k])
        t.append(time.perf_counter() - t0)
        st.append(a)
    gs = s.gyro_stats()[0]
    s.close()
    return t, st, gs


def kernel_ms(w, h, n, lens):
    code, D = {"pinhole": (0, None), "radtan": (1, (-0.12, 0.03, 0.001, -0.0005)), "fisheye": (2, G.FISHEYE)}[lens]
    K = synth.intrinsics(w, h)
    rng = np.random.default_rng(n)
    u, v = rng.uniform(0, w, n), rng.uniform(0, h, n)
    bv = np.stack([(u - K[2]) / K[0], (v - K[3]) / K[1], np.ones(n)], 1)
    bv /= np.linalg.norm(bv, axis=1, keepdims=True)
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()  # noqa: E731
    bvd, fl = d(bv, np.float64), d(np.ones(n), np.uint8)
    pr, rot = d(np.stack([u, v], 1), np.float32), torch.zeros(n, dtype=torch.uint8, device="cuda")
    R = G._ry(np.radians(4.0)) @ G._rx(np.radians(2.0))
    ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    call = lambda: ctx.rotate_priors(bvd, fl, n, w, h, K, D, code, R.reshape(9), pr, rot)  # noqa: E731
    for _ in range(20):
        call()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(200)]
    for a, b in ev:
        a.record(); call(); b.record()
    torch.cuda.synchronize()
    ctx.close()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_gyro_bench.py needs an H100")
    res = dict(card())
    res.update(sequence="tests/gyro_util.py pan_sequence(90, peak_dps=90), 200 Hz samples", system={}, kernel_ms={})
    for w, h in ((640, 480), (1280, 720), (1920, 1080)):
        seq = G.pan_sequence(90, peak_dps=90.0, w=w, h=h)
        one_pass(w, h, (seq[0][:3], seq[1][:3], seq[2][:3], None), True)   # warm-up: module loads, first launches
        r = {}
        for i, gyro in enumerate((False, True, False, True)):
            t, st, gs = one_pass(w, h, seq, gyro)
            tracked = [t[k] for k in range(20, len(t)) if st[k] == 1]
            r[f"pass{i // 2 + 1}_{'on' if gyro else 'off'}"] = {"tracked": stats(tracked), "statuses": "".join(map(str, st)),
                                                               **({"gyro_stats": gs} if gyro else {})}
        for m in ("off", "on"):
            a1, a2 = r[f"pass1_{m}"]["tracked"], r[f"pass2_{m}"]["tracked"]
            r[f"spread_{m}_median_ms"] = abs(a1["median_ms"] - a2["median_ms"])
        on = np.mean([r[f"pass{p}_on"]["tracked"]["median_ms"] for p in (1, 2)])
        off = np.mean([r[f"pass{p}_off"]["tracked"]["median_ms"] for p in (1, 2)])
        r["on_minus_off_median_ms"] = float(on - off)
        res["system"][f"{w}x{h}"] = r
        cells = -(-w // 40) * -(-h // 40)
        for lens in ("pinhole", "radtan", "fisheye"):
            for n in (cells, 2 * cells):
                res["kernel_ms"][f"{w}x{h}_{lens}_n{n}"] = kernel_ms(w, h, n, lens)
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
