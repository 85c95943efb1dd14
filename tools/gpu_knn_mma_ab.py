"""The tensor-core Hamming 2-NN on the bench's problem (64 frames x 1536 query slots, 1 000 live, 10 000 map descriptors):
the whole `alva_k_hamming_knn2_batch` call per operand layout (`knn_mma_mode`) and operand kind (`knn_mma_kind`), with
CUDA events (median of 20 calls after 3 warm-up calls, every configuration in one process), each launch's time
(`torch.profiler`, a separate pass), and the card, its power limit and its highest SM clock, read in the same run.  Every
configuration's output is compared with the first one's.

    python tools/gpu_knn_mma_ab.py --out profiles/knn_h100.json"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import alvaar_b200

ap = argparse.ArgumentParser()
ap.add_argument("--out", default="")
ap.add_argument("--calls", type=int, default=20)
args = ap.parse_args()

dev = "cuda:0"
ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
L = ctx.L


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


rng = np.random.default_rng(5)
nb, qcap, live, nt = 64, 1536, 1000, 10000
q = rng.integers(0, 256, (nb * qcap, 32), dtype=np.uint8)
t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
q[::3] = t[rng.integers(0, nt, len(q[::3]))] ^ (rng.random((len(q[::3]), 32)) < 0.05).astype(np.uint8)
dq, dt = torch.from_numpy(q).to(dev), torch.from_numpy(t).to(dev)
counts = torch.full((nb,), live, dtype=torch.int32, device=dev)
out = torch.zeros((nb * qcap, 4), dtype=torch.int32, device=dev)
macs = nb * live * nt * 256


def call():
    ctx.hamming_knn2_batch(dq, counts, nb, qcap, dt, nt, out)


def time_calls(n):
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1000.0)
    return statistics.median(ts), min(ts)


def per_launch(n=10):
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            call()
        torch.cuda.synchronize()
    res = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us > 0 and "knn2" in e.key:
            m = re.search(r"knn2_\w+(<\d>)?", e.key)
            name = m.group(0) if m else e.key
            res[name] = {"us_per_call": round(us / n, 1), "launches_per_call": e.count // n}
    return res


# kind 2 (1-bit operands) has one layout: knn_mma_mode does not apply to it
configs = [dict(knn_mma_mode=mode, knn_mma_kind=kind) for mode in (0, 1) for kind in (0, 1)] + [dict(knn_mma_mode=0, knn_mma_kind=2)]
result = {"card": card(), "problem": f"{nb} x {qcap} slots, {live} live, {nt} map rows", "macs": macs,
          "int8_tensor_floor_us_at_1979_tops": round(2 * macs / 1979e12 * 1e6, 1), "configs": [], "per_launch": []}
print(result["card"], flush=True)
assert L.alva_set_option(b"knn_mma", 2) == 0
ref = None
for cfg in configs:
    for k, v in cfg.items():
        assert L.alva_set_option(k.encode(), v) == 0
    med, best = time_calls(args.calls)
    got = out.cpu().numpy()
    if ref is None:
        ref = got
    row = dict(cfg, median_us=round(med, 1), min_us=round(best, 1), tops=round(2 * macs / (med * 1e-6) / 1e12),
               same_output=bool(np.array_equal(got, ref)))
    print(row, flush=True)
    result["configs"].append(row)
for mode, kind in ((0, 0), (1, 0), (0, 2)):
    assert L.alva_set_option(b"knn_mma_mode", mode) == 0
    assert L.alva_set_option(b"knn_mma_kind", kind) == 0
    result["per_launch"].append({"knn_mma_mode": mode, "knn_mma_kind": kind, "kernels": per_launch()})
    print(result["per_launch"][-1], flush=True)
for k, v in (("knn_mma", 1), ("knn_mma_mode", 0), ("knn_mma_kind", 2)):
    L.alva_set_option(k.encode(), v)
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
ok = all(r["same_output"] for r in result["configs"])
print("RESULT", "PASS" if ok else "FAIL")
sys.exit(0 if ok else 1)
