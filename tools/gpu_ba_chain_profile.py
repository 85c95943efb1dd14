"""Where the local-BA chain of the headline step (bench.py, config c2) spends its time, in one process on the bench shapes
(13 problems of 20 KF x 3000 landmarks x 12 000 observations, LM <= 5 iterations):

  step split      ms per pipeline step (CUDA events, 20 steps after 3 warm-ups) with BA overlapped, with BA serial after the
                  frame stages, and without BA (kf_interval 0): if the no-BA step is close to the full one, BA does not bound it
  chain           one standalone 13-problem alva_k_ba_solve, CUDA events (as tools/gpu_ba_bench.py)
  kernels         the same solve under torch.profiler (CUDA activities), in a pass of its own: each ba_* kernel's total time
                  and call count per solve, and its duration per launch in launch order (us_per_launch)
  dense_schur     chain and kernels again with alva_set_option("ba_dense_schur", 1): the Schur term as an FP64 tensor-core SYRK
  card            name and power limit, read in the same run

    python tools/gpu_ba_chain_profile.py --out profiles/ba_chain_h100.json
"""
import argparse, json, os, re, subprocess, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alvaar_b200
from alvaar_b200 import synth
from alvaar_b200.pipeline import Pipeline

W, H, B = 1280, 720, 64                       # bench.py c2
MAP_SIZE, KF_INTERVAL, FAST_THR, NFEAT = 10000, 5, 20, 1000
BA_NKF, BA_NLM, BA_OBS_PER_LM, BA_ITERS = 20, 3000, 4, 5
NPROB = 13                                    # keyframes per 64-frame step at kf_interval 5


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["sm_max_clock"] = [s.strip() for s in q.split(",")[:2]]
    except Exception as e:   # nvidia-smi missing: say so rather than guess
        out["power_limit"] = f"not read ({type(e).__name__})"
    return out


def step_ms(ctx, stream, d_in, mapd, ba, kf_interval, overlap, warmup=3, steps=20):
    ctx.L.alva_set_option(b"pipeline_graphs", 1)
    ctx.L.alva_set_option(b"pipeline_ba_overlap", overlap)
    pipe = Pipeline(ctx, W, H, B, fast_thr=FAST_THR, nfeatures=NFEAT, orb_flags=alvaar_b200.ORB_IC_ANGLE | alvaar_b200.ORB_HARRIS,
                    map_size=MAP_SIZE, kf_interval=kf_interval, ba_nkf=BA_NKF, ba_nlm=BA_NLM, ba_nobs=len(ba["obs_kf"]),
                    ba_max_iter=BA_ITERS, ba_huber=ba["huber"], derivatives=True)
    pipe.set_map(mapd[:MAP_SIZE])
    for s in range(pipe.nprob):
        pipe.set_ba(s, ba)
    with torch.cuda.stream(stream):
        for _ in range(warmup):
            pipe.step_dev(d_in)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            pipe.step_dev(d_in)
        e1.record(stream)
        torch.cuda.synchronize()
    pipe.close()
    ctx.L.alva_set_option(b"pipeline_ba_overlap", 1)
    return e0.elapsed_time(e1) / steps


def kernel_name(key):
    # "void (anonymous namespace)::ba_linearize_kernel<true>(...)" -> "ba_linearize_kernel<true>"
    m = re.search(r"(ba_\w+(?:<[^>]*>)?)\s*\(", key)
    return m.group(1) if m else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="", help="write the JSON result here (else stdout only)")
    ap.add_argument("--reps", type=int, default=20, help="timed standalone solves")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"card": card(), "shapes": f"{NPROB} problems x {BA_NKF} KF x {BA_NLM} landmarks x {BA_NLM * BA_OBS_PER_LM} obs, "
                                     f"max_iter {BA_ITERS}"}

    # ---- step split
    stream = torch.cuda.Stream()
    ctx = alvaar_b200.Context(0, stream.cuda_stream)
    frames, _ = synth.make_frames(B, W, H, seed=99, texture_seed=1234)
    _, mapd = synth.make_descriptors(8, MAP_SIZE, seed=7)
    ba = synth.make_ba_problem(BA_NKF, BA_NLM, BA_OBS_PER_LM, seed=42)
    d_in = torch.from_numpy(frames).cuda()
    full = step_ms(ctx, stream, d_in, mapd, ba, KF_INTERVAL, 1)
    serial = step_ms(ctx, stream, d_in, mapd, ba, KF_INTERVAL, 0)
    nob = step_ms(ctx, stream, d_in, mapd, ba, 0, 1)
    res["step_ms"] = {"ba_overlapped": full, "ba_serial": serial, "no_ba": nob, "no_ba_over_full": nob / full,
                      "note": "CUDA events over 20 steps after 3 warm-ups, CUDA graphs on"}
    ctx.close()

    # ---- standalone chain, CUDA events (inputs reset on the device before each solve, outside the timed window)
    ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    ctx.L.alva_set_option(b"pipeline_graphs", 0)
    st = lambda k: torch.from_numpy(np.stack([ba[k]] * NPROB)).cuda()  # noqa: E731
    calib, poses0, const, invd0 = st("calib"), st("poses"), st("pose_const"), st("invd")
    akf, auv, okf, olm, ouv = st("anch_kf"), st("anch_uv"), st("obs_kf"), st("obs_lm"), st("obs_uv")
    summ = torch.zeros((NPROB, 8), dtype=torch.float64, device="cuda")
    nobs = len(ba["obs_kf"])

    def solve():
        poses, invd = poses0.clone(), invd0.clone()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ctx.ba_solve(NPROB, BA_NKF, BA_NLM, nobs, calib, poses, const, invd, akf, auv, okf, olm, ouv, ba["huber"], BA_ITERS, summ)
        e1.record()
        return e0, e1

    def timed(dense):
        ctx.L.alva_set_option(b"ba_dense_schur", dense)
        for _ in range(3):
            solve()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            l0 = ctx.launches
            e0, e1 = solve()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
            launches = ctx.launches - l0
        s = summ.cpu().numpy()[0]
        out = {"median": float(np.median(ts)), "min": float(np.min(ts)), "max": float(np.max(ts)), "reps": args.reps,
               "launches_per_solve_incl_summary": int(launches),
               "summary_problem0": {"initial_cost": float(s[0]), "final_cost": float(s[1]), "n_success": int(s[2]),
                                    "n_iter": int(s[3]), "term": int(s[4])}}
        ctx.L.alva_set_option(b"ba_dense_schur", 0)
        return out

    # ---- per-kernel times, torch.profiler in a pass of its own: totals per solve, and every launch in launch order (a launch
    # whose problems are all finished returns at once, so the active ones stand apart)
    nprof = 10

    def profiled(dense):
        from torch.profiler import profile, ProfilerActivity
        from torch.autograd import DeviceType
        ctx.L.alva_set_option(b"ba_dense_schur", dense)
        for _ in range(3):
            solve()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(nprof):
                solve()
            torch.cuda.synchronize()
        ctx.L.alva_set_option(b"ba_dense_schur", 0)
        evs = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and kernel_name(e.name)),
                     key=lambda e: e.time_range.start)
        solves = []   # per solve: kernel -> [us of launch 1, 2, ...]
        for e in evs:
            name = kernel_name(e.name)
            if name == "ba_setup_kernel":
                solves.append({})
            if solves:
                solves[-1].setdefault(name, []).append(e.time_range.elapsed_us())
        assert len(solves) == nprof, len(solves)
        kern, launch = {}, {}
        for name in solves[0]:
            per = np.array([sv[name] for sv in solves], dtype=np.float64)   # [solve][launch]
            kern[name] = {"us_per_solve": float(per.sum(1).mean()), "calls_per_solve": per.shape[1],
                          "us_per_call": float(per.mean())}
            launch[name] = [round(float(v), 2) for v in per.mean(0)]
        kern = dict(sorted(kern.items(), key=lambda kv: -kv[1]["us_per_solve"]))
        return {"kernels": kern, "kernels_total_us_per_solve": sum(k["us_per_solve"] for k in kern.values()),
                "us_per_launch": {k: launch[k] for k in kern},
                "kernels_note": f"torch.profiler, CUDA activities, {nprof} solves after the timed pass; times are kernel durations, "
                                "us_per_launch in launch order, averaged over the solves"}

    res["chain_ms"] = timed(0)
    res.update(profiled(0))
    # the same with the Schur term as an FP64 tensor-core SYRK (alva_set_option("ba_dense_schur", 1))
    res["dense_schur"] = {"chain_ms": timed(1), **profiled(1)}
    ctx.close()

    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
