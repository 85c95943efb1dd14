"""GPU tests (H100) of the cross-stream loop-closure detector (csrc/loopclosure.cu).  The reference has no loop closure
(SURVEY 8e: parity unpinned): what is checked is the wire format, determinism, detection of PLANTED revisits (the remote stream
shows the same scene a few frames apart) with the temporal rule, and silence on unrelated streams."""
import numpy as np
import pytest
import torch

from alvaar_b200 import synth
from alvaar_b200.loopclosure import HEADER_BYTES, MAGIC, VERSION, LoopClosure, block_bytes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W, H, NMAX, CAP = 640, 480, 1024, 1024


def features(ctx, frames_rgba):
    """ORB keypoints + descriptors of a batch of RGBA frames through the kernels of the hot path -> desc, pts, counts (device)"""
    n = len(frames_rgba)
    rgba = torch.from_numpy(np.ascontiguousarray(frames_rgba)).to(DEV)
    gray = torch.zeros((n, H, W), dtype=torch.uint8, device=DEV)
    ctx.gray(rgba, gray, W, H, n)
    kp = torch.zeros((n, CAP, 4), dtype=torch.float32, device=DEV)
    desc = torch.zeros((n, CAP, 32), dtype=torch.uint8, device=DEV)
    cnt = torch.zeros(n, dtype=torch.int32, device=DEV)
    ctx.orb_detect(gray, W, H, n, 700, 20, 2, kp, desc, cnt, CAP)      # 2 = ALVA_ORB_IC_ANGLE: steered descriptors
    torch.cuda.synchronize()
    cnt = torch.clamp(cnt, max=CAP)
    return desc, kp[:, :, :2].contiguous(), cnt


def run_steps(ctx, local, remote, kf, nsteps, world=2, **kw):
    """world ranks on one GPU: rank 0 = `local` features, ranks 1.. = `remote[r - 1]`; per step K = len(kf[s]) keyframes"""
    K4 = synth.intrinsics(W, H)
    K = len(kf[0])
    dets = [LoopClosure(ctx, NMAX, K, world, r, K4, **kw) for r in range(world)]
    bb = block_bytes(NMAX)
    events, scores, sends = [], [], []
    for s in range(nsteps):
        idx = torch.tensor(kf[s], dtype=torch.int32, device=DEV)
        gathered = torch.zeros(world * K * bb, dtype=torch.uint8, device=DEV)
        for r in range(world):
            d, p, c = local if r == 0 else remote[r - 1]
            send = gathered[r * K * bb:(r + 1) * K * bb]
            dets[r].pack(d, p, c, idx, send)
        dets[0].detect(gathered)
        events += dets[0].poll(wait=True)
        scores.append(dets[0].last_scores())
        sends.append(gathered.cpu().numpy())
    for d in dets:
        d.close()
    return events, scores, sends


def test_wire_format_and_planted_revisit(gpu_ctx):
    frames, _ = synth.make_frames(14, W, H, seed=7, rgba=True)
    other, _ = synth.make_frames(14, W, H, seed=23, rgba=True, texture_seed=777)
    a = features(gpu_ctx, frames[:12])                # local stream: frames 0..11
    b = features(gpu_ctx, frames[2:14])               # remote stream 1: the same scene two frames later (the planted revisit)
    c = features(gpu_ctx, other[:12])                 # remote stream 2: an unrelated scene
    kf = [[0, 1, 2], [3, 4, 5], [6, 7, 8]]
    ev, sc, sends = run_steps(gpu_ctx, a, [b, c], kf, 3, world=3)
    # wire format of rank 0's first block
    bb = block_bytes(NMAX)
    blk = sends[0][:bb]
    hdr = blk[:HEADER_BYTES].view(np.int32)
    n0 = int(a[2][0].item())
    assert hdr[0] == MAGIC and hdr[1] == VERSION and hdr[2] == 0 and hdr[3] == 0 and hdr[4] == n0 and hdr[5] == NMAX
    K4 = synth.intrinsics(W, H)
    assert np.allclose(blk[:HEADER_BYTES].view(np.float32)[6:10], np.asarray(K4, np.float32))
    px = blk[HEADER_BYTES:HEADER_BYTES + 8 * NMAX].view(np.float32).reshape(NMAX, 2)
    assert (px[:n0] == a[1][0, :n0].cpu().numpy()).all() and (px[n0:] == 0).all()
    dsc = blk[HEADER_BYTES + 8 * NMAX:].reshape(NMAX, 32)
    assert (dsc[:n0] == a[0][0, :n0].cpu().numpy()).all()
    hdr2 = sends[1][bb:bb + HEADER_BYTES].view(np.int32)
    assert hdr2[3] == 4                                # keyframe sequence numbers run on across steps (step 1, event 1)
    # the revisit is found against stream 1 and only there; the temporal rule holds the report back until 3 events in a row passed
    assert len(ev) >= 1 and all(e["remote_rank"] == 1 for e in ev)
    assert ev[0]["local_kf"] == 2 and ev[0]["consecutive"] == 3 and ev[0]["n_inliers"] >= 20
    for s in sc:
        assert (s[:, 1, 0] >= 30).all() and s[-1, 1, 1] == 1 and (s[:-1, 1, 1] == 2).all()   # stream 1: many putative matches (verdict 2); RANSAC runs on the step's newest keyframe and succeeds (1)
        assert (4 * s[:, 2, 0] < s[:, 1, 0]).all() and (s[:, 2, 1] == 0).all()   # stream 2: a few chance matches (~6 % of the keypoints), no geometry
        assert (s[:, 0, :3] == 0).all()                                  # a stream is not matched against itself (field 3: the block's keyframe number)
    R = ev[0]["Rt"][:, :3]
    assert np.abs(R @ R.T - np.eye(3)).max() < 1e-9 and np.abs(R - np.eye(3)).max() < 0.05    # two frames apart: nearly the same view


def test_detection_is_deterministic_and_interrupted_runs_do_not_report(gpu_ctx):
    frames, _ = synth.make_frames(12, W, H, seed=7, rgba=True)
    other, _ = synth.make_frames(12, W, H, seed=31, rgba=True, texture_seed=778)
    a = features(gpu_ctx, frames[:10])
    b = features(gpu_ctx, frames[1:11])
    kf = [[0, 1, 2], [3, 4, 5]]
    e1, s1, g1 = run_steps(gpu_ctx, a, [b], kf, 2)
    e2, s2, g2 = run_steps(gpu_ctx, a, [b], kf, 2)
    assert len(e1) == len(e2) >= 1 and all(np.array_equal(x, y) for x, y in zip(s1, s2)) and all(np.array_equal(x, y) for x, y in zip(g1, g2))
    for x, y in zip(e1, e2):
        assert {k: v for k, v in x.items() if k != "Rt"} == {k: v for k, v in y.items() if k != "Rt"} and np.array_equal(x["Rt"], y["Rt"])
    # a remote stream whose every second keyframe is unrelated never gets 3 passes in a row
    mix_d, mix_p, mix_c = [t.clone() for t in b]
    od, op, oc = features(gpu_ctx, other[:10])
    for f in (1, 3, 5):
        mix_d[f], mix_p[f], mix_c[f] = od[f], op[f], oc[f]
    e3, s3, _ = run_steps(gpu_ctx, a, [(mix_d, mix_p, mix_c)], kf, 2)
    assert e3 == []
    assert s3[0][0, 1, 0] >= 30 and s3[0][1, 1, 0] < s3[0][0, 1, 0] / 4 and s3[0][2, 1, 1] == 1   # the streak is broken by match counts, not by the geometry
