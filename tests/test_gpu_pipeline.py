"""GPU parity test (H100): the whole per-frame hot path as one object (alva_pipeline_*) against the stage-by-stage
oracle: gray -> pyramid -> FAST -> retainBest -> ORB (IC angle) -> Hamming 2-NN -> local BA."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import P
from alvaar_b200 import synth, unpack_keys, ORB_IC_ANGLE
from alvaar_b200.pipeline import Pipeline

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("w,h,batch,nfeat", [(640, 480, 3, 300), (1280, 720, 2, 1000), (1920, 1080, 2, 2000)])   # C2 and C3 of BASELINE.json
def test_pipeline_vs_oracle(gpu_ctx, oracle, w, h, batch, nfeat):
    frames, _ = synth.make_frames(batch, w, h, seed=5)
    q, mapd = synth.make_descriptors(8, 2000, seed=3)
    ba = synth.make_ba_problem(8, 300, 3, seed=7)
    pipe = Pipeline(gpu_ctx, w, h, batch, fast_thr=20, nfeatures=nfeat, orb_flags=ORB_IC_ANGLE, map_size=2000, kf_interval=2,
                    ba_nkf=8, ba_nlm=300, ba_nobs=len(ba["obs_kf"]), ba_max_iter=5, ba_huber=ba["huber"], derivatives=True)
    pipe.set_map(mapd)
    for s in range(pipe.nprob):
        pipe.set_ba(s, ba)
    host_in = torch.from_numpy(frames).pin_memory()
    nfeat_h = torch.zeros(batch, dtype=torch.int32).pin_memory()
    match_h = torch.zeros((batch, pipe.fcap, 4), dtype=torch.int32).pin_memory()
    poses_h = torch.zeros((pipe.nprob, 8, 7), dtype=torch.float64).pin_memory()
    summ_h = torch.zeros((pipe.nprob, 8), dtype=torch.float64).pin_memory()
    pipe.step_host(host_in, nfeat_h, match_h, poses_h, summ_h)
    # and the device-resident entry point gives the same answer
    pipe.step_dev(host_in.to(DEV))
    torch.cuda.synchronize()
    fcap = pipe.fcap
    sel = pipe.buffer("sel", (batch, fcap), torch.int32).cpu().numpy().view(np.uint32)
    selc = pipe.buffer("selcounts", (batch,), torch.int32).cpu().numpy()
    desc = pipe.buffer("desc", (batch, fcap, 32), torch.uint8).cpu().numpy()
    kept = pipe.buffer("kept", (batch, fcap), torch.uint8).cpu().numpy()
    matches = pipe.buffer("matches", (batch, fcap, 4), torch.int32).cpu().numpy()
    assert (selc == nfeat_h.numpy()).all() and (matches == match_h.numpy()).all()
    sizes = [(w, h)]
    for _ in range(3):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    lv = [pipe.buffer(f"l{k}", (batch, sizes[k][1], sizes[k][0]), torch.uint8).cpu().numpy() for k in range(4)]
    dv = [pipe.buffer(f"d{k}", (batch, sizes[k][1], sizes[k][0], 2), torch.int16).cpu().numpy() for k in range(4)]
    for f in range(batch):
        gray = np.empty((h, w), np.uint8)
        oracle.orc_gray(P(frames[f]), w, h, P(gray))
        assert (lv[0][f] == gray).all()
        cur = gray
        for k in (1, 2, 3):
            nxt = np.empty((sizes[k][1], sizes[k][0]), np.uint8)
            oracle.orc_pyrdown(P(cur), cur.shape[1], cur.shape[0], P(nxt))
            assert (lv[k][f] == nxt).all()
            cur = nxt
        for k in range(4):   # derivative pyramid (buildOpticalFlowPyramid withDerivatives)
            want = np.zeros((sizes[k][1], sizes[k][0], 2), np.int16)
            oracle.orc_scharr(P(np.ascontiguousarray(lv[k][f])), sizes[k][0], sizes[k][1], P(want))
            assert (dv[k][f] == want).all()
        xs = np.zeros((w * h // 4, 3), np.int32)
        n = oracle.orc_fast9(P(gray), w, h, 20, 1, P(xs), len(xs))
        k = xs[:n]
        k = np.ascontiguousarray(k[(k[:, 0] >= 31) & (k[:, 0] < w - 31) & (k[:, 1] >= 31) & (k[:, 1] < h - 31)])
        thr = oracle.orc_retain_best_threshold(P(k), len(k), nfeat)
        want = k[k[:, 2] >= thr]
        c = int(selc[f])
        assert c == len(want) and nfeat <= c <= fcap
        assert (unpack_keys(sel[f, :c]) == want).all()
        pts = np.ascontiguousarray(want[:, :2].astype(np.float32))
        ang = np.zeros(c, np.float32)
        oracle.orc_ic_angles(P(gray), w, h, P(pts), c, P(ang))
        blur = np.empty_like(gray)
        oracle.orc_orb_blur(P(gray), w, h, 0, P(blur))
        wd, wk = np.zeros((c, 32), np.uint8), np.zeros(c, np.uint8)
        oracle.orc_orb_describe(P(blur), w, h, P(pts), P(ang), c, P(wd), P(wk))
        assert wk.all() and (kept[f, :c] == 1).all() and (kept[f, c:] == 0).all()
        assert (desc[f, :c] == wd).all()
        wm = np.zeros((c, 4), np.int32)
        oracle.orc_knn2(P(wd), c, P(mapd), len(mapd), P(wm))
        assert (matches[f, :c] == wm).all() and (matches[f, c:] == -1).all()
    wp, wdpt = ba["poses"].copy(), ba["invd"].copy()
    ws = np.zeros(8)
    oracle.orc_ba_solve(P(ba["calib"]), P(wp), P(ba["pose_const"]), 8, P(wdpt), P(ba["anch_kf"]), P(ba["anch_uv"]), 300,
                        P(ba["obs_kf"]), P(ba["obs_lm"]), P(ba["obs_uv"]), len(ba["obs_kf"]), C.c_double(ba["huber"]), 5, P(ws),
                        None)
    for s in range(pipe.nprob):
        assert np.allclose(poses_h[s].numpy(), wp, rtol=1e-4, atol=1e-9)
        assert (summ_h[s].numpy()[2:5] == ws[2:5]).all()
    pipe.close()


@pytest.mark.parametrize("w,h,batch,nfeat", [(640, 480, 3, 300), (1280, 720, 2, 1000), (1920, 1080, 2, 2000)])
def test_pipeline_detect_and_compute_mode(gpu_ctx, oracle, w, h, batch, nfeat):
    """orb_flags = IC_ANGLE | HARRIS: the pipeline's feature set per frame is exactly ORB::detectAndCompute(nfeat, 1 level)'s
    (oracle composition pinned bit-for-bit to the reference in tests/test_oracle.py), and the matches follow from it."""
    from alvaar_b200 import ORB_HARRIS
    frames, _ = synth.make_frames(batch, w, h, seed=8)
    _, mapd = synth.make_descriptors(8, 1500, seed=4)
    pipe = Pipeline(gpu_ctx, w, h, batch, fast_thr=20, nfeatures=nfeat, orb_flags=ORB_IC_ANGLE | ORB_HARRIS, map_size=1500)
    pipe.set_map(mapd)
    pipe.step_dev(torch.from_numpy(frames).to(DEV))
    torch.cuda.synchronize()
    fcap = pipe.fcap
    sel = pipe.buffer("sel", (batch, fcap), torch.int32).cpu().numpy().view(np.uint32)
    selc = pipe.buffer("selcounts", (batch,), torch.int32).cpu().numpy()
    desc = pipe.buffer("desc", (batch, fcap, 32), torch.uint8).cpu().numpy()
    ang = pipe.buffer("angles", (batch, fcap), torch.float32).cpu().numpy()
    matches = pipe.buffer("matches", (batch, fcap, 4), torch.int32).cpu().numpy()
    for f in range(batch):
        gray = np.empty((h, w), np.uint8)
        oracle.orc_gray(P(frames[f]), w, h, P(gray))
        wk, wd = np.zeros((4096, 4), np.float32), np.zeros((4096, 32), np.uint8)
        n = oracle.orc_orb_detect(P(gray), w, h, nfeat, 20, 0, P(wk), P(wd), 4096)
        assert n == selc[f] and nfeat <= n <= fcap
        k = unpack_keys(sel[f, :n])
        assert (k[:, 0] == wk[:n, 0]).all() and (k[:, 1] == wk[:n, 1]).all()
        assert (ang[f, :n].view(np.uint32) == wk[:n, 3].copy().view(np.uint32)).all()
        assert (desc[f, :n] == wd[:n]).all()
        wm = np.zeros((n, 4), np.int32)
        oracle.orc_knn2(P(np.ascontiguousarray(wd[:n])), n, P(mapd), len(mapd), P(wm))
        assert (matches[f, :n] == wm).all() and (matches[f, n:] == -1).all()
    pipe.close()


def test_submit_wait_equals_step_host(gpu_ctx):
    """The asynchronous host step (two submissions in flight) delivers exactly what the synchronous one does."""
    import alvaar_b200
    from alvaar_b200.pipeline import Pipeline
    w, h, B = 640, 480, 16
    frames, _ = synth.make_frames(B, w, h, seed=5)
    _, mapd = synth.make_descriptors(8, 2000, seed=7)
    pipe = Pipeline(gpu_ctx, w, h, B, fast_thr=20, nfeatures=300, orb_flags=alvaar_b200.ORB_IC_ANGLE, map_size=2000)
    pipe.set_map(mapd)
    host = torch.from_numpy(frames).pin_memory()
    mk = lambda: (torch.zeros(B, dtype=torch.int32).pin_memory(), torch.zeros((B, pipe.fcap, 4), dtype=torch.int32).pin_memory())  # noqa: E731
    a, b, c = mk(), mk(), mk()
    pipe.step_host(host, *a)
    pipe.submit_host(host, *b)
    pipe.submit_host(host, *c)
    with pytest.raises(alvaar_b200.AlvaError):
        pipe.submit_host(host, *a)            # at most two outstanding
    pipe.wait(); pipe.wait(); pipe.wait()     # the third wait is a no-op
    assert a[0].sum() > 0
    for x in (b, c):
        assert torch.equal(x[0], a[0]) and torch.equal(x[1], a[1])
    pipe.close()


def test_lagged_ba_delivers_the_same_results_one_step_later(gpu_ctx):
    """alva_set_option("pipeline_ba_lag", 1): the BA chain of step s is joined at the end of step s + 1 (two chains in flight).
    Same numbers as the same-step schedule, one step later; alva_pipeline_drain joins the last one."""
    w, h, B = 640, 480, 4
    frames, _ = synth.make_frames(B, w, h, seed=5)
    _, mapd = synth.make_descriptors(8, 2000, seed=7)
    ba = synth.make_ba_problem(8, 300, 3, seed=7)
    ba2 = synth.make_ba_problem(8, 300, 3, seed=11)
    L = gpu_ctx.L

    def make():
        pipe = Pipeline(gpu_ctx, w, h, B, fast_thr=20, nfeatures=300, orb_flags=ORB_IC_ANGLE, map_size=2000, kf_interval=2,
                        ba_nkf=8, ba_nlm=300, ba_nobs=len(ba["obs_kf"]), ba_max_iter=5, ba_huber=ba["huber"])
        pipe.set_map(mapd)
        for s in range(pipe.nprob):
            pipe.set_ba(s, ba)
        return pipe

    def ba_out(pipe):
        torch.cuda.synchronize()
        return (pipe.buffer("ba_poses", (pipe.nprob, 8, 7), torch.float64).cpu().numpy().copy(),
                pipe.buffer("ba_summary", (pipe.nprob, 8), torch.float64).cpu().numpy().copy())

    d_in = torch.from_numpy(frames).to(DEV)
    try:
        assert L.alva_set_option(b"pipeline_ba_lag", 0) == 0
        ref = make()
        ref.step_dev(d_in)
        want1 = ba_out(ref)
        for s in range(ref.nprob):
            ref.set_ba(s, ba2)
        ref.step_dev(d_in)
        want2 = ba_out(ref)
        ref.close()
        assert not np.array_equal(want1[0], want2[0])

        assert L.alva_set_option(b"pipeline_ba_lag", 1) == 0
        pipe = make()
        pipe.step_dev(d_in)                       # step 0: its chain is still in flight when the step returns
        torch.cuda.synchronize()
        for s in range(pipe.nprob):
            pipe.set_ba(s, ba2)                   # (synchronous upload: both chains idle)
        pipe.drain()
        got = ba_out(pipe)
        assert np.array_equal(got[0], want1[0]) and np.array_equal(got[1], want1[1])
        pipe.step_dev(d_in)                       # step 1 (problem 2) joins nothing new: step 0 was drained
        pipe.step_dev(d_in)                       # step 2 joins step 1
        got = ba_out(pipe)
        assert np.array_equal(got[0], want2[0]) and np.array_equal(got[1], want2[1])
        for _ in range(4):                        # graphs captured by now: replays keep delivering the same
            pipe.step_dev(d_in)
        pipe.drain()
        got = ba_out(pipe)
        assert np.array_equal(got[0], want2[0]) and np.array_equal(got[1], want2[1])
        # matches / counts are the step's own in either mode
        pipe.close()
    finally:
        L.alva_set_option(b"pipeline_ba_lag", 0)
