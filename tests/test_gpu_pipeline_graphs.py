"""GPU parity tests (H100) of the batched pipeline's CUDA-graph replays against the stage-by-stage oracle.

alva_pipeline_* captures the per-frame stages of each (input pointer, frame range) and each BA slot into a CUDA graph after a
first direct run, and replays it from then on.  A graph bakes in the addresses of the context workspaces its kernels use
and the kernel variants the library options chose; the pipeline replays it only while those are unchanged and captures it
anew otherwise.  These tests step the pipeline through the sequences that change them -- the chunked host path next to the
device path, other calls on the pipeline's context, two pipelines on one context, option changes -- with different inputs at
every step, and check every step's output against the oracle: levels, derivatives, selected keys, descriptors, `kept`, angle
bits and matches exactly, BA poses at rtol 1e-4 / atol 1e-9 and the BA summary's counts exactly."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

from conftest import P
import alvaar_b200
from alvaar_b200 import synth, unpack_keys, ORB_IC_ANGLE, ORB_HARRIS
from alvaar_b200.pipeline import Pipeline

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W, H, NFEAT, MAPN, THR = 640, 480, 300, 2000, 20
BA_NKF, BA_NLM, BA_ITER = 8, 300, 5
MODES = [ORB_IC_ANGLE, ORB_IC_ANGLE | ORB_HARRIS]

_frames = {}


def frames(n, w=W, h=H, seed=31):
    """n distinct frames along one camera path (cached: rendering is the slow part of the set-up)"""
    key = (n, w, h, seed)
    if key not in _frames:
        _frames[key] = synth.make_frames(n, w, h, seed=seed)[0]
    return _frames[key]


def pick(pool, step, batch, stride=7):
    """the frames of submission `step`: a different selection from the pool at every step"""
    return np.ascontiguousarray(pool[[(step * stride + i) % len(pool) for i in range(batch)]])


def ba_problem(seed):
    pb = synth.make_ba_problem(BA_NKF, BA_NLM, 3, seed=seed)
    pb["seed"] = seed
    return pb


class Oracle:
    """The oracle's answer for one frame, composed from the same calls test_gpu_pipeline.py makes (cached per frame)."""

    def __init__(self, orc, w, h, nfeat, flags):
        self.o, self.w, self.h, self.nfeat, self.flags = orc, w, h, nfeat, flags
        self.cache, self.ba_cache = {}, {}
        self.sizes = [(w, h)]
        for _ in range(3):
            self.sizes.append(((self.sizes[-1][0] + 1) // 2, (self.sizes[-1][1] + 1) // 2))

    def frame(self, rgba):
        key = hashlib.blake2b(rgba.tobytes(), digest_size=16).digest()
        if key not in self.cache:
            self.cache[key] = self._frame(rgba)
        return self.cache[key]

    def _frame(self, rgba):
        o, w, h, nfeat = self.o, self.w, self.h, self.nfeat
        gray = np.empty((h, w), np.uint8)
        o.orc_gray(P(np.ascontiguousarray(rgba)), w, h, P(gray))
        levels, cur = [gray], gray
        for k in (1, 2, 3):
            nxt = np.empty((self.sizes[k][1], self.sizes[k][0]), np.uint8)
            o.orc_pyrdown(P(cur), cur.shape[1], cur.shape[0], P(nxt))
            levels.append(nxt)
            cur = nxt
        derivs = []
        for k in range(4):
            d = np.zeros((self.sizes[k][1], self.sizes[k][0], 2), np.int16)
            o.orc_scharr(P(levels[k]), self.sizes[k][0], self.sizes[k][1], P(d))
            derivs.append(d)
        xs = np.zeros((w * h // 4, 3), np.int32)
        n = o.orc_fast9(P(gray), w, h, THR, 1, P(xs), len(xs))
        k = xs[:n]
        k = np.ascontiguousarray(k[(k[:, 0] >= 31) & (k[:, 0] < w - 31) & (k[:, 1] >= 31) & (k[:, 1] < h - 31)])
        inborder = len(k)   # FAST corners inside ORB's border: what the selection chooses from
        if self.flags & ORB_HARRIS:
            wk, wd = np.zeros((4096, 4), np.float32), np.zeros((4096, 32), np.uint8)
            c = o.orc_orb_detect(P(gray), w, h, nfeat, THR, 0, P(wk), P(wd), 4096)
            xy = wk[:c, :2].astype(np.int32)
            score = None
            ang = np.ascontiguousarray(wk[:c, 3])
            desc = np.ascontiguousarray(wd[:c])
        else:
            thr = o.orc_retain_best_threshold(P(k), len(k), nfeat)
            want = k[k[:, 2] >= thr]
            c = len(want)
            xy, score = want[:, :2], want[:, 2]
            pts = np.ascontiguousarray(xy.astype(np.float32))
            ang = np.zeros(c, np.float32)
            o.orc_ic_angles(P(gray), w, h, P(pts), c, P(ang))
            blur = np.empty_like(gray)
            o.orc_orb_blur(P(gray), w, h, 0, P(blur))
            desc, kept = np.zeros((c, 32), np.uint8), np.zeros(c, np.uint8)
            o.orc_orb_describe(P(blur), w, h, P(pts), P(ang), c, P(desc), P(kept))
            assert kept.all()   # every selected key lies inside the border
        return dict(levels=levels, derivs=derivs, count=int(c), inborder=int(inborder), xy=xy, score=score,
                    ang=ang.view(np.uint32), desc=desc)

    def matches(self, want, mapd):
        c = want["count"]
        m = np.zeros((c, 4), np.int32)
        if c:
            self.o.orc_knn2(P(want["desc"]), c, P(np.ascontiguousarray(mapd)), len(mapd), P(m))
        return m

    def ba(self, pb):
        """orc_ba_solve of one problem: (poses, summary)"""
        if pb["seed"] not in self.ba_cache:
            wp, wd, ws = pb["poses"].copy(), pb["invd"].copy(), np.zeros(8)
            self.o.orc_ba_solve(P(pb["calib"]), P(wp), P(pb["pose_const"]), BA_NKF, P(wd), P(pb["anch_kf"]), P(pb["anch_uv"]),
                                BA_NLM, P(pb["obs_kf"]), P(pb["obs_lm"]), P(pb["obs_uv"]), len(pb["obs_kf"]),
                                C.c_double(pb["huber"]), BA_ITER, P(ws), None)
            self.ba_cache[pb["seed"]] = (wp, ws)
        return self.ba_cache[pb["seed"]]


_oracles = {}


def get_oracle(orc, w, h, nfeat, flags):
    key = (w, h, nfeat, flags)
    if key not in _oracles:
        _oracles[key] = Oracle(orc, w, h, nfeat, flags)
    return _oracles[key]


def make_pipe(ctx, w=W, h=H, batch=4, nfeat=NFEAT, flags=ORB_IC_ANGLE, mapd=None, pb=None, kf_interval=2, derivatives=True):
    nobs = len(pb["obs_kf"]) if pb is not None else 0
    pipe = Pipeline(ctx, w, h, batch, fast_thr=THR, nfeatures=nfeat, orb_flags=flags,
                    map_size=len(mapd) if mapd is not None else 0, kf_interval=kf_interval if pb is not None else 0,
                    ba_nkf=BA_NKF if pb is not None else 0, ba_nlm=BA_NLM if pb is not None else 0, ba_nobs=nobs,
                    ba_max_iter=BA_ITER, ba_huber=pb["huber"] if pb is not None else 0.0, derivatives=derivatives)
    if mapd is not None:
        pipe.set_map(mapd)
    if pb is not None:
        set_ba(pipe, pb)
    return pipe


def set_ba(pipe, pb):
    for s in range(pipe.nprob):
        pipe.set_ba(s, pb)


class HostOut:
    """pinned result buffers of one host submission"""

    def __init__(self, pipe):
        B = pipe.cfg.batch
        self.nfeat = torch.full((B,), -7, dtype=torch.int32).pin_memory()
        self.matches = torch.full((B, pipe.fcap, 4), -7, dtype=torch.int32).pin_memory()
        self.poses = torch.zeros((max(pipe.nprob, 1), BA_NKF, 7), dtype=torch.float64).pin_memory()
        self.summary = torch.zeros((max(pipe.nprob, 1), 8), dtype=torch.float64).pin_memory()

    def args(self):
        return self.nfeat, self.matches, self.poses, self.summary


def step_host(pipe, batch_frames, out=None):
    out = out or HostOut(pipe)
    pipe.step_host(torch.from_numpy(batch_frames).pin_memory(), *out.args())
    return out


def check_frame_sel(want, f, selc, sel, kept, desc, ang, matches, fcap, mapd, ora):
    c = want["count"]
    assert int(selc[f]) == c, (f, int(selc[f]), c)
    assert c <= fcap
    k = unpack_keys(sel[f, :c])
    assert (k[:, :2] == want["xy"]).all(), f
    if want["score"] is not None:
        assert (k[:, 2] == want["score"]).all(), f
    assert (kept[f, :c] == 1).all() and (kept[f, c:] == 0).all(), f
    assert (desc[f, :c] == want["desc"]).all(), f
    assert (ang[f, :c].view(np.uint32) == want["ang"]).all(), f
    if mapd is not None:
        assert (matches[f, :c] == ora.matches(want, mapd)).all(), f
        assert (matches[f, c:] == -1).all(), f


def check_device(pipe, ora, batch_frames, mapd, derivatives=True):
    """every per-frame buffer the last step left on the device against the oracle"""
    torch.cuda.synchronize()
    B, fcap, sz = pipe.cfg.batch, pipe.fcap, ora.sizes
    sel = pipe.buffer("sel", (B, fcap), torch.int32).cpu().numpy().view(np.uint32)
    selc = pipe.buffer("selcounts", (B,), torch.int32).cpu().numpy()
    desc = pipe.buffer("desc", (B, fcap, 32), torch.uint8).cpu().numpy()
    kept = pipe.buffer("kept", (B, fcap), torch.uint8).cpu().numpy()
    ang = pipe.buffer("angles", (B, fcap), torch.float32).cpu().numpy()
    matches = pipe.buffer("matches", (B, fcap, 4), torch.int32).cpu().numpy() if mapd is not None else None
    lv = [pipe.buffer(f"l{k}", (B, sz[k][1], sz[k][0]), torch.uint8).cpu().numpy() for k in range(4)]
    dv = [pipe.buffer(f"d{k}", (B, sz[k][1], sz[k][0], 2), torch.int16).cpu().numpy() for k in range(4)] if derivatives else None
    for f in range(B):
        want = ora.frame(batch_frames[f])
        for k in range(4):
            assert (lv[k][f] == want["levels"][k]).all(), (f, k)
            if derivatives:
                assert (dv[k][f] == want["derivs"][k]).all(), (f, k)
        check_frame_sel(want, f, selc, sel, kept, desc, ang, matches, fcap, mapd, ora)


def check_host(pipe, ora, batch_frames, out, mapd, pb):
    """what a host submission delivered: per-frame counts and matches, and the step's BA"""
    fcap = pipe.fcap
    nf, m = out.nfeat.numpy(), out.matches.numpy()
    for f in range(pipe.cfg.batch):
        want = ora.frame(batch_frames[f])
        c = want["count"]
        assert int(nf[f]) == c, (f, int(nf[f]), c)
        if mapd is not None:
            assert (m[f, :c] == ora.matches(want, mapd)).all(), f
            assert (m[f, c:fcap] == -1).all(), f
    if pb is not None:
        check_ba(pipe, ora, pb, out.poses.numpy(), out.summary.numpy())


def check_ba(pipe, ora, pb, poses=None, summary=None):
    if poses is None:
        torch.cuda.synchronize()
        poses = pipe.buffer("ba_poses", (pipe.nprob, BA_NKF, 7), torch.float64).cpu().numpy()
        summary = pipe.buffer("ba_summary", (pipe.nprob, 8), torch.float64).cpu().numpy()
    wp, ws = ora.ba(pb)
    for s in range(pipe.nprob):
        assert np.allclose(poses[s], wp, rtol=1e-4, atol=1e-9), s
        assert (summary[s][2:5] == ws[2:5]).all(), s


@pytest.fixture
def ctx():
    """A context of its own, so that its workspaces start empty and which call grows them is known.  It runs on a stream of
    its own, which torch uses as well for the test: CUDA cannot capture a graph from the legacy default stream, so a pipeline
    on a context of that stream launches kernel by kernel and never replays."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        c = alvaar_b200.Context(0, s.cuda_stream)
        yield c
        torch.cuda.synchronize()
        c.close()


@pytest.fixture(scope="module")
def mapd():
    return synth.make_descriptors(8, MAPN, seed=3)[1]


@pytest.mark.parametrize("flags", MODES, ids=["ic", "harris"])
@pytest.mark.parametrize("batch", [16, 17, 18])
def test_chunked_host_path_replays(ctx, oracle, mapd, batch, flags):
    """step_host / submit_host run the batch in 4 chunks (16: 4 x 4, 17: 5, 5, 5, 2, 18: 5, 5, 5, 3), each at a frame offset into
    every buffer, from two staging slots.  Six submissions with different frames, two of them outstanding together: the
    first two run directly, the next two capture each slot's chunk graphs, the last two replay them.  Every frame of every
    chunk equals the oracle."""
    ora = get_oracle(oracle, W, H, NFEAT, flags)
    pool = frames(24)
    pb = ba_problem(7)
    pipe = make_pipe(ctx, batch=batch, flags=flags, mapd=mapd, pb=pb, kf_interval=8)
    try:
        for s in range(2):
            fr = pick(pool, s, batch)
            check_host(pipe, ora, fr, step_host(pipe, fr), mapd, pb)
            check_device(pipe, ora, fr, mapd)
        fr2, fr3 = pick(pool, 2, batch), pick(pool, 3, batch)
        o2, o3 = HostOut(pipe), HostOut(pipe)
        h2, h3 = torch.from_numpy(fr2).pin_memory(), torch.from_numpy(fr3).pin_memory()
        pipe.submit_host(h2, *o2.args())
        pipe.submit_host(h3, *o3.args())
        pipe.wait()
        pipe.wait()
        check_host(pipe, ora, fr2, o2, mapd, pb)
        check_host(pipe, ora, fr3, o3, mapd, pb)
        check_device(pipe, ora, fr3, mapd)
        captured_before, replays_before, _ = pipe.graph_stats()
        for s in (4, 5):
            fr = pick(pool, s, batch)
            check_host(pipe, ora, fr, step_host(pipe, fr), mapd, pb)
            check_device(pipe, ora, fr, mapd)
        captured, replays, failed = pipe.graph_stats()
        assert not failed
        assert captured == 2 * 4 + 1                     # 4 chunk graphs per staging slot and the BA chain's
        assert captured == captured_before               # the last two submissions captured nothing ...
        assert replays == replays_before + 2 * (4 + 1)   # ... they replayed every chunk and the BA chain
    finally:
        pipe.close()


def test_replays_read_new_inputs_map_and_ba(ctx, oracle, mapd):
    """step_dev on one device buffer whose frames are rewritten between steps; a new map and a new BA problem uploaded after
    the graphs were captured.  Every step equals the oracle for the inputs current at that step."""
    ora = get_oracle(oracle, W, H, NFEAT, ORB_IC_ANGLE)
    pool = frames(24)
    map2 = synth.make_descriptors(8, MAPN, seed=13)[1]
    pb1, pb2 = ba_problem(7), ba_problem(11)
    B = 4
    pipe = make_pipe(ctx, batch=B, mapd=mapd, pb=pb1)
    d_in = torch.empty((B, H, W, 4), dtype=torch.uint8, device=DEV)
    cur_map, cur_pb = mapd, pb1
    try:
        for s in range(7):
            if s == 3:
                pipe.set_map(map2)
                cur_map = map2
            if s == 5:
                set_ba(pipe, pb2)
                cur_pb = pb2
            fr = pick(pool, s, B, stride=5)
            d_in.copy_(torch.from_numpy(fr))
            pipe.step_dev(d_in)
            check_device(pipe, ora, fr, cur_map)
            check_ba(pipe, ora, cur_pb)
        captured, replays, failed = pipe.graph_stats()
        assert not failed and captured == 2 and replays == 2 * 6   # frame graph and BA graph: captured on step 1, replayed since
    finally:
        pipe.close()


def test_host_dev_host_recaptures_after_workspace_growth(ctx, oracle, mapd):
    """step_host x 3, step_dev, step_host x 4, step_dev x 2.  The full-batch direct run of step_dev needs more selection and
    matcher scratch than a chunk and reallocates it; the chunk graphs captured before it baked in the old buffers.  They are
    dropped and captured again instead of replayed (the captured count rises), and every step equals the oracle."""
    ora = get_oracle(oracle, W, H, NFEAT, ORB_IC_ANGLE)
    pool = frames(24)
    pb = ba_problem(7)
    B = 16
    pipe = make_pipe(ctx, batch=B, mapd=mapd, pb=pb, kf_interval=8)
    d_in = torch.empty((B, H, W, 4), dtype=torch.uint8, device=DEV)
    step = iter(range(100))

    def host():
        fr = pick(pool, next(step), B)
        check_host(pipe, ora, fr, step_host(pipe, fr), mapd, pb)
        check_device(pipe, ora, fr, mapd)

    def dev():
        fr = pick(pool, next(step), B)
        d_in.copy_(torch.from_numpy(fr))
        pipe.step_dev(d_in)
        check_device(pipe, ora, fr, mapd)
        check_ba(pipe, ora, pb)

    try:
        for _ in range(3):
            host()
        captured0 = pipe.graph_stats()[0]
        assert captured0 == 4 + 1   # slot 0's chunks and the BA chain
        dev()
        for _ in range(4):
            host()
        captured1, _, failed = pipe.graph_stats()
        assert not failed
        assert captured1 == captured0 + 2 * 4   # both slots' chunk graphs captured (again) after the direct full-batch run
        dev()
        dev()
        captured2, _, failed = pipe.graph_stats()
        assert not failed and captured2 == captured1 + 1   # the full-batch graph; nothing else changed
    finally:
        pipe.close()


def test_dev_host_dev(ctx, oracle, mapd):
    """step_dev, step_host, step_dev, repeated until every key has been captured and replayed: all equal the oracle."""
    ora = get_oracle(oracle, W, H, NFEAT, ORB_IC_ANGLE)
    pool = frames(24)
    pb = ba_problem(7)
    B = 16
    pipe = make_pipe(ctx, batch=B, mapd=mapd, pb=pb, kf_interval=8)
    d_in = torch.empty((B, H, W, 4), dtype=torch.uint8, device=DEV)
    try:
        for s in range(7):
            fr = pick(pool, s, B)
            if s % 2 == 0:
                d_in.copy_(torch.from_numpy(fr))
                pipe.step_dev(d_in)
                check_ba(pipe, ora, pb)
            else:
                check_host(pipe, ora, fr, step_host(pipe, fr), mapd, pb)
            check_device(pipe, ora, fr, mapd)
        captured, replays, failed = pipe.graph_stats()
        assert not failed and captured >= 2 and replays > 0
    finally:
        pipe.close()


def test_other_calls_on_the_context_between_steps(ctx, oracle, mapd):
    """The pipeline's matcher runs on the caller's context (tensor-core matcher forced: knn_mma = 2).  A larger Hamming 2-NN
    and a P3P-LMedS on that context between steps reallocate its workspaces; the pipeline's graphs are captured again and
    every step equals the oracle."""
    L = ctx.L
    ora = get_oracle(oracle, W, H, NFEAT, ORB_IC_ANGLE)
    pool = frames(24)
    pb = ba_problem(7)
    B = 4
    try:
        assert L.alva_set_option(b"knn_mma", 2) == 0
        pipe = make_pipe(ctx, batch=B, mapd=mapd, pb=pb)
        d_in = torch.empty((B, H, W, 4), dtype=torch.uint8, device=DEV)
        step = iter(range(100))

        def steps(n):
            for _ in range(n):
                fr = pick(pool, next(step), B, stride=3)
                d_in.copy_(torch.from_numpy(fr))
                pipe.step_dev(d_in)
                check_device(pipe, ora, fr, mapd)
                check_ba(pipe, ora, pb)

        try:
            steps(3)
            c0 = pipe.graph_stats()[0]
            assert c0 == 2
            # a larger matcher call on the same context: its scratch and tensor-core workspace grow
            q, t = synth.make_descriptors(20000, 6000, seed=17)
            out = torch.zeros((20000, 4), dtype=torch.int32, device=DEV)
            ctx.hamming_knn2(torch.from_numpy(q).to(DEV), 20000, torch.from_numpy(t).to(DEV), 6000, out)
            steps(3)
            c1, _, failed = pipe.graph_stats()
            assert not failed and c1 == c0 + 1   # the frame graph again (the BA chain runs on a context of its own)
            # a pose solve on the same context: its sampler table and scratch
            n = 3000
            pr = synth.make_pose_problem(n=n, seed=21, w=1280, h=720, outlier_frac=0.2)
            T = torch.zeros((16, 12), dtype=torch.float64, device=DEV)
            o = torch.zeros((16, n), dtype=torch.uint8, device=DEV)
            info = torch.zeros((16, 4), dtype=torch.float64, device=DEV)
            bv = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(pr["bv"], (16,) + pr["bv"].shape))).to(DEV)
            X = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(pr["X"], (16,) + pr["X"].shape))).to(DEV)
            fx = float(pr["K"][0])
            ctx.p3p_lmeds(16, n, bv, X, None, T, o, info, max_iter=100, fx=fx, fy=fx, seed=4242)
            steps(3)
            c2, _, failed = pipe.graph_stats()
            assert not failed and c2 == c1 + 1
        finally:
            pipe.close()
    finally:
        L.alva_set_option(b"knn_mma", 1)


def test_two_pipelines_on_one_context(ctx, oracle, mapd):
    """A 640x480 and a 1280x720 pipeline share one context (and so its matcher scratch), stepped in turn: each one's graphs
    are captured again whenever the other has grown the shared workspaces, and both equal the oracle at every step."""
    oa = get_oracle(oracle, W, H, NFEAT, ORB_IC_ANGLE)
    ob = get_oracle(oracle, 1280, 720, 1000, ORB_IC_ANGLE)
    pa_pool, pb_pool = frames(24), frames(4, 1280, 720)
    pb = ba_problem(7)
    map_b = synth.make_descriptors(8, 3000, seed=23)[1]
    A = make_pipe(ctx, batch=4, mapd=mapd, pb=pb)
    B = make_pipe(ctx, 1280, 720, batch=2, nfeat=1000, mapd=map_b, kf_interval=0)
    da = torch.empty((4, H, W, 4), dtype=torch.uint8, device=DEV)
    db = torch.empty((2, 720, 1280, 4), dtype=torch.uint8, device=DEV)
    try:
        for s in range(5):
            fa = pick(pa_pool, s, 4, stride=5)
            da.copy_(torch.from_numpy(fa))
            A.step_dev(da)
            check_device(A, oa, fa, mapd)
            check_ba(A, oa, pb)
            fb = pick(pb_pool, s, 2, stride=1)
            db.copy_(torch.from_numpy(fb))
            B.step_dev(db)
            check_device(B, ob, fb, map_b)
        # interleaved steps on one stream, checked only at the end
        fa, fb = pick(pa_pool, 9, 4, stride=5), pick(pb_pool, 3, 2, stride=1)
        da.copy_(torch.from_numpy(fa))
        db.copy_(torch.from_numpy(fb))
        A.step_dev(da)
        B.step_dev(db)
        check_device(A, oa, fa, mapd)
        check_device(B, ob, fb, map_b)
        for p in (A, B):
            assert not p.graph_stats()[2]
    finally:
        A.close()
        B.close()


def test_option_changes_recapture(ctx, oracle, mapd):
    """knn_mma 1 -> 0 -> 2, knn_qpw 4 -> 8, frontend_variant 2 -> 0 between replayed steps select other kernels: each change
    makes the pipeline capture its graphs again (a stale replay would keep running the old kernel).  The outputs stay
    bit-identical and equal the oracle."""
    L = ctx.L
    ora = get_oracle(oracle, W, H, NFEAT, ORB_IC_ANGLE)
    pool = frames(24)
    pb = ba_problem(7)
    B = 4
    fr = pick(pool, 0, B)
    pipe = make_pipe(ctx, batch=B, mapd=mapd, pb=pb)
    d_in = torch.from_numpy(fr).to(DEV)

    def step():
        pipe.step_dev(d_in)
        check_device(pipe, ora, fr, mapd)
        check_ba(pipe, ora, pb)

    try:
        for _ in range(3):
            step()
        captured = pipe.graph_stats()[0]
        assert captured == 2
        for name, value in ((b"knn_mma", 0), (b"knn_mma", 2), (b"knn_qpw", 8), (b"frontend_variant", 0)):
            assert L.alva_set_option(name, value) == 0
            step()   # direct run under the new option
            step()   # capture
            step()   # replay
            now, _, failed = pipe.graph_stats()
            assert not failed
            assert now == captured + 2, name   # the frame graph and the BA chain, captured again
            captured = now
    finally:
        pipe.close()
        L.alva_set_option(b"knn_mma", 1)
        L.alva_set_option(b"knn_qpw", 4)
        L.alva_set_option(b"frontend_variant", 2)


def test_graphs_and_profile_change_nothing(ctx, oracle, mapd):
    """The same four steps (new frames and a new BA problem between them) with graphs, without graphs
    (pipeline_graphs = 0) and while profiling: every buffer bit-identical, BA poses and summaries included."""
    L = ctx.L
    pool = frames(24)
    pb1, pb2 = ba_problem(7), ba_problem(11)
    B = 4

    def run(mode):
        pipe = make_pipe(ctx, batch=B, mapd=mapd, pb=pb1)
        if mode == "profile":
            pipe.profile(True)
        d_in = torch.empty((B, H, W, 4), dtype=torch.uint8, device=DEV)
        res = []
        try:
            for s in range(4):
                if s == 2:
                    set_ba(pipe, pb2)
                d_in.copy_(torch.from_numpy(pick(pool, s, B, stride=3)))
                pipe.step_dev(d_in)
                torch.cuda.synchronize()
                fcap, sz = pipe.fcap, get_oracle(oracle, W, H, NFEAT, ORB_IC_ANGLE).sizes
                selc = pipe.buffer("selcounts", (B,), torch.int32).cpu().numpy().copy()
                r = dict(selc=selc, counts=pipe.buffer("counts", (B,), torch.int32).cpu().numpy().copy())
                for name, shape, dt in (("sel", (B, fcap), torch.int32), ("pts", (B, fcap, 2), torch.float32),
                                        ("angles", (B, fcap), torch.float32), ("desc", (B, fcap, 32), torch.uint8)):
                    a = pipe.buffer(name, shape, dt).cpu().numpy()
                    r[name] = [a[f, :selc[f]].copy() for f in range(B)]   # live slots only
                r["kept"] = pipe.buffer("kept", (B, fcap), torch.uint8).cpu().numpy().copy()
                r["matches"] = pipe.buffer("matches", (B, fcap, 4), torch.int32).cpu().numpy().copy()
                r["blur"] = pipe.buffer("blur", (B, H, W), torch.uint8).cpu().numpy().copy()
                for k in range(4):
                    r[f"l{k}"] = pipe.buffer(f"l{k}", (B, sz[k][1], sz[k][0]), torch.uint8).cpu().numpy().copy()
                    r[f"d{k}"] = pipe.buffer(f"d{k}", (B, sz[k][1], sz[k][0], 2), torch.int16).cpu().numpy().copy()
                r["ba_poses"] = pipe.buffer("ba_poses", (pipe.nprob, BA_NKF, 7), torch.float64).cpu().numpy().copy()
                r["ba_invd"] = pipe.buffer("ba_invd", (pipe.nprob, BA_NLM), torch.float64).cpu().numpy().copy()
                r["ba_summary"] = pipe.buffer("ba_summary", (pipe.nprob, 8), torch.float64).cpu().numpy().copy()
                res.append(r)
            stats = pipe.graph_stats()
        finally:
            pipe.close()
        return res, stats

    try:
        want, stats = run("graphs")
        assert stats[0] == 2 and stats[1] == 2 * 3 and not stats[2]
        assert L.alva_set_option(b"pipeline_graphs", 0) == 0
        nograph, stats = run("direct")
        assert stats[:2] == (0, 0)
        assert L.alva_set_option(b"pipeline_graphs", 1) == 0
        prof, stats = run("profile")
        assert stats[:2] == (0, 0)
    finally:
        L.alva_set_option(b"pipeline_graphs", 1)
    assert not np.array_equal(want[0]["ba_poses"], want[2]["ba_poses"])   # the new BA problem was solved
    for got in (nograph, prof):
        for s in range(4):
            for k, v in want[s].items():
                g = got[s][k]
                if isinstance(v, list):
                    assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(v, g)), (s, k)
                else:
                    assert np.array_equal(v.view(np.uint8), g.view(np.uint8)), (s, k)


def degenerate_batch(B, at):
    """B frames from the pool with a flat frame and a frame with few corners (a small textured window in a flat frame)
    at the chunk boundary `at` (frames at - 1 and at), and a flat last frame"""
    fr = pick(frames(24), 0, B).copy()
    flat = np.full((H, W, 4), 255, np.uint8)
    flat[..., :3] = 117
    sparse = flat.copy()
    sparse[200:240, 300:350] = fr[0][200:240, 300:350]
    fr[at - 1], fr[at], fr[-1] = flat, sparse, flat
    return np.ascontiguousarray(fr)


@pytest.mark.parametrize("flags", MODES, ids=["ic", "harris"])
def test_degenerate_frames_at_a_chunk_boundary(ctx, oracle, mapd, flags):
    """A flat frame (no corner: count 0, every slot kept = 0 and matches = -1) and a frame with fewer in-border corners than
    nfeatures (all of them kept) at the boundary of two chunks, through both entry points and their replays."""
    ora = get_oracle(oracle, W, H, NFEAT, flags)
    pb = ba_problem(7)
    B = 16
    fr = degenerate_batch(B, 4)
    wz, ws = ora.frame(fr[3]), ora.frame(fr[4])
    assert wz["count"] == 0
    assert 0 < ws["count"] == ws["inborder"] < NFEAT
    pipe = make_pipe(ctx, batch=B, flags=flags, mapd=mapd, pb=pb, kf_interval=8)
    d_in = torch.from_numpy(fr).to(DEV)
    try:
        for _ in range(3):
            check_host(pipe, ora, fr, step_host(pipe, fr), mapd, pb)
            check_device(pipe, ora, fr, mapd)
            pipe.step_dev(d_in)
            check_device(pipe, ora, fr, mapd)
            check_ba(pipe, ora, pb)
        assert not pipe.graph_stats()[2]
    finally:
        pipe.close()


@pytest.mark.parametrize("with_map,with_ba", [(False, False), (False, True), (True, False)], ids=["bare", "ba-only", "map-only"])
def test_map_size_0_and_kf_interval_0(ctx, oracle, mapd, with_map, with_ba):
    """map_size 0 (no matching) and kf_interval 0 (no BA): both entry points succeed, replays included, and the stages
    still enabled equal the oracle."""
    ora = get_oracle(oracle, W, H, NFEAT, ORB_IC_ANGLE)
    pb = ba_problem(7) if with_ba else None
    m = mapd if with_map else None
    B = 16
    fr = degenerate_batch(B, 8)
    pipe = make_pipe(ctx, batch=B, mapd=m, pb=pb, kf_interval=8, derivatives=False)
    assert pipe.map_size == (MAPN if with_map else 0) and pipe.nprob == (2 if with_ba else 0)
    d_in = torch.from_numpy(fr).to(DEV)
    try:
        for _ in range(3):
            out = step_host(pipe, fr)
            check_host(pipe, ora, fr, out, m, pb)
            if not with_map:
                assert (out.matches.numpy() == -7).all()   # nothing written
            check_device(pipe, ora, fr, m, derivatives=False)
            pipe.step_dev(d_in)
            check_device(pipe, ora, fr, m, derivatives=False)
            if pb is not None:
                check_ba(pipe, ora, pb)
        assert not pipe.graph_stats()[2]
    finally:
        pipe.close()
