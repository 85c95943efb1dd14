"""GPU tests (H100) of the cross-stream loop-closure detector (csrc/loopclosure.cu, knn2_blockpair_kernel in csrc/hamming.cu)
stage by stage against the host model of tests/lc_util.py, at its structural limits: the wire format of alva_lc_pack, the 2-NN
lists, ratio test, gates, ordered compaction and PAIR_CAP truncation, the bearing vectors, the geometric check, and the temporal
rule and event queue of alva_lc_poll.  Bars: wire bytes, 2-NN rows of the live local descriptors, match counts and
correspondence counts exact; bearing vectors bitwise; verdicts and inlier counts exact; RANSAC [R | t] within 1e-9 of the
oracle's (the optimize=0 bar of test_gpu_init.py), except over the 20 checks of the temporal test (see there)."""
import ctypes as C

import numpy as np
import pytest
import torch

from alvaar_b200 import synth
from alvaar_b200.lib import AlvaError
from alvaar_b200.loopclosure import LoopClosure
from lc_util import (HDR, PAIR_CAP, block_bytes, config, detect_model, flip_bits, local_keyframe, make_block, pack_model, poll_model,
                     remote_view)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E_STATE = -4
K4A = tuple(float(v) for v in np.float32(synth.intrinsics(640, 480)))
THRESHOLDS = ("min_matches", "max_dist", "ratio_num", "ratio_den", "min_consecutive", "min_inliers", "err_px")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def detector(ctx, cfg, K4=None):
    """K4: the intrinsics alva_lc_pack writes; its focal is the geometric check's (cfg's fx_hint / fy_hint when K4 is None)"""
    K4 = (cfg["fx_hint"], cfg["fy_hint"], 0.0, 0.0) if K4 is None else K4
    assert (K4[0], K4[1]) == (cfg["fx_hint"], cfg["fy_hint"])
    return LoopClosure(ctx, cfg["n_max"], cfg["K"], cfg["world"], cfg["rank"], K4, **{k: cfg[k] for k in THRESHOLDS})


def readback(lc):
    nn, npair, bvl, bvr = lc.last_matches()
    return dict(scores=lc.last_scores(), nn=nn, npair=npair, bvl=bvl, bvr=bvr)


def run_step(ctx, gathered, cfg):
    """one detection on a host-built gathered buffer -> the device's per-pair state and the step's events"""
    lc = detector(ctx, cfg)
    try:
        g = dev(gathered)
        lc.detect(g)
        ev = lc.poll(wait=True)
        return dict(readback(lc), events=ev)
    finally:
        lc.close()


def check(d, m, cfg, skip_nn=()):
    """every stage of every pair (e, r) of one step: device `d` against the model `m`; skip_nn: pairs whose 2-NN rows the header does
    not define (a bad magic or version)"""
    sc = d["scores"]
    for e in range(cfg["K"]):
        for r in range(cfg["world"]):
            at = (e, r)
            assert sc[e, r, 0] == m["nmatch"][e, r], (at, sc[e, r], m["nmatch"][e, r])
            assert sc[e, r, 1] == m["verdict"][e, r], (at, sc[e, r], m["verdict"][e, r])
            assert sc[e, r, 2] == m["inliers"][e, r], (at, sc[e, r], m["inliers"][e, r])
            assert sc[e, r, 3] == m["remote_kf"][e, r], (at, sc[e, r])
            assert d["npair"][e, r] == m["npair"][e, r], (at, d["npair"][e, r], m["npair"][e, r])
            if r == cfg["rank"]:
                continue
            if at not in skip_nn:
                want = m["nn"][e][r]
                got = d["nn"][e, r, :len(want)]
                bad = np.nonzero((got != want).any(1))[0]
                assert len(bad) == 0, (at, bad[:4], got[bad[:4]], want[bad[:4]])
            k = min(int(m["nmatch"][e, r]), PAIR_CAP)
            if k:
                for side in ("bvl", "bvr"):
                    got, want = d[side][e, r, :k], m[side][e][r]
                    assert np.array_equal(got.view(np.int64), want.view(np.int64)), (at, side, np.abs(got - want).max())


def check_events(got, want, rt_tol=1e-9):
    assert len(got) == len(want), ([(e["local_kf"], e["remote_rank"]) for e in got], [(e["local_kf"], e["remote_rank"]) for e in want])
    for g, w in zip(got, want):
        assert {k: v for k, v in g.items() if k != "Rt"} == {k: v for k, v in w.items() if k != "Rt"}, (g, w)
        assert np.abs(g["Rt"] - w["Rt"]).max() < rt_tol, (g["Rt"], w["Rt"])


def build(rng, cfg, lcounts, rcounts, planted, K4s, seq=lambda r, e: 100 * r + e, **view):
    """host-built gathered buffer: local keyframe e has lcounts[e] keypoints, remote block (r, e) rcounts[r][e] entries of which
    planted[r][e] are true matches of the local keyframe; K4s[r]: the intrinsics of rank r"""
    n_max, K, world, rank = cfg["n_max"], cfg["K"], cfg["world"], cfg["rank"]
    blocks = [[None] * K for _ in range(world)]
    for e in range(K):
        loc = local_keyframe(rng, lcounts[e], K4s[rank])
        blocks[rank][e] = make_block(n_max, loc["px"], loc["desc"], K4s[rank], rank, seq(rank, e))
        for r in range(world):
            if r != rank:
                px, desc, _ = remote_view(rng, loc, rcounts[r][e], planted[r][e], K4s[r], **view)
                blocks[r][e] = make_block(n_max, px, desc, K4s[r], r, seq(r, e))
    return np.concatenate([b for row in blocks for b in row])


def shape_bench(rng):
    cfg = config(1536, 13, 2, 0, min_matches=100, min_consecutive=1, fx_hint=K4A[0], fy_hint=K4A[1])
    lc = rng.integers(900, 1301, 13)
    rc = [lc, rng.integers(900, 1301, 13)]
    frac = [0.0, 0.05, 0.08, 0.1, 0.12, 0.15, 0.2, 0.3, 0.09, 0.11, 0.13, 0.4, 0.35]
    pl = [None, [int(f * min(a, b)) for f, a, b in zip(frac, lc, rc[1])]]
    return cfg, build(rng, cfg, lc, rc, pl, [K4A] * 2, shifted=0.1, dups=4)


def shape_smallest(rng):
    cfg = config(8, 1, 2, 0, min_matches=1, min_consecutive=1, fx_hint=K4A[0], fy_hint=K4A[1])
    return cfg, build(rng, cfg, [8], [None, [1]], [None, [1]], [K4A] * 2)


def shape_largest(rng):
    cfg = config(8192, 1, 2, 1, min_consecutive=1, fx_hint=K4A[0], fy_hint=K4A[1])
    return cfg, build(rng, cfg, [8192], [[8192], None], [[3000], None], [K4A] * 2, shifted=0.1, dups=6)


def shape_wide(rng):
    # local counts per keyframe: the 32-query CTA tile +-1, none at all, and a full newest keyframe; remote counts: none, one (no
    # second neighbour), the 32-wide train tail +-1, full
    cfg = config(256, 4, 8, 5, min_matches=10, min_consecutive=1, fx_hint=K4A[0], fy_hint=K4A[1])
    lc = [33, 0, 31, 256]
    vals = [0, 1, 31, 32, 33, 256, 200, 97, 150, 64]
    rc = [[vals[(4 * r + e) % len(vals)] for e in range(4)] for r in range(8)]
    pl = [[int(0.6 * min(lc[e], rc[r][e])) for e in range(4)] for r in range(8)]
    return cfg, build(rng, cfg, lc, rc, pl, [K4A] * 8, dups=2)


def shape_last_rank_other_intrinsics(rng):
    # the local stream is the last rank; the remote cameras have their own intrinsics, which their bearings must use
    cfg = config(512, 2, 3, 2, min_consecutive=1, fx_hint=K4A[0], fy_hint=K4A[1])
    K4s = [(420.5, 431.25, 300.5, 250.75), (610.0, 602.5, 331.0, 236.5), K4A]
    return cfg, build(rng, cfg, [400, 480], [[500, 450], [300, 512], None], [[60, 200], [40, 240], None], K4s, shifted=0.15, dups=3)


SHAPES = {"bench": shape_bench, "smallest": shape_smallest, "largest": shape_largest, "wide": shape_wide,
          "last_rank_other_intrinsics": shape_last_rank_other_intrinsics}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_shapes_stage_by_stage(gpu_ctx, oracle, shape):
    rng = np.random.default_rng(list(SHAPES).index(shape) + 11)
    cfg, gathered = SHAPES[shape](rng)
    m = detect_model(oracle, gathered, cfg)
    d = run_step(gpu_ctx, gathered, cfg)
    check(d, m, cfg)
    check_events(d["events"], poll_model([(0, m)], cfg))
    K, rank = cfg["K"], cfg["rank"]
    others = [r for r in range(cfg["world"]) if r != rank]
    if shape == "bench":      # every verdict occurs, and counts between min_matches and nq / 8 are among them
        v = m["verdict"][:, 1]
        assert v[-1] == 1 and (v[:-1] == 2).any() and (v[:-1] == 0).any()
        assert any(100 <= m["nmatch"][e, 1] < 1536 and m["verdict"][e, 1] == 0 for e in range(K - 1))
    if shape == "largest":    # truncation to PAIR_CAP ahead of the geometric check
        assert m["nmatch"][0, 0] > PAIR_CAP and m["npair"][0, 0] == PAIR_CAP and m["verdict"][0, 0] == 1
    if shape in ("wide", "last_rank_other_intrinsics"):
        assert all(m["verdict"][K - 1, r] == 1 for r in others if m["npair"][K - 1, r] >= 40)
        assert len(d["events"]) >= 1


@pytest.mark.parametrize("n_max,cap", [(64, 40), (64, 96)])
def test_pack_wire_format(gpu_ctx, n_max, cap):
    """alva_lc_pack byte for byte: cap below and above n_max, counts above cap and above n_max, a negative count (no live entries),
    repeated and out-of-order keyframe frames, padding written over whatever the send buffer held, sequence numbers running on"""
    rng = np.random.default_rng(cap)
    desc = rng.integers(0, 256, (5, cap, 32), dtype=np.uint8)
    pts = rng.uniform(0, 640, (5, cap, 2)).astype(np.float32)
    counts = np.array([cap, cap + 30, 7, -3, n_max + 5], np.int32)
    kf = np.array([4, 1, 1, 0, 3, 2], np.int32)
    K4 = (612.5, 598.25, 321.75, 243.5)
    lc = LoopClosure(gpu_ctx, n_max, len(kf), 3, 1, K4)
    try:
        send = torch.full((len(kf) * block_bytes(n_max),), 0xAB, dtype=torch.uint8, device=DEV)
        for step in range(2):
            lc.pack(dev(desc), dev(pts), dev(counts), dev(kf), send)
            torch.cuda.synchronize()
            got, want = send.cpu().numpy(), pack_model(desc, pts, counts, cap, kf, step * len(kf), K4, n_max, 1)
            assert np.array_equal(got, want), np.nonzero(got != want)[0][:8]
    finally:
        lc.close()


def boundary_pairs(rng, ldesc, rdesc, queries, slots, cases):
    """plants, for query queries[i], remote descriptors at exactly the Hamming distances of cases[i] = (best, second) in free remote
    slots; second None: an exact duplicate of the best.  -> {query: remote slots}"""
    out, s = {}, iter(slots)
    for q, (d0, d1) in zip(queries, cases):
        a = flip_bits(rng, ldesc[q], d0)
        j0, j1 = next(s), next(s)
        rdesc[j0] = a
        rdesc[j1] = a if d1 is None else flip_bits(rng, ldesc[q], d1)
        out[q] = (j0, j1)
    return out


def test_gate_boundaries(gpu_ctx, oracle):
    """max_dist 40, ratio 3/4, min_matches 20 with 800 local keypoints (nq / 8 = 100): best == max_dist is kept and max_dist + 1
    dropped; best * den == second * num is dropped (the test is strict), one below it kept; an exact duplicate gives the lowest
    index and fails the ratio test; 99 matches (between min_matches and nq / 8) give verdict 0 with no geometric check, 100 are
    enough -- on an older keyframe (verdict 2) and on the newest (checked)"""
    rng = np.random.default_rng(5)
    n_max, n = 1024, 800
    cfg = config(n_max, 2, 3, 0, min_matches=20, max_dist=40, ratio_num=3, ratio_den=4, min_consecutive=1, fx_hint=K4A[0], fy_hint=K4A[1])
    cases = [(40, 60), (41, 60), (30, 40), (29, 40), (3, None), (0, None)]
    blocks = [[None] * 2 for _ in range(3)]
    dup_rows = {}
    for e in range(2):
        loc = local_keyframe(rng, n, K4A)
        blocks[0][e] = make_block(n_max, loc["px"], loc["desc"], K4A, 0, e)
        for r, planted in ((1, 97), (2, 100)):
            px, desc, (li, ri) = remote_view(rng, loc, 900, planted, K4A)
            if r == 1:
                q = [i for i in range(n) if i not in set(li)][:len(cases)]
                slots = sorted(set(range(900)) - set(ri))[::7]
                placed = boundary_pairs(rng, loc["desc"], desc, q, slots, cases)
                dup_rows[e] = [(q[i], placed[q[i]]) for i in (4, 5)]
            blocks[r][e] = make_block(n_max, px, desc, K4A, r, 10 * r + e)
    gathered = np.concatenate([b for row in blocks for b in row])
    m = detect_model(oracle, gathered, cfg)
    # the construction does what it says: 97 + 2 kept boundary queries on stream 1, 100 planted matches on stream 2
    assert list(m["nmatch"][:, 1]) == [99, 99] and list(m["nmatch"][:, 2]) == [100, 100]
    assert list(m["verdict"][0]) == [0, 0, 2] and list(m["npair"][1]) == [0, 0, 100] and m["verdict"][1, 2] == 1
    for e, rows in dup_rows.items():
        for q, (j0, j1) in rows:
            d0 = m["nn"][e][1][q][1]
            assert tuple(m["nn"][e][1][q]) == (min(j0, j1), d0, max(j0, j1), d0)
    d = run_step(gpu_ctx, gathered, cfg)
    check(d, m, cfg)
    check_events(d["events"], poll_model([(0, m)], cfg))


def test_bad_headers(gpu_ctx, oracle):
    """remote blocks with a bad magic, a bad version, a count above n_max (clamped: all entries live) and a count of -1 (no live
    entries); the other pairs of the step are unaffected.  The -1 block is built so that a kernel that trusted the count could not
    leave the gathered buffer: its tail step would read at most 32 descriptors (1 KB) before the descriptor array, i.e. inside the
    block's own pixel array (n_max >= 128), filled with 0xFF against all-zero local descriptors -- every stray candidate sits at
    distance 256, beyond the default max_dist, so it can only show in the 2-NN rows, which must all read -1"""
    rng = np.random.default_rng(9)
    n_max, world = 128, 6
    cfg = config(n_max, 2, world, 0, min_matches=10, min_consecutive=1, fx_hint=K4A[0], fy_hint=K4A[1])
    blocks = [[None] * 2 for _ in range(world)]
    for e in range(2):
        loc = local_keyframe(rng, n_max, K4A)
        if e == 0:
            loc["desc"][:] = 0
        blocks[0][e] = make_block(n_max, loc["px"], loc["desc"], K4A, 0, e)
        for r in range(1, world):
            px, desc, _ = remote_view(rng, loc, n_max, 60 if e == 1 else 0, K4A)
            kw = {}
            if e == 1 and r == 1:
                kw = dict(magic=0x12345678)
            elif e == 1 and r == 2:
                kw = dict(version=2)
            elif e == 1 and r == 3:
                kw = dict(count=n_max + 5)
            elif e == 0 and r == 4:
                kw = dict(count=-1)
            blocks[r][e] = make_block(n_max, px, desc, K4A, r, 10 * r + e, **kw)
            if e == 0 and r == 4:
                blocks[r][e][HDR:HDR + 8 * n_max] = 0xFF
    gathered = np.concatenate([b for row in blocks for b in row])
    m = detect_model(oracle, gathered, cfg)
    assert [m["verdict"][1, r] for r in range(1, world)] == [0, 0, 1, 1, 1]
    d = run_step(gpu_ctx, gathered, cfg)
    assert (d["nn"][0, 4] == -1).all(), d["nn"][0, 4][(d["nn"][0, 4] != -1).any(1)][:4]
    for r in (1, 2):
        assert d["scores"][1, r, 0] == 0 and d["scores"][1, r, 1] == 0 and d["npair"][1, r] == 0
    check(d, m, cfg, skip_nn={(1, 1), (1, 2)})
    check_events(d["events"], poll_model([(0, m)], cfg))


def drain(lc):
    """poll with room for one event at a time until the queue is empty"""
    out = []
    while True:
        ev = lc.poll(wait=True, cap=1)
        assert len(ev) <= 1
        if not ev:
            return out
        out += ev


@pytest.mark.parametrize("K", [1, 3])
def test_temporal_rule_and_queue(gpu_ctx, oracle, K):
    """8 steps, 3 remote streams with scripted related (R) / unrelated (U) keyframes; the local blocks go through alva_lc_pack.
    Events equal the model's in every field; poll(cap=1) hands them out one at a time; a fifth step enqueued with four in flight
    is refused with ALVA_E_STATE (through the C call: the Python wrapper drains on its own)"""
    rng = np.random.default_rng(20 + K)
    n_max, world, nsteps, n = 256, 4, 8, 200
    cfg = config(n_max, K, world, 0, fx_hint=K4A[0], fy_hint=K4A[1])
    script = {1: "R" * 24, 2: "RRRRU" * 5, 3: "RRU" * 8}
    bb = block_bytes(n_max)
    lc = detector(gpu_ctx, cfg, K4A)
    L, h = lc.L, lc.h
    L.alva_lc_inflight.argtypes = [C.c_void_p]
    events, steps, bufs, refused = [], [], [], 0
    try:
        for s in range(nsteps):
            locs = [local_keyframe(rng, n, K4A) for _ in range(K)]
            desc = np.zeros((K, n_max, 32), np.uint8)
            pts = np.zeros((K, n_max, 2), np.float32)
            for e, loc in enumerate(locs):
                desc[e, :n], pts[e, :n] = loc["desc"], loc["px"]
            counts, kf = np.full(K, n, np.int32), np.arange(K, dtype=np.int32)
            parts = [pack_model(desc, pts, counts, n_max, kf, s * K, K4A, n_max, 0)]
            for r in range(1, world):
                for e in range(K):
                    related = script[r][s * K + e] == "R"
                    px, dsc, _ = remote_view(rng, locs[e], 230, 120 if related else 0, K4A, shifted=0.1)
                    parts.append(make_block(n_max, px, dsc, K4A, r, 1000 * r + s * K + e))
            gathered = np.concatenate(parts)
            g = dev(gathered)
            g[:K * bb] = 0xEE                     # the local blocks come from the pack kernel
            lc.pack(dev(desc), dev(pts), dev(counts), dev(kf), g[:K * bb])
            rc = L.alva_lc_detect(h, C.c_void_p(g.data_ptr()))
            if rc == E_STATE:
                assert L.alva_lc_inflight(h) == 4
                refused += 1
                events += drain(lc)
                rc = L.alva_lc_detect(h, C.c_void_p(g.data_ptr()))
            assert rc == 0
            bufs.append(g)
            steps.append((s * K, detect_model(oracle, gathered, cfg)))
        events += drain(lc)
        assert refused == 1
        assert np.array_equal(bufs[-1].cpu().numpy(), gathered)
        check(readback(lc), steps[-1][1], cfg)
    finally:
        lc.close()
    want = poll_model(steps, cfg)
    assert len(want) >= 3 and {e["remote_rank"] for e in want} >= {1, 2}
    # the pose at the seeded-problem bar of test_gpu_init.py (1e-4), not 1e-9: alva_k_essential_5pt is compiled with FMA contraction
    # and the oracle is not, and over these 20 checks some five-point sample has two near-identical solutions whose order the
    # contraction swaps (measured on H100: 5e-6 in t, 4e-7 in R, same inlier count); every other field stays exact
    check_events(events, want, rt_tol=1e-4)


def test_create_checks_and_defaults(gpu_ctx, oracle):
    """bad sizes are refused; zero thresholds fall back to the documented defaults (min_matches 30, max_dist 64, ratio 4/5,
    min_consecutive 3, min_inliers 20, err_px 3, focal 500): the gates and the ratio by matches on their boundaries, min_matches
    by 29 matches against nq / 8 = 25, the temporal rule by the step of the first event, the threshold by the exact inlier count"""
    for n_max, K, world, rank in [(0, 1, 2, 0), (7, 1, 2, 0), (12, 1, 2, 0), (8200, 1, 2, 0), (64, 0, 2, 0), (64, 1, 2, 2)]:
        with pytest.raises(AlvaError):
            LoopClosure(gpu_ctx, n_max, K, world, rank, K4A)
    for n_max in (8, 8192):
        LoopClosure(gpu_ctx, n_max, 1, 2, 0, K4A).close()
    rng = np.random.default_rng(3)
    n_max, n = 256, 200                         # nq / 8 = 25 < 30
    cfg = config(n_max, 1, 3, 0)
    loc = local_keyframe(rng, n, K4A)
    blocks = [make_block(n_max, loc["px"], loc["desc"], K4A, 0, 0)]
    px, desc, (li, ri) = remote_view(rng, loc, 256, 100, K4A, shifted=0.3)
    q = [i for i in range(n) if i not in set(li)][:4]
    boundary_pairs(rng, loc["desc"], desc, q, sorted(set(range(256)) - set(ri)), [(64, 90), (65, 90), (40, 50), (39, 50)])
    blocks.append(make_block(n_max, px, desc, K4A, 1, 5))
    px, desc, _ = remote_view(rng, loc, 256, 29, K4A)
    blocks.append(make_block(n_max, px, desc, K4A, 2, 7))
    gathered = np.concatenate(blocks)
    m = detect_model(oracle, gathered, cfg)
    assert m["nmatch"][0, 1] == 102 and m["verdict"][0, 1] == 1 and m["nmatch"][0, 2] == 29 and m["verdict"][0, 2] == 0
    lc = LoopClosure(gpu_ctx, n_max, 1, 3, 0, (0.0, 0.0, 0.0, 0.0), **{k: 0 for k in THRESHOLDS})
    try:
        g = dev(gathered)
        events = []
        for s in range(3):
            lc.detect(g)
            events.append(lc.poll(wait=True))
        check(readback(lc), m, cfg)
    finally:
        lc.close()
    assert events[0] == [] and events[1] == []
    check_events(events[2], poll_model([(0, m)] * 3, cfg))
