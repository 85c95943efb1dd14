"""The tensor-core Hamming 2-NN matcher with 1-bit operands (knn_mma_kind 2, the default): each query row is stored as
[a | ~a] and each train row as [~b | b], so one `wgmma ... .b1.and.popc` over the 512 bits gives popc(a & ~b) + popc(~a & b),
the Hamming distance itself, and the selection keeps the smallest distances.  The zero rows that pad the last train tile are
at distance 0 from every query under this encoding: only the tail mask keeps them out, so train counts that are not a
multiple of 128 are covered throughout.  Every output is compared bit for bit with the oracle (orc_knn2), with the answer
known by construction, or with the LOP3/POPC kernel and the int8 operands on the same inputs."""
import ctypes as C

import numpy as np
import pytest
import torch

import knn_limits_util as U
from alvaar_b200 import synth, ORB_IC_ANGLE, ORB_HARRIS
from alvaar_b200.pipeline import Pipeline

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DEFAULTS = {"knn_mma": 1, "knn_mma_kind": 2, "knn_mma_mode": 0, "knn_qpw": 4}


def set_options(ctx, opts):
    for k, v in dict(DEFAULTS, **opts).items():
        assert ctx.L.alva_set_option(k.encode(), v) == 0, (k, v)


@pytest.fixture
def b1(gpu_ctx):
    """the tensor-core matcher forced (knn_mma 2) with 1-bit operands; the process-wide options go back to their defaults"""
    set_options(gpu_ctx, {"knn_mma": 2, "knn_mma_kind": 2})
    yield gpu_ctx
    set_options(gpu_ctx, {})


def knn2(ctx, q, t):
    """alva_k_hamming_knn2 into an output that starts as -7 everywhere, so a row the matcher never writes shows up"""
    dq = torch.from_numpy(np.ascontiguousarray(q)).to(DEV)
    dt = torch.from_numpy(np.ascontiguousarray(t)).to(DEV)
    out = torch.full((len(q), 4), -7, dtype=torch.int32, device=DEV)
    ctx.hamming_knn2(dq, len(q), dt, len(t), out)
    return out.cpu().numpy()


def descriptors(nq, nt, seed):
    """random rows, a third of the queries copies of train rows with up to 3 bits flipped"""
    rng = np.random.default_rng(seed)
    q, t = synth.make_descriptors(nq, nt, seed=seed, planted=0.0)
    n = len(q[::3])
    q[::3] = t[rng.integers(0, nt, n)] ^ np.packbits(rng.random((n, 256)) < 3 / 256, axis=1)
    return q, t


def check(got, want, what):
    bad = np.argwhere((got != want).any(1)).ravel()
    assert not len(bad), (what, bad[:5], got[bad[:3]], want[bad[:3]])


@pytest.mark.parametrize("name", [n for n in U.SCENES if n != "batch_pool"])
def test_b1_scene(b1, oracle, name):
    """ties across every tile edge, complement scenes (every real row farther than a zero row), the nearest row last at
    nt % 128 in {0, 1, 31, 127}, train sets of 1 to 7 repeated descriptors, query counts 1 ... 513"""
    q, t = U.SCENES[name]()
    check(knn2(b1, q, t), U.oracle_knn2(oracle, q, t), name)


@pytest.mark.parametrize("nq,nt", [(1, 1), (1, 129), (2, 127), (129, 1), (256, 257), (257, 256), (257, 255), (7, 20000),
                                   (1000, 20000), (20000, 1000), (20000, 1)])
def test_b1_sizes(b1, oracle, nq, nt):
    q, t = descriptors(nq, nt, nq * 7 + nt)
    want = U.oracle_knn2(oracle, q, t)
    got = knn2(b1, q, t)
    check(got, want, (nq, nt))
    if nt == 1:
        assert (got[:, 0] == 0).all() and (got[:, 2] == -1).all() and (got[:, 3] == -1).all()


@pytest.mark.parametrize("nt", [1, 2, 100, 128, 129, 1000])
def test_b1_all_zero_and_all_ones(b1, oracle, nt):
    """descriptors of all zeros and all ones: distances 0 and 256 only, exactly as far as and farther than the zero rows that
    pad the last train tile"""
    z, o = np.zeros(32, np.uint8), np.full(32, 255, np.uint8)
    t = np.stack([o if i % 3 else z for i in range(nt)])
    q = np.stack([z, o, o, z] * 80)
    check(knn2(b1, q, t), U.oracle_knn2(oracle, q, t), ("mixed", nt))
    t1 = np.tile(o, (nt, 1))
    got = knn2(b1, np.stack([z] * 64), t1)
    check(got, U.oracle_knn2(oracle, np.stack([z] * 64), t1), ("ones", nt))
    assert (got[:, 0] == 0).all() and (got[:, 1] == 256).all()


@pytest.mark.parametrize("distinct,nt", [(1, 1000), (2, 3000), (3, 257), (7, 10000)])
def test_b1_repeated_train_rows(b1, oracle, distinct, nt):
    rng = np.random.default_rng(distinct * 1000 + nt)
    q, base = synth.make_descriptors(600, distinct, seed=distinct + nt, planted=0.0)
    q[::2] = base[rng.integers(0, distinct, 300)]
    t = np.ascontiguousarray(base[rng.integers(0, distinct, nt)])
    check(knn2(b1, q, t), U.oracle_knn2(oracle, q, t), (distinct, nt))


def test_b1_best_match_in_a_late_tile(b1, oracle):
    """every query's exact match sits in the last train tiles, behind 9 000 rows at one shared distance"""
    nq, nt = 1024, 10000
    q, t = synth.make_descriptors(nq, nt, seed=77, planted=0.0)
    t[:9000] = t[0]
    t[nt - nq:] = q
    got = knn2(b1, q, t)
    check(got, U.oracle_knn2(oracle, q, t), "late")
    assert (got[:, 0] == np.arange(nt - nq, nt)).all() and (got[:, 1] == 0).all()


@pytest.mark.parametrize("key", U.PLANTED, ids=[f"nt{k[0]}_{'below' if k[2] else 'high'}" for k in U.PLANTED])
def test_b1_planted_high_indices(b1, key):
    """answers at train indices >= 2^21 up to nt = 2^22 - 1 and index 2^22 - 2, distance-1 ties broken by index"""
    nt, nq, below = key
    q, t, rows = U.planted(nt, nq, nt + below, below)
    check(knn2(b1, q, t), U.planted_answer(q, t, rows), key)


@pytest.mark.parametrize("nbatch,qcap", U.BATCH_SHAPES)
def test_b1_batch_ragged(b1, oracle, nbatch, qcap):
    """[nbatch][qcap] slots with counts of 0, 1, 7, 8, 9, qcap - 1, qcap, qcap + 5 and -3: live queries compacted, dead
    slots four -1s"""
    t = U.batch_train()
    pool = U.batch_pool(t)
    pool_ans = U.oracle_knn2(oracle, pool, t)
    counts = U.batch_counts(nbatch, qcap, nbatch + qcap)
    slots = U.batch_slots(nbatch, qcap, nbatch + qcap, len(pool))
    q = pool[slots]
    want = U.batch_answer(pool_ans, slots, counts, qcap)
    out = torch.full((len(q), 4), -7, dtype=torch.int32, device=DEV)
    b1.hamming_knn2_batch(torch.from_numpy(np.ascontiguousarray(q)).to(DEV), torch.from_numpy(counts).to(DEV), nbatch, qcap,
                          torch.from_numpy(t).to(DEV), len(t), out)
    check(out.cpu().numpy(), want, (nbatch, qcap))


def test_b1_bench_shape_equals_lop3_and_int8(gpu_ctx):
    """the bench's matcher problem (64 frames x 1 536 slots, ragged live counts around 1 000, 10 000 map rows) through the
    batch entry point: 1-bit operands, int8 operands and the LOP3/POPC kernel give the same array"""
    rng = np.random.default_rng(11)
    nb, qcap, nt = 64, 1536, 10000
    q, t = descriptors(nb * qcap, nt, 12)
    counts = rng.integers(900, 1100, nb).astype(np.int32)
    counts[:3] = (0, qcap, qcap + 9)
    dq, dt, dc = torch.from_numpy(q).to(DEV), torch.from_numpy(t).to(DEV), torch.from_numpy(counts).to(DEV)
    outs = []
    try:
        for opts in ({"knn_mma": 2, "knn_mma_kind": 2}, {"knn_mma": 1}, {"knn_mma": 2, "knn_mma_kind": 0}, {"knn_mma": 0}):
            set_options(gpu_ctx, opts)
            out = torch.full((nb * qcap, 4), -7, dtype=torch.int32, device=DEV)
            n0 = gpu_ctx.launches
            gpu_ctx.hamming_knn2_batch(dq, dc, nb, qcap, dt, nt, out)
            if opts["knn_mma"]:
                assert gpu_ctx.launches - n0 == 4   # offsets, expand, match, merge
            outs.append(out.cpu().numpy())
    finally:
        set_options(gpu_ctx, {})
    for o in outs[1:]:
        assert np.array_equal(outs[0], o)
    assert (outs[0].reshape(nb, qcap, 4)[0] == -1).all()


def test_b1_ignores_the_swizzle_option(b1, oracle):
    """knn_mma_mode selects the shared-memory layout of the 8-bit kinds; the 64-byte rows of kind 2 have one layout"""
    q, t = synth.make_descriptors(700, 3000, seed=3)
    want = U.oracle_knn2(oracle, q, t)
    for mode in (0, 1):
        set_options(b1, {"knn_mma": 2, "knn_mma_kind": 2, "knn_mma_mode": mode})
        check(knn2(b1, q, t), want, mode)


def test_b1_option_values(gpu_ctx):
    L = gpu_ctx.L
    try:
        for v in (0, 1, 2):
            assert L.alva_set_option(b"knn_mma_kind", v) == 0
        for v in (-1, 3):
            assert L.alva_set_option(b"knn_mma_kind", v) != 0
    finally:
        set_options(gpu_ctx, {})


def test_b1_debug_entry_returns_distances(b1):
    """alva_debug_knn2_mma returns the raw accumulators of the first 128 x 128 tile: Hamming distances under kind 2"""
    L = b1.L
    vp, i32 = C.c_void_p, C.c_int
    L.alva_debug_knn2_mma.argtypes = [vp, vp, i32, vp, i32, vp, vp]
    q, t = synth.make_descriptors(300, 1000, seed=8)
    dq, dt = torch.from_numpy(q).to(DEV), torch.from_numpy(t).to(DEV)
    out = torch.full((300, 4), -7, dtype=torch.int32, device=DEV)
    dbg = torch.full((128, 128), -1, dtype=torch.int32, device=DEV)
    assert L.alva_debug_knn2_mma(b1.h, C.c_void_p(dq.data_ptr()), 300, C.c_void_p(dt.data_ptr()), 1000,
                                 C.c_void_p(out.data_ptr()), C.c_void_p(dbg.data_ptr())) == 0
    torch.cuda.synchronize()
    assert np.array_equal(dbg.cpu().numpy(), U.hamming_numpy(q[:128], t[:128]))


def _pipeline_outputs(ctx, kind, frames, mapd, flags):
    set_options(ctx, {"knn_mma": 2, "knn_mma_kind": kind})
    B, (h, w) = len(frames), frames.shape[1:3]
    pipe = Pipeline(ctx, w, h, B, fast_thr=20, nfeatures=1000, orb_flags=flags, map_size=len(mapd))
    try:
        pipe.set_map(mapd)
        d_in = torch.from_numpy(frames).to(DEV)
        pipe.step_dev(d_in)
        pipe.step_dev(d_in)
        torch.cuda.synchronize()
        cnt = pipe.buffer("selcounts", (B,), torch.int32).cpu().numpy().copy()
        live = np.arange(pipe.fcap)[None, :] < cnt[:, None]
        out = {"selcounts": cnt}
        for name, shape, dt in (("pts", (B, pipe.fcap, 2), torch.float32), ("desc", (B, pipe.fcap, 32), torch.uint8),
                                ("matches", (B, pipe.fcap, 4), torch.int32)):
            a = pipe.buffer(name, shape, dt).cpu().numpy().copy()
            a[~live] = 0
            out[name] = a
        return out
    finally:
        pipe.close()


@pytest.mark.parametrize("flags", [ORB_IC_ANGLE, ORB_IC_ANGLE | ORB_HARRIS], ids=["ic_angle", "harris"])
def test_b1_pipeline_step_equals_int8(gpu_ctx, flags):
    """one batched pipeline step with the matcher on 1-bit operands equals the step on int8 operands: counts, keys,
    descriptors and matches against a 10 000-row map"""
    frames, _ = synth.make_frames(4, 1280, 720, seed=5)
    _, mapd = synth.make_descriptors(8, 10000, seed=7)
    try:
        a = _pipeline_outputs(gpu_ctx, 2, frames, mapd, flags)
        b = _pipeline_outputs(gpu_ctx, 0, frames, mapd, flags)
    finally:
        set_options(gpu_ctx, {})
    assert (a["selcounts"] > 0).all()
    for k in a:
        assert np.array_equal(a[k], b[k]), k
