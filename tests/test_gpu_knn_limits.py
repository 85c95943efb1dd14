"""The Hamming 2-NN matcher at its structural limits, on both kernels and every option that shapes them: the LOP3/POPC kernel
(knn_mma 0) with 4 and 8 queries per warp, and the tensor-core kernel (knn_mma 2) with int8 and E4M3 operands, unswizzled and
128-byte-swizzled.  The scenes (tests/knn_limits_util.py) put equal-distance ties across every warp-step, tile and chunk edge,
make every real row farther than the zero rows that pad the last train tile, put the answer last, plant it at train indices
>= 2^21 up to the largest train set, and drive the batch entry point through ragged, empty, over-full and negative counts.
Every output column is compared bit for bit with the oracle (orc_knn2), or with the answer known by construction where the
oracle would take minutes.  knn_mma_mode 2 is a debugging variant and is not run."""
import numpy as np
import pytest
import torch

import knn_limits_util as U
from alvaar_b200.lib import AlvaError

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

DEFAULTS = {"knn_mma": 1, "knn_mma_kind": 0, "knn_mma_mode": 0, "knn_qpw": 4}
PATHS = {"lop3_qpw4": {"knn_mma": 0, "knn_qpw": 4}, "lop3_qpw8": {"knn_mma": 0, "knn_qpw": 8},
         "mma_i8": {"knn_mma": 2}, "mma_i8_swz": {"knn_mma": 2, "knn_mma_mode": 1},
         "mma_e4m3": {"knn_mma": 2, "knn_mma_kind": 1}, "mma_e4m3_swz": {"knn_mma": 2, "knn_mma_kind": 1, "knn_mma_mode": 1}}


def set_options(ctx, opts):
    for k, v in dict(DEFAULTS, **opts).items():
        assert ctx.L.alva_set_option(k.encode(), v) == 0, (k, v)


@pytest.fixture
def ctx(gpu_ctx):
    """the matcher options are process-wide: every test leaves them at their defaults for the tests that run after it"""
    yield gpu_ctx
    set_options(gpu_ctx, {})


# every scene and its answer once per module, shared by all paths; device copies too
_host, _dev = {}, {}


def scene(oracle, name):
    if name not in _host:
        q, t = U.SCENES[name]()
        _host[name] = (q, t, U.oracle_knn2(oracle, q, t))
    return _host[name]


def planted(key):
    if key not in _host:
        nt, nq, below = key
        q, t, rows = U.planted(nt, nq, nt + below, below)
        _host[key] = (q, t, U.planted_answer(q, t, rows))
    return _host[key]


def dev(key, a):
    if key not in _dev:
        _dev[key] = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return _dev[key]


def knn2(ctx, q, t, qkey=None, tkey=None):
    """alva_k_hamming_knn2 into an output that starts as -7 everywhere, so a row the matcher never writes shows up"""
    dq = dev(qkey, q) if qkey is not None else torch.from_numpy(np.ascontiguousarray(q)).to(DEV)
    dt = dev(tkey, t) if tkey is not None else torch.from_numpy(np.ascontiguousarray(t)).to(DEV)
    out = torch.full((len(q), 4), -7, dtype=torch.int32, device=DEV)
    ctx.hamming_knn2(dq, len(q), dt, len(t), out)
    return out.cpu().numpy()


@pytest.mark.parametrize("name", list(U.SCENES))
@pytest.mark.parametrize("path", list(PATHS))
def test_knn2_scene(ctx, oracle, path, name):
    q, t, want = scene(oracle, name)
    set_options(ctx, PATHS[path])
    got = knn2(ctx, q, t, (name, "q"), (name, "t"))
    assert np.array_equal(got, want), (path, name, np.argwhere((got != want).any(1))[:5].ravel(), got[(got != want).any(1)][:3])


@pytest.mark.parametrize("key", U.PLANTED, ids=[f"nt{k[0]}_{'below' if k[2] else 'high'}" for k in U.PLANTED])
@pytest.mark.parametrize("path", list(PATHS))
def test_knn2_planted_high_indices(ctx, path, key):
    """answers at train indices >= 2^21 (bit 21 of the index shares the tensor-core key's bits with the distance) up to
    nt = 2^22 - 1 and index 2^22 - 2, with distance-1 ties broken by index, one of them just below 2^21"""
    q, t, want = planted(key)
    set_options(ctx, PATHS[path])
    got = knn2(ctx, q, t, (key, "q"), (key, "t"))
    assert np.array_equal(got, want), (path, key, np.argwhere((got != want).any(1))[:5].ravel())


# ---- the batch entry point ------------------------------------------------------------------------------------------------------

def batch_case(oracle, nbatch, qcap, all_zero=False):
    key = ("batch", nbatch, qcap, all_zero)
    if key not in _host:
        pool, t, pool_ans = scene(oracle, "batch_pool")
        counts = U.batch_counts(nbatch, qcap, nbatch + qcap, all_zero)
        slots = U.batch_slots(nbatch, qcap, nbatch + qcap, len(pool))
        _host[key] = (pool[slots], counts, U.batch_answer(pool_ans, slots, counts, qcap))
    return _host[key]


def knn2_batch(ctx, oracle, nbatch, qcap, all_zero=False):
    q, counts, want = batch_case(oracle, nbatch, qcap, all_zero)
    t = scene(oracle, "batch_pool")[1]
    key = ("batch", nbatch, qcap, all_zero)
    out = torch.full((len(q), 4), -7, dtype=torch.int32, device=DEV)
    ctx.hamming_knn2_batch(dev(key + ("q",), q), dev(key + ("c",), counts), nbatch, qcap, dev("batch_t", t), len(t), out)
    return out.cpu().numpy(), counts, want


@pytest.mark.parametrize("nbatch,qcap", U.BATCH_SHAPES)
@pytest.mark.parametrize("path", list(PATHS))
def test_knn2_batch_ragged(ctx, oracle, path, nbatch, qcap):
    """[nbatch][qcap] slots, counts[b] of them live: counts above qcap mean every slot, counts below 0 none; dead slots are
    four -1s"""
    set_options(ctx, PATHS[path])
    got, counts, want = knn2_batch(ctx, oracle, nbatch, qcap)
    assert np.array_equal(got, want), (path, nbatch, qcap, np.argwhere((got != want).any(1))[:5].ravel())
    g = got.reshape(nbatch, qcap, 4)
    assert (g[counts > qcap] >= 0).all() and (g[counts <= 0] == -1).all()


@pytest.mark.parametrize("path", list(PATHS))
def test_knn2_batch_all_empty(ctx, oracle, path):
    set_options(ctx, PATHS[path])
    got, _, _ = knn2_batch(ctx, oracle, 257, 16, all_zero=True)
    assert (got == -1).all()


# ---- dispatch, workspace, arguments ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nq,nt", U.CROSSOVER)
@pytest.mark.parametrize("mma", [0, 1, 2])
def test_knn2_dispatch_crossover(ctx, oracle, mma, nq, nt):
    """around the automatic choice (knn_mma 1: the tensor cores from nq >= 1024, nt >= 1024 and nq * nt >= 2^22 on) every
    setting gives the oracle's answer; the launch count (tensor cores: expand, match, merge; LOP3: match, merge) shows which
    kernel ran"""
    name = f"crossover_{nq}x{nt}"
    q, t, want = scene(oracle, name)
    set_options(ctx, {"knn_mma": mma})
    n0 = ctx.launches
    got = knn2(ctx, q, t, (name, "q"), (name, "t"))
    used_mma = ctx.launches - n0 == 3
    assert ctx.launches - n0 in (2, 3)
    assert used_mma == (mma == 2 or (mma == 1 and U.mma_wanted(nq, nt)))
    assert np.array_equal(got, want), (mma, nq, nt)


def test_knn2_workspace_lifecycle(ctx, oracle):
    """the tensor-core path keeps its workspace and grows it only for a larger problem: large -> small -> batch -> large again
    with another operand layout -> tiny, on one context, every output checked"""
    set_options(ctx, {"knn_mma": 2})
    big = (U.NT_MAX, 256, False)
    q, t, want = planted(big)
    assert np.array_equal(knn2(ctx, q, t, (big, "q"), (big, "t")), want)
    q, t, _ = scene(oracle, "repeated_3_1024")
    q2, t2 = q[:200], np.ascontiguousarray(t[:300])
    assert np.array_equal(knn2(ctx, q2, t2), U.oracle_knn2(oracle, q2, t2))
    got, _, want = knn2_batch(ctx, oracle, 257, 16)
    assert np.array_equal(got, want)
    set_options(ctx, {"knn_mma": 2, "knn_mma_mode": 1, "knn_mma_kind": 1})
    q, t, want = planted(big)
    assert np.array_equal(knn2(ctx, q, t, (big, "q"), (big, "t")), want)
    q, t = U.repeated(1, 1, 7, 3)
    assert np.array_equal(knn2(ctx, q, t), U.oracle_knn2(oracle, q, t))


def test_knn2_argument_checks(ctx):
    """nt outside [1, 2^22), nq or nbatch or qcap below 1, qcap not a multiple of 8 and buffers not 16-byte aligned are refused
    before anything runs"""
    raw = torch.zeros(((1 << 22) + 1) * 32, dtype=torch.uint8, device=DEV)
    t = raw[:(1 << 22) * 32]
    q = raw[:64 * 32]
    out = torch.zeros((65, 4), dtype=torch.int32, device=DEV)
    counts = torch.full((8,), 8, dtype=torch.int32, device=DEV)
    ctx.hamming_knn2(q, 64, t, (1 << 22) - 1, out)    # the largest train set is accepted
    torch.cuda.synchronize()
    bad = [lambda: ctx.hamming_knn2(q, 64, t, 1 << 22, out),
           lambda: ctx.hamming_knn2(q, 64, t, 0, out),
           lambda: ctx.hamming_knn2(q, 0, t, 64, out),
           lambda: ctx.hamming_knn2(raw[1:64 * 32 + 1], 64, t, 64, out),
           lambda: ctx.hamming_knn2(q, 64, raw[8:64 * 32 + 8], 64, out),
           lambda: ctx.hamming_knn2(q, 64, t, 64, out.view(-1)[1:]),
           lambda: ctx.hamming_knn2_batch(q, counts, 8, 12, t, 64, out),
           lambda: ctx.hamming_knn2_batch(q, counts, 0, 8, t, 64, out),
           lambda: ctx.hamming_knn2_batch(q, counts, 8, 0, t, 64, out),
           lambda: ctx.hamming_knn2_batch(q, counts, 8, 8, t, 1 << 22, out),
           lambda: ctx.hamming_knn2_batch(raw[4:64 * 32 + 4], counts, 8, 8, t, 64, out)]
    for call in bad:
        with pytest.raises(AlvaError):
            call()
