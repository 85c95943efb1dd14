"""Input scenes of the Hamming 2-NN structural-limit tests (tests/test_gpu_knn_limits.py runs them through both matcher kernels,
tests/test_oracle_knn_limits.py checks the oracle and a plain NumPy restatement against the reference on them), that NumPy
reference, and the store of the reference's outputs on these scenes (tests/golden/ref_live_knn_limits.npz).

Every scene is deterministic by its seed and returns (q, t): uint8 [nq][32] query and [nt][32] train descriptors.  An answer is
an int32 [nq][4] array {idx0, d0, idx1, d1}, -1 where there are fewer than one / two train rows: BFMatcher(NORM_HAMMING)'s
knnMatch(k = 2), ties to the lower train index."""
import ctypes as C
import os

import numpy as np

from conftest import P

STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_live_knn_limits.npz")
_stored = {}

NT_MAX = (1 << 22) - 1   # the largest train set alva_k_hamming_knn2 accepts (keys hold a 22-bit index)
HIGH = 1 << 21           # train indices from here on set bit 21 of the index, which the tensor-core key shares with the distance


def ref_outputs(ref, key, compute):
    """compute(ref) -> {name: array} from the live reference (oracle/_ref/libalva_ref.so built in the tree), else the stored
    arrays of `key`; with the reference built, ALVA_RECORD_REF=1 rewrites the stored entries of `key`.  The same rule as
    ref_golden.ref_outputs, over this file's own store."""
    if not _stored and os.path.exists(STORE):
        _stored.update(dict(np.load(STORE)))
    if ref is not None:
        out = {k: np.asarray(v) for k, v in compute(ref).items()}
        if os.environ.get("ALVA_RECORD_REF") == "1":
            for k in [k for k in _stored if k.startswith(key + "/")]:
                del _stored[k]
            _stored.update({f"{key}/{k}": v for k, v in out.items()})
            np.savez_compressed(STORE, **_stored)
        return out
    out = {k[len(key) + 1:]: v for k, v in _stored.items() if k.startswith(key + "/")}
    assert out, f"no stored reference outputs for {key}: build oracle/_ref and record them (ALVA_RECORD_REF=1)"
    return out


# ---- references -------------------------------------------------------------------------------------------------------------

POPC8 = np.array([bin(i).count("1") for i in range(256)], np.uint16)
POPC16 = (POPC8[:, None] + POPC8[None, :]).ravel()   # the byte table over both bytes of a 16-bit word


def hamming_numpy(q, t):
    """[nq][nt] Hamming distances (uint16) from a byte-popcount table on the XOR, two bytes per lookup"""
    return POPC16[(q[:, None, :] ^ t[None, :, :]).view(np.uint16)].sum(-1, dtype=np.uint16)


def knn2_numpy(q, t):
    """The 2-NN by a stable sort of each query's distances: equal distances stay in train-index order.  Shares no code with
    orc_knn2.  Blocked over the queries so that the [block][nt][32] XOR stays small."""
    q, t = np.ascontiguousarray(q, np.uint8), np.ascontiguousarray(t, np.uint8)
    nq, nt = len(q), len(t)
    out = np.full((nq, 4), -1, np.int32)
    blk = max(1, (1 << 22) // max(1, 32 * nt))
    for i in range(0, nq, blk):
        d = hamming_numpy(q[i:i + blk], t)
        o = np.argsort(d, axis=1, kind="stable")[:, :2]
        for k in range(min(2, nt)):
            out[i:i + blk, 2 * k] = o[:, k]
            out[i:i + blk, 2 * k + 1] = np.take_along_axis(d, o[:, k:k + 1], 1)[:, 0]
    return out


def oracle_knn2(oracle, q, t):
    q, t = np.ascontiguousarray(q, np.uint8), np.ascontiguousarray(t, np.uint8)
    out = np.zeros((len(q), 4), np.int32)
    oracle.orc_knn2(P(q), len(q), P(t), len(t), P(out))
    return out


def ref_knn2(R, q, t):
    """cv::BFMatcher(NORM_HAMMING).knnMatch(k = 2) (oracle/ref_harness.cpp)"""
    q, t = np.ascontiguousarray(q, np.uint8), np.ascontiguousarray(t, np.uint8)
    out = np.zeros((len(q), 4), np.int32)
    R.ref_knn2.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    R.ref_knn2(P(q), len(q), P(t), len(t), P(out))
    return out


# ---- scenes -----------------------------------------------------------------------------------------------------------------

def _rand(rng, n):
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


def _flip(d, bits):
    """d with the given bit positions (0..255, LSB first within each byte) inverted"""
    d = d.copy()
    for b in np.atleast_1d(bits):
        d[..., b >> 3] ^= np.uint8(1 << (b & 7))
    return d


def _flip_random(rng, rows, max_bits):
    """each row with 0..max_bits random bits inverted"""
    rows = rows.copy()
    for i in range(len(rows)):
        rows[i] = _flip(rows[i], rng.choice(256, int(rng.integers(0, max_bits + 1)), replace=False))
    return rows


def runs(seed, n_runs=80):
    """Runs of identical train rows, 33 and 129 long alternately, laid end to end, every run its own descriptor: a query equal to
    a run's descriptor ties at distance 0 with the whole run, and the runs start at every residue modulo 32 and 128 and at many
    modulo 512, so the tie straddles each warp step, train tile, query-pair chunk and LOP3 chunk boundary somewhere.  Queries:
    one copy of every run's descriptor, one with 1-3 bits flipped, and random ones."""
    rng = np.random.default_rng(seed)
    base = _rand(rng, n_runs)
    lens = np.where(np.arange(n_runs) % 2 == 0, 33, 129)
    t = np.repeat(base, lens, axis=0)
    q = np.concatenate([base, _flip_random(rng, base, 3), _rand(rng, 40)])
    return np.ascontiguousarray(q[rng.permutation(len(q))]), np.ascontiguousarray(t)


def complement(nq, nt, seed, max_bits=4):
    """Every train row within max_bits bits of one base descriptor and every query within max_bits bits of its complement: every
    distance is at least 256 - 2 max_bits, farther than the zero rows that pad the last train tile (distance 128).  Queries that
    are the exact complement of a train row that is the base itself meet distance 256 (dot product -256)."""
    rng = np.random.default_rng(seed)
    base = _rand(rng, 1)[0]
    t = _flip_random(rng, np.repeat(base[None], nt, 0), max_bits)
    t[rng.integers(0, nt, max(1, nt // 16))] = base
    q = _flip_random(rng, np.repeat(~base[None], nq, 0), max_bits)
    q[: max(1, nq // 8)] = ~base
    return q, t


def complement_all(nq, nt):
    """Every train row the same descriptor, every query its complement: every distance is 256, the largest key, and the answer
    is the two lowest indices"""
    rng = np.random.default_rng(nt)
    base = _rand(rng, 1)[0]
    return np.repeat(~base[None], nq, 0), np.repeat(base[None], nt, 0)


def nearest_last(nq, nt, seed):
    """The complement scene with its nearest row, the exact complement of the queries' base, last (t[nt - 1]): the row every
    query must find sits in the ragged end of the last warp step and train tile"""
    q, t = complement(nq, nt, seed)
    t[nt - 1] = q[0]   # ~base: within max_bits bits of every query
    return q, t


NEAREST_LAST_NT = [1, 2, 31, 32, 127, 128, 129, 159, 1025, 1055, 1151, 2048, 4097, 4223]   # nt % 128 in {0, 1, 31, 127}


def planted(nt, nq, seed, below=False):
    """Random train rows and, for each query, planted rows at indices in [2^21, nt): an exact copy, a 1-bit flip and another 1-bit
    flip (the second best is a distance-1 tie broken by index); with `below`, a third 1-bit flip at an index just below 2^21,
    which must win that tie.  Random rows have their first two bytes 0xFF and queries 0x00 there, and the flips stay out of
    those bytes, so every random row is at least 16 bits from every query and cannot take part in an answer.  Where [2^21, nt)
    is too short for three rows per query, the queries share one set of planted rows (four or five queries of different
    answers, repeated).  Returns (q, t, planted indices, ascending)."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    t[:, :2] = 0xFF
    q = _rand(rng, nq)
    q[:, :2] = 0
    bits = lambda k: rng.choice(np.arange(16, 256), k, replace=False)   # noqa: E731
    if nt - HIGH >= 3 * nq:
        idx = rng.choice(nt - HIGH, 3 * nq, replace=False).reshape(nq, 3) + HIGH
        idx[0, 0] = nt - 1              # the largest index a key can hold, as an exact copy
        idx[min(1, nq - 1), 0] = HIGH   # and bit 21 alone
        for i in range(nq):
            b = bits(3)
            t[idx[i, 0]] = q[i]
            t[idx[i, 1]] = _flip(q[i], b[0])
            t[idx[i, 2]] = _flip(q[i], b[1])
        rows = list(idx.ravel())
        if below:
            low = rng.choice(4096, nq, replace=False) + HIGH - 4096
            low[0] = HIGH - 1
            for i in range(nq):
                t[low[i]] = _flip(q[i], bits(1)[0])
            rows += list(low)
    else:
        assert nt - HIGH >= 3
        base = q[0].copy()
        b = bits(3)
        rows = [nt - 1, HIGH, HIGH + 1]
        t[nt - 1], t[HIGH], t[HIGH + 1] = base, _flip(base, b[0]), _flip(base, b[1])
        kinds = [base, _flip(base, b[0]), _flip(base, b[1]), _flip(_flip(base, b[0]), b[1])]
        if below:
            t[HIGH - 1] = _flip(base, b[2])
            rows.append(HIGH - 1)
            kinds.append(_flip(base, b[2]))
        q = np.ascontiguousarray(np.stack([kinds[i % len(kinds)] for i in range(nq)]))
    return q, t, np.array(sorted(set(int(r) for r in rows)), np.int64)


def planted_answer(q, t, rows):
    """The answer of a planted scene, known by construction: the 2-NN among the planted rows (knn2_numpy; `rows` ascending, so
    index order is kept), after checking that every other row is farther from every query than that answer's second best"""
    assert (t[np.setdiff1d(np.arange(len(t)), rows)][:, :2] == 0xFF).all() and (q[:, :2] == 0).all()   # >= 16 bits away
    a = knn2_numpy(q, t[rows])
    assert (a[:, 3] >= 0).all() and a[:, 3].max() < 16
    a[:, 0], a[:, 2] = rows[a[:, 0]], rows[a[:, 2]]
    return a


def repeated(distinct, nt, nq, seed):
    """A train set of `distinct` descriptors repeated in random order; half the queries are copies of them (distance-0 ties across
    the whole set), half random"""
    rng = np.random.default_rng(seed)
    base = _rand(rng, distinct)
    t = np.ascontiguousarray(base[rng.integers(0, distinct, nt)])
    q = _rand(rng, nq)
    q[::2] = base[rng.integers(0, distinct, (nq + 1) // 2)]
    return q, t


REPEATED_NT = [1, 2, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025]


def batch_train(seed=5, nt=1000):
    """the train set of the batch scenes: 200 descriptors, each at about five scattered indices"""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(_rand(rng, 200)[rng.integers(0, 200, nt)])


def batch_pool(t, seed=6, n=256):
    """the descriptors the batch scenes' query slots are drawn from: copies of train rows, copies with a few bits flipped, random"""
    rng = np.random.default_rng(seed)
    pool = _rand(rng, n)
    pool[: n // 2] = t[rng.integers(0, len(t), n // 2)]
    pool[n // 4: n // 2] = _flip_random(rng, pool[n // 4: n // 2], 3)
    return pool


COUNT_MIX = lambda qcap: [0, 1, 7, 8, 9, qcap - 1, qcap, qcap + 5, -3]   # noqa: E731


def batch_counts(nbatch, qcap, seed, all_zero=False):
    """counts[nbatch] cycling through 0, 1, 7, 8, 9, qcap - 1, qcap, qcap + 5 and -3 in a seeded order.  The last batch is never
    over-full and the counts sum to at most nbatch * qcap, so even a matcher that forgot to clamp them to [0, qcap] stays inside
    the arrays and fails by its answers."""
    if all_zero:
        return np.zeros(nbatch, np.int32)
    rng = np.random.default_rng(seed)
    mix = COUNT_MIX(qcap)
    c = np.array([mix[i % len(mix)] for i in rng.permutation(nbatch) + seed], np.int64)
    if c[-1] > qcap:
        c[-1] = qcap - 1
    while c.sum() > nbatch * qcap:
        c[np.argmax(c)] = 0
    return c.astype(np.int32)


def batch_slots(nbatch, qcap, seed, npool):
    """pool index of every query slot [nbatch * qcap] (dead slots too: they hold descriptors the matcher must ignore)"""
    return np.random.default_rng(seed + 1).integers(0, npool, nbatch * qcap)


def batch_answer(pool_answer, slots, counts, qcap):
    """the answer of every slot: its pool descriptor's where the slot is live (slot < counts clamped to [0, qcap]), -1 x 4 where not"""
    live = (np.arange(len(slots)) % qcap) < np.repeat(np.clip(counts, 0, qcap), qcap)
    out = np.full((len(slots), 4), -1, np.int32)
    out[live] = pool_answer[slots[live]]
    return out


BATCH_SHAPES = [(nb, qc) for nb in (1, 255, 256, 257, 300) for qc in (8, 16, 1536, 4096)]


def nq_train(seed=9, nt=3000):
    """the fixed train set of the query-count sweep: random rows, a tenth of them repeated"""
    rng = np.random.default_rng(seed)
    t = _rand(rng, nt)
    t[rng.integers(0, nt, nt // 10)] = t[rng.integers(0, nt, nt // 10)]
    return t


def nq_queries(nq, t, seed=10):
    rng = np.random.default_rng(seed + nq)
    q = _rand(rng, nq)
    q[::3] = _flip_random(rng, t[rng.integers(0, len(t), len(q[::3]))], 2)
    return q


NQ_SWEEP = [1, 7, 8, 9, 255, 256, 257, 511, 512, 513]
# (nq, nt) around the tensor-core dispatch rule (nq >= 1024, nt >= 1024, nq * nt >= 2^22)
CROSSOVER = [(1023, 1023), (1023, 1024), (1024, 1023), (1024, 1024), (1024, 4095), (1024, 4096), (2049, 2048)]


def mma_wanted(nq, nt):
    return nq >= 1024 and nt >= 1024 and nq * nt >= (1 << 22)


def _batch_scene():
    t = batch_train()
    return batch_pool(t), t


# the scenes both kernels and the oracle run on whole (name -> () -> (q, t))
SCENES = {"runs": lambda: runs(1)}
SCENES.update({f"complement_{nt}": (lambda nt=nt: complement(300, nt, nt)) for nt in (1, 2, 129, 1000, 4097)})
SCENES.update({f"complement_all_{nt}": (lambda nt=nt: complement_all(64, nt)) for nt in (1, 2, 129, 1000)})
SCENES.update({f"nearest_last_{nt}": (lambda nt=nt: nearest_last(200, nt, nt)) for nt in NEAREST_LAST_NT})
SCENES.update({f"repeated_{k}_{nt}": (lambda k=k, nt=nt: repeated(k, nt, 300, 100 * k + nt)) for k in (1, 3, 7) for nt in REPEATED_NT})
SCENES["batch_pool"] = _batch_scene
SCENES.update({f"nq_{nq}": (lambda nq=nq: (nq_queries(nq, nq_train()), nq_train())) for nq in NQ_SWEEP})
SCENES.update({f"crossover_{nq}x{nt}": (lambda nq=nq, nt=nt: repeated(5, nt, nq, nq + nt)) for nq, nt in CROSSOVER})
# the planted high-index scenes: (nt, nq, below) -> seed nt + below
PLANTED = [(HIGH + 3, 64, False), (HIGH + 3, 64, True), (NT_MAX, 256, False), (NT_MAX, 256, True)]
