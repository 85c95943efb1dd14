"""CPU tests: the Hamming 2-NN oracle (orc_knn2) against a plain NumPy restatement (knn_limits_util.knn2_numpy) and against the
reference's own cv::BFMatcher(NORM_HAMMING).knnMatch(k = 2), on the structural-limit scenes that tests/test_gpu_knn_limits.py
drives both matcher kernels through: runs of identical rows across every tile edge, complements (every distance >= 248, and 256),
the nearest row last at every ragged end, planted answers at train indices >= 2^21 up to the largest train set, train sets of a few
repeated descriptors, and the batch, query-count and dispatch-crossover shapes.  The reference's outputs are stored in
tests/golden/ref_live_knn_limits.npz, so this runs without it.  Every value is an integer: bit-exact.

This pins the tie rule (equal distances to the lower train index) and the "-1 where there are fewer than two rows" convention
against OpenCV itself on these scenes, not only against the project's restatement of it."""
import numpy as np
import pytest

import knn_limits_util as U
from ref_golden import digest

BIG = 256   # answers of more rows than this are stored as their row count and digest


def stored(a):
    return {"n": np.int64(len(a)), "d": digest(a)} if len(a) > BIG else {"n": np.int64(len(a)), "a": a}


def same(a, want):
    if "a" in want:
        return len(a) == len(want["a"]) and np.array_equal(a, want["a"])
    return len(a) == int(want["n"]) and (digest(a) == want["d"]).all()


@pytest.mark.parametrize("name", list(U.SCENES))
def test_knn2_oracle_numpy_reference(oracle, ref, name):
    q, t = U.SCENES[name]()
    got = U.oracle_knn2(oracle, q, t)
    assert np.array_equal(got, U.knn2_numpy(q, t)), name
    want = ref_outputs_knn(ref, f"knn_limits_{name}", q, t)
    assert same(got, want), name
    if len(t) < 2:
        assert (got[:, 2:] == -1).all() and (got[:, 0] == 0).all()
    if name.startswith("complement"):
        assert got[:, 1].min() >= 248 and (len(t) < 2 or got[:, 3].min() >= 248)
    if name.startswith("complement_all"):
        assert (got[:, 1] == 256).all() and (got[:, 0] == 0).all() and (got[:, 2] == (1 if len(t) > 1 else -1)).all()
    if name.startswith("nearest_last"):
        assert (got[:, 0] == len(t) - 1).all() and got[:, 1].max() <= 4


def ref_outputs_knn(ref, key, q, t):
    return U.ref_outputs(ref, key, lambda R: stored(U.ref_knn2(R, q, t)))


@pytest.mark.parametrize("nt,nq,nchk", [(U.HIGH + 3, 64, 32), (U.NT_MAX, 256, 8)])
@pytest.mark.parametrize("below", [False, True])
def test_knn2_planted_high_indices(oracle, ref, nt, nq, nchk, below):
    """the known answers of the planted scenes (indices >= 2^21, up to the largest train set) are the oracle's on the first nchk
    queries; the second best is a distance-1 tie broken by index.  BFMatcher refuses train sets of 2^18 rows or more
    (matchers.cpp:860, CV_Assert(rows < IMGIDX_ONE)), so the reference runs on the planted rows alone -- every other row is at
    least 16 bits from every query -- with its indices mapped back: the tie rule is OpenCV's, the index range this project's."""
    q, t, rows = U.planted(nt, nq, nt + below, below)
    want = U.planted_answer(q, t, rows)
    assert (rows[-1] >= 1 << 18) and len(rows) < 1 << 18
    assert (want[:, 3] <= 1).all() and (want[:, 0] >= U.HIGH).any()
    if below:
        assert (want[:, 2] < U.HIGH).any()
    if nt == U.NT_MAX:
        assert (want[:, 1] == 0).all() and (want[:, 0] >= U.HIGH).all() and want[0, 0] == U.NT_MAX - 1
        assert (want[:, 2] < U.HIGH).all() if below else (want[:, 2] >= U.HIGH).all()
    got = U.oracle_knn2(oracle, q[:nchk], t)
    assert np.array_equal(got, want[:nchk])
    r = U.ref_outputs(ref, f"knn_limits_planted_{nt}_{int(below)}", lambda R: stored(U.ref_knn2(R, q, t[rows])))
    mapped = want.copy()
    mapped[:, 0], mapped[:, 2] = np.searchsorted(rows, want[:, 0]), np.searchsorted(rows, want[:, 2])
    assert same(mapped, r)


@pytest.mark.parametrize("nbatch,qcap", [(257, 8), (300, 16), (3, 1536)])
def test_batch_answer_rule(nbatch, qcap):
    """the batch scenes' expected answers: a slot is live below its batch's count clamped to [0, qcap], else four -1s; the counts
    mix every edge and keep the last batch at most full"""
    counts = U.batch_counts(nbatch, qcap, nbatch + qcap)
    assert counts[-1] <= qcap and counts.sum() <= nbatch * qcap
    if nbatch >= 9:
        assert set(U.COUNT_MIX(qcap)) <= set(counts.tolist())
    pool_ans = np.arange(4 * 256, dtype=np.int32).reshape(256, 4)
    slots = U.batch_slots(nbatch, qcap, 1, 256)
    a = U.batch_answer(pool_ans, slots, counts, qcap).reshape(nbatch, qcap, 4)
    for b in range(nbatch):
        n = min(max(int(counts[b]), 0), qcap)
        assert (a[b, n:] == -1).all() and np.array_equal(a[b, :n], pool_ans[slots[b * qcap:b * qcap + n]])
