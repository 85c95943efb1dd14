"""The tensor-core matcher's selection under heavy ties.  The four threads that hold one query row share a bound on the
row's second best between train tiles, so a candidate that only equals that bound must lose to the earlier, lower train
index that set it, whichever thread saw it.  Train sets made of a few distinct descriptors, repeated across tiles and
across the columns of every thread, put many exact ties at the top of each row; the lists must equal the oracle's."""
import numpy as np
import pytest
import torch

from conftest import P
from alvaar_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture
def knn_mma(gpu_ctx):
    assert gpu_ctx.L.alva_set_option(b"knn_mma", 2) == 0
    yield gpu_ctx
    gpu_ctx.L.alva_set_option(b"knn_mma", 1)
    gpu_ctx.L.alva_set_option(b"knn_mma_mode", 0)
    gpu_ctx.L.alva_set_option(b"knn_mma_kind", 0)


@pytest.mark.parametrize("kind,mode", [(0, 0), (1, 1)])
@pytest.mark.parametrize("distinct,nt", [(1, 1000), (2, 3000), (3, 257), (7, 10000)])
def test_knn2_mma_repeated_train_rows(knn_mma, oracle, kind, mode, distinct, nt):
    assert knn_mma.L.alva_set_option(b"knn_mma_kind", kind) == 0
    assert knn_mma.L.alva_set_option(b"knn_mma_mode", mode) == 0
    rng = np.random.default_rng(distinct * 1000 + nt)
    q, base = synth.make_descriptors(600, distinct, seed=distinct + nt, planted=0.0)
    q[::2] = base[rng.integers(0, distinct, 300)]   # distance 0 to every copy of a train descriptor
    t = np.ascontiguousarray(base[rng.integers(0, distinct, nt)])
    want = np.zeros((len(q), 4), np.int32)
    oracle.orc_knn2(P(q), len(q), P(t), nt, P(want))
    out = torch.full((len(q), 4), -7, dtype=torch.int32, device=DEV)
    knn_mma.hamming_knn2(torch.from_numpy(q).to(DEV), len(q), torch.from_numpy(t).to(DEV), nt, out)
    assert (out.cpu().numpy() == want).all()


@pytest.mark.parametrize("kind", [0, 1])
def test_knn2_mma_best_match_in_a_late_tile(knn_mma, oracle, kind):
    """every query's exact match sits in the last train tiles, behind 9 000 rows at one shared distance: the shared bound
    rises early and must not hide the later, strictly better candidates"""
    assert knn_mma.L.alva_set_option(b"knn_mma_kind", kind) == 0
    nq, nt = 1024, 10000
    q, t = synth.make_descriptors(nq, nt, seed=77, planted=0.0)
    t[:9000] = t[0]
    t[nt - nq:] = q
    want = np.zeros((nq, 4), np.int32)
    oracle.orc_knn2(P(q), nq, P(t), nt, P(want))
    out = torch.full((nq, 4), -7, dtype=torch.int32, device=DEV)
    knn_mma.hamming_knn2(torch.from_numpy(q).to(DEV), nq, torch.from_numpy(t).to(DEV), nt, out)
    got = out.cpu().numpy()
    assert (got == want).all()
    assert (got[:, 0] == np.arange(nt - nq, nt)).all() and (got[:, 1] == 0).all()
