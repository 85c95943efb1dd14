"""GPU tests (H100): the reduced camera system S, rhs that the gather-form Schur assembly (ba_lm_kernel's landmark pass +
ba_gather_kernel) builds, against the FP64-atomic per-landmark path on the same linearisation (alva_k_ba_schur_dump: the first
Levenberg-Marquardt iteration of alva_k_ba_solve).  The two sum the same products in different orders, so they agree to
rounding: max |dS| <= 1e-12 max |S| and the same for rhs.  Cases: the bench's problem shape and make_ba_edge_problem's
structural edges (1 to 21 free poses, tracks of 6 and 13, more than 128 keyframes, shuffled observations).  The gather result
is also bit-reproducible, and a problem in a batch gets the bits it gets alone."""
import numpy as np
import pytest
import torch

import ba_util as B
from alvaar_b200 import synth
from test_gpu_ba_edges import high_layout, tracks

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NMAX = 128
RTOL = 1e-12


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def schur(ctx, pbs, atomic):
    """-> S [n][128][128], rhs [n][128], info [n][2] (width, gather path) of the first LM iteration"""
    n = len(pbs)
    nkf, nlm, nobs = len(pbs[0]["poses"]), len(pbs[0]["invd"]), len(pbs[0]["obs_kf"])
    st = lambda k: dev(np.stack([p[k] for p in pbs]))  # noqa: E731
    S = torch.full((n, NMAX, NMAX), np.nan, dtype=torch.float64, device=DEV)
    rhs = torch.full((n, NMAX), np.nan, dtype=torch.float64, device=DEV)
    info = torch.full((n, 2), -1.0, dtype=torch.float64, device=DEV)
    ctx.ba_schur_dump(n, nkf, nlm, nobs, st("calib"), st("poses"), st("pose_const"), st("invd"), st("anch_kf"), st("anch_uv"),
                      st("obs_kf"), st("obs_lm"), st("obs_uv"), pbs[0]["huber"], atomic, S, rhs, info)
    torch.cuda.synchronize()
    return S.cpu().numpy(), rhs.cpu().numpy(), info.cpu().numpy()


def check_against_atomic(ctx, pbs):
    gS, gr, gi = schur(ctx, pbs, False)
    aS, ar, ai = schur(ctx, pbs, True)
    for i, pb in enumerate(pbs):
        n = 6 * B.nfree(pb)
        assert gi[i, 0] == n and ai[i, 0] == n
        assert gi[i, 1] == 1 and ai[i, 1] == 0, (gi[i], ai[i])   # the gather path assembled the first, the atomic path the second
        assert n > 0 and np.abs(aS[i, :n, :n]).max() > 0
        assert np.abs(gS[i, :n, :n] - aS[i, :n, :n]).max() <= RTOL * np.abs(aS[i, :n, :n]).max()
        assert np.abs(gr[i, :n] - ar[i, :n]).max() <= RTOL * np.abs(ar[i, :n]).max()
        # block (bi, bj) and its mirror are stored together: S is symmetric up to the atomic path's rounding
        assert np.abs(gS[i, :n, :n] - gS[i, :n, :n].T).max() <= RTOL * np.abs(aS[i, :n, :n]).max()
        assert (gS[i, n:, :] == 0).all() and (gS[i, :, n:] == 0).all() and (gr[i, n:] == 0).all()
    return gS, gr


def bench_problem(seed):
    """the headline step's local-BA shape (bench.py c2): 20 keyframes (2 constant), 3000 landmarks, 9000 observations"""
    return B.problem_only(synth.make_ba_problem(20, 3000, 4, seed=seed))


def test_bench_shape(gpu_ctx):
    pbs = [bench_problem(s) for s in (42, 43, 44)]
    for pb in pbs:
        pb["free_ref"] = pb["pose_const"] == 0
    gS, gr = check_against_atomic(gpu_ctx, pbs)
    # bit-reproducible, and a problem in a batch gets the bits it gets alone
    gS2, gr2, _ = schur(gpu_ctx, pbs, False)
    assert (gS2 == gS).all() and (gr2 == gr).all()
    for i, pb in enumerate(pbs):
        sS, sr, _ = schur(gpu_ctx, [pb], False)
        assert (sS[0] == gS[i]).all() and (sr[0] == gr[i]).all()


@pytest.mark.parametrize("nf", [1, 2, 3, 5, 18, 21])
def test_width(gpu_ctx, nf):
    pb = B.make_ba_edge_problem(nfree=nf, nconst=2, nlm=600, track=tracks(nf, 600, min(8, nf + 1)), seed=100 + nf)
    assert B.nfree(pb) == nf and B.takes_gather_path(pb)
    check_against_atomic(gpu_ctx, [pb])


@pytest.mark.parametrize("t", [6, 13])
def test_track_length(gpu_ctx, t):
    """every landmark seen t times (13: the longest track whose entries still fit the gather's entry buffer)"""
    pb = B.make_ba_edge_problem(nfree=21, nconst=2, nlm=600, track=t, seed=300 + t, tie_frac=0.05)
    assert B.takes_gather_path(pb)
    check_against_atomic(gpu_ctx, [pb])


@pytest.mark.parametrize("nkf", [140, 256])
def test_many_keyframes(gpu_ctx, nkf):
    nfree, nconst = 9, 3
    nunref = nkf - nfree - nconst
    pb = B.make_ba_edge_problem(nfree=nfree, nconst=nconst, nlm=400, track=tracks(nkf, 400, 6), seed=nkf,
                                unref_free=nunref // 2, unref_const=nunref - nunref // 2,
                                kf_index=high_layout(nfree, nconst, nkf, seed=nkf))
    assert B.takes_gather_path(pb)
    check_against_atomic(gpu_ctx, [pb])


def test_shuffled_observations(gpu_ctx):
    pb = B.make_ba_edge_problem(nfree=7, nconst=2, nlm=500, track=tracks(8, 500, 6), seed=700, shuffle=True, pad=50)
    assert B.takes_gather_path(pb)
    check_against_atomic(gpu_ctx, [pb])
