"""Local BA through the Levenberg-Marquardt paths that do not accept the step: rejected steps and tolerance terminations, through
alva_k_ba_solve and alva_k_ba_local, against the FP64 oracle (oracle/ba_oracle.c) at the bar of test_gpu_ba.py.

A rejected step keeps the current point and its linearisation and solves again with the smaller radius; a tolerance
termination ends the solve without accepting the candidate.  The bench-shaped problems accept every step, so these cases are
built to leave that path (tests/ba_util.make_ba_edge_problem), and the CPU tests below check, from the oracle's own summary
counters, that each case takes the path it names.  No invalid step (failed factorisation, non-positive model change) is
covered: none of the generator's problems tried produced one."""
import numpy as np
import pytest

import ba_util as B
from test_gpu_ba_edges import gpu_local, gpu_solve

MAX_ITER = 10
# no robust loss and 30 % gross outliers: the first steps overshoot and are rejected (successful steps < iterations)
REJECTED = [dict(nfree=6, nconst=2, nlm=300, track=4, seed=s, huber=False, outlier_frac=0.3, outlier_px=300.0) for s in (0, 2)]
# poses far from the solution: every step is accepted and a tolerance ends the solve before MAX_ITER
TOLERANCE = [dict(nfree=6, nconst=2, nlm=300, track=4, seed=2, pose_noise_t=0.5, pose_noise_r_deg=15.0, noise_px=10.0)]
CASES = [("rejected", kw) for kw in REJECTED] + [("tolerance", kw) for kw in TOLERANCE]
IDS = [f"{name}-{kw['seed']}" for name, kw in CASES]


def takes_path(name, s):
    """summary[0..4] of one solve: initial cost, final cost, successful steps, iterations (incl. iteration 0), termination"""
    if name == "rejected":
        return s[2] < s[3]
    return s[4] == 0 and s[3] - 1 < MAX_ITER   # CONVERGENCE before the iteration limit


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_oracle_takes_the_path(oracle, name, kw):
    _, _, ws = B.oracle_solve(oracle, B.make_ba_edge_problem(**kw), max_iter=MAX_ITER)
    assert takes_path(name, ws), ws


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_oracle_local_takes_the_path(oracle, name, kw):
    nbad, _, _, _, ws = B.oracle_local(oracle, B.make_ba_edge_problem(**kw), max_iter=MAX_ITER)
    assert takes_path(name, ws[:5]), ws
    if name == "tolerance":
        assert nbad > 0 and ws[8] > 0   # the outliers are removed and the second solve runs


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_solve_vs_oracle(gpu_ctx, oracle, name, kw):
    pb = B.make_ba_edge_problem(**kw)
    wp, wd, ws = B.oracle_solve(oracle, pb, max_iter=MAX_ITER)
    gp, gd, gs = gpu_solve(gpu_ctx, [pb], max_iter=MAX_ITER)
    assert (gs[0, 2:5] == ws[2:5]).all(), (gs[0], ws)
    assert np.allclose(gs[0, :2], ws[:2], rtol=1e-8)
    assert np.allclose(gp[0], wp, rtol=1e-4, atol=1e-9) and np.allclose(gd[0], wd, rtol=1e-4, atol=1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_local_vs_oracle(gpu_ctx, oracle, name, kw):
    pb = B.make_ba_edge_problem(**kw)
    _, wp, wd, wf, ws = B.oracle_local(oracle, pb, max_iter=MAX_ITER)
    gp, gd, gf, gs = gpu_local(gpu_ctx, [pb], max_iter=MAX_ITER)
    assert (gf[0] == wf).all()
    assert (gs[0][[2, 3, 4, 7, 8, 9]] == ws[[2, 3, 4, 7, 8, 9]]).all(), (gs[0], ws)
    assert np.allclose(gs[0], ws, rtol=1e-8)
    assert np.allclose(gp[0], wp, rtol=1e-4, atol=1e-9) and np.allclose(gd[0], wd, rtol=1e-4, atol=1e-9)


@pytest.mark.gpu
def test_mixed_batch_equals_solo(gpu_ctx):
    """problems whose steps are rejected at different iterations, in one batch, give their solo results bit for bit (one
    problem's state must not leak into another's choice of linearisation)"""
    pbs = [B.make_ba_edge_problem(**kw) for kw in REJECTED]   # one batch shares the robust loss: these are all without it
    bp, bd, bs = gpu_solve(gpu_ctx, pbs, max_iter=MAX_ITER)
    for i, pb in enumerate(pbs):
        sp, sd, ss = gpu_solve(gpu_ctx, [pb], max_iter=MAX_ITER)
        assert (bp[i] == sp[0]).all() and (bd[i] == sd[0]).all() and (bs[i] == ss[0]).all()
