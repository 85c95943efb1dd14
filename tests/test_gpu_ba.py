"""GPU parity tests (H100): local BA through the C ABI vs the CPU oracle (itself pinned to ceres::Solve at 1e-14)
and the golden Ceres solution.  FP64; tolerance 1e-4 relative on poses / inverse depths (north_star), plus equal
iteration counts and termination reason."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import P, golden
from alvaar_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def oracle_solve(oracle, pb, max_iter=5, huber=None):
    poses, invd = pb["poses"].copy(), pb["invd"].copy()
    summary, costs = np.zeros(8), np.zeros(64)
    oracle.orc_ba_solve(P(pb["calib"]), P(poses), P(pb["pose_const"]), len(poses), P(invd), P(pb["anch_kf"]),
                        P(pb["anch_uv"]), len(invd), P(pb["obs_kf"]), P(pb["obs_lm"]), P(pb["obs_uv"]), len(pb["obs_kf"]),
                        C.c_double(pb["huber"] if huber is None else huber), max_iter, P(summary), P(costs))
    return poses, invd, summary


def gpu_solve(ctx, pbs, max_iter=5, huber=None):
    n = len(pbs)
    nkf, nlm, nobs = len(pbs[0]["poses"]), len(pbs[0]["invd"]), len(pbs[0]["obs_kf"])
    st = lambda k: dev(np.stack([p[k] for p in pbs]))  # noqa: E731
    poses, invd = st("poses"), st("invd")
    summary = torch.zeros((n, 8), dtype=torch.float64, device=DEV)
    ctx.ba_solve(n, nkf, nlm, nobs, st("calib"), poses, st("pose_const"), invd, st("anch_kf"), st("anch_uv"), st("obs_kf"),
                 st("obs_lm"), st("obs_uv"), pbs[0]["huber"] if huber is None else huber, max_iter, summary)
    torch.cuda.synchronize()
    return poses.cpu().numpy(), invd.cpu().numpy(), summary.cpu().numpy()


def test_linearize_vs_oracle(gpu_ctx, oracle):
    pb = synth.make_ba_problem(20, 3000, 4, seed=42)
    nobs = len(pb["obs_kf"])
    res, Ja, Jp, Jd = np.zeros(2 * nobs), np.zeros(12 * nobs), np.zeros(12 * nobs), np.zeros(2 * nobs)
    oracle.orc_ba_linearize.restype = C.c_double
    cost = oracle.orc_ba_linearize(P(pb["calib"]), P(pb["poses"]), 20, P(pb["invd"]), P(pb["anch_kf"]), P(pb["anch_uv"]), 3000,
                                   P(pb["obs_kf"]), P(pb["obs_lm"]), P(pb["obs_uv"]), nobs, C.c_double(pb["huber"]), P(res),
                                   P(Ja), P(Jp), P(Jd))
    z = lambda k: torch.zeros(k, dtype=torch.float64, device=DEV)  # noqa: E731
    g_res, g_Ja, g_Jp, g_Jd, g_c = z(2 * nobs), z(12 * nobs), z(12 * nobs), z(2 * nobs), z(nobs)
    gpu_ctx.ba_linearize(20, 3000, nobs, dev(pb["calib"]), dev(pb["poses"]), dev(pb["invd"]), dev(pb["anch_kf"]),
                         dev(pb["anch_uv"]), dev(pb["obs_kf"]), dev(pb["obs_lm"]), dev(pb["obs_uv"]), pb["huber"], g_res, g_Ja,
                         g_Jp, g_Jd, g_c)
    for a, b in ((res, g_res), (Ja, g_Ja), (Jp, g_Jp), (Jd, g_Jd)):
        assert np.allclose(a, b.cpu().numpy(), rtol=1e-10, atol=1e-9)
    assert np.isclose(cost, g_c.sum().item(), rtol=1e-12)


@pytest.mark.parametrize("nkf,nlm,k,seed,huber", [(20, 3000, 4, 42, None), (8, 300, 3, 7, None), (6, 120, 4, 9, 0.0),
                                                  (20, 3000, 4, 43, None), (12, 1000, 5, 5, None)])
def test_solve_vs_oracle(gpu_ctx, oracle, nkf, nlm, k, seed, huber):
    pb = synth.make_ba_problem(nkf, nlm, k, seed=seed)
    wp, wd, ws = oracle_solve(oracle, pb, huber=huber)
    gp, gd, gs = gpu_solve(gpu_ctx, [pb], huber=huber)
    assert (gs[0, 2:5] == ws[2:5]).all(), (gs[0], ws)               # successful steps, iterations, termination
    assert np.allclose(gs[0, :2], ws[:2], rtol=1e-8)
    assert ws[1] < 0.9 * ws[0]
    assert np.allclose(gp[0], wp, rtol=1e-4, atol=1e-9) and np.allclose(gd[0], wd, rtol=1e-4, atol=1e-9)
    assert np.abs(gp[0] - wp).max() < 1e-7 and np.abs(gd[0] - wd).max() < 1e-6


def test_solve_golden_ceres(gpu_ctx):
    g = golden("ba")
    pb = {k: np.ascontiguousarray(g[k]) for k in ("calib", "poses", "pose_const", "invd", "anch_kf", "anch_uv", "obs_kf",
                                                   "obs_lm", "obs_uv")}
    pb["huber"] = float(g["huber"])
    gp, gd, gs = gpu_solve(gpu_ctx, [pb])
    assert (gs[0, 2:5] == g["summary"][2:5]).all()
    assert np.allclose(gs[0, :2], g["summary"][:2], rtol=1e-8)
    assert np.allclose(gp[0], g["poses_out"], rtol=1e-4, atol=1e-9) and np.allclose(gd[0], g["invd_out"], rtol=1e-4, atol=1e-9)


def test_solve_batch_and_padding(gpu_ctx, oracle):
    """Several problems in one call; unused observation slots (obs_lm = -1), a landmark without residuals and a
    keyframe nobody observes must be left untouched."""
    pbs = [synth.make_ba_problem(10, 500, 4, seed=s) for s in (1, 2, 3)]
    for pb in pbs:
        pb["obs_lm"] = np.concatenate([pb["obs_lm"], -np.ones(37, np.int32)])
        pb["obs_kf"] = np.concatenate([pb["obs_kf"], np.zeros(37, np.int32)])
        pb["obs_uv"] = np.concatenate([pb["obs_uv"], np.zeros((37, 2))])
        pb["invd"] = np.concatenate([pb["invd"], [0.25]])                    # landmark 500: no observation
        pb["anch_kf"] = np.concatenate([pb["anch_kf"], np.zeros(1, np.int32)])
        pb["anch_uv"] = np.concatenate([pb["anch_uv"], np.zeros((1, 2))])
        pb["poses"] = np.concatenate([pb["poses"], [[9, 9, 9, 0, 0, 0, 1.0]]])  # keyframe 10: unreferenced, free
        pb["pose_const"] = np.concatenate([pb["pose_const"], np.zeros(1, np.uint8)])
    gp, gd, gs = gpu_solve(gpu_ctx, pbs)
    for i, pb in enumerate(pbs):
        clean = {k: v for k, v in pb.items()}
        m = pb["obs_lm"] >= 0
        clean["obs_lm"], clean["obs_kf"], clean["obs_uv"] = pb["obs_lm"][m], pb["obs_kf"][m], np.ascontiguousarray(pb["obs_uv"][m])
        wp, wd, ws = oracle_solve(oracle, clean)
        assert (gs[i, 2:5] == ws[2:5]).all()
        assert np.allclose(gp[i], wp, rtol=1e-4, atol=1e-9) and np.allclose(gd[i], wd, rtol=1e-4, atol=1e-9)
        assert (gp[i][10] == pb["poses"][10]).all() and gd[i][500] == 0.25
        assert (gp[i][:2] == pb["poses"][:2]).all()                          # the two fixed keyframes


def test_solve_improves_ground_truth_error(gpu_ctx):
    """Property at the BASELINE size (20 KF x 3000 landmarks x 9000 residual obs + 3000 anchors = 12000 observations):
    the robust cost drops and stays finite."""
    pb = synth.make_ba_problem(20, 3000, 4, seed=77)
    gp, gd, gs = gpu_solve(gpu_ctx, [pb])
    assert np.isfinite(gp).all() and np.isfinite(gd).all()
    assert gs[0, 1] < 0.5 * gs[0, 0] and gs[0, 4] in (0.0, 1.0)


def test_solve_dense_schur_tensor_cores(gpu_ctx, oracle):
    """Same solve with the Schur term computed by the FP64 tensor-core SYRK (S -= Wt'Wt, DMMA) instead of atomics."""
    from alvaar_b200 import lib
    L = lib()
    pb = synth.make_ba_problem(20, 3000, 4, seed=42)
    wp, wd, ws = oracle_solve(oracle, pb)
    assert L.alva_set_option(b"ba_dense_schur", 1) == 0
    try:
        gp, gd, gs = gpu_solve(gpu_ctx, [pb, pb])
    finally:
        L.alva_set_option(b"ba_dense_schur", 0)
    for i in range(2):
        assert (gs[i, 2:5] == ws[2:5]).all(), (gs[i], ws)
        assert np.allclose(gp[i], wp, rtol=1e-4, atol=1e-9) and np.allclose(gd[i], wd, rtol=1e-4, atol=1e-9)
        assert np.abs(gp[i] - wp).max() < 1e-7
    assert L.alva_set_option(b"no_such_option", 1) == -1


def test_solve_duplicate_pose_falls_back(gpu_ctx, oracle):
    """A landmark observed twice from the same keyframe (two slots on one pose) is outside what the gather-form Schur
    assembles; the solver must detect it and take the atomic path -- same answer as the oracle."""
    pb = synth.make_ba_problem(8, 200, 3, seed=11)
    # duplicate the first residual observation of 20 landmarks (keeping observations grouped by landmark)
    order = []
    for o in range(len(pb["obs_lm"])):
        order.append(o)
        l = pb["obs_lm"][o]
        if l < 20 and (o == 0 or pb["obs_lm"][o - 1] != l):
            order.append(o)
    order = np.array(order)
    pb["obs_lm"], pb["obs_kf"] = pb["obs_lm"][order], pb["obs_kf"][order]
    uv = pb["obs_uv"][order].copy()
    dup = np.r_[False, order[1:] == order[:-1]]
    uv[dup] += 0.3
    pb["obs_uv"] = np.ascontiguousarray(uv)
    wp, wd, ws = oracle_solve(oracle, pb)
    gp, gd, gs = gpu_solve(gpu_ctx, [pb])
    assert (gs[0, 2:5] == ws[2:5]).all(), (gs[0], ws)
    assert np.allclose(gp[0], wp, rtol=1e-4, atol=1e-9) and np.allclose(gd[0], wd, rtol=1e-4, atol=1e-9)


def oracle_local(oracle, pb, max_iter=5, thr=5.9915):
    poses, invd = pb["poses"].copy(), pb["invd"].copy()
    summary, flags = np.zeros(10), np.zeros(len(pb["obs_kf"]), np.int32)
    oracle.orc_ba_local.restype = C.c_int
    nbad = oracle.orc_ba_local(P(pb["calib"]), P(poses), P(pb["pose_const"]), len(poses), P(invd), P(pb["anch_kf"]),
                               P(pb["anch_uv"]), len(invd), P(pb["obs_kf"]), P(pb["obs_lm"]), P(pb["obs_uv"]),
                               len(pb["obs_kf"]), C.c_double(pb["huber"]), C.c_double(thr), max_iter, P(flags), P(summary))
    return nbad, poses, invd, flags, summary


def gpu_local(ctx, pbs, max_iter=5, thr=5.9915):
    n = len(pbs)
    nkf, nlm, nobs = len(pbs[0]["poses"]), len(pbs[0]["invd"]), len(pbs[0]["obs_kf"])
    st = lambda k: dev(np.stack([p[k] for p in pbs]))  # noqa: E731
    poses, invd, obs_lm = st("poses"), st("invd"), st("obs_lm")
    summary = torch.full((n, 10), -7.0, dtype=torch.float64, device=DEV)
    flags = torch.full((n, nobs), -9, dtype=torch.int32, device=DEV)
    ctx.ba_local(n, nkf, nlm, nobs, st("calib"), poses, st("pose_const"), invd, st("anch_kf"), st("anch_uv"), st("obs_kf"),
                 obs_lm, st("obs_uv"), pbs[0]["huber"], thr, max_iter, flags, summary)
    torch.cuda.synchronize()
    assert (obs_lm.cpu().numpy() == np.stack([p["obs_lm"] for p in pbs])).all()   # the caller's obs_lm is not touched
    return poses.cpu().numpy(), invd.cpu().numpy(), flags.cpu().numpy(), summary.cpu().numpy()


@pytest.mark.parametrize("nkf,nlm,k,seed", [(20, 3000, 4, 42), (8, 300, 3, 7), (12, 800, 5, 3), (10, 400, 3, 11)])
def test_local_ba_vs_oracle(gpu_ctx, oracle, nkf, nlm, k, seed):
    """Optimizer::localBA steps 2-4 on the device: identical outlier sets (both passes), iteration counts and
    termination, solution within the north-star 1e-4 (observed ~1e-9)."""
    pb = synth.make_ba_problem(nkf, nlm, k, seed=seed)
    nb, wp, wd, wf, ws = oracle_local(oracle, pb)
    gp, gd, gf, gs = gpu_local(gpu_ctx, [pb])
    assert nb > 0 and (gf[0] == wf).all()
    assert (gs[0][[2, 3, 4, 7, 8, 9]] == ws[[2, 3, 4, 7, 8, 9]]).all(), (gs[0], ws)
    assert np.allclose(gs[0], ws, rtol=1e-8)
    assert np.allclose(gp[0], wp, rtol=1e-4, atol=1e-9) and np.allclose(gd[0], wd, rtol=1e-4, atol=1e-9)
    assert np.abs(gp[0] - wp).max() < 1e-7 and np.abs(gd[0] - wd).max() < 1e-6


def test_local_ba_golden_ceres(gpu_ctx):
    g = golden("ba_local")
    pb = {k: np.ascontiguousarray(g[k]) for k in ("calib", "poses", "pose_const", "invd", "anch_kf", "anch_uv", "obs_kf",
                                                   "obs_lm", "obs_uv")}
    pb["huber"] = float(g["huber"])
    gp, gd, gf, gs = gpu_local(gpu_ctx, [pb])
    assert (gf[0] == g["flags"]).all() and (g["flags"] == 2).sum() >= 1
    assert (gs[0][[2, 3, 4, 7, 8, 9]] == g["summary"][[2, 3, 4, 7, 8, 9]]).all()
    assert np.allclose(gp[0], g["poses_out"], rtol=1e-4, atol=1e-9) and np.allclose(gd[0], g["invd_out"], rtol=1e-4, atol=1e-9)


def test_local_ba_batch_mixed_skip(gpu_ctx, oracle):
    """A batch where one problem loses no residual: its second solve must be skipped on the device (summary[5:] = 0,
    result = first solve) while its neighbours run theirs."""
    clean = synth.make_ba_problem(8, 300, 3, seed=7, outlier_frac=0.0, noise_px=0.05, pose_noise_t=0.002, pose_noise_r_deg=0.05)
    dirty = [synth.make_ba_problem(8, 300, 3, seed=s) for s in (21, 22)]
    pbs = [dirty[0], clean, dirty[1]]
    n = min(len(p["obs_kf"]) for p in pbs)
    assert all(len(p["obs_kf"]) == n for p in pbs)
    gp, gd, gf, gs = gpu_local(gpu_ctx, pbs)
    for i, pb in enumerate(pbs):
        nb, wp, wd, wf, ws = oracle_local(oracle, pb)
        assert (gf[i] == wf).all() and (gs[i][[2, 3, 4, 7, 8, 9]] == ws[[2, 3, 4, 7, 8, 9]]).all()
        assert np.abs(gp[i] - wp).max() < 1e-7 and np.abs(gd[i] - wd).max() < 1e-6
        if i == 1:
            assert nb == 0 and (gs[i][5:] == 0).all()

