"""GPU parity tests (H100): the map-initialisation kernels (alva_k_essential_5pt, alva_k_triangulate) through the C ABI vs the
CPU oracle and the golden vectors dumped from the reference's own MultiViewGeometry + OpenGV.  Bars as in
tests/test_oracle_init.py: RANSAC model 1e-9 and outlier set exact; refined pose inside the reference's own 1-ulp band and a
cost no worse than the reference's; triangulated points 1e-11 relative."""
import numpy as np
import pytest
import torch

from conftest import golden
from init_util import TAGS, orc_essential, pose_error, refine_cost
from test_oracle_init import spread
from alvaar_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def run(ctx, problems, cap, K32, opt, seed=12345):
    nprob = len(problems)
    b1 = np.zeros((nprob, cap, 3)); b2 = np.zeros((nprob, cap, 3)); cnt = np.zeros(nprob, np.int32)
    for i, (a, b) in enumerate(problems):
        b1[i, :len(a)] = a; b2[i, :len(b)] = b; cnt[i] = len(a)
    Rt = torch.zeros((nprob, 12), dtype=torch.float64, device=DEV)
    out = torch.zeros((nprob, cap), dtype=torch.uint8, device=DEV)
    info = torch.zeros((nprob, 4), dtype=torch.float64, device=DEV)
    ctx.essential_5pt(nprob, cap, dev(b1), dev(b2), dev(cnt), Rt, out, info, max_iter=100, err_px=3.0, optimize=int(opt), fx=float(K32[0]),
                      fy=float(K32[1]), seed=seed)
    torch.cuda.synchronize()
    return Rt.cpu().numpy(), out.cpu().numpy(), info.cpu().numpy()


@pytest.mark.parametrize("opt", [0, 1, 2])
def test_essential_golden_batched(gpu_ctx, opt):
    """the 640x480 golden problems in one batched launch (one CTA per problem).  opt 1: LM on central differences (block-parallel,
    the default of System); opt 2: the reference's own minimiser restated (MINPACK LM on forward differences, lmdif_core.h, one
    thread) -- both inside the reference's own spread"""
    g = golden("init")
    tags = [t for t in TAGS if t != "d"]
    cap = max(len(g[f"{t}_bv1"]) for t in tags)
    Rt, out, info = run(gpu_ctx, [(g[f"{t}_bv1"], g[f"{t}_bv2"]) for t in tags], cap, g["a_K"], opt)
    for i, t in enumerate(tags):
        n = len(g[f"{t}_bv1"])
        assert info[i, 0] == 1 and info[i, 1] == (g[f"{t}_outlier"] == 0).sum()
        assert (out[i, :n] == g[f"{t}_outlier"]).all() and (out[i, n:] == 1).all()
        if not opt:
            assert np.abs(Rt[i] - g[f"{t}_ransac_Rt"]).max() < 1e-9
        else:
            tolR, tolt = spread(g, t)
            dR, dt = pose_error(Rt[i], g[f"{t}_refined_Rt"])
            assert dR < tolR and dt < tolt, (t, dR, dt)
            inl = g[f"{t}_outlier"] == 0
            assert refine_cost(Rt[i], g[f"{t}_bv1"], g[f"{t}_bv2"], inl) <= refine_cost(g[f"{t}_refined_Rt"], g[f"{t}_bv1"], g[f"{t}_bv2"], inl) * (1 + (1e-4 if opt == 1 else 0.5))


def test_essential_1080p_golden_and_oracle(gpu_ctx, oracle):
    g = golden("init")
    n = len(g["d_bv1"])
    Rt, out, info = run(gpu_ctx, [(g["d_bv1"], g["d_bv2"])], n, g["d_K"], False)
    assert (out[0] == g["d_outlier"]).all() and np.abs(Rt[0] - g["d_ransac_Rt"]).max() < 1e-9
    _, _, _, oinfo = orc_essential(oracle, g["d_bv1"], g["d_bv2"], g["d_K"], 0)
    assert info[0, 1] == oinfo[0] and info[0, 2] == oinfo[1] and info[0, 3] == oinfo[2]      # inliers, iterations, draws


def test_essential_against_oracle_seeds(gpu_ctx, oracle):
    """fresh seeded problems, incl. ones that need more than one CHUNK of hypotheses (many outliers) and failing ones"""
    cases = [dict(n=300, seed=41, outlier_frac=0.45), dict(n=80, seed=42, outlier_frac=0.5, noise_px=0.8), dict(n=7, seed=43),
             dict(n=500, seed=44, outlier_frac=0.2), dict(n=40, seed=45, outlier_frac=0.9)]
    prs = [synth.make_twoview_problem(**c) for c in cases]
    K32 = prs[0]["K"].astype(np.float32)
    Rt, out, info = run(gpu_ctx, [(p["bv1"], p["bv2"]) for p in prs], 512, K32, True)
    for i, p in enumerate(prs):
        n = len(p["bv1"])
        ok, Rt_o, o_o, oinfo = orc_essential(oracle, p["bv1"], p["bv2"], K32, 1)
        assert info[i, 0] == ok
        assert info[i, 2] == oinfo[1] and info[i, 3] == oinfo[2]
        if ok:
            assert (out[i, :n] == o_o).all()
            dR, dt = pose_error(Rt[i], Rt_o)
            assert dR < 1e-4 and dt < 1e-3, (i, dR, dt)


def test_triangulate_golden(gpu_ctx):
    g = golden("init")
    n = len(g["tri_points"])
    out = torch.zeros((n, 3), dtype=torch.float64, device=DEV)
    gpu_ctx.triangulate(dev(g["tri_Tlr"]), dev(g["a_bv1"]), dev(g["a_bv2"]), n, out)
    torch.cuda.synchronize()
    assert np.abs(out.cpu().numpy() - g["tri_points"]).max() < 1e-11 * np.abs(g["tri_points"]).max()
