"""GPU parity tests (H100): batched P3P-LMedS and PnP through the C ABI vs the CPU oracle and the golden vectors dumped
from the reference's own MultiViewGeometry.  fp64: pose within 1e-4 relative (BASELINE north_star; observed ~1e-12),
inlier / outlier sets exact."""
import numpy as np
import pytest
import torch

from conftest import golden
from pose_util import make_pose_problem
from test_oracle_pose import orc_p3p, orc_pnp, HUBER, CHI2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4   # relative, on pose entries of O(1)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def run_p3p(ctx, problems, cap, K32, seed=12345):
    nprob = len(problems)
    bv = np.zeros((nprob, cap, 3)); X = np.zeros((nprob, cap, 3)); cnt = np.zeros(nprob, np.int32)
    for i, (b, x) in enumerate(problems):
        bv[i, :len(b)] = b; X[i, :len(x)] = x; cnt[i] = len(b)
    T = torch.zeros((nprob, 12), dtype=torch.float64, device=DEV)
    out = torch.zeros((nprob, cap), dtype=torch.uint8, device=DEV)
    info = torch.zeros((nprob, 4), dtype=torch.float64, device=DEV)
    ctx.p3p_lmeds(nprob, cap, dev(bv), dev(X), dev(cnt), T, out, info, max_iter=100, err_px=3.0, fx=float(K32[0]), fy=float(K32[1]), seed=seed)
    torch.cuda.synchronize()
    return T.cpu().numpy(), out.cpu().numpy(), info.cpu().numpy()


def run_pnp(ctx, problems, cap, K, rob=True, l2=True, max_iter=5):
    nprob = len(problems)
    uv = np.zeros((nprob, cap, 2)); X = np.zeros((nprob, cap, 3)); cnt = np.zeros(nprob, np.int32); poses = np.zeros((nprob, 7))
    for i, (u, x, p0) in enumerate(problems):
        uv[i, :len(u)] = u; X[i, :len(x)] = x; cnt[i] = len(u); poses[i] = p0
    Kd = np.tile(np.asarray(K, np.float64), (nprob, 1))
    d_pose = dev(poses)
    out = torch.zeros((nprob, cap), dtype=torch.uint8, device=DEV)
    summ = torch.zeros((nprob, 12), dtype=torch.float64, device=DEV)
    ctx.pnp(nprob, cap, dev(Kd), dev(uv), dev(X), dev(cnt), d_pose, out, summ, HUBER, CHI2, max_iter, rob, l2)
    torch.cuda.synchronize()
    return d_pose.cpu().numpy(), out.cpu().numpy(), summ.cpu().numpy()


def test_p3p_lmeds_golden(gpu_ctx):
    g = golden("pose")
    tags = ["a", "b", "c"]
    T, out, info = run_p3p(gpu_ctx, [(g[f"{t}_bv"], g[f"{t}_X"]) for t in tags], 576, g["a_K"])
    for i, t in enumerate(tags):
        n = len(g[f"{t}_bv"])
        assert info[i, 0] == 1 == int(g[f"{t}_p3p_ok"])
        assert (out[i, :n] == g[f"{t}_p3p_outlier"]).all() and (out[i, n:] == 1).all()
        assert np.abs(T[i] - g[f"{t}_p3p_T"]).max() < TOL
        assert info[i, 3] == 100


@pytest.mark.parametrize("rob,l2", [(1, 1), (1, 0), (0, 0)])
def test_pnp_golden(gpu_ctx, rob, l2):
    g = golden("pose")
    tags = ["a", "b", "c"]
    poses, out, summ = run_pnp(gpu_ctx, [(g[f"{t}_uv"], g[f"{t}_X"], g[f"{t}_pose0"]) for t in tags], 600,
                               g["a_K"].astype(np.float64), bool(rob), bool(l2))
    for i, t in enumerate(tags):
        n = len(g[f"{t}_uv"])
        assert summ[i, 10] == 1 == int(g[f"{t}_pnp{rob}{l2}_ok"])
        assert (out[i, :n] == g[f"{t}_pnp{rob}{l2}_outlier"]).all() and (out[i, n:] == 0).all()
        assert np.abs(poses[i] - g[f"{t}_pnp{rob}{l2}_pose"]).max() < TOL


def test_pose_vs_oracle_batch(gpu_ctx, oracle):
    """C3-sized batch: 16 problems of up to 2000 points (ragged), P3P-LMedS then PnP on the P3P inliers, as computePose does."""
    rng = np.random.default_rng(0)
    sizes = [int(x) for x in rng.integers(40, 2000, 16)]
    prs = [make_pose_problem(n, 100 + i, w=1920, h=1080, outlier_frac=0.05 + 0.02 * i) for i, n in enumerate(sizes)]
    K32 = prs[0]["K"].astype(np.float32)
    T, out, info = run_p3p(gpu_ctx, [(p["bv"], p["X"]) for p in prs], 2000, K32)
    pnp_in = []
    for i, p in enumerate(prs):
        ok, To, oo, io = orc_p3p(oracle, p["bv"], p["X"], K32)
        n = sizes[i]
        assert ok == info[i, 0] == 1
        assert (out[i, :n] == oo).all(), (i, int((out[i, :n] != oo).sum()))
        assert np.abs(T[i] - To).max() < TOL
        assert abs(info[i, 2] - io[1]) <= 1e-6 * io[1] + 1e-300
        keep = oo == 0
        # pose from P3P as the initial value (visual_frontend.cpp:326): quaternion of R
        R, t = To.reshape(3, 4)[:, :3], To.reshape(3, 4)[:, 3]
        qw = np.sqrt(max(0.0, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
        q = np.array([(R[2, 1] - R[1, 2]) / (4 * qw), (R[0, 2] - R[2, 0]) / (4 * qw), (R[1, 0] - R[0, 1]) / (4 * qw), qw])
        pnp_in.append((p["uv"][keep], p["X"][keep], np.concatenate([t, q])))
    poses, pout, summ = run_pnp(gpu_ctx, pnp_in, 2000, K32.astype(np.float64))
    for i, (u, x, p0) in enumerate(pnp_in):
        ok, po, oo, so = orc_pnp(oracle, u, x, K32.astype(np.float64), p0)
        assert ok == summ[i, 10] == 1
        assert (pout[i, :len(u)] == oo).all()
        assert np.abs(poses[i] - po).max() < TOL
        assert (summ[i, [3, 4, 8, 9]] == so[[3, 4, 8, 9]]).all()   # same iteration counts / terminations
        # and the refined pose is the generating one to the noise level
        assert np.abs(poses[i][:3] - prs[i]["pose_true"][:3]).max() < 5e-3


def test_pose_edge_cases(gpu_ctx, oracle):
    # fewer than 4 points: p3pRansac returns false; all-outlier PnP leaves the pose untouched
    pr = make_pose_problem(3, 1, outlier_frac=0.0)
    T, out, info = run_p3p(gpu_ctx, [(pr["bv"], pr["X"])], 8, pr["K"].astype(np.float32))
    assert info[0, 0] == 0
    pr = make_pose_problem(50, 2, outlier_frac=0.0)
    bad_uv = pr["uv"] + 500.0
    poses, pout, summ = run_pnp(gpu_ctx, [(bad_uv, pr["X"], pr["pose0"])], 64, pr["K"])
    ok, po, oo, _ = orc_pnp(oracle, bad_uv, pr["X"], pr["K"], pr["pose0"])
    assert ok == summ[0, 10]
    assert (pout[0, :50] == oo).all()
    assert np.abs(poses[0] - po).max() < TOL


def test_p3p_seed_changes_draws_not_result_quality(gpu_ctx):
    """Property at full size: a different sampler seed gives a different best sample but the same inlier set up to
    borderline points (LMedS on 10 % outliers)."""
    pr = make_pose_problem(2000, 7, w=1920, h=1080, outlier_frac=0.1)
    K32 = pr["K"].astype(np.float32)
    _, o1, i1 = run_p3p(gpu_ctx, [(pr["bv"], pr["X"])], 2000, K32, seed=12345)
    _, o2, i2 = run_p3p(gpu_ctx, [(pr["bv"], pr["X"])], 2000, K32, seed=999)
    assert i1[0, 0] == i2[0, 0] == 1
    assert (o1[0] != o2[0]).mean() < 0.1
    assert ((o1[0] == 1) & pr["outlier_true"]).sum() > 0.8 * pr["outlier_true"].sum()
