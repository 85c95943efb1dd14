"""GPU tests (H100): local BA at its structural edges against the FP64 oracle (oracle/ba_oracle.c).

tests/test_gpu_ba.py covers the reference's own problem shape (synth.make_ba_problem: <= 20 keyframes, an even number of
free poses, short grouped tracks).  This file drives alva_k_ba_solve and alva_k_ba_local through the shapes where the
solver's control flow changes (tests/ba_util.make_ba_edge_problem): every width of the reduced camera system up to its
21-pose maximum and the refusal beyond it, up to 256 keyframes, the gather-form Schur complement's capacity and 16-bit
limits against its FP64-atomic fallback, anchor = observer, unordered observations, 0 and 1 iterations, and batches whose
problems take different paths.

The bar is test_gpu_ba.py's: the integer summary fields equal and the costs to rtol 1e-8, |d pose| < 1e-7, |d invd| < 1e-6,
identical outlier flags, summary[5] = 6 x free poses; constant and unreferenced poses and unobserved inverse depths come
back bit-identical to the input."""
import numpy as np
import pytest
import torch

import ba_util as B
from alvaar_b200 import AlvaError, lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def gpu_solve(ctx, pbs, max_iter=5):
    n = len(pbs)
    nkf, nlm, nobs = len(pbs[0]["poses"]), len(pbs[0]["invd"]), len(pbs[0]["obs_kf"])
    st = lambda k: dev(np.stack([p[k] for p in pbs]))  # noqa: E731
    poses, invd = st("poses"), st("invd")
    summary = torch.full((n, 8), -7.0, dtype=torch.float64, device=DEV)
    ctx.ba_solve(n, nkf, nlm, nobs, st("calib"), poses, st("pose_const"), invd, st("anch_kf"), st("anch_uv"), st("obs_kf"),
                 st("obs_lm"), st("obs_uv"), pbs[0]["huber"], max_iter, summary)
    torch.cuda.synchronize()
    return poses.cpu().numpy(), invd.cpu().numpy(), summary.cpu().numpy()


def gpu_local(ctx, pbs, max_iter=5, thr=B.CHI2):
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


@pytest.fixture
def dense_schur():
    """the tensor-core SYRK form of the Schur term (alva_set_option("ba_dense_schur", 1)) for one test"""
    L = lib()
    assert L.alva_set_option(b"ba_dense_schur", 1) == 0
    yield
    L.alva_set_option(b"ba_dense_schur", 0)


def assert_untouched(pb, gp, gd):
    fixed = ~pb["free_ref"]                                  # constant, and unreferenced free, keyframes
    assert (gp[fixed] == pb["poses"][fixed]).all()
    unobs = ~pb["observed"]
    assert (gd[unobs] == pb["invd"][unobs]).all()


def check_solve(pb, g, w):
    (gp, gd, gs), (wp, wd, ws) = g, w
    assert (gs[2:5] == ws[2:5]).all(), (gs, ws)              # successful steps, iterations, termination
    assert np.allclose(gs[:2], ws[:2], rtol=1e-8), (gs, ws)
    assert gs[5] == 6 * B.nfree(pb)
    assert np.abs(gp - wp).max() < 1e-7 and np.abs(gd - wd).max() < 1e-6
    assert_untouched(pb, gp, gd)


def check_local(pb, g, w):
    (gp, gd, gf, gs), (nb, wp, wd, wf, ws) = g, w
    assert (gf == wf).all(), np.flatnonzero(gf != wf)[:20]
    assert (gs[[2, 3, 4, 7, 8, 9]] == ws[[2, 3, 4, 7, 8, 9]]).all(), (gs, ws)
    assert np.allclose(gs, ws, rtol=1e-8), (gs, ws)
    assert np.abs(gp - wp).max() < 1e-7 and np.abs(gd - wd).max() < 1e-6
    assert_untouched(pb, gp, gd)


def run_both(ctx, oracle, pb, max_iter=5):
    """alva_k_ba_solve and alva_k_ba_local against orc_ba_solve / orc_ba_local; returns the oracle's local result"""
    g = gpu_solve(ctx, [pb], max_iter)
    check_solve(pb, tuple(a[0] for a in g), B.oracle_solve(oracle, pb, max_iter))
    wl = B.oracle_local(oracle, pb, max_iter)
    g = gpu_local(ctx, [pb], max_iter)
    check_local(pb, tuple(a[0] for a in g), wl)
    return wl


def tracks(seed, n, hi):
    return np.random.default_rng(seed).integers(1, hi + 1, n)


# ------------------------------------------------------------------ width of the reduced camera system
# n = 6 nfree: every class of n mod 4 (the right-hand side row shares a 4 x 4 tile with matrix rows when n = 2 mod 4),
# the 126-wide maximum and a structure-only problem (no free pose, n = 0)
@pytest.mark.parametrize("nf", [0, 1, 2, 3, 5, 7, 11, 13, 17, 19, 20, 21])
def test_width(gpu_ctx, oracle, nf):
    pb = B.make_ba_edge_problem(nfree=nf, nconst=2, nlm=600, track=tracks(nf, 600, min(8, nf + 1)), seed=100 + nf)
    assert B.nfree(pb) == nf and B.takes_gather_path(pb)
    nb = run_both(gpu_ctx, oracle, pb)[0]
    assert nb > 0                                            # the second solve of alva_k_ba_local ran too


@pytest.mark.parametrize("nf", [1, 7, 21])
def test_width_dense_schur(gpu_ctx, oracle, dense_schur, nf):
    """the same through the FP64 tensor-core SYRK, with nlm = 1001 (not a multiple of the MMA's k = 4)"""
    pb = B.make_ba_edge_problem(nfree=nf, nconst=2, nlm=1001, track=tracks(nf, 1001, min(6, nf + 1)), seed=200 + nf)
    run_both(gpu_ctx, oracle, pb)


# ------------------------------------------------------------------ more free poses than the solver takes
REFUSED_SOLVE = np.array([0, 0, 0, 0, 2, 0, 1e4, 0])       # costs, steps, iterations, termination, width, radius, iteration
REFUSED_LOCAL = np.array([0, 0, 0, 0, 2] * 2)
# initial poses close to the truth: few observations fail the outlier test at the input, so every free pose keeps some
LOW_NOISE = dict(pose_noise_t=0.001, pose_noise_r_deg=0.01)


def test_refused_beyond_21_free_poses(gpu_ctx, oracle):
    """22 free poses: termination 2, parameters bit-untouched, the documented summary -- also right after a solved problem of
    the same dimensions, whose costs are still in the workspace.  alva_k_ba_local tests the outliers at the untouched input,
    so it loses residuals and runs its second solve on the rest, which still references 22 free poses and is refused too."""
    ok = B.make_ba_edge_problem(nfree=21, nconst=3, nlm=500, track=4, seed=22)
    big = B.make_ba_edge_problem(nfree=22, nconst=2, nlm=500, track=4, seed=23, **LOW_NOISE)
    assert len(ok["poses"]) == len(big["poses"]) and len(ok["obs_lm"]) == len(big["obs_lm"])
    bad = B.outliers_at_input(oracle, big)
    assert bad.sum() > 0 and B.after_removal(big, bad)[0] == 22
    gs_ok = gpu_solve(gpu_ctx, [ok])[2][0]
    assert gs_ok[4] != 2 and gs_ok[0] > 0
    gp, gd, gs = gpu_solve(gpu_ctx, [big])
    assert (gs[0] == REFUSED_SOLVE).all(), gs[0]
    assert (gp[0] == big["poses"]).all() and (gd[0] == big["invd"]).all()
    gl_ok = gpu_local(gpu_ctx, [ok])[3][0]
    assert gl_ok[4] != 2 and gl_ok[0] > 0
    gp, gd, gf, gs = gpu_local(gpu_ctx, [big])
    assert (gs[0] == REFUSED_LOCAL).all(), gs[0]
    assert (gp[0] == big["poses"]).all() and (gd[0] == big["invd"]).all()
    assert (gf[0] == bad.astype(np.int32)).all()


# ------------------------------------------------------------------ more than 128 keyframes
def high_layout(nfree, nconst, nkf, seed):
    """kf_index with the referenced constants, two free poses and as many unreferenced keyframes as fit at indices >= 128"""
    rng = np.random.default_rng(seed)
    high, low = list(rng.permutation(np.arange(128, nkf))), list(rng.permutation(np.arange(min(128, nkf))))
    take = lambda src, n: [src.pop() for _ in range(min(n, len(src)))]  # noqa: E731
    const = take(high, nconst)
    const += take(low, nconst - len(const))
    free = take(high, 2)
    free += take(low, nfree - len(free))
    rest = high + low
    return np.array(const + free + rest)


@pytest.mark.parametrize("nkf", [129, 140, 200, 256])
def test_many_keyframes(gpu_ctx, oracle, nkf):
    nfree, nconst = 9, 3
    nunref = nkf - nfree - nconst
    kf_index = high_layout(nfree, nconst, nkf, seed=nkf)
    pb = B.make_ba_edge_problem(nfree=nfree, nconst=nconst, nlm=400, track=tracks(nkf, 400, 6), seed=nkf,
                                unref_free=nunref // 2, unref_const=nunref - nunref // 2, kf_index=kf_index)
    assert len(pb["poses"]) == nkf and (pb["pose_const"][128:] & pb["referenced"][128:]).any()
    assert nkf == 129 or (pb["free_ref"][128:].any() and (~pb["referenced"][128:]).any())
    run_both(gpu_ctx, oracle, pb)


def test_widest_system_vs_ceres(gpu_ctx):
    """21 free poses among 140 keyframes, tracks of 20 (atomic path), against what ceres::Solve computed for the same problem
    (tests/golden/ba_edges.npz)"""
    pb = B.wide_problem()
    want = B.ceres_outputs(None, pb)
    gp, gd, gs = (a[0] for a in gpu_solve(gpu_ctx, [pb]))
    ws = want["solve_summary"]
    assert (gs[2:5] == ws[2:5]).all() and np.allclose(gs[:2], ws[:2], rtol=1e-8) and gs[5] == 126
    assert np.abs(gp - want["solve_poses"]).max() < 1e-7 and np.abs(gd - want["solve_invd"]).max() < 1e-6
    assert_untouched(pb, gp, gd)
    gp, gd, gf, gs = (a[0] for a in gpu_local(gpu_ctx, [pb]))
    ws = want["local_summary"]
    assert (gf == want["local_flags"]).all()
    assert (gs[[2, 3, 4, 7, 8, 9]] == ws[[2, 3, 4, 7, 8, 9]]).all() and np.allclose(gs, ws, rtol=1e-8)
    assert np.abs(gp - want["local_poses"]).max() < 1e-7 and np.abs(gd - want["local_invd"]).max() < 1e-6
    assert_untouched(pb, gp, gd)


def test_257_keyframes_rejected(gpu_ctx):
    pb = B.make_ba_edge_problem(nfree=4, nconst=2, nlm=100, track=3, seed=257, unref_free=251)
    assert len(pb["poses"]) == 257
    with pytest.raises(AlvaError):
        gpu_solve(gpu_ctx, [pb])
    with pytest.raises(AlvaError):
        gpu_local(gpu_ctx, [pb])


# ------------------------------------------------------------------ gather-form Schur complement: capacity and 16-bit fields
@pytest.mark.parametrize("t", [6, 13, 14, 20])
def test_gather_capacity(gpu_ctx, oracle, t):
    """21 free poses, every landmark seen t times (all-free tracks but for a 5 % share that ties in the constants).  The entry
    buffer holds 8 nobs + 2 nlm entries (ba_prepare) and a track of t free observations plus a free anchor lists
    (t + 1)(t + 2) / 2 of them: t = 13 lists 105 against 106 and still fits, t = 14 lists 120 against 114 and takes the
    atomic path (ba_pairs_kernel's total > ecap test)."""
    pb = B.make_ba_edge_problem(nfree=21, nconst=2, nlm=600, track=t, seed=300 + t, tie_frac=0.05)
    assert B.takes_gather_path(pb) == (t <= 13), (B.gather_entries(pb), B.gather_capacity(pb))
    run_both(gpu_ctx, oracle, pb)


@pytest.mark.parametrize("nobs", [65534, 65535])
def test_obs_index_limit(gpu_ctx, oracle, nobs):
    """observation indices travel in 16 bits (0xffff marks the anchor slot): 65 534 slots is the largest gather problem,
    65 535 the first that falls back"""
    pb = B.make_ba_edge_problem(nfree=6, nconst=2, nlm=21844, track=3, seed=400, nobs=nobs)
    assert B.takes_gather_path(pb) == (nobs == 65534)
    run_both(gpu_ctx, oracle, pb)


@pytest.mark.parametrize("nlm", [65535, 65536])
def test_landmark_index_limit(gpu_ctx, oracle, nlm):
    """landmark indices travel in 16 bits: 65 535 landmarks is the largest gather problem, 65 536 the first that falls back;
    all but 3 000 of them are unobserved, so nobs stays far below its own limit"""
    pb = B.make_ba_edge_problem(nfree=6, nconst=2, nlm=3000, track=3, seed=500, unobserved=nlm - 3000)
    assert len(pb["invd"]) == nlm and B.takes_gather_path(pb) == (nlm == 65535)
    run_both(gpu_ctx, oracle, pb)


# ------------------------------------------------------------------ structure the packed lists cannot express, unordered input
def test_anchor_is_observer(gpu_ctx, oracle):
    """60 landmarks whose anchor keyframe also observes them: two slots on one pose, the atomic Schur path"""
    pb = B.make_ba_edge_problem(nfree=7, nconst=2, nlm=500, track=tracks(7, 500, 6) + 1, seed=600, anchor_observer=60)
    assert pb["anch_obs"].sum() == 60 and not B.takes_gather_path(pb)
    assert_depths_determined(oracle, pb)
    run_both(gpu_ctx, oracle, pb)


def assert_depths_determined(oracle, pb):
    """premise of a comparison that involves anchor = observer landmarks: none of them is left, after alva_k_ba_local's first
    outlier removal, with its anchor's own observation alone -- its depth would then be set by rounding noise (B.after_removal)"""
    flags = B.oracle_local(oracle, pb)[3]
    assert len(B.after_removal(pb, flags == 1)[1]) == 0


def test_shuffled_observations_with_unused_slots(gpu_ctx, oracle):
    """observations in random order with 50 unused slots among them: the landmark -> observation index takes the linear scan"""
    pb = B.make_ba_edge_problem(nfree=7, nconst=2, nlm=500, track=tracks(8, 500, 6), seed=700, shuffle=True, pad=50)
    run_both(gpu_ctx, oracle, pb)


# ------------------------------------------------------------------ iteration count edges
@pytest.mark.parametrize("max_iter", [0, 1])
def test_iteration_edges(gpu_ctx, oracle, max_iter):
    pb = B.make_ba_edge_problem(nfree=5, nconst=2, nlm=500, track=tracks(9, 500, 5), seed=800 + max_iter)
    run_both(gpu_ctx, oracle, pb, max_iter=max_iter)
    gp, gd, gs = gpu_solve(gpu_ctx, [pb], max_iter)
    if max_iter == 0:                                        # no step: the input comes back, with its cost
        assert (gp[0] == pb["poses"]).all() and (gd[0] == pb["invd"]).all()
        assert gs[0][0] == gs[0][1] and np.isclose(gs[0][0], B.oracle_solve(oracle, pb, 0)[2][0], rtol=1e-12)
        assert gs[0][3] == 1 and gs[0][4] == 1


# ------------------------------------------------------------------ one batch, four paths
def mixed_batch():
    """equal dimensions (24 keyframes, 500 landmarks, 7 000 slots), four different paths through the solver"""
    kw = dict(nlm=500, nobs=7000)
    normal = B.make_ba_edge_problem(nfree=10, nconst=2, unref_free=6, unref_const=6, track=4, seed=901, **kw)
    long_tracks = B.make_ba_edge_problem(nfree=21, nconst=2, unref_free=1, track=14, tie_frac=0.05, seed=902, **kw)
    refused = B.make_ba_edge_problem(nfree=22, nconst=2, track=4, seed=903, **LOW_NOISE, **kw)
    anchor_obs = B.make_ba_edge_problem(nfree=8, nconst=2, unref_free=7, unref_const=7, track=5, anchor_observer=50, seed=904,
                                        **kw)
    pbs = [normal, long_tracks, refused, anchor_obs]
    assert [B.takes_gather_path(p) for p in (normal, long_tracks, anchor_obs)] == [True, False, False]
    return pbs


def test_mixed_batch_equals_solo(gpu_ctx, oracle):
    pbs = mixed_batch()
    assert B.after_removal(pbs[2], B.outliers_at_input(oracle, pbs[2]))[0] == 22   # its second solve is refused as well
    assert_depths_determined(oracle, pbs[3])
    for run, ncols in ((gpu_solve, 8), (gpu_local, 10)):
        batch = run(gpu_ctx, pbs)
        for i, pb in enumerate(pbs):
            solo = tuple(a[0] for a in run(gpu_ctx, [pb]))
            got = tuple(a[i] for a in batch)
            if i == 0:                                       # gather path: bit for bit
                assert all((a == b).all() for a, b in zip(got, solo))
            elif i == 2:                                     # refused
                assert (got[0] == pb["poses"]).all() and (got[1] == pb["invd"]).all()
                assert (got[-1] == (REFUSED_SOLVE if ncols == 8 else REFUSED_LOCAL)).all(), got[-1]
            else:                                            # atomic path: FP64 atomics sum in any order
                gs, ss = got[-1], solo[-1]
                exact = [2, 3, 4] if ncols == 8 else [2, 3, 4, 7, 8, 9]
                assert (gs[exact] == ss[exact]).all() and np.allclose(gs, ss, rtol=1e-8)
                assert np.abs(got[0] - solo[0]).max() < 1e-7 and np.abs(got[1] - solo[1]).max() < 1e-6
                if ncols == 10:
                    assert (got[2] == solo[2]).all()
            assert_untouched(pb, got[0], got[1])


# ------------------------------------------------------------------ reproducibility (DESIGN 4.5)
def test_gather_path_bit_reproducible(gpu_ctx):
    """the gather path has no floating-point atomics: the same problem twice gives the same bits"""
    pb = B.make_ba_edge_problem(nfree=13, nconst=2, nlm=1500, track=tracks(10, 1500, 8), seed=1000)
    assert B.takes_gather_path(pb)
    for run in (gpu_solve, gpu_local):
        a, b = run(gpu_ctx, [pb]), run(gpu_ctx, [pb])
        assert all((x == y).all() for x, y in zip(a, b))
