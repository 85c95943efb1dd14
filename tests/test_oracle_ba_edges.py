"""CPU tests for the local-BA edge-shape suite: the problem generator (tests/ba_util.py) builds what it is asked for, and the
FP64 oracle (oracle/ba_oracle.c) is invariant, to 1e-10, under rewrites that leave the problem the same -- keyframe
relabelling with unreferenced padding, observation order, unobserved landmarks.  That is what makes it a fair reference for
tests/test_gpu_ba_edges.py at shapes it has not been pinned to Ceres on.  Where the reference is built in this tree
(oracle/_ref), the oracle is also pinned to ceres::Solve at the widest reduced system (21 free poses, 140 keyframes, tracks
of 20); elsewhere against tests/golden/ba_edges.npz, which tools/make_golden_ba_edges.py writes from the reference."""
import time

import numpy as np
import pytest

import ba_util as B


def _rng_tracks(seed, n, lo, hi):
    return np.random.default_rng(seed).integers(lo, hi + 1, n)


# ------------------------------------------------------------------ generator
@pytest.mark.parametrize("kw", [
    dict(nfree=5, nconst=2, nlm=300, track=3),
    dict(nfree=0, nconst=3, nlm=200, track=2, unref_free=2),
    dict(nfree=21, nconst=2, nlm=400, track=20, tie_frac=0.05, unobserved=17),
    dict(nfree=7, nconst=2, nlm=300, track=_rng_tracks(1, 300, 1, 8), anchor_observer=40, pad=25, unref_const=3),
    dict(nfree=4, nconst=3, nlm=250, track=5, shuffle=True, pad=30, nobs=1400),
])
def test_generator_structure(kw):
    pb = B.make_ba_edge_problem(seed=3, **kw)
    nkf, nlm_all = len(pb["poses"]), len(pb["invd"])
    nref = kw["nfree"] + kw["nconst"]
    track = np.broadcast_to(kw["track"], (kw["nlm"],))
    m = pb["obs_lm"] >= 0
    # exact track lengths, unobserved landmarks without observations and with their distinctive inverse depths
    counts = np.bincount(pb["obs_lm"][m], minlength=nlm_all)
    assert (counts[pb["observed"]] == track).all() and (counts[~pb["observed"]] == 0).all()
    assert (pb["n_obs"] == counts).all() and (~pb["observed"]).sum() == kw.get("unobserved", 0)
    assert (pb["invd"][~pb["observed"]] == 0.25 + 1e-3 * np.arange(kw.get("unobserved", 0))).all()
    # distinct observers; the anchor observes only the anchor = observer landmarks
    lm, kf = pb["obs_lm"][m], pb["obs_kf"][m]
    assert len(np.unique(lm.astype(np.int64) * 1000 + kf)) == m.sum()
    self_obs = np.bincount(lm[kf == pb["anch_kf"][lm]], minlength=nlm_all) > 0
    assert (self_obs == pb["anch_obs"]).all() and pb["anch_obs"].sum() == kw.get("anchor_observer", 0)
    # keyframe roles and counts
    assert pb["free_ref"].sum() == kw["nfree"] and pb["referenced"].sum() == nref
    assert nkf == nref + kw.get("unref_free", 0) + kw.get("unref_const", 0)
    unref = np.flatnonzero(~pb["referenced"])
    assert (pb["poses"][unref] == np.array([B.unref_pose(i) for i in range(len(unref))]).reshape(-1, 7)).all()
    assert (pb["pose_const"][unref] == 0).sum() == kw.get("unref_free", 0)
    # every observed landmark in front of its observers' ground truth: the generator asserts it; constants only in the tie share
    if kw.get("tie_frac", 1.0) < 1:
        n_tie = int(np.ceil(kw["tie_frac"] * kw["nlm"]))
        late = np.flatnonzero(pb["observed"])[n_tie:]
        on_late = np.isin(pb["obs_lm"], late)
        assert pb["free_ref"][pb["obs_kf"][on_late]].all() and pb["free_ref"][pb["anch_kf"][late]].all()
    # order: grouped by landmark (keyframe order inside) unless shuffled; -1 slots interleaved, then the tail up to nobs
    if kw.get("shuffle"):
        assert (np.diff(lm) < 0).any()
    else:
        assert (np.diff(lm) >= 0).all()
        assert (np.diff(kf)[np.diff(lm) == 0] > 0).all()
    n_pad = (~m).sum()
    assert n_pad == kw.get("pad", 0) + (kw["nobs"] - track.sum() - kw.get("pad", 0) if "nobs" in kw else 0)
    if kw.get("pad"):
        first_pad = np.argmin(m)
        assert m[first_pad:].any(), "unused slots must be interleaved, not only appended"
    assert len(pb["obs_lm"]) == kw.get("nobs", track.sum() + kw.get("pad", 0))


def test_generator_index_layout():
    """chosen keyframes at chosen indices: referenced constants and unreferenced keyframes at >= 128, nkf = 256"""
    nfree, nconst, uf, uc = 9, 4, 120, 123
    nkf = nfree + nconst + uf + uc
    rng = np.random.default_rng(0)
    high = rng.permutation(np.arange(128, nkf))
    low = rng.permutation(np.arange(128))
    kf_index = np.empty(nkf, np.int64)
    kf_index[:nconst] = high[:nconst]                                  # referenced constants >= 128
    kf_index[nconst:nconst + 3] = high[nconst:nconst + 3]              # three free referenced >= 128 as well
    kf_index[nconst + 3:nconst + nfree] = low[:nfree - 3]
    rest = np.concatenate([high[nconst + 3:], low[nfree - 3:]])
    kf_index[nconst + nfree:] = rest
    pb = B.make_ba_edge_problem(nfree=nfree, nconst=nconst, nlm=300, track=4, unref_free=uf, unref_const=uc, kf_index=kf_index)
    assert nkf == 256 and len(pb["poses"]) == 256
    assert (pb["pose_const"][kf_index[:nconst]] == 1).all() and pb["referenced"][kf_index[:nconst]].all()
    assert pb["free_ref"][kf_index[nconst:nconst + nfree]].all()
    assert (pb["poses"][kf_index[nconst + nfree:]] == np.array([B.unref_pose(i) for i in range(uf + uc)])).all()
    assert (pb["pose_const"][kf_index[nconst + nfree:]] == np.r_[np.zeros(uf), np.ones(uc)]).all()
    assert set(np.unique(np.r_[pb["obs_kf"], pb["anch_kf"]])) == set(kf_index[:nfree + nconst].tolist())


def test_generator_70k_observations_fast():
    t = time.perf_counter()
    pb = B.make_ba_edge_problem(nfree=21, nconst=2, nlm=3500, track=20, tie_frac=0.05, seed=5)
    dt = time.perf_counter() - t
    assert len(pb["obs_lm"]) == 70000 and dt < 5.0, dt


def test_gather_capacity_arithmetic():
    """ba_prepare sizes the entry buffer 8 nobs + 2 nlm (ecap) and ba_pairs_kernel drops to the atomic path when the lists
    hold more (ba.cu, the total > ecap test).  A uniform all-free track of t observations lists (t + 1)(t + 2) / 2 entries
    against a capacity of 8 t + 2: t = 13 is the last that fits (105 <= 106), t = 14 the first that overflows (120 > 114)."""
    fits = [t for t in range(1, 40) if (t + 1) * (t + 2) // 2 <= 8 * t + 2]
    assert fits == list(range(1, 14))
    for t, ok in ((6, True), (13, True), (14, False), (20, False)):
        pb = B.make_ba_edge_problem(nfree=21, nconst=2, nlm=600, track=t, seed=t, tie_frac=0.05)
        assert (B.gather_entries(pb) <= B.gather_capacity(pb)) == ok and B.takes_gather_path(pb) == ok


# ------------------------------------------------------------------ oracle invariances
def _base():
    return B.make_ba_edge_problem(nfree=7, nconst=2, nlm=400, track=_rng_tracks(2, 400, 1, 6), seed=21)


def _same(a, b, kf_map=None, lm_map=None, obs_perm=None):
    """(poses, invd, summary[, flags]) of a rewritten problem == those of the original, mapped back"""
    pa, da, sa = a[:3]
    pb_, db, sb = b[:3]
    n = len(sa)
    exact = [2, 3, 4] if n == 8 else [2, 3, 4, 7, 8, 9]
    assert (sa[exact] == sb[exact]).all(), (sa, sb)
    assert np.allclose(sa, sb, rtol=1e-10, atol=0)
    pb_ = pb_ if kf_map is None else pb_[kf_map]
    db = db if lm_map is None else db[lm_map]
    assert np.abs(pa - pb_).max() < 1e-10 and np.abs(da - db).max() < 1e-10
    if len(a) > 3:
        fb = b[3] if obs_perm is None else b[3][np.argsort(obs_perm)]
        assert (a[3] == fb).all()


def _runs(oracle, pb):
    p, d, s = B.oracle_solve(oracle, pb)
    nb, lp, ld, lf, ls = B.oracle_local(oracle, pb)
    assert nb > 0
    return (p, d, s), (lp, ld, ls, lf)


def test_oracle_invariant_to_keyframe_relabelling(oracle):
    pb = _base()
    solve0, local0 = _runs(oracle, pb)
    kf_map = np.random.default_rng(4).choice(np.arange(3, 150), len(pb["poses"]), replace=False)
    pr = B.relabel_keyframes(pb, kf_map, 150)
    solve1, local1 = _runs(oracle, pr)
    _same(solve0, solve1, kf_map=kf_map)
    _same(local0, local1, kf_map=kf_map)
    spare = np.setdiff1d(np.arange(150), kf_map)
    for res in (solve1, local1):
        assert (res[0][spare] == pr["poses"][spare]).all()


def test_oracle_invariant_to_observation_order(oracle):
    pb = _base()
    solve0, local0 = _runs(oracle, pb)
    perm = np.random.default_rng(5).permutation(len(pb["obs_lm"]))
    ps = dict(pb)
    ps["obs_lm"], ps["obs_kf"], ps["obs_uv"] = pb["obs_lm"][perm], pb["obs_kf"][perm], np.ascontiguousarray(pb["obs_uv"][perm])
    solve1, local1 = _runs(oracle, ps)
    _same(solve0, solve1)
    _same(local0, local1, obs_perm=perm)


def test_oracle_invariant_to_unobserved_landmarks(oracle):
    pb = _base()
    solve0, local0 = _runs(oracle, pb)
    pu, lm_map = B.add_unobserved_landmarks(pb, 123, seed=6)
    solve1, local1 = _runs(oracle, pu)
    _same(solve0, solve1, lm_map=lm_map)
    _same(local0, local1, lm_map=lm_map)
    fresh = ~pu["observed"]
    for res in (solve1, local1):
        assert (res[1][fresh] == pu["invd"][fresh]).all()


# ------------------------------------------------------------------ the oracle against Ceres at the widest system
def test_oracle_vs_ceres_widest_system(oracle, ref):
    """observed agreement ~2e-14"""
    pb = B.wide_problem()
    assert B.nfree(pb) == 21 and len(pb["poses"]) == 140
    want = B.ceres_outputs(ref, pb)
    p, d, s = B.oracle_solve(oracle, pb)
    sw = want["solve_summary"]
    assert (s[2:5] == sw[2:5]).all(), (s, sw)
    assert np.allclose(s[:2], sw[:2], rtol=1e-9) and s[1] < 0.9 * s[0]
    assert np.abs(p - want["solve_poses"]).max() < 1e-11 and np.abs(d - want["solve_invd"]).max() < 1e-11
    nb, lp, ld, lf, ls = B.oracle_local(oracle, pb)
    lw = want["local_summary"]
    assert nb == int(want["local_nbad"]) and nb > 0 and (lf == want["local_flags"]).all()
    assert (ls[[2, 3, 4, 7, 8, 9]] == lw[[2, 3, 4, 7, 8, 9]]).all() and np.allclose(ls, lw, rtol=1e-9)
    assert np.abs(lp - want["local_poses"]).max() < 1e-11 and np.abs(ld - want["local_invd"]).max() < 1e-11
