"""Local-BA problems at the solver's structural edges, shared by tests/test_gpu_ba_edges.py, tests/test_oracle_ba_edges.py
and tools/make_golden_ba_edges.py.

`make_ba_edge_problem` builds a problem in the layout of include/alva_b200.h (the same dict as synth.make_ba_problem, which
stays untouched because existing goldens depend on it) with control over what synth.make_ba_problem fixes: the number of
free and constant referenced keyframes, unreferenced keyframes and where every keyframe sits in the index range, the exact
track length of every landmark, landmarks without observations, anchor = observer landmarks, observation order and unused
(-1) slots.  The referenced cameras sit on a short baseline facing a 3-8 m point cloud, so every landmark projects in front
of every camera and any track length up to the number of referenced cameras can be drawn.  Vectorised numpy: a
70 000-observation problem takes well under a second.

Besides the problem arrays the dict carries its structure: `referenced` / `free_ref` [nkf] bool, `observed` [nlm] bool,
`n_obs` [nlm] residuals per landmark, `anch_obs` [nlm] bool (the anchor keyframe also observes the landmark)."""
import ctypes as C
import os

import numpy as np

from alvaar_b200 import synth
from ref_golden import digest

HUBER = float(np.sqrt(5.9915))
CHI2 = 5.9915
PROBLEM_KEYS = ("calib", "poses", "pose_const", "invd", "anch_kf", "anch_uv", "obs_kf", "obs_lm", "obs_uv")
NBMAX = 21   # free referenced poses the device solver takes (csrc/ba.cu: NMAX = 128 columns, 6 per pose)


def unref_pose(i):
    """distinctive pose of the i-th unreferenced keyframe: far from the scene, identity rotation"""
    return np.array([9.0, 9.0, 9.0 + i, 0.0, 0.0, 0.0, 1.0])


def make_ba_edge_problem(nfree=5, nconst=2, nlm=400, track=4, seed=0, unref_free=0, unref_const=0, kf_index=None,
                         unobserved=0, anchor_observer=0, tie_frac=1.0, shuffle=False, pad=0, nobs=None, noise_px=0.5,
                         outlier_frac=0.05, outlier_px=20.0, pose_noise_t=0.01, pose_noise_r_deg=0.2, huber=True, w=1280,
                         h=720):
    """nfree / nconst referenced keyframes (free / fixed), unref_free / unref_const keyframes no observation touches.

    Logical keyframe j -- referenced constants, referenced free, unreferenced free, unreferenced constants, in that order --
    sits at index kf_index[j] (default: j); kf_index must be a permutation of range(nkf).
    nlm observed landmarks with track[l] residual observations each (an int or an [nlm] array), plus `unobserved` landmarks
    without any, inserted at random landmark indices (inverse depth 0.25 + 1e-3 i).  Observers are distinct keyframes other
    than the anchor, except for `anchor_observer` landmarks (a count, or the observed-landmark ordinals) whose anchor keyframe
    is one of their observers.  Only the first ceil(tie_frac * nlm) landmarks may be seen by constant keyframes; the others
    are anchored and observed on free keyframes alone (a track of length t then fills t + 1 slots of the reduced system).
    Observations are grouped by landmark (keyframe order inside a group) unless `shuffle`; `pad` unused slots (obs_lm = -1)
    are interleaved at random positions and, with `nobs`, more are appended up to that many slots."""
    rng = np.random.default_rng(seed)
    nref, nunref = nfree + nconst, unref_free + unref_const
    nkf = nref + nunref
    kf_index = np.arange(nkf) if kf_index is None else np.asarray(kf_index, np.int64)
    assert sorted(kf_index.tolist()) == list(range(nkf)), "kf_index must be a permutation of range(nkf)"
    fx, fy, cx, cy = synth.intrinsics(w, h)
    K_inv = np.array([[1 / fx, 0, -cx / fx], [0, 1 / fy, -cy / fy], [0, 0, 1]])

    # ground-truth referenced cameras: a 0.8 m baseline, every one looking down +z within a few degrees
    j = np.arange(nref)
    xs = np.linspace(-0.4, 0.4, nref) if nref > 1 else np.zeros(1)
    t_gt = np.stack([xs, 0.05 * np.sin(1.7 * j), 0.05 * np.cos(1.3 * j)], 1)
    R_gt = np.stack([synth._rot(0.02 * np.sin(j_), 0.03 * np.cos(0.7 * j_), 0.01 * np.sin(2.1 * j_)) for j_ in range(nref)]) \
        if nref else np.zeros((0, 3, 3))

    # per-landmark pools: tie landmarks may use every referenced camera, the rest the free ones only
    n_tie = nlm if (nfree == 0 or tie_frac >= 1) else int(np.ceil(tie_frac * nlm))
    track = np.broadcast_to(np.asarray(track, np.int64), (nlm,)).copy()
    assert (track >= 1).all(), "an observed landmark needs at least one residual"
    ao = np.zeros(nlm, bool)
    if np.ndim(anchor_observer) == 0:
        if anchor_observer:
            cand = np.flatnonzero(track >= 2)
            ao[rng.choice(cand, int(anchor_observer), replace=False)] = True
    else:
        ao[np.asarray(anchor_observer, np.int64)] = True
    pool = np.zeros((nlm, nref), bool)
    pool[:n_tie] = True
    pool[n_tie:, nconst:] = True
    npool = pool.sum(1)
    assert (track <= npool - 1 + ao).all(), "track longer than the keyframes a landmark can be seen from"
    lm = np.arange(nlm)
    anchor = np.where(lm < n_tie, lm % max(nref, 1), nconst + (lm - n_tie) % max(nfree, 1))
    keys = rng.random((nlm, nref))
    keys[~pool] = 3.0
    keys[lm, anchor] = np.where(ao, -1.0, 2.0)               # anchor = observer: the anchor is always drawn
    sel_rank = np.argsort(keys, 1)
    chosen = np.zeros((nlm, nref), bool)
    np.put_along_axis(chosen, sel_rank, np.arange(nref)[None, :] < track[:, None], 1)

    # landmarks: a pixel in the centre of the anchor image and a depth of 3-8 m
    u = rng.uniform(0.35 * w, 0.65 * w, nlm)
    v = rng.uniform(0.35 * h, 0.65 * h, nlm)
    z = rng.uniform(3.0, 8.0, nlm)
    pc_a = (K_inv @ np.stack([u, v, np.ones(nlm)])).T * z[:, None]
    X = np.einsum("lij,lj->li", R_gt[anchor], pc_a) + t_gt[anchor]
    anch_uv_o = np.stack([u, v], 1) + rng.normal(0, noise_px, (nlm, 2))
    invd_o = 1.0 / (z * (1 + rng.normal(0, 0.02, nlm)))

    # observations, grouped by landmark, keyframe order inside a group
    ol, ok_ = np.nonzero(chosen)
    pc = np.einsum("oji,oj->oi", R_gt[ok_], X[ol] - t_gt[ok_])
    assert (pc[:, 2] > 1.0).all()
    uv = np.stack([fx * pc[:, 0] / pc[:, 2] + cx, fy * pc[:, 1] / pc[:, 2] + cy], 1)
    sig = np.where(rng.random(len(ol)) < outlier_frac, outlier_px, noise_px)
    uv = uv + rng.normal(0, 1, (len(ol), 2)) * sig[:, None]

    # landmark indices with the unobserved ones interleaved
    nlm_all = nlm + unobserved
    unobs_at = np.sort(rng.choice(nlm_all, unobserved, replace=False)) if unobserved else np.zeros(0, np.int64)
    observed = np.ones(nlm_all, bool)
    observed[unobs_at] = False
    lm_id = np.flatnonzero(observed)                         # observed ordinal -> landmark index
    invd = np.zeros(nlm_all)
    invd[lm_id] = invd_o
    invd[unobs_at] = 0.25 + 1e-3 * np.arange(unobserved)
    anch_kf = np.zeros(nlm_all, np.int32)
    anch_kf[lm_id] = kf_index[anchor]
    anch_kf[unobs_at] = kf_index[rng.integers(0, nkf, unobserved)]
    anch_uv = np.zeros((nlm_all, 2))
    anch_uv[lm_id] = anch_uv_o
    anch_uv[unobs_at] = rng.uniform(0, w, (unobserved, 2))

    obs_lm, obs_kf = lm_id[ol].astype(np.int32), kf_index[ok_].astype(np.int32)
    if shuffle:
        p = rng.permutation(len(ol))
        obs_lm, obs_kf, uv = obs_lm[p], obs_kf[p], uv[p]
    n_used = len(ol)
    n_total = n_used + pad if nobs is None else nobs
    assert n_total >= n_used + pad, "nobs below the observations plus the requested padding"
    if pad:   # unused slots at random positions among the observations
        slot = np.sort(rng.choice(n_used + pad, pad, replace=False))
        keep = np.ones(n_used + pad, bool)
        keep[slot] = False
        lm2, kf2, uv2 = np.full(n_used + pad, -1, np.int32), np.zeros(n_used + pad, np.int32), np.zeros((n_used + pad, 2))
        lm2[keep], kf2[keep], uv2[keep] = obs_lm, obs_kf, uv
        obs_lm, obs_kf, uv = lm2, kf2, uv2
    tail = n_total - len(obs_lm)
    obs_lm = np.concatenate([obs_lm, np.full(tail, -1, np.int32)])
    obs_kf = np.concatenate([obs_kf, np.zeros(tail, np.int32)])
    uv = np.concatenate([uv, np.zeros((tail, 2))])

    # poses: referenced ones perturbed (free) or exact (constant), unreferenced ones distinctive
    poses = np.zeros((nkf, 7))
    pose_const = np.zeros(nkf, np.uint8)
    for jj in range(nref):
        R, t = R_gt[jj], t_gt[jj]
        if jj >= nconst:
            R = synth._rot(*np.deg2rad(rng.normal(0, pose_noise_r_deg, 3))) @ R
            t = t + rng.normal(0, pose_noise_t, 3)
        poses[kf_index[jj], :3] = t
        poses[kf_index[jj], 3:] = synth._quat_from_R(R)
        pose_const[kf_index[jj]] = jj < nconst
    for i in range(nunref):
        poses[kf_index[nref + i]] = unref_pose(i)
        pose_const[kf_index[nref + i]] = i >= unref_free

    referenced = np.zeros(nkf, bool)
    referenced[kf_index[:nref]] = True
    got = np.zeros(nkf, bool)
    got[obs_kf[obs_lm >= 0]] = True
    got[anch_kf[observed]] = True
    assert (got == referenced).all(), "some referenced keyframe ended up unreferenced: more landmarks needed"
    n_obs = np.zeros(nlm_all, np.int64)
    n_obs[lm_id] = track
    anch_obs = np.zeros(nlm_all, bool)
    anch_obs[lm_id] = ao
    return dict(calib=np.array([fx, fy, cx, cy]), poses=poses, pose_const=pose_const, invd=invd, anch_kf=anch_kf,
                anch_uv=np.ascontiguousarray(anch_uv), obs_kf=obs_kf, obs_lm=obs_lm, obs_uv=np.ascontiguousarray(uv),
                huber=HUBER if huber else 0.0, referenced=referenced, free_ref=referenced & (pose_const == 0),
                observed=observed, n_obs=n_obs, anch_obs=anch_obs)


def problem_only(pb):
    """the solver's inputs of pb (structure metadata dropped)"""
    return {k: pb[k] for k in PROBLEM_KEYS + ("huber",)}


def nfree(pb):
    return int(pb["free_ref"].sum())


# ------------------------------------------------------------------ gather-form Schur capacity (csrc/ba.cu)
def gather_entries(pb):
    """entries the gather-form Schur complement lists for pb: a landmark whose anchor and observations occupy f slots on
    distinct free poses contributes one entry per unordered slot pair plus one per slot, f (f + 1) / 2
    (ba_pairs_kernel: block (bi, bj >= bi), slot_v >= slot_u on the diagonal)"""
    free = pb["free_ref"]
    m = pb["obs_lm"] >= 0
    f = np.bincount(pb["obs_lm"][m], weights=free[pb["obs_kf"][m]], minlength=len(pb["invd"]))
    f = f + (free[pb["anch_kf"]] & pb["observed"])
    f = f * pb["observed"]
    return int((f * (f + 1) // 2).sum())


def gather_capacity(pb):
    """size of the entry buffer: 8 nobs + 2 nlm (ba_prepare's ecap); more entries send the problem to the atomic path"""
    return 8 * len(pb["obs_lm"]) + 2 * len(pb["invd"])


def takes_gather_path(pb):
    """the conditions under which ba_setup_kernel / ba_pairs_kernel keep a problem on the gather path"""
    return bool(pb["n_obs"].max() < 255 and len(pb["invd"]) < 65536 and len(pb["obs_lm"]) < 65535
                and not pb["anch_obs"].any() and gather_entries(pb) <= gather_capacity(pb))


def after_removal(pb, removed):
    """structure left once the observations `removed` ([nobs] bool) are dropped: (free referenced poses, landmarks whose only
    residuals are their anchor keyframe's own observations).  Such a landmark has no depth information left (the ray through
    its anchor pixel projects to that pixel at every depth), so its inverse depth follows rounding noise."""
    m = (pb["obs_lm"] >= 0) & ~removed
    lm, kf = pb["obs_lm"][m], pb["obs_kf"][m]
    nlm = len(pb["invd"])
    used = np.bincount(lm, minlength=nlm) > 0
    ref = np.zeros(len(pb["poses"]), bool)
    ref[kf] = True
    ref[pb["anch_kf"][used]] = True
    other = np.bincount(lm[kf != pb["anch_kf"][lm]], minlength=nlm)
    return int((ref & (pb["pose_const"] == 0)).sum()), np.flatnonzero(used & (other == 0))


# ------------------------------------------------------------------ structure-preserving rewrites (oracle invariances)
def relabel_keyframes(pb, kf_map, nkf_new, seed=0):
    """keyframe k -> kf_map[k] in a problem of nkf_new keyframes; the new indices no one maps to hold unreferenced
    keyframes (free and constant alternately)"""
    kf_map = np.asarray(kf_map, np.int64)
    out = dict(pb)
    poses = np.zeros((nkf_new, 7))
    pc = np.zeros(nkf_new, np.uint8)
    spare = np.setdiff1d(np.arange(nkf_new), kf_map)
    for i, k in enumerate(spare):
        poses[k] = unref_pose(i)
        pc[k] = i % 2
    poses[kf_map] = pb["poses"]
    pc[kf_map] = pb["pose_const"]
    out["poses"], out["pose_const"] = poses, pc
    out["anch_kf"] = kf_map[pb["anch_kf"]].astype(np.int32)
    out["obs_kf"] = kf_map[pb["obs_kf"]].astype(np.int32)
    for k in ("referenced", "free_ref"):
        a = np.zeros(nkf_new, bool)
        a[kf_map] = pb[k]
        out[k] = a
    return out


def shuffle_observations(pb, seed=0):
    p = np.random.default_rng(seed).permutation(len(pb["obs_lm"]))
    out = dict(pb)
    out["obs_lm"], out["obs_kf"], out["obs_uv"] = pb["obs_lm"][p], pb["obs_kf"][p], np.ascontiguousarray(pb["obs_uv"][p])
    return out


def add_unobserved_landmarks(pb, n, seed=0):
    """n landmarks without observations inserted at random landmark indices; returns (problem, old -> new landmark index)"""
    rng = np.random.default_rng(seed)
    nlm = len(pb["invd"])
    at = np.sort(rng.choice(nlm + n, n, replace=False))
    keep = np.ones(nlm + n, bool)
    keep[at] = False
    lm_map = np.flatnonzero(keep)
    out = dict(pb)
    for k, fill in (("invd", 0.5), ("anch_kf", 0), ("anch_uv", 7.0), ("observed", False), ("n_obs", 0), ("anch_obs", False)):
        a = np.full((nlm + n,) + pb[k].shape[1:], fill, pb[k].dtype)
        a[lm_map] = pb[k]
        out[k] = a
    out["anch_kf"][at] = rng.integers(0, len(pb["poses"]), n)
    m = pb["obs_lm"] >= 0
    out["obs_lm"] = np.where(m, lm_map[np.maximum(pb["obs_lm"], 0)], -1).astype(np.int32)
    return out, lm_map


# ------------------------------------------------------------------ the FP64 oracle (oracle/ba_oracle.c) and its Ceres harness
def oracle_solve(L, pb, max_iter=5, huber=None, prefix="orc"):
    """prefix "orc": the plain-C oracle, "ref": ceres::Solve with the reference's functor.  -> poses, invd, summary[8]"""
    poses, invd = pb["poses"].copy(), pb["invd"].copy()
    summary, costs = np.zeros(8), np.zeros(64)
    fn = getattr(L, prefix + "_ba_solve")
    fn.restype = C.c_int
    P = _P
    fn(P(pb["calib"]), P(poses), P(pb["pose_const"]), len(poses), P(invd), P(pb["anch_kf"]), P(pb["anch_uv"]), len(invd),
       P(pb["obs_kf"]), P(pb["obs_lm"]), P(pb["obs_uv"]), len(pb["obs_kf"]), C.c_double(pb["huber"] if huber is None else huber),
       max_iter, P(summary), P(costs))
    return poses, invd, summary


def oracle_local(L, pb, max_iter=5, thr=CHI2, prefix="orc"):
    """-> nbad, poses, invd, flags, summary[10]"""
    poses, invd = pb["poses"].copy(), pb["invd"].copy()
    summary, flags = np.zeros(10), np.zeros(len(pb["obs_kf"]), np.int32)
    fn = getattr(L, prefix + "_ba_local")
    fn.restype = C.c_int
    P = _P
    nbad = fn(P(pb["calib"]), P(poses), P(pb["pose_const"]), len(poses), P(invd), P(pb["anch_kf"]), P(pb["anch_uv"]), len(invd),
              P(pb["obs_kf"]), P(pb["obs_lm"]), P(pb["obs_uv"]), len(pb["obs_kf"]), C.c_double(pb["huber"]), C.c_double(thr),
              max_iter, P(flags), P(summary))
    return nbad, poses, invd, flags, summary


def outliers_at_input(L, pb, thr=CHI2):
    """observations the outlier test flags at the input point: chi2 = |r|^2 > thr or depth not positive"""
    L.orc_ba_evaluate.restype = C.c_int
    out = np.zeros(len(pb["obs_lm"]), bool)
    r, s = np.zeros(2), np.zeros(1)
    for o in np.flatnonzero(pb["obs_lm"] >= 0):
        l = pb["obs_lm"][o]
        obs = np.array([*pb["obs_uv"][o], *pb["anch_uv"][l]])
        front = L.orc_ba_evaluate(_P(pb["calib"]), _P(np.ascontiguousarray(pb["poses"][pb["anch_kf"][l]])),
                                  _P(np.ascontiguousarray(pb["poses"][pb["obs_kf"][o]])), C.c_double(pb["invd"][l]), _P(obs),
                                  _P(r), None, None, None, _P(s))
        out[o] = s[0] > thr or not front
    return out


# ------------------------------------------------------------------ the widest reduced system, pinned to Ceres
def wide_problem():
    """21 free poses (the widest reduced system, 126 columns) among 140 keyframes, every landmark seen 20 times; referenced
    constants, two free poses and unreferenced keyframes sit at indices >= 128"""
    nfree, nconst, uf, uc = 21, 3, 60, 56
    rng = np.random.default_rng(140)
    high, low = rng.permutation(np.arange(128, 140)), rng.permutation(np.arange(128))
    kf_index = np.concatenate([high[:nconst], high[nconst:nconst + 2], low[:nfree - 2], high[nconst + 2:], low[nfree - 2:]])
    return make_ba_edge_problem(nfree=nfree, nconst=nconst, nlm=500, track=20, seed=140, unref_free=uf, unref_const=uc,
                                kf_index=kf_index, tie_frac=0.1)


def problem_digest(pb):
    return digest(np.concatenate([np.ascontiguousarray(pb[k]).view(np.uint8).ravel() for k in PROBLEM_KEYS]))


def ceres_outputs(ref, pb):
    """ceres::Solve's results for pb (ref_ba_solve, ref_ba_local): live from oracle/_ref when `ref` is loaded, else as
    tools/make_golden_ba_edges.py stored them for wide_problem() in tests/golden/ba_edges.npz"""
    if ref is not None:
        p, d, s = oracle_solve(ref, pb, prefix="ref")
        nb, lp, ld, lf, ls = oracle_local(ref, pb, prefix="ref")
        return dict(solve_poses=p, solve_invd=d, solve_summary=s, local_nbad=np.array(nb), local_poses=lp, local_invd=ld,
                    local_flags=lf, local_summary=ls)
    g = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ba_edges.npz")))
    assert (g["problem_digest"] == problem_digest(pb)).all(), "tests/ba_util.py no longer builds the stored problem"
    return g


def _P(a):
    assert a.flags.c_contiguous
    return a.ctypes.data_as(C.c_void_p)
