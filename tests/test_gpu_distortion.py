"""GPU tests (H100) of the lens distortion: alva_k_undistort_points / alva_k_project_points against the host side of
camera_model.h and the reference's digests (tests/golden/camera.npz), alva_k_match_to_map_dist against orc_match_to_map_dist,
and the System with alva_system_set_distortion against the reference System's trace (tests/golden/system_dist.npz).

Exact: both kernels on every case (NaN payloads aside); the matcher's maps; the System's status codes, track ids in the
reference's order, 3-D flags and counters over all 100 frames given the reference's initialisation (poses then 1e-7), and
everything including pixels and getFramePoints up to its own initialisation when free-running."""
import ctypes as C

import numpy as np
import pytest
import torch

from camera_util import (CASES, SYSTEM_DIST, case_K, case_pixels, case_points, cdigest, cpu_dist_system_lib, oracle_lib,
                         run_points, same_bits)
from conftest import P, golden
from match_util import ORC_ARGS
from system_util import CAP, PoseReport, frame_slice, quat_dist
from test_oracle_distortion import NAMES, frames_and_golden
from alvaar_b200 import AlvaError, System, lib, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("k", range(len(CASES)), ids=NAMES)
def test_kernels_are_bit_exact(gpu_ctx, k):
    g = golden("camera")
    name, w, h, dist = CASES[k]
    K, D = case_K(k)
    px, X = case_pixels(k), case_points(k)
    S = cpu_dist_system_lib()
    want_un, want_uv = run_points(S.cpu_radtan_undistort_points, px, K, D), run_points(S.cpu_radtan_project_points, X, K, D)
    d_un = torch.full((len(px), 2), 7.0, dtype=torch.float32, device=DEV)
    gpu_ctx.undistort_points(dev(px), None, 1, len(px), K, D, d_un)
    d_uv = torch.full((len(X), 2), 7.0, dtype=torch.float32, device=DEV)
    gpu_ctx.project_points(dev(X), len(X), K, D, d_uv)
    un, uv = d_un.cpu().numpy(), d_uv.cpu().numpy()
    assert same_bits(un, want_un), np.argwhere(un != want_un)[:4]
    assert same_bits(uv, want_uv), np.argwhere((uv != want_uv) & ~(np.isnan(uv) & np.isnan(want_uv)))[:4]
    assert (cdigest(un) == g[f"{name}/unpx"]).all() and (cdigest(uv) == g[f"{name}/uv"]).all()


def test_undistort_batched_with_counts(gpu_ctx):
    """[nframes][cap] layout: each frame's first counts[f] points, the rest left alone"""
    K, D = case_K(0)
    px = case_pixels(0)[:4 * 3000].reshape(4, 3000, 2)
    counts = np.array([3000, 1234, 0, 2999], np.int32)
    out = torch.full((4, 3000, 2), -5.0, dtype=torch.float32, device=DEV)
    gpu_ctx.undistort_points(dev(px), dev(counts), 4, 3000, K, D, out)
    got = out.cpu().numpy()
    want = run_points(cpu_dist_system_lib().cpu_radtan_undistort_points, np.ascontiguousarray(px.reshape(-1, 2)), K, D).reshape(4, 3000, 2)
    for f in range(4):
        assert (got[f, :counts[f]] == want[f, :counts[f]]).all() and (got[f, counts[f]:] == -5.0).all(), f


def test_kernels_reject_bad_arguments(gpu_ctx):
    K, D = case_K(0)
    px = torch.zeros((8, 2), dtype=torch.float32, device=DEV)
    X = torch.ones((8, 3), dtype=torch.float64, device=DEV)
    out = torch.zeros((8, 2), dtype=torch.float32, device=DEV)
    for KK, DD in ((K, [float("nan"), 0, 0, 0]), (K, [0, float("inf"), 0, 0]), ([0.0, K[1], K[2], K[3]], D), ([K[0], K[1], float("nan"), K[3]], D)):
        with pytest.raises(AlvaError):
            gpu_ctx.undistort_points(px, None, 1, 8, KK, DD, out)
        with pytest.raises(AlvaError):
            gpu_ctx.project_points(X, 8, KK, DD, out)
    for nf, cap in ((0, 8), (1, 0)):
        with pytest.raises(AlvaError):
            gpu_ctx.undistort_points(px, None, nf, cap, K, D, out)
    with pytest.raises(AlvaError):
        gpu_ctx.project_points(X, 0, K, D, out)
    with pytest.raises(AlvaError):
        gpu_ctx.undistort_points(px, None, 1, 7, K, D, out.view(-1)[1:15])    # misaligned float2 output


# ------------------------------------------------------------------------------------------------ local-map matching
def distort_px(px, K, D, w, h):
    """pinhole pixels -> the pixels a lens D shows them at (forward radial-tangential model), kept inside the image"""
    x, y = (px[:, 0] - K[2]) / K[0], (px[:, 1] - K[3]) / K[1]
    r2 = x * x + y * y
    c = 1 + D[0] * r2 + D[1] * r2 * r2
    xd = x * c + 2 * D[2] * x * y + D[3] * (r2 + 2 * x * x)
    yd = y * c + D[2] * (r2 + 2 * y * y) + 2 * D[3] * x * y
    out = np.stack([np.clip(xd * K[0] + K[2], 1.0, w - 2.0), np.clip(yd * K[1] + K[3], 1.0, h - 2.0)], 1)
    return np.ascontiguousarray(out.astype(np.float32))


def oracle_match_dist(O, p, order, nkp3d, dist):
    O.orc_match_to_map_dist.argtypes = ORC_ARGS + [C.c_void_p]
    mk, mm = np.zeros(len(p["kp_id"]) + 1, np.int32), np.zeros(len(p["kp_id"]) + 1, np.int32)
    order = np.ascontiguousarray(order, np.int32)
    d4 = np.ascontiguousarray(dist, np.float64)
    n = O.orc_match_to_map_dist(p["w"], p["h"], p["K"][0], p["K"][1], p["K"][2], p["K"][3], P(p["cur_T"]), len(p["kp_id"]), P(p["kp_id"]),
                                P(p["kp_px"]), nkp3d, len(p["kf_id"]), P(p["kf_id"]), P(p["kf_T"]), len(p["mp_id"]), P(p["mp_id"]),
                                P(p["mp_wpt"]), P(p["mp_is3d"]), P(p["obs_start"]), P(p["obs_kf"]), P(p["obs_px"]), P(p["desc_start"]),
                                P(p["desc_kf"]), P(p["desc"]), len(order), P(order), 2.0, 0.2, P(mk), P(mm), P(d4))
    return dict(zip(mk[:n].tolist(), mm[:n].tolist()))


def gpu_match_dist(ctx, p, order, nkp3d, dist):
    idx = {int(i): k for k, i in enumerate(p["mp_id"])}
    kp_mp = np.array([idx.get(int(i), -1) for i in p["kp_id"]], np.int32)
    local_mp = np.array([idx.get(int(i), -1) for i in order], np.int32)
    out = torch.full((len(kp_mp),), -7, dtype=torch.int32, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    ctx.match_to_map(p["w"], p["h"], 40, [float(v) for v in p["K"]], dev(p["cur_T"]), dev(kp_mp), dev(p["kp_px"]), nkp3d, dev(p["kf_T"]),
                     dev(p["mp_wpt"]), dev(p["mp_is3d"]), dev(p["obs_start"]), dev(p["obs_kf"]), dev(p["obs_px"]), dev(p["desc_start"]),
                     dev(p["desc"]), dev(local_mp), out, None, cnt, dist=dist)
    o = out.cpu().numpy()
    assert int(cnt.item()) == int((o >= 0).sum())
    return {int(p["kp_id"][k]): int(p["mp_id"][o[k]]) for k in range(len(o)) if o[k] >= 0}


@pytest.mark.parametrize("seed,nkp,nloc,w,h", [(31, 576, 5760, 1280, 720), (32, 1296, 6000, 1920, 1080), (33, 150, 400, 640, 480)])
def test_match_to_map_dist_vs_oracle(gpu_ctx, seed, nkp, nloc, w, h):
    """C2 / C3-sized maps seen through the lens: the keypoints' and observations' pixels are where the lens puts them, so
    matching needs the distorted projections; without them (the pinhole matcher) fewer keypoints match"""
    O = oracle_lib()
    p = synth.make_match_problem(seed, w=w, h=h, n_kf=30 if nkp > 200 else 6, n_frame_kp=nkp, n_local=nloc, dup_frac=0.3)
    p["kp_px"] = distort_px(p["kp_px"].astype(np.float64), p["K"], SYSTEM_DIST, w, h)
    p["obs_px"] = distort_px(p["obs_px"].astype(np.float64), p["K"], SYSTEM_DIST, w, h)
    order = p["local_ids"][np.random.default_rng(seed).permutation(len(p["local_ids"]))]
    for nk in (200, 7):
        want = oracle_match_dist(O, p, order, nk, SYSTEM_DIST)
        got = gpu_match_dist(gpu_ctx, p, order, nk, SYSTEM_DIST)
        assert got == want and len(want) > min(20, nkp // 8), (len(got), len(want))
        assert gpu_match_dist(gpu_ctx, p, order, nk, (0.0, 0.0, 0.0, 0.0)) == oracle_match_dist(O, p, order, nk, (0.0, 0.0, 0.0, 0.0))
    assert len(gpu_match_dist(gpu_ctx, p, order, 200, (0.0, 0.0, 0.0, 0.0))) < len(gpu_match_dist(gpu_ctx, p, order, 200, SYSTEM_DIST))
    with pytest.raises(AlvaError):
        gpu_match_dist(gpu_ctx, p, order, 200, (float("nan"), 0.0, 0.0, 0.0))


# ------------------------------------------------------------------------------------------------ System
def bind():
    L = lib()
    L.alva_system_create.restype = C.c_void_p
    L.alva_system_destroy.argtypes = [C.c_void_p]
    L.alva_system_reset.argtypes = [C.c_void_p]
    L.alva_system_configure.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_double] * 8
    L.alva_system_set_distortion.argtypes = [C.c_void_p] + [C.c_double] * 4
    L.alva_system_find_camera_pose_ts.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    L.alva_system_get_tracks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.alva_system_get_frame_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.alva_system_get_pose.argtypes = [C.c_void_p, C.c_void_p]
    L.alva_system_get_info.argtypes = [C.c_void_p, C.c_void_p]
    L.alva_system_debug_set_initialisation.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    return L


def step(L, s, frame, t):
    pose = np.zeros(16, np.float32)
    st = L.alva_system_find_camera_pose_ts(s, P(np.ascontiguousarray(frame)), t, P(pose))
    ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3))
    n = L.alva_system_get_tracks(s, P(ids), P(px), P(d3), P(wp), CAP)
    xy = np.zeros((CAP, 2), np.int32)
    m = L.alva_system_get_frame_points(s, P(xy), CAP)
    T = np.zeros(7); info = np.zeros(8, np.int32)
    L.alva_system_get_pose(s, P(T)); L.alva_system_get_info(s, P(info))
    return st, T, info, ids[:n], px[:n], d3[:n], wp[:n], pose, xy[:m]


def configured(L, g, dist=SYSTEM_DIST):
    s = C.c_void_p(L.alva_system_create(0))
    K = g["K"]
    assert L.alva_system_configure(s, int(g["w"]), int(g["h"]), K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    if dist is not None:
        assert L.alva_system_set_distortion(s, *dist) == 0
    return s


def ref_xy(g, k):
    a, b = int(g["ref_xy_start"][k]), int(g["ref_xy_start"][k + 1])
    return g["ref_xy"][a:b]


def test_system_with_distortion_lockstep_given_the_reference_initialisation():
    g, frames = frames_and_golden()
    L = bind()
    s = configured(L, g)
    Rt = np.ascontiguousarray(g["ref_init_Rt"]); outl = np.ascontiguousarray(g["ref_init_outlier"])
    assert L.alva_system_debug_set_initialisation(s, P(Rt), P(outl), len(outl)) == 0
    worst_T = worst_px = 0.0
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp, pose, xy = step(L, s, frames[k], k * 33.333)
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k] and (info == g["ref_info"][k]).all(), (k, st, info)
        assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
        assert len(xy) == len(ref_xy(g, k)), k
        worst_px = max(worst_px, float(np.abs(px - rpx).max(initial=0)))
        worst_T = max(worst_T, float(np.abs(T[:3] - g["ref_Twc"][k][:3]).max()) / max(1.0, float(np.linalg.norm(g["ref_Twc"][k][:3]))),
                      quat_dist(T[3:], g["ref_Twc"][k][3:]))
        assert np.abs(wp - rwp).max(initial=0) < 1e-6 * max(1.0, np.abs(rwp).max(initial=0)), k
    assert worst_T < 1e-7 and worst_px < 1e-3, (worst_T, worst_px)
    L.alva_system_destroy(s)


def test_system_with_distortion_follows_the_reference():
    """Free-running (its own initialisation): every field exact through the initialisation frame -- pixels, getFramePoints and
    the API pose bit for bit before it.  After it the five-point refinement is noise-limited (DESIGN 4.11): the status stays
    exact and the pose inside system_util.PoseReport's band (1e-4, or 10x the reference's own 1-ulp spread on this trace)."""
    g, frames = frames_and_golden()
    L = bind()
    s = configured(L, g)
    init = int(np.argmax(g["ref_status"] == 1))
    rep = PoseReport("System with lens distortion on the GPU vs the reference System, free-running")
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp, pose, xy = step(L, s, frames[k], k * 33.333)
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k], (k, st)
        if k <= init:
            assert (info == g["ref_info"][k]).all(), (k, info, g["ref_info"][k])
            assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
            assert len(xy) == len(ref_xy(g, k)), k
        if k < init:
            assert (px.view(np.uint32) == rpx.view(np.uint32)).all(), k
            assert (xy == ref_xy(g, k)).all(), k
            assert (pose == g["ref_pose16"][k]).all(), k
        else:
            rep.check(g, k, T)
    print(rep.summary(g))
    L.alva_system_destroy(s)


def test_without_the_lens_model_the_undistorted_points_differ():
    """negative control: the same frames on a pinhole System give other getFramePoints than the reference before its
    initialisation (the keypoints themselves are the same: the detector and KLT see the same pixels)"""
    g, frames = frames_and_golden()
    L = bind()
    s = configured(L, g, dist=None)
    init = int(np.argmax(g["ref_status"] == 1))
    seen = 0
    for k in range(init):
        st, T, info, ids, px, d3, wp, pose, xy = step(L, s, frames[k], k * 33.333)
        if st != 3:   # the pinhole System's own initialisation: the frames are no longer comparable
            break
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert (ids == rids).all() and (px.view(np.uint32) == rpx.view(np.uint32)).all(), k
        assert len(xy) != len(ref_xy(g, k)) or (xy != ref_xy(g, k)).any(), k
        seen += 1
    assert seen >= 3, seen
    L.alva_system_destroy(s)


def plain_frames(n=None):
    g = golden("system")
    frames, _ = synth.make_frames(n or int(g["nframes"]), int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True)
    return g, frames


def test_zero_distortion_is_bit_identical_to_never_setting_it():
    g, frames = plain_frames()
    L = bind()
    a, b = configured(L, g, dist=None), configured(L, g, dist=(0.0, 0.0, 0.0, 0.0))
    for k in range(len(frames)):
        ra, rb = step(L, a, frames[k], k * 33.333), step(L, b, frames[k], k * 33.333)
        assert ra[0] == rb[0] and (ra[2] == rb[2]).all() and (ra[3] == rb[3]).all() and (ra[5] == rb[5]).all(), k
        assert (ra[4].view(np.uint32) == rb[4].view(np.uint32)).all() and (ra[8] == rb[8]).all(), k
        assert (ra[1] == rb[1]).all() and (ra[7] == rb[7]).all(), k
    L.alva_system_destroy(a); L.alva_system_destroy(b)


def test_configure_clears_reset_keeps_and_a_change_restarts_the_tracker():
    g, frames = frames_and_golden()
    L = bind()
    K = g["K"]
    # configure clears it: a System configured again tracks like one that never had it
    gp, plain = plain_frames(4)
    a, b = configured(L, gp, dist=None), configured(L, gp)
    assert L.alva_system_configure(b, int(gp["w"]), int(gp["h"]), K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    for k in range(4):
        ra, rb = step(L, a, plain[k], k * 33.3), step(L, b, plain[k], k * 33.3)
        assert (ra[3] == rb[3]).all() and (ra[4].view(np.uint32) == rb[4].view(np.uint32)).all() and (ra[8] == rb[8]).all(), k
    L.alva_system_destroy(a); L.alva_system_destroy(b)
    # reset keeps it: after a reset the undistorted positions are still the lens model's
    s = configured(L, g)
    for k in range(3):
        step(L, s, frames[k], k * 33.3)
    assert L.alva_system_reset(s) == 0
    st, T, info, ids, px, d3, wp, pose, xy = step(L, s, frames[0], 200.0)
    assert st == 3 and len(xy) == len(px) > 100
    un = run_points(cpu_dist_system_lib().cpu_radtan_undistort_points, np.ascontiguousarray(px), np.array(K), np.array(SYSTEM_DIST))
    assert (xy == un.astype(np.int32)).all()
    L.alva_system_destroy(s)
    # a change mid-stream restarts the tracker and the map: status 3, a first frame with one keyframe
    s = configured(L, g)
    init = int(np.argmax(g["ref_status"] == 1))
    for k in range(init + 3):
        r = step(L, s, frames[k], k * 33.333)
    assert r[0] == 1
    assert L.alva_system_set_distortion(s, -0.2, 0.05, 0.0, 0.0) == 0
    st, T, info, ids, px, d3, wp, pose, xy = step(L, s, frames[init + 3], (init + 3) * 33.333)
    assert st == 3 and info[0] == 0 and info[5] == 1 and not d3.any()
    L.alva_system_destroy(s)


def test_switch_argument_checks():
    g, frames = frames_and_golden()
    L = bind()
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_distortion(s, *SYSTEM_DIST) == -4                  # not configured: ALVA_E_STATE
    L.alva_system_destroy(s)
    s = configured(L, g, dist=None)
    for bad in ((float("nan"), 0, 0, 0), (0, float("inf"), 0, 0), (0, 0, float("-inf"), 0), (0, 0, 0, float("nan"))):
        assert L.alva_system_set_distortion(s, *bad) == -1
    assert L.alva_system_set_distortion(None, *SYSTEM_DIST) == -1
    L.alva_system_destroy(s)
    sysobj = System(int(g["w"]), int(g["h"]), *g["K"])
    with pytest.raises(AlvaError):
        sysobj.set_distortion(float("nan"), 0, 0, 0)
    sysobj.set_distortion(*SYSTEM_DIST)
    st, _ = sysobj.find_camera_pose(np.ascontiguousarray(frames[0]), 0.0)
    assert st == 3 and (sysobj.frame_points() == ref_xy(g, 0)).all()
    sysobj.close()
