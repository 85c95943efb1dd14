"""GPU tests (H100) of the reference's presets (alva_system_set_preset, state.hpp:9-17): the grid detector and the local-map
matcher at the preset cell sizes 35, 45 and 50 against the reference's digests / the CPU oracle, and the System under each preset
against the reference System's trace (tests/golden/system_preset_*.npz, tools/make_golden_presets.py).

Exact: detector output bit for bit at every cell size, matcher maps identical; the System's status codes, track ids in the
reference's order, 3-D flags and counters over all 100 frames given the reference's initialisation (poses then 1e-7).  With its
own initialisation: exact through the initialisation frame, then inside the band of test_gpu_clahe.py (|dt| < 1e-2 of the
baseline, |dq| < 1e-3) with exact status codes."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import P, golden
from detect_util import oracle_detect
from preset_util import PRESETS, match_cell_oracle_lib
from system_util import CAP, frame_slice
from test_gpu_detect import bits, gpu_detect
from alvaar_b200 import AlvaError, System, lib, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DETECT_TAGS = ["c35", "c45", "c50", "c35b"]
NAMES = ["fast", "average", "accurate"]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ------------------------------------------------------------------------------------------------ detector and matcher
@pytest.mark.parametrize("tag", DETECT_TAGS)
def test_detect_grid_at_preset_cells(gpu_ctx, oracle, tag):
    g = golden("detect_presets")
    img, cs = np.ascontiguousarray(g[f"{tag}_img"]), int(g[f"{tag}_cell"])
    roi = [int(v) for v in g[f"{tag}_roi"]]
    out, oi, cnt, q = gpu_detect(gpu_ctx, img[None], cs, [g[f"{tag}_cur"]], roi, 0.001)
    want = g[f"{tag}_pts"]
    assert cnt[0] == len(want) > 0
    assert (bits(out[0, :cnt[0]]) == bits(want)).all()
    pts, ints, qo = oracle_detect(oracle, img, cs, g[f"{tag}_cur"], roi, 0.001)
    assert (oi[0, :cnt[0]] == ints).all() and q[0] == qo


def oracle_match_cell(O, p, order, nkp3d, cell):
    C.c_int.in_dll(O, "orc_match_cell").value = cell
    mk, mm = np.zeros(len(p["kp_id"]) + 1, np.int32), np.zeros(len(p["kp_id"]) + 1, np.int32)
    order = np.ascontiguousarray(order, np.int32)
    n = O.orc_match_to_map_cell(p["w"], p["h"], p["K"][0], p["K"][1], p["K"][2], p["K"][3], P(p["cur_T"]), len(p["kp_id"]), P(p["kp_id"]),
                                P(p["kp_px"]), nkp3d, len(p["kf_id"]), P(p["kf_id"]), P(p["kf_T"]), len(p["mp_id"]), P(p["mp_id"]),
                                P(p["mp_wpt"]), P(p["mp_is3d"]), P(p["obs_start"]), P(p["obs_kf"]), P(p["obs_px"]), P(p["desc_start"]),
                                P(p["desc_kf"]), P(p["desc"]), len(order), P(order), 2.0, 0.2, P(mk), P(mm), None)
    return dict(zip(mk[:n].tolist(), mm[:n].tolist()))


def gpu_match_cell(ctx, p, order, nkp3d, cell):
    idx = {int(i): k for k, i in enumerate(p["mp_id"])}
    kp_mp = np.array([idx.get(int(i), -1) for i in p["kp_id"]], np.int32)
    local_mp = np.array([idx.get(int(i), -1) for i in order], np.int32)
    out = torch.full((len(kp_mp),), -7, dtype=torch.int32, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    ctx.match_to_map(p["w"], p["h"], cell, [float(v) for v in p["K"]], dev(p["cur_T"]), dev(kp_mp), dev(p["kp_px"]), nkp3d, dev(p["kf_T"]),
                     dev(p["mp_wpt"]), dev(p["mp_is3d"]), dev(p["obs_start"]), dev(p["obs_kf"]), dev(p["obs_px"]), dev(p["desc_start"]),
                     dev(p["desc"]), dev(local_mp), out, None, cnt)
    o = out.cpu().numpy()
    assert int(cnt.item()) == int((o >= 0).sum())
    return {int(p["kp_id"][k]): int(p["mp_id"][o[k]]) for k in range(len(o)) if o[k] >= 0}


@pytest.mark.parametrize("cell", [35, 45, 50])
@pytest.mark.parametrize("seed,nkp,nloc,w,h", [(41, 784, 7840, 1280, 720), (42, 1296, 6000, 1920, 1080), (43, 150, 400, 640, 480)])
def test_match_to_map_at_preset_cells(gpu_ctx, seed, nkp, nloc, w, h, cell):
    """C2 / C3-sized maps: alva_k_match_to_map on a frame grid of the preset's cells gives the oracle's map"""
    O = match_cell_oracle_lib()
    p = synth.make_match_problem(seed, w=w, h=h, n_kf=30 if nkp > 200 else 6, n_frame_kp=nkp, n_local=nloc, dup_frac=0.3)
    order = p["local_ids"][np.random.default_rng(seed).permutation(len(p["local_ids"]))]
    for nk in (200, 7):
        want = oracle_match_cell(O, p, order, nk, cell)
        got = gpu_match_cell(gpu_ctx, p, order, nk, cell)
        assert got == want and len(want) > min(20, nkp // 8), (len(got), len(want))
    assert oracle_match_cell(O, p, order, 200, 40) == gpu_match_cell(gpu_ctx, p, order, 200, 40)


# ------------------------------------------------------------------------------------------------ System
def bind():
    L = lib()
    L.alva_system_create.restype = C.c_void_p
    L.alva_system_destroy.argtypes = [C.c_void_p]
    L.alva_system_reset.argtypes = [C.c_void_p]
    L.alva_system_configure.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_double] * 8
    L.alva_system_set_preset.argtypes = [C.c_void_p, C.c_int]
    L.alva_system_set_clahe.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int]
    L.alva_system_set_distortion.argtypes = [C.c_void_p] + [C.c_double] * 4
    L.alva_system_find_camera_pose_ts.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    L.alva_system_get_tracks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.alva_system_get_pose.argtypes = [C.c_void_p, C.c_void_p]
    L.alva_system_get_info.argtypes = [C.c_void_p, C.c_void_p]
    L.alva_system_debug_set_initialisation.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    return L


def step(L, s, frame, t):
    pose = np.zeros(16, np.float32)
    st = L.alva_system_find_camera_pose_ts(s, P(np.ascontiguousarray(frame)), t, P(pose))
    ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3))
    n = L.alva_system_get_tracks(s, P(ids), P(px), P(d3), P(wp), CAP)
    T = np.zeros(7); info = np.zeros(8, np.int32)
    L.alva_system_get_pose(s, P(T)); L.alva_system_get_info(s, P(info))
    return st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy(), wp[:n].copy(), pose


def configured(L, g, preset=None):
    s = C.c_void_p(L.alva_system_create(0))
    K = g["K"]
    assert L.alva_system_configure(s, int(g["w"]), int(g["h"]), K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    if preset is not None:
        assert L.alva_system_set_preset(s, preset) == 0
    return s


def preset_golden(name):
    g = golden(f"system_preset_{name}")
    frames, _ = synth.make_frames(int(g["nframes"]), int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True)
    return g, frames


@pytest.mark.parametrize("name", NAMES)
def test_system_under_preset_follows_the_reference(name):
    g, frames = preset_golden(name)
    L = bind()
    s = configured(L, g, PRESETS[name][0])
    init = int(np.argmax(g["ref_status"] == 1))
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp, pose = step(L, s, frames[k], k * 33.333)
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k], (k, st)
        if k <= init:
            assert (info == g["ref_info"][k]).all(), (k, info, g["ref_info"][k])
            assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
        if k < init:
            assert (px.view(np.uint32) == rpx.view(np.uint32)).all(), k
        else:
            sc = max(1.0, float(np.linalg.norm(g["ref_Twc"][k][:3])))
            assert np.abs(T[:3] - g["ref_Twc"][k][:3]).max() < 1e-2 * sc and min(np.abs(T[3:] - g["ref_Twc"][k][3:]).max(),
                                                                                  np.abs(T[3:] + g["ref_Twc"][k][3:]).max()) < 1e-3, k
    L.alva_system_destroy(s)


@pytest.mark.parametrize("name", NAMES)
def test_system_under_preset_lockstep_given_the_reference_initialisation(name):
    g, frames = preset_golden(name)
    L = bind()
    s = configured(L, g, PRESETS[name][0])
    Rt = np.ascontiguousarray(g["ref_init_Rt"]); outl = np.ascontiguousarray(g["ref_init_outlier"])
    assert L.alva_system_debug_set_initialisation(s, P(Rt), P(outl), len(outl)) == 0
    worst_T = 0.0
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp, pose = step(L, s, frames[k], k * 33.333)
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k] and (info == g["ref_info"][k]).all(), (k, st, info, g["ref_info"][k])
        assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
        worst_T = max(worst_T, float(np.abs(T[:3] - g["ref_Twc"][k][:3]).max()) / max(1.0, float(np.linalg.norm(g["ref_Twc"][k][:3]))),
                      float(min(np.abs(T[3:] - g["ref_Twc"][k][3:]).max(), np.abs(T[3:] + g["ref_Twc"][k][3:]).max())))
        assert np.abs(wp - rwp).max(initial=0) < 1e-6 * max(1.0, np.abs(rwp).max(initial=0)), k
    assert worst_T < 1e-7, worst_T
    L.alva_system_destroy(s)


def plain_frames(n):
    g = golden("system")
    frames, _ = synth.make_frames(n, int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True)
    return g, frames


def run(L, s, frames, t0=0.0):
    return [step(L, s, frames[k], t0 + k * 33.333) for k in range(len(frames))]


def same(a, b):
    return all(x[0] == y[0] and (x[1] == y[1]).all() and (x[3] == y[3]).all() and (x[4].view(np.uint32) == y[4].view(np.uint32)).all()
               and (x[5] == y[5]).all() and (x[6] == y[6]).all() for x, y in zip(a, b))


def test_default_is_bit_identical_to_never_calling_it():
    """ALVA_PRESET_DEFAULT on system.npz: every frame's status, pose, tracks and world points bit for bit as without the call,
    also after a round trip through ACCURATE (its larger buffers stay, its CLAHE switch goes off again)"""
    g, frames = plain_frames(100)
    L = bind()
    a, b, c = configured(L, g), configured(L, g, 0), configured(L, g, 3)
    assert L.alva_system_set_preset(c, 0) == 0
    ra, rb, rc = run(L, a, frames), run(L, b, frames), run(L, c, frames)
    assert same(ra, rb) and same(ra, rc)
    for k in range(len(frames)):
        assert ra[k][0] == g["ref_status"][k]
    for s in (a, b, c):
        L.alva_system_destroy(s)


def test_configure_restores_default_and_reset_keeps_the_preset():
    g, frames = plain_frames(16)
    L = bind()
    K = g["K"]
    a, b = configured(L, g), configured(L, g, 2)
    assert L.alva_system_configure(b, int(g["w"]), int(g["h"]), K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    assert same(run(L, a, frames), run(L, b, frames))
    # reset keeps it: after some frames and a reset, the first frame is detected on AVERAGE's 45-px grid (640 / 45 x 480 / 45 =
    # 14 x 10 detector cells, one keypoint per empty cell), not on DEFAULT's 40-px one (16 x 12).  (reset() keeps the motion model
    # and the detector's adapted quality, as the reference's does, so later frames are not compared with a fresh System's.)
    c = configured(L, g, 2)
    run(L, c, frames[:6])
    assert L.alva_system_reset(c) == 0
    n_avg = len(step(L, c, frames[0], 1000.0)[3])
    e = configured(L, g)
    n_def = len(step(L, e, frames[0], 0.0)[3])
    assert 100 < n_avg <= 14 * 10 < n_def <= 16 * 12, (n_avg, n_def)
    for s in (a, b, c, e):
        L.alva_system_destroy(s)


def test_set_clahe_after_a_preset_overrides_it_and_a_preset_composes_with_distortion():
    g, frames = plain_frames(12)
    L = bind()
    acc, acc_off, avg = configured(L, g, 3), configured(L, g, 3), configured(L, g, 2)
    assert L.alva_system_set_clahe(acc_off, 0, 3.0, 50) == 0
    r_acc, r_off, r_avg = run(L, acc, frames), run(L, acc_off, frames), run(L, avg, frames)
    assert not same(r_acc, r_off)                                   # the preset turned CLAHE on, set_clahe turned it off
    # with CLAHE off, ACCURATE's 35-px grid detects more keypoints on the first frame than AVERAGE's 45-px one
    assert len(r_off[0][3]) > len(r_avg[0][3])
    # composes with the lens model: the preset after set_distortion keeps it, set_distortion after the preset keeps the preset
    D = (-0.05, 0.01, 0.0005, -0.0003)
    p, q = configured(L, g), configured(L, g, 1)
    assert L.alva_system_set_distortion(p, *D) == 0 and L.alva_system_set_preset(p, 1) == 0
    assert L.alva_system_set_distortion(q, *D) == 0
    rp, rq = run(L, p, frames), run(L, q, frames)
    assert same(rp, rq)
    # the lens model is in effect: the keypoints' undistorted positions (getFramePoints) differ from a FAST System without it
    r = configured(L, g, 1)
    run(L, r, frames)
    L.alva_system_get_frame_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    xy_p, xy_r = np.zeros((CAP, 2), np.int32), np.zeros((CAP, 2), np.int32)
    n_p, n_r = L.alva_system_get_frame_points(p, P(xy_p), CAP), L.alva_system_get_frame_points(r, P(xy_r), CAP)
    assert n_p == n_r > 50 and not (xy_p[:n_p] == xy_r[:n_r]).all()
    L.alva_system_destroy(r)
    for s in (acc, acc_off, avg, p, q):
        L.alva_system_destroy(s)


def test_argument_and_state_errors():
    g, frames = plain_frames(1)
    L = bind()
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_preset(s, 1) == -4                    # not configured: ALVA_E_STATE
    L.alva_system_destroy(s)
    assert L.alva_system_set_preset(None, 1) == -1                 # null handle: ALVA_E_INVALID
    s = configured(L, g)
    for bad in (-1, 4, 1000):
        assert L.alva_system_set_preset(s, bad) == -1
    st = step(L, s, frames[0], 0.0)
    assert st[0] == 3 and len(st[3]) > 50                          # a refused preset leaves the handle usable
    L.alva_system_destroy(s)
    sysobj = System(int(g["w"]), int(g["h"]), *g["K"])
    with pytest.raises(ValueError):
        sysobj.set_preset("turbo")
    for name in ("fast", "average", "accurate", "default"):
        sysobj.set_preset(name)
    st, _ = sysobj.find_camera_pose(np.ascontiguousarray(frames[0]), 0.0)
    assert st == 3 and sysobj.info()["keypoints"] > 50
    sysobj.close()
