"""CPU tests of the lens distortion (the reference's CameraCalibration with non-zero k1 k2 p1 p2, camera_calibration.cpp:34-72).

The host side of alvaar_b200/csrc/camera_model.h (what the state machine and, compiled for the device, the kernels run), the
plain-C oracle (oracle/camera_oracle.c) and the reference's own CameraCalibration agree bit for bit on every case of
tests/golden/camera.npz -- live when oracle/_ref/libalva_ref_camera.so is built, else through the stored digests.  With zero
coefficients the radial-tangential path gives the pinhole path's bits.  The host-side System state machine over the CPU oracle
with the lens (tests/host/system_cpu_dist.cpp), given the reference's own initialisation, follows the reference System's
100-frame trace (tests/golden/system_dist.npz, tools/make_golden_distortion.py)."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from camera_util import (CASES, SYSTEM_DIST, case_K, case_pixels, case_points, cdigest, cpu_dist_system_lib, oracle_lib,
                         ref_camera_lib, run_points, run_ref, same_bits)
from conftest import P, golden
from ref_golden import digest
from system_util import CAP, frame_slice
from test_oracle_clahe import ReplayHook

NAMES = [c[0] for c in CASES]


@pytest.mark.parametrize("k", range(len(CASES)), ids=NAMES)
def test_header_oracle_and_reference_agree(k):
    g = golden("camera")
    name, w, h, dist = CASES[k]
    K, D = case_K(k)
    px, X = case_pixels(k), case_points(k)
    assert (digest(px) == g[f"{name}/px"]).all() and (digest(X) == g[f"{name}/X"]).all(), "case generator changed: re-dump camera.npz"
    assert (g[f"{name}/K"] == K).all() and (g[f"{name}/D"] == D).all()
    S, O = cpu_dist_system_lib(), oracle_lib()
    hu, hp = run_points(S.cpu_cam_undistort_points, px, K, D), run_points(S.cpu_cam_project_points, X, K, D)
    ou, op = run_points(O.orc_undistort_points, px, K, D), run_points(O.orc_project_points, X, K, D)
    assert same_bits(hu, ou) and same_bits(hp, op)
    RC = ref_camera_lib()
    if RC is not None:
        ru, rp = run_ref(RC.ref_undistort_points, px, K, D, w, h), run_ref(RC.ref_project_points, X, K, D, w, h)
        assert same_bits(hu, ru), np.argwhere((hu != ru) & ~(np.isnan(hu) & np.isnan(ru)))[:4]
        assert same_bits(hp, rp), np.argwhere((hp != rp) & ~(np.isnan(hp) & np.isnan(rp)))[:4]
    assert (cdigest(hu) == g[f"{name}/unpx"]).all() and (cdigest(hp) == g[f"{name}/uv"]).all()


def test_cases_cover_the_fold_back_and_the_camera_plane():
    g = golden("camera")
    assert int(g["fold_back_640x480/n_fold"]) > 100 and int(g["webcam_640x480/n_fold"]) == 0
    k = NAMES.index("fold_back_640x480")
    K, D = case_K(k)
    px = case_pixels(k)
    S = cpu_dist_system_lib()
    un, pinhole = run_points(S.cpu_cam_undistort_points, px, K, D), run_points(S.cpu_cam_undistort_points, px, K, np.zeros(4))
    x, y = (px[:, 0].astype(np.float64) - K[2]) / K[0], (px[:, 1].astype(np.float64) - K[3]) / K[1]
    fold = 1 + (D[1] * (x * x + y * y) + D[0]) * (x * x + y * y) < 0
    assert (un[fold] == pinhole[fold]).all()                              # the fallback returns the pinhole point
    X = case_points(k)
    assert (X[:, 2] == 0).sum() >= 1000 and (X[:, 2] < 0).sum() >= 1000


@pytest.mark.parametrize("k", range(len(CASES)), ids=NAMES)
def test_zero_coefficients_give_the_pinhole_bits(k):
    """the radial-tangential model with k1 = k2 = p1 = p2 = 0 (camera_model.h) and the state machine's pinhole forms (what runs
    without distortion, unchanged) give the same bits -- at z = 0 both are non-finite, so outside the image either way"""
    S = cpu_dist_system_lib()
    K, _ = case_K(k)
    z = np.zeros(4)
    px, X = case_pixels(k), case_points(k)
    assert same_bits(run_points(S.cpu_radtan_undistort_points, px, K, z), run_points(S.cpu_cam_undistort_points, px, K, z))
    a, b = run_points(S.cpu_radtan_project_points, X, K, z), run_points(S.cpu_cam_project_points, X, K, z)
    front = X[:, 2] != 0
    assert same_bits(a[front], b[front])
    assert not np.isfinite(a[~front]).all(1).any() and not np.isfinite(b[~front]).all(1).any()
    RC = ref_camera_lib()
    if RC is not None:
        name, w, h, _ = CASES[k]
        assert same_bits(run_ref(RC.ref_project_points, X, K, z, w, h), a)


def frames_and_golden():
    from alvaar_b200 import synth
    g = golden("system_dist")
    w, h, nf = int(g["w"]), int(g["h"]), int(g["nframes"])
    assert tuple(g["dist"]) == SYSTEM_DIST
    frames = synth.make_frames(nf, w, h, seed=int(g["seed"]), rgba=True, dist=SYSTEM_DIST)[0]
    assert hashlib.sha256(frames.tobytes()).hexdigest() == str(g["sha256"]), "synthetic frames changed: re-dump the golden"
    return g, frames


def test_pinhole_renderer_is_unchanged():
    """make_frames without a lens is byte for byte the renderer system.npz was recorded with"""
    from alvaar_b200 import synth
    g = golden("system")
    frames, _ = synth.make_frames(int(g["nframes"]), int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True, dist=None)
    assert hashlib.sha256(frames.tobytes()).hexdigest() == str(g["sha256"])


def test_golden_trace_initialises_and_runs_a_local_ba():
    g, frames = frames_and_golden()
    init = int(np.argmax(g["ref_status"] == 1))
    assert (g["ref_status"] == 1).any() and 0 < init
    kf_init = int(g["ref_info"][init][1])
    assert int(g["ref_info"][:, 1].max()) >= kf_init + 2                       # keyframes after the initialisation
    assert init < int(g["first_ba_frame"]) < len(frames)                        # and a local BA
    assert (g["ref_status"][init:] == 1).all()


def run(S, frames, K, dist=SYSTEM_DIST, hook=None):
    s = S.cpu_dist_system_create(frames.shape[2], frames.shape[1], K[0], K[1], K[2], K[3])
    if dist is not None:
        S.cpu_system_set_distortion(s, *dist)
    if hook is not None:
        S.cpu_dist_system_set_essential_hook(s, hook)
    out = []
    for k in range(len(frames)):
        T = np.zeros(7)
        st = S.cpu_dist_system_process(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); info = np.zeros(8, np.int32)
        n = S.cpu_dist_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP)
        xy = np.zeros((CAP, 2), np.int32)
        m = S.cpu_dist_system_frame_points(s, P(xy), CAP)
        S.cpu_dist_system_info(s, P(info))
        out.append((st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy(), wp[:n].copy(), xy[:m].copy()))
    S.cpu_dist_system_destroy(s)
    return out


def test_state_machine_with_distortion_given_the_reference_initialisation(oracle, ref):
    g, frames = frames_and_golden()
    hook = ReplayHook(ref, g)
    tr = run(cpu_dist_system_lib(), frames, g["K"], hook=hook.ptr)
    hook.finish()
    init = int(np.argmax(g["ref_status"] == 1))
    for k, (st, T, info, ids, px, d3, wp, xy) in enumerate(tr):
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k] and (info == g["ref_info"][k]).all(), (k, st, info, g["ref_info"][k])
        assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
        a, b = int(g["ref_xy_start"][k]), int(g["ref_xy_start"][k + 1])
        if k < init:
            assert (px.view(np.uint32) == rpx.view(np.uint32)).all(), k
            assert len(xy) == b - a and (xy == g["ref_xy"][a:b]).all(), k           # getFramePoints: the undistorted positions
        assert np.abs(T - g["ref_Twc"][k]).max() < 1e-9, k
        assert np.abs(wp - rwp).max(initial=0) < 1e-9 * max(1.0, np.abs(rwp).max(initial=0)), k


def test_committed_cpu_trace_is_this_state_machine(oracle):
    """the `cpu_*` trace (its own initialisation) is this very state machine"""
    g, frames = frames_and_golden()
    tr = run(cpu_dist_system_lib(), frames, g["K"])
    for k, (st, T, info, ids, px, d3, wp, xy) in enumerate(tr):
        cids, cpx, cd3, cwp = frame_slice(g, "cpu_", k)
        assert st == g["cpu_status"][k] and (info == g["cpu_info"][k]).all(), k
        assert (ids == cids).all() and (d3 == cd3).all() and (px.view(np.uint32) == cpx.view(np.uint32)).all(), k
        assert np.abs(T - g["cpu_Twc"][k]).max() < 1e-12, k


def test_zero_distortion_is_the_plain_backend(oracle):
    """set to zero, the distortion build is the plain one: the first 20 frames of system.npz's `cpu_*` trace, bit for bit"""
    g = golden("system")
    from alvaar_b200 import synth
    frames, _ = synth.make_frames(20, int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True)
    tr = run(cpu_dist_system_lib(), frames, g["K"], dist=(0.0, 0.0, 0.0, 0.0))
    for k, (st, T, info, ids, px, d3, wp, xy) in enumerate(tr):
        cids, cpx, cd3, cwp = frame_slice(g, "cpu_", k)
        assert st == g["cpu_status"][k] and (ids == cids).all() and (px.view(np.uint32) == cpx.view(np.uint32)).all(), k
        assert (T == g["cpu_Twc"][k]).all(), k


def test_system_switch_error_codes_without_a_device():
    """alva_system_set_distortion before configure -> ALVA_E_STATE; a null handle -> ALVA_E_INVALID"""
    from alvaar_b200 import lib
    L = lib()
    L.alva_system_create.restype = C.c_void_p
    L.alva_system_destroy.argtypes = [C.c_void_p]
    L.alva_system_set_distortion.argtypes = [C.c_void_p] + [C.c_double] * 4
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_distortion(s, *SYSTEM_DIST) == -4
    assert L.alva_system_set_distortion(s, float("nan"), 0, 0, 0) == -4               # the state is checked first
    assert L.alva_system_set_distortion(None, *SYSTEM_DIST) == -1
    L.alva_system_destroy(s)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_match_dist_oracle_without_a_lens_is_the_match_oracle(oracle, seed):
    """orc_match_to_map_dist (oracle/match_dist_oracle.c) with no or all-zero coefficients gives orc_match_to_map's maps (the
    oracle pinned to the reference's Mapper by tests/test_oracle_match.py); with the lens it gives others"""
    from alvaar_b200 import synth
    from match_util import ORC_ARGS, oracle_match
    O = oracle_lib()
    O.orc_match_to_map_dist.argtypes = ORC_ARGS + [C.c_void_p]
    p = synth.make_match_problem(seed, n_frame_kp=150 + 20 * seed, n_local=350 + 50 * seed)
    order = np.ascontiguousarray(p["local_ids"][np.random.default_rng(seed).permutation(len(p["local_ids"]))], np.int32)

    def dist_match(d, nk):
        mk, mm = np.zeros(len(p["kp_id"]) + 1, np.int32), np.zeros(len(p["kp_id"]) + 1, np.int32)
        d4 = None if d is None else np.ascontiguousarray(d, np.float64)
        n = O.orc_match_to_map_dist(p["w"], p["h"], p["K"][0], p["K"][1], p["K"][2], p["K"][3], P(p["cur_T"]), len(p["kp_id"]), P(p["kp_id"]),
                                    P(p["kp_px"]), nk, len(p["kf_id"]), P(p["kf_id"]), P(p["kf_T"]), len(p["mp_id"]), P(p["mp_id"]),
                                    P(p["mp_wpt"]), P(p["mp_is3d"]), P(p["obs_start"]), P(p["obs_kf"]), P(p["obs_px"]), P(p["desc_start"]),
                                    P(p["desc_kf"]), P(p["desc"]), len(order), P(order), 2.0, 0.2, P(mk), P(mm),
                                    None if d4 is None else P(d4))
        return dict(zip(mk[:n].tolist(), mm[:n].tolist()))
    for nk in (100, 10):
        want = oracle_match(oracle, p, order, nk)
        assert dist_match(None, nk) == want and dist_match((0.0, 0.0, 0.0, 0.0), nk) == want and len(want) > 10
        assert dist_match(SYSTEM_DIST, nk) != want
