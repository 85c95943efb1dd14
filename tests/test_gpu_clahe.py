"""GPU tests (H100) of the CLAHE pre-processing: alva_k_clahe against orc_clahe and the reference's digests
(tests/golden/clahe.npz), and the System with CLAHE on against the reference System's trace (tests/golden/system_clahe.npz).

Exact: the kernel's output on every case, run to run and in place; the System's status codes, track ids in the reference's
order, 3-D flags and counters over all 100 frames given the reference's initialisation (poses then 1e-7), pixel positions bit
for bit before the initialisation.  With its own initialisation, see test_system_with_clahe_follows_the_reference."""
import ctypes as C

import numpy as np
import pytest

from clahe_util import CASES
from conftest import P, golden
from ref_golden import digest
from system_util import CAP, frame_slice
from test_oracle_clahe import NAMES, frames_and_golden, run_orc
from alvaar_b200 import AlvaError, System, lib, synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k", range(len(CASES)), ids=NAMES)
def test_kernel_is_bit_exact(gpu_ctx, k):
    import torch
    g = golden("clahe")
    name, w, h, n, clip, tx, ty, kind = CASES[k]
    x, want = run_orc(k)
    d_in = torch.from_numpy(x).cuda()
    d_out = torch.zeros_like(d_in)
    gpu_ctx.clahe(d_in, d_out, w, h, n, clip, tx, ty)
    got = d_out.cpu().numpy()
    bad = np.argwhere(got != want)
    assert len(bad) == 0, f"{len(bad)} pixels differ from orc_clahe, first {bad[:4].tolist()}"
    assert (digest(got) == g[f"{name}/out"]).all()
    d_out2 = torch.full_like(d_in, 7)
    gpu_ctx.clahe(d_in, d_out2, w, h, n, clip, tx, ty)                   # run to run
    assert torch.equal(d_out, d_out2)
    gpu_ctx.clahe(d_in, d_in, w, h, n, clip, tx, ty)                     # in place
    assert torch.equal(d_in, d_out)


def test_kernel_rejects_bad_arguments(gpu_ctx):
    import torch
    x = torch.zeros((1, 48, 64), dtype=torch.uint8, device="cuda")
    for clip, tx, ty in ((3.0, 0, 4), (3.0, 4, 0), (3.0, 65, 4), (3.0, 4, 49), (-1.0, 4, 4), (float("nan"), 4, 4)):
        with pytest.raises(AlvaError):
            gpu_ctx.clahe(x, x, 64, 48, 1, clip, tx, ty)


def bind():
    L = lib()
    L.alva_system_create.restype = C.c_void_p
    L.alva_system_destroy.argtypes = [C.c_void_p]
    L.alva_system_reset.argtypes = [C.c_void_p]
    L.alva_system_configure.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_double] * 8
    L.alva_system_set_clahe.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int]
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
    return st, T, info, ids[:n], px[:n], d3[:n], wp[:n], pose


def configured(L, g, clahe=True):
    s = C.c_void_p(L.alva_system_create(0))
    K = g["K"]
    assert L.alva_system_configure(s, int(g["w"]), int(g["h"]), K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    if clahe:
        assert L.alva_system_set_clahe(s, 1, 3.0, 50) == 0                # the ACCURATE preset's setting, as in system_clahe.npz
    return s


def test_system_with_clahe_follows_the_reference():
    """Free-running (its own initialisation): every field exact through the initialisation frame, pixels bit for bit before it.
    After it the five-point refinement is noise-limited (DESIGN 4.11): on this trace the device's result ends ~7e-4 of the
    baseline away from the CPU build's and, ten frames later, one keypoint's gate decides differently -- so from there on the
    status is exact and the pose stays inside the band |dt| < 1e-2 of the baseline, |dq| < 1e-3.  The lockstep test below pins
    everything downstream of the initialisation exactly, with the reference's initialisation plugged in."""
    g, frames = frames_and_golden()
    L = bind()
    s = configured(L, g)
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
            assert (pose == g["ref_pose16"][k]).all()
        else:
            sc = max(1.0, float(np.linalg.norm(g["ref_Twc"][k][:3])))
            assert np.abs(T[:3] - g["ref_Twc"][k][:3]).max() < 1e-2 * sc and min(np.abs(T[3:] - g["ref_Twc"][k][3:]).max(),
                                                                                  np.abs(T[3:] + g["ref_Twc"][k][3:]).max()) < 1e-3, k
    L.alva_system_destroy(s)


def test_system_with_clahe_lockstep_given_the_reference_initialisation():
    g, frames = frames_and_golden()
    L = bind()
    s = configured(L, g)
    Rt = np.ascontiguousarray(g["ref_init_Rt"]); outl = np.ascontiguousarray(g["ref_init_outlier"])
    assert L.alva_system_debug_set_initialisation(s, P(Rt), P(outl), len(outl)) == 0
    worst_T = worst_px = 0.0
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp, pose = step(L, s, frames[k], k * 33.333)
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k] and (info == g["ref_info"][k]).all(), (k, st, info)
        assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
        worst_px = max(worst_px, float(np.abs(px - rpx).max(initial=0)))
        worst_T = max(worst_T, float(np.abs(T[:3] - g["ref_Twc"][k][:3]).max()) / max(1.0, float(np.linalg.norm(g["ref_Twc"][k][:3]))),
                      float(min(np.abs(T[3:] - g["ref_Twc"][k][3:]).max(), np.abs(T[3:] + g["ref_Twc"][k][3:]).max())))
        assert np.abs(wp - rwp).max(initial=0) < 1e-6 * max(1.0, np.abs(rwp).max(initial=0)), k
    assert worst_T < 1e-7 and worst_px < 1e-3, (worst_T, worst_px)
    L.alva_system_destroy(s)


def plain_frames(n):
    g = golden("system")
    frames, _ = synth.make_frames(n, int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True)
    return g, frames


def test_switch_default_off_and_configure_turns_it_off():
    """a new System, and a System configured again after CLAHE was on, track system.npz's frames exactly as without CLAHE"""
    g, frames = plain_frames(4)
    L = bind()
    a = configured(L, g, clahe=False)
    b = configured(L, g, clahe=True)
    K = g["K"]
    assert L.alva_system_configure(b, int(g["w"]), int(g["h"]), K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    for k in range(4):
        for s in (a, b):
            st, T, info, ids, px, d3, wp, pose = step(L, s, frames[k], k * 33.333)
            rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
            assert st == g["ref_status"][k] and (ids == rids).all() and (px.view(np.uint32) == rpx.view(np.uint32)).all(), k
    L.alva_system_destroy(a); L.alva_system_destroy(b)


def test_switch_reset_keeps_it_and_it_applies_from_the_next_frame():
    # on from the next frame: switched on after frame 2 of an unequalised run (system.npz's frames), frame 3 is tracked on
    # equalised images -- against the raw images of frame 2 most tracks are lost
    gp, plain = plain_frames(5)
    L = bind()
    on, off = configured(L, gp, clahe=False), configured(L, gp, clahe=False)
    for k in range(3):
        ra, rb = step(L, on, plain[k], k * 33.3), step(L, off, plain[k], k * 33.3)
        assert len(ra[3]) > 100 and (ra[4] == rb[4]).all()
    assert L.alva_system_set_clahe(on, 1, 3.0, 50) == 0
    ra, rb = step(L, on, plain[3], 100.0), step(L, off, plain[3], 100.0)
    assert len(ra[3]) != len(rb[3]) or not (ra[4] == rb[4]).all()
    assert L.alva_system_set_clahe(on, 0, 3.0, 50) == 0                    # and off again: the plain graphs are still valid
    ra, rb = step(L, on, plain[4], 133.3), step(L, off, plain[4], 133.3)
    assert ra[0] in (1, 2, 3) and np.isfinite(ra[1]).all()
    L.alva_system_destroy(on); L.alva_system_destroy(off)
    g, frames = frames_and_golden()
    # reset keeps it: after a reset the first frame is detected on the equalised image
    a, b = configured(L, g, clahe=True), configured(L, g, clahe=True)
    for s in (a, b):
        for k in range(3):
            step(L, s, frames[k], k * 33.3)
        assert L.alva_system_reset(s) == 0
    assert L.alva_system_set_clahe(b, 0, 3.0, 50) == 0
    ra, rb = step(L, a, frames[0], 200.0), step(L, b, frames[0], 200.0)
    assert ra[0] == 3 and rb[0] == 3
    assert len(ra[3]) != len(rb[3]) or not (ra[4] == rb[4]).all()
    c = configured(L, g, clahe=True)
    for k in range(3):
        step(L, c, frames[k], k * 33.3)
    assert L.alva_system_reset(c) == 0
    rc = step(L, c, frames[0], 200.0)
    assert (rc[3] == ra[3]).all() and (rc[4] == ra[4]).all()              # deterministic
    for s in (a, b, c):
        L.alva_system_destroy(s)


def test_switch_argument_checks():
    g, frames = frames_and_golden()
    L = bind()
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_clahe(s, 1, 3.0, 50) == -4                    # not configured: ALVA_E_STATE
    L.alva_system_destroy(s)
    s = configured(L, g, clahe=False)
    assert L.alva_system_set_clahe(s, 1, 3.0, 481) == -1                   # 640x480 / 481: an empty grid
    assert L.alva_system_set_clahe(s, 1, 3.0, 0) == -1
    assert L.alva_system_set_clahe(s, 1, -1.0, 50) == -1
    assert L.alva_system_set_clahe(s, 1, 3.0, 480) == 0                    # a 1x1 grid
    L.alva_system_destroy(s)
    sysobj = System(int(g["w"]), int(g["h"]), *g["K"])
    with pytest.raises(AlvaError):
        sysobj.set_clahe(True, 3.0, 1000)
    sysobj.set_clahe(True)
    st, _ = sysobj.find_camera_pose(np.ascontiguousarray(frames[0]), 0.0)
    assert st == 3 and sysobj.info()["keypoints"] > 50
    sysobj.close()
