"""CPU tests of the System state machine under the reference's presets (state.hpp:9-17), over the CPU oracle
(tests/host/system_cpu_preset.cpp).

Against the committed traces of the reference System under FAST, AVERAGE and ACCURATE (tests/golden/system_preset_*.npz,
tools/make_golden_presets.py), given the reference's own initialisation through the five-point hook: status, track ids in the
reference's order, 3-D flags and counters exact on every frame, poses and world points 1e-9.  Against the live reference (where
it is built in this tree, else skipped): a sequence with jumps under AVERAGE, so that p3pReq_ is set and P3P runs after frames
posed by PnP from the motion prior, and a long FAST run past keyframe id 20, so that the 0.9 keyframe filter runs."""
import hashlib

import numpy as np
import pytest

from conftest import golden
from preset_util import PRESETS, CpuRun, cpu_preset_system_lib, ref_frame, ref_preset_lib, ref_system_create
from system_util import frame_slice
from test_oracle_clahe import ReplayHook
from alvaar_b200 import synth

NAMES = ["fast", "average", "accurate"]


def preset_golden(name):
    g = golden(f"system_preset_{name}")
    w, h, nf = int(g["w"]), int(g["h"]), int(g["nframes"])
    frames, _ = synth.make_frames(nf, w, h, seed=int(g["seed"]), rgba=True)
    assert hashlib.sha256(frames.tobytes()).hexdigest() == str(g["sha256"]), "synthetic frames changed: re-dump the golden"
    return g, frames


@pytest.mark.parametrize("name", NAMES)
def test_golden_trace_covers_the_preset(name):
    """each trace initialises, runs local BAs, never reaches the 21-free-pose limit; AVERAGE and ACCURATE pose frames by PnP
    from the motion prior"""
    g, frames = preset_golden(name)
    assert int(g["cell"]) == PRESETS[name][1] and int(g["p3p"]) == PRESETS[name][3]
    init = int(np.argmax(g["ref_status"] == 1))
    assert 0 < init < int(g["first_ba_frame"]) < len(frames)
    assert int(g["counters_lockstep_local_ba"]) > 0 and int(g["counters_lockstep_free_pose_clamp"]) == 0
    assert int(g["counters_own_free_pose_clamp"]) == 0
    if PRESETS[name][3]:
        assert int(g["counters_lockstep_pnp_prior"]) == 0
    else:
        assert int(g["counters_lockstep_pnp_prior"]) > 50


@pytest.mark.parametrize("name", NAMES)
def test_state_machine_under_preset_given_the_reference_initialisation(oracle, ref, name):
    g, frames = preset_golden(name)
    hook = ReplayHook(ref, g)
    r = CpuRun(cpu_preset_system_lib(), name, int(g["w"]), int(g["h"]), g["K"], hook.ptr)
    init = int(np.argmax(g["ref_status"] == 1))
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp = r.frame(frames[k], k * 33.333)
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k] and (info == g["ref_info"][k]).all(), (k, st, info, g["ref_info"][k])
        assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
        if k < init:
            assert (px.view(np.uint32) == rpx.view(np.uint32)).all(), k
        assert np.abs(T - g["ref_Twc"][k]).max() < 1e-9, k
        assert np.abs(wp - rwp).max(initial=0) < 1e-9 * max(1.0, np.abs(rwp).max(initial=0)), k
    c = r.counters()
    r.close()
    hook.finish()
    assert c["free_pose_clamp"] == 0 and c["pnp_prior"] == int(g["counters_lockstep_pnp_prior"])


@pytest.mark.parametrize("name", NAMES)
def test_committed_cpu_trace_is_this_state_machine(oracle, name):
    """the `cpu_*` trace (its own initialisation) is this very state machine"""
    g, frames = preset_golden(name)
    r = CpuRun(cpu_preset_system_lib(), name, int(g["w"]), int(g["h"]), g["K"])
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp = r.frame(frames[k], k * 33.333)
        cids, cpx, cd3, cwp = frame_slice(g, "cpu_", k)
        assert st == g["cpu_status"][k] and (info == g["cpu_info"][k]).all(), k
        assert (ids == cids).all() and (d3 == cd3).all() and (px.view(np.uint32) == cpx.view(np.uint32)).all(), k
        assert np.abs(T - g["cpu_Twc"][k]).max() < 1e-12, k
    r.close()


def test_default_preset_is_the_plain_backend(oracle):
    """DEFAULT through the preset backend: system.npz's `cpu_*` trace bit for bit"""
    g = golden("system")
    frames, _ = synth.make_frames(int(g["nframes"]), int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True)
    r = CpuRun(cpu_preset_system_lib(), "default", int(g["w"]), int(g["h"]), g["K"])
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp = r.frame(frames[k], k * 33.333)
        cids, cpx, cd3, cwp = frame_slice(g, "cpu_", k)
        assert st == g["cpu_status"][k] and (ids == cids).all() and (px.view(np.uint32) == cpx.view(np.uint32)).all(), k
        assert (T == g["cpu_Twc"][k]).all(), k
    r.close()


def test_unknown_preset_is_refused(oracle):
    S = cpu_preset_system_lib()
    s = S.cpu_preset_system_create(640, 480, 500.0, 500.0, 320.0, 240.0)
    assert S.cpu_preset_system_set_preset(s, 4) == -1 and S.cpu_preset_system_set_preset(s, -1) == -1
    assert S.cpu_preset_system_set_preset(s, 3) == 0
    S.cpu_preset_system_destroy(s)


# ------------------------------------------------------------------------------------------------ live reference
def live(ref):
    RP = ref_preset_lib(ref)
    if RP is None:
        pytest.skip("the reference and its preset harness are not built in this tree (oracle/build_ref_preset.sh)")
    return RP


def lockstep(ref, RP, name, seq, w, h, K):
    """the CPU state machine (the reference's five-point stage plugged in) against the reference System, frame by frame;
    returns the reference's p3pReq_ after each frame, its status codes and the CPU run's counters"""
    import ctypes as C
    ref.ref_essential_5pt.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    PROTO = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p)
    cb = PROTO(lambda *a: ref.ref_essential_5pt(*a))
    r = CpuRun(cpu_preset_system_lib(), name, w, h, K, C.cast(cb, C.c_void_p))
    s = ref_system_create(ref, RP, name, w, h, K)
    reqs, sts, kfs = [], [], []
    for k, f in enumerate(seq):
        st, T, info, ids, px, d3, wp = r.frame(f, k * 33.333)
        rst, rT, rinfo, rids, rpx, rd3, rwp, req = ref_frame(ref, RP, s, f, k * 33.333)
        assert st == rst and (info == rinfo).all(), (k, st, rst, info, rinfo)
        assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
        assert (px.view(np.uint32) == rpx.view(np.uint32)).all(), k
        assert np.abs(T - rT).max() < 1e-6, k
        reqs.append(req); sts.append(st); kfs.append(int(info[1]))
    c = r.counters()
    r.close()
    ref.ref_system_destroy(s)
    return np.array(reqs), np.array(sts), np.array(kfs), c


def test_average_pnp_from_the_prior_and_its_p3p_fallback_with_the_live_reference(oracle, ref):
    """AVERAGE (p3pEnabled_ off) on system.npz's scene, then a jump to an unrelated sequence and back: tracked frames are posed
    by PnP from the motion prior; at each jump p3pReq_ is set and the following frames run P3P until a pose succeeds -- both
    state machines take every decision alike (status, ids, 3-D flags, counters, pixels bit for bit, poses 1e-6).  On this
    sequence it is the KLT gate that sets p3pReq_ (fewer than a third of the 3-D keypoints tracked, visual_frontend.cpp:196-199);
    the PnP-failure branch that also sets it (visual_frontend.cpp:384-389) is counted, and did not fire here."""
    RP = live(ref)
    w, h = 640, 480
    K = synth.intrinsics(w, h)
    A, _ = synth.make_frames(40, w, h, seed=7, rgba=True)
    B, _ = synth.make_frames(26, w, h, seed=33, rgba=True)
    seq = [A[k] for k in range(30)] + [B[k] for k in range(26)] + [A[k] for k in range(30, 40)]
    reqs, sts, kfs, c = lockstep(ref, RP, "average", seq, w, h, K)
    assert c["pnp_prior"] > 10
    assert reqs[:30].sum() == 0 and reqs[30] == 1 and reqs[56] == 1, reqs.nonzero()     # set at both jumps, in lockstep
    print(f"AVERAGE with jumps: frames posed by PnP from the prior {c['pnp_prior']}, p3pReq_ set after {int(reqs.sum())} frames, "
          f"of which by a failed PnP from the prior: {c['p3p_fallback']}")


def test_fast_past_keyframe_20_with_the_live_reference(oracle, ref):
    """FAST (filtering ratio 0.9) long enough for keyframe ids past 20, where Mapper::optimize filters keyframes.  On this
    synthetic scene the filter runs on every keyframe from id 20 on; whether it removes one is reported, not asserted -- a
    removal needs a keyframe whose 3-D points are more than 90 % seen by more than four keyframes."""
    RP = live(ref)
    w, h = 640, 480
    K = synth.intrinsics(w, h)
    frames, _ = synth.make_frames(400, w, h, seed=7, rgba=True)
    reqs, sts, kfs, c = lockstep(ref, RP, "fast", frames, w, h, K)
    assert kfs.max() >= 20, kfs.max()
    print(f"FAST: keyframe ids up to {kfs.max()}, local BAs {c['local_ba']}, 21-free-pose limit engaged {c['free_pose_clamp']} times")
