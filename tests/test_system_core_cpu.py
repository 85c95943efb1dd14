"""CPU tests of the host-side System state machine (alvaar_b200/csrc/system_core.h) -- the code that, in the product, drives
the CUDA kernels -- instantiated over the CPU oracle backend (test infrastructure) and compared with a 100-frame trace of the
reference's own System (tests/golden/system.npz, dumped by tools/make_golden_system.py: initialisation at frame 13, eight keyframes,
the first local BA at frame 27).

What is exact over all 100 frames: status codes, track ids IN THE REFERENCE'S ITERATION ORDER (it decides RANSAC sample indices
and Ceres residual order), 3-D flags, keyframe events, frame / map counters -- and, before the initialisation, every pixel
position bit for bit.
What is toleranced: after the initialisation, poses / world points carry the reference's own noise-limited 5-point refinement
(tests/test_oracle_init.py: a 1-ulp input change moves ITS result by 1e-6 .. 1e-3).  The bar is data-driven (system_util.
pose_deviation): 1e-4 relative (north_star), or 4 x the reference's OWN spread on this trace under a 1-ulp change of one intrinsic
(stored in the golden) where that spread is larger; the worst observed deviation is printed.
With the reference's OWN initialisation stage plugged in (live, or replayed call by call from its stored outputs:
tests/ref_golden.py) everything downstream -- KLT with projected
priors, P3P-LMedS, PnP, keyframe decisions, triangulation, local-map matching, local BA, culling -- is in lockstep: poses and
world points 1e-9, pixel positions bit-identical, over the whole trace (tools/compare_system_cpu.py shows the same over 140
frames / 11 keyframes / 9 local BAs)."""
import ctypes as C

import numpy as np

from conftest import P
from ref_golden import EssentialHook, digest, ref_outputs
from system_util import CAP, PoseReport, cpu_system_lib, frame_slice, frames_and_golden, quat_dist


def run(S, frames, K, hook=None):
    w, h = frames.shape[2], frames.shape[1]
    s = S.cpu_system_create(w, h, K[0], K[1], K[2], K[3])
    if hook is not None:
        S.cpu_system_set_essential_hook(s, hook)
    out = []
    for k in range(len(frames)):
        T = np.zeros(7)
        st = S.cpu_system_process(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); info = np.zeros(8, np.int32)
        n = S.cpu_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP)
        S.cpu_system_info(s, P(info))
        out.append((st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy(), wp[:n].copy()))
    S.cpu_system_destroy(s)
    return out


def test_state_machine_follows_the_reference(oracle):
    g, frames = frames_and_golden()
    tr = run(cpu_system_lib(), frames, g["K"])
    fb = int(g["first_ba_frame"])
    init = int(np.argmax(g["ref_status"] == 1))
    assert 10 <= init < fb < len(frames)
    rep = PoseReport("state machine over the CPU oracle vs the reference System, free-running")
    for k, (st, T, info, ids, px, d3, wp) in enumerate(tr):
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k], k
        assert (info == g["ref_info"][k]).all(), (k, info, g["ref_info"][k])
        assert (ids == rids).all() and (d3 == rd3).all(), k                 # ids in the reference's iteration order, 3-D flags
        if k < init:
            assert (px.view(np.uint32) == rpx.view(np.uint32)).all()        # bit-identical tracks before the initialisation
            assert (T == g["ref_Twc"][k]).all()
        else:
            assert np.abs(px - rpx).max() < 0.02
            rep.check(g, k, T)                                               # 1e-4, or SPREAD_K x the reference's own 1-ulp spread where that is larger
        # the committed cpu_* trace (what the GPU build is compared with) is this very run
        cids, cpx, cd3, cwp = frame_slice(g, "cpu_", k)
        assert (ids == cids).all() and (px.view(np.uint32) == cpx.view(np.uint32)).all() and np.abs(T - g["cpu_Twc"][k]).max() < 1e-12
    rep.summary(g)


def test_lockstep_given_the_reference_initialisation(oracle, ref):
    g, frames = frames_and_golden()
    hook = EssentialHook(ref, "system_essential_640x480")
    tr = run(cpu_system_lib(), frames, g["K"], hook.ptr)
    hook.finish()
    assert int(g["first_ba_frame"]) < len(frames) - 5                        # the trace does contain a local BA
    for k in range(len(frames)):
        st, T, info, ids, px, d3, wp = tr[k]
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k] and (ids == rids).all() and (d3 == rd3).all()
        assert (px.view(np.uint32) == rpx.view(np.uint32)).all()
        assert np.abs(T - g["ref_Twc"][k]).max() < 1e-9
        assert np.abs(wp - rwp).max() < 1e-9 * max(1.0, np.abs(rwp).max())


def test_reset_when_tracks_are_lost(oracle):
    """visual_frontend.cpp:54-58: fewer than 50 tracked keypoints before initialisation -> reset, status 2, a fresh first frame"""
    from alvaar_b200 import synth
    w, h = 640, 480
    frames, _ = synth.make_frames(1, w, h, seed=3, rgba=True)
    other = synth.random_rgba(w, h, 1, seed=5)[0]
    K = synth.intrinsics(w, h)
    S = cpu_system_lib()
    s = S.cpu_system_create(w, h, K[0], K[1], K[2], K[3])
    T = np.zeros(7)
    assert S.cpu_system_process(s, P(np.ascontiguousarray(frames[0])), 0.0, P(T)) == 3
    assert S.cpu_system_process(s, P(np.ascontiguousarray(other)), 33.3, P(T)) == 2
    info = np.zeros(8, np.int32)
    S.cpu_system_info(s, P(info))
    assert info[0] == -1 and info[2] == 0 and info[5] == 0
    assert S.cpu_system_process(s, P(np.ascontiguousarray(frames[0])), 66.6, P(T)) == 3
    S.cpu_system_info(s, P(info))
    assert info[0] == 0 and info[2] > 100 and info[5] == 1
    S.cpu_system_destroy(s)


WSTRIDE = 16   # world points: every 16th keypoint of a frame is stored (compared in full when the reference runs live)


def reference_trace(ref, key, seq, w, h, K):
    """The reference System over `seq`, frame by frame: status, keypoint count, info, pose (stored), track ids, pixel
    positions and 3-D flags (digests), world points of every WSTRIDE-th keypoint -- of every keypoint when the reference is live."""
    full_wp = []

    def compute(R):
        R.ref_system_create.restype = C.c_void_p
        R.ref_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 8
        R.ref_system_find_camera_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
        R.ref_system_keypoints.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
        R.ref_system_info8.argtypes = [C.c_void_p, C.c_void_p]
        R.ref_system_destroy.argtypes = [C.c_void_p]
        r = R.ref_system_create(w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0)
        out = {k: [] for k in ("st", "n", "info", "T", "ids", "px", "d3", "wp")}
        for k, f in enumerate(seq):
            f = np.ascontiguousarray(f)
            pose = np.zeros(16, np.float32); T_r = np.zeros(7)
            st_r = R.ref_system_find_camera_pose(r, P(f), k * 33.333, P(pose))
            ids_r = np.zeros(CAP, np.int32); px_r = np.zeros((CAP, 2), np.float32); d3_r = np.zeros(CAP, np.uint8); w_r = np.zeros((CAP, 3))
            n_r = R.ref_system_keypoints(r, P(ids_r), P(px_r), P(d3_r), P(w_r), CAP, P(T_r))
            i_r = np.zeros(8, np.int32)
            R.ref_system_info8(r, P(i_r))
            for name, v in (("st", st_r), ("n", n_r), ("info", i_r), ("T", T_r), ("ids", digest(ids_r[:n_r])),
                            ("px", digest(px_r[:n_r].view(np.uint32))), ("d3", digest(d3_r[:n_r])), ("wp", w_r[:n_r:WSTRIDE])):
                out[name].append(v)
            full_wp.append(w_r[:n_r].copy())
        R.ref_system_destroy(r)
        out["wp"] = np.concatenate(out["wp"])
        return {k: np.array(v) if k != "wp" else v for k, v in out.items()}
    t = ref_outputs(ref, key, compute)
    starts = np.concatenate([[0], np.cumsum((t["n"] + WSTRIDE - 1) // WSTRIDE)])
    stride = 1 if full_wp else WSTRIDE
    return [dict(st=int(t["st"][k]), n=int(t["n"][k]), info=t["info"][k], T=t["T"][k], ids=t["ids"][k], px=t["px"][k], d3=t["d3"][k],
                 wp=full_wp[k] if full_wp else t["wp"][starts[k]:starts[k + 1]], wstride=stride) for k in range(len(seq))]


def test_failure_paths_in_lockstep_with_the_live_reference(oracle, ref):
    """Blackout frame, a jump to an unrelated sequence, a jump back: lost tracks, P3P / PnP outlier removal, failed poses,
    resets (status 2) with a stale motion model, re-initialisations -- against the live reference System frame by frame
    (its own initialisation stage plugged in): every discrete quantity equal, poses 1e-6."""
    from alvaar_b200 import synth
    w, h = 640, 480
    K = synth.intrinsics(w, h)
    A, _ = synth.make_frames(40, w, h, seed=7, rgba=True)
    B, _ = synth.make_frames(26, w, h, seed=33, rgba=True)
    black = np.zeros_like(A[0]); black[..., 3] = 255
    seq = [A[k] for k in range(24)] + [black] + [B[k] for k in range(26)] + [A[k] for k in range(20, 40)]
    trace = reference_trace(ref, "system_failure_paths", seq, w, h, K)
    S = cpu_system_lib()
    s = S.cpu_system_create(w, h, K[0], K[1], K[2], K[3])
    hook = EssentialHook(ref, "system_failure_paths_essential")
    S.cpu_system_set_essential_hook(s, hook.ptr)
    seen = set()
    for k, f in enumerate(seq):
        f = np.ascontiguousarray(f)
        T_s = np.zeros(7)
        st_s = S.cpu_system_process(s, P(f), k * 33.333, P(T_s))
        ids_s = np.zeros(CAP, np.int32); px_s = np.zeros((CAP, 2), np.float32); d3_s = np.zeros(CAP, np.uint8); w_s = np.zeros((CAP, 3))
        n_s = S.cpu_system_keypoints(s, P(ids_s), P(px_s), P(d3_s), P(w_s), CAP)
        i_s = np.zeros(8, np.int32)
        S.cpu_system_info(s, P(i_s))
        r = trace[k]
        assert r["st"] == st_s and r["n"] == n_s and (r["info"] == i_s).all(), (k, r["st"], st_s, r["info"], i_s)
        assert (r["ids"] == digest(ids_s[:n_s])).all() and (r["d3"] == digest(d3_s[:n_s])).all(), k
        assert (r["px"] == digest(px_s[:n_s].view(np.uint32))).all(), k
        assert np.abs(r["T"] - T_s).max() < 1e-6, k
        seen.add(r["st"])
    hook.finish()
    assert seen == {1, 2, 3}                                              # the sequence did exercise resets and re-initialisation
    S.cpu_system_destroy(s)


def test_lockstep_at_720p_with_the_live_reference(oracle, ref):
    """BASELINE's frame size (1280x720, 784 keypoints / frame): 36 frames through initialisation (frame 12), two more keyframes
    and the first local BA against the live reference System, its own initialisation stage plugged in: lockstep as at 640x480."""
    from alvaar_b200 import synth
    w, h, nf = 1280, 720, 36
    K = synth.intrinsics(w, h)
    frames, _ = synth.make_frames(nf, w, h, seed=7, rgba=True)
    trace = reference_trace(ref, "system_720p", frames, w, h, K)
    S = cpu_system_lib()
    s = S.cpu_system_create(w, h, K[0], K[1], K[2], K[3])
    hook = EssentialHook(ref, "system_720p_essential")
    S.cpu_system_set_essential_hook(s, hook.ptr)
    last = None
    for k in range(nf):
        f = np.ascontiguousarray(frames[k])
        T_s = np.zeros(7)
        st_s = S.cpu_system_process(s, P(f), k * 33.333, P(T_s))
        ids_s = np.zeros(CAP, np.int32); px_s = np.zeros((CAP, 2), np.float32); d3_s = np.zeros(CAP, np.uint8); w_s = np.zeros((CAP, 3))
        n_s = S.cpu_system_keypoints(s, P(ids_s), P(px_s), P(d3_s), P(w_s), CAP)
        i_s = np.zeros(8, np.int32)
        S.cpu_system_info(s, P(i_s))
        r = trace[k]
        assert r["st"] == st_s and r["n"] == n_s and (r["info"] == i_s).all(), (k, r["st"], st_s, r["info"], i_s)
        assert (r["ids"] == digest(ids_s[:n_s])).all() and (r["d3"] == digest(d3_s[:n_s])).all(), k
        assert (r["px"] == digest(px_s[:n_s].view(np.uint32))).all(), k
        w_r = r["wp"]
        assert np.abs(r["T"] - T_s).max() < 1e-9 and np.abs(w_r - w_s[:n_s:r["wstride"]]).max(initial=0) < 1e-9 * max(1.0, np.abs(w_r).max(initial=0)), k
        last = r["info"]
    hook.finish()
    assert last[4] == 1 and last[1] >= 2 and last[2] > 500          # initialised, at least keyframe 2 (a local BA ran), 720p-sized
    S.cpu_system_destroy(s)


def test_find_plane_on_the_planar_scene(oracle):
    """System::findPlane as intended (system_core.h lists the defects of the reference's own processPlane, which make it
    unpinnable): 0 before the initialisation; afterwards the synthetic scene -- a textured plane facing the first camera -- is
    found: unit rotation whose first column (the image of `up` = (1, 0, 0) under R1) is the plane normal ~ +-z, origin at the
    inliers' centroid, normal pointing away from the camera; repeatable call to call."""
    g, frames = frames_and_golden()
    S = cpu_system_lib()
    S.cpu_system_find_plane.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    K = g["K"]
    s = S.cpu_system_create(frames.shape[2], frames.shape[1], K[0], K[1], K[2], K[3])
    out = np.zeros(16, np.float32)
    T = np.zeros(7)
    for k in range(40):
        S.cpu_system_process(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(T))
        if k == 5:
            assert S.cpu_system_find_plane(s, P(out), 250) == 0          # fewer than 32 map points: no plane
    assert S.cpu_system_find_plane(s, P(out), 250) == 1
    M = out.reshape(4, 4).T                                              # Utils::toPoseArray(Mat) writes column-major
    R, t = M[:3, :3].astype(np.float64), M[:3, 3]
    assert np.abs(R.T @ R - np.eye(3)).max() < 1e-5 and abs(np.linalg.det(R) - 1) < 1e-5 and M[3, 3] == 1
    n = R[:, 0]
    assert abs(n[2]) > 0.999                                             # the plane z = const of the first camera
    ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3))
    m = S.cpu_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP)
    pts = wp[:m][d3[:m] == 1]
    assert np.abs(t - pts.mean(0)).max() < 0.5 and np.abs((pts - t) @ n).mean() < 0.2   # on the plane of the map points
    cam = T[:3]
    assert (cam - t) @ n < 0                                             # turned away from the camera
    S.cpu_system_destroy(s)
