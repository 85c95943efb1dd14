"""GPU tests (H100): the System facade (alva_system_*) -- the reference's public API (system.hpp:28-38) on the CUDA kernels --
against the 100-frame trace of the reference's own System (tests/golden/system.npz `ref_*`) and against the same host-side state
machine run over the CPU oracle (`cpu_*`, tools/make_golden_system.py).

Exact: status codes, track ids in the reference's iteration order, 3-D flags, keyframe events and frame counters over all 100
frames; every pixel position bit for bit before the initialisation; getFramePoints.  Tight (same arithmetic, same
initialisation up to the summation order of its refinement): poses vs `cpu_*` to 1e-4, world points 1e-3, pixels 2e-3 px.  Bounded by the reference's own
noise-limited initialisation (tests/test_oracle_init.py; `test_system_lockstep_given_the_reference_initialisation` plugs the
reference's own initialisation result in and gets 1e-7 over the whole trace): poses vs `ref_*` |dt| < 1e-2 max(1, |t|), |dq| < 1e-3 -- over the whole trace,
which contains two keyframes after the initialisation and a local BA (tests/test_system_core_cpu.py shows that, given the
reference's own initialisation result, the same state machine is in lockstep with the reference to 1e-9)."""
import ctypes as C

import numpy as np
import pytest

from conftest import P
from system_util import CAP, PoseReport, frame_slice, frames_and_golden, quat_dist
from alvaar_b200 import synth, lib

pytestmark = pytest.mark.gpu


def bind():
    L = lib()
    L.alva_system_create.restype = C.c_void_p
    for f in ("alva_system_destroy", "alva_system_reset", "alva_system_num_matched"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.alva_system_configure.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_double] * 8
    L.alva_system_find_camera_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.alva_system_find_camera_pose_ts.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    L.alva_system_find_camera_pose_imu.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.alva_system_get_frame_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.alva_system_get_tracks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.alva_system_get_descriptors.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.alva_system_get_pose.argtypes = [C.c_void_p, C.c_void_p]
    L.alva_system_get_info.argtypes = [C.c_void_p, C.c_void_p]
    L.alva_system_find_plane.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    return L


def pose16_of(T):
    R = synth.quat_to_R(T[3:])
    p = np.zeros(16, np.float32)
    for r in range(3):
        p[4 * r:4 * r + 3] = R[r]
    p[12:15] = T[:3]
    p[15] = 1
    return p


def test_system_follows_the_reference():
    g, frames = frames_and_golden()
    w, h, nf = frames.shape[2], frames.shape[1], len(frames)
    L = bind()
    s = C.c_void_p(L.alva_system_create(0))
    pose = np.zeros(16, np.float32)
    assert L.alva_system_find_camera_pose(s, P(frames[0]), P(pose)) == -4          # not configured -> ALVA_E_STATE
    K = g["K"]
    assert L.alva_system_configure(s, w, h, K[0], K[1], K[2], K[3], 0.1, 0, 0, 0) == -1   # lens distortion: rejected, not ignored
    assert L.alva_system_configure(s, w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    fb = int(g["first_ba_frame"])
    init = int(np.argmax(g["ref_status"] == 1))
    assert init < fb < nf
    rep = PoseReport("System on the GPU vs the reference System, free-running")
    for k in range(nf):
        st = L.alva_system_find_camera_pose_ts(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(pose))
        assert st == g["ref_status"][k], (k, st)
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3))
        n = L.alva_system_get_tracks(s, P(ids), P(px), P(d3), P(wp), CAP)
        ids, px, d3, wp = ids[:n], px[:n], d3[:n], wp[:n]
        info = np.zeros(8, np.int32); T = np.zeros(7)
        L.alva_system_get_info(s, P(info)); L.alva_system_get_pose(s, P(T))
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        cids, cpx, cd3, cwp = frame_slice(g, "cpu_", k)
        assert (info == g["ref_info"][k]).all(), (k, info, g["ref_info"][k])
        assert n == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k          # ids in the reference's order, 3-D flags
        assert n == L.alva_system_num_matched(s)
        xy = np.zeros((CAP, 2), np.int32)
        m = L.alva_system_get_frame_points(s, P(xy), CAP)
        a, b = int(g["ref_xy_start"][k]), int(g["ref_xy_start"][k + 1])
        assert m == b - a
        assert np.abs(pose - pose16_of(T)).max() < 1e-6                                 # Utils::toPoseArray layout
        if k < init:
            assert (px.view(np.uint32) == rpx.view(np.uint32)).all()                    # pixel positions, float bits
            assert (xy[:m] == g["ref_xy"][a:b]).all()                                   # getFramePoints
            assert (pose == g["ref_pose16"][k]).all()                                   # identity, as the reference writes it
        else:
            # same arithmetic, but the initialisation's refinement sums its normal equations in another order on the device and
            # ends 5e-6 away in its flat valley (DESIGN 4.11); everything downstream inherits that
            # (pixels: KLT stops at 0.01 px updates, so priors that differ in the last digits may end a few 1e-3 px apart)
            sc = max(1.0, float(np.linalg.norm(g["ref_Twc"][k][:3])))                     # the trajectory is measured in units of the initial baseline
            assert np.abs(px - cpx).max() < 0.02 and np.abs(T - g["cpu_Twc"][k]).max() < 1e-4 * sc
            assert np.abs(wp - cwp).max() < 1e-3 * max(1.0, np.abs(cwp).max())
            assert np.abs(px - rpx).max() < 0.02                                        # also after the local BA at frame fb
            rep.check(g, k, T)   # vs the reference: 1e-4, or SPREAD_K x the reference's own 1-ulp spread on this trace where that is larger
            assert np.abs(xy[:m] - g["ref_xy"][a:b]).max() <= 1
        if k == 0:                                                                      # 256-bit ORB descriptors of the keypoints
            desc = np.zeros((CAP, 32), np.uint8); has = np.zeros(CAP, np.uint8)
            assert L.alva_system_get_descriptors(s, P(desc), P(has), CAP) == n
            assert (has[:n] == g["f0_has_desc"]).all() and has[:n].sum() > 100
            mk = g["f0_has_desc"] == 1
            assert (desc[:n][mk] == g["f0_desc"][mk]).all()
    rep.summary(g)
    out = np.zeros(16, np.float32)
    assert L.alva_system_find_plane(s, P(out), 250) == 1                             # the scene is a plane facing the first camera
    M = out.reshape(4, 4).T
    assert np.abs(M[:3, :3].T @ M[:3, :3] - np.eye(3)).max() < 1e-5 and abs(M[2, 0]) > 0.99   # R1 maps (1,0,0) onto the normal ~ +-z
    assert np.abs(M[:3, 3] - wp[d3 == 1].mean(0)).max() < 0.5                        # origin = centroid of the inliers
    assert L.alva_system_reset(s) == 0
    # after a reset the next frame is a first frame again: same keypoints as frame 0 except for the adapted detector quality
    assert L.alva_system_find_camera_pose_ts(s, P(np.ascontiguousarray(frames[0])), 5000.0, P(pose)) == 3
    assert L.alva_system_num_matched(s) > 100
    assert (pose == np.eye(4, dtype=np.float32).ravel()).all()
    imu = np.array([1.0, 0, 0, 0, 0], np.float64)
    assert L.alva_system_find_camera_pose_imu(s, P(np.ascontiguousarray(frames[0])), P(imu), P(pose)) == 1
    assert np.allclose(pose, np.eye(4, dtype=np.float32).ravel())
    L.alva_system_destroy(s)


def test_system_lockstep_given_the_reference_initialisation():
    """The reference's own initialisation result (recorded inside the golden run: what compute5ptEssentialMatrix returned)
    is handed to the System through the test hook; everything else -- KLT with projected priors, P3P-LMedS, PnP, keyframes,
    triangulation, local-map matching, local BA, culling -- runs on the GPU and must reproduce the reference's trajectory:
    poses 1e-7 (fp64 solvers agree with Ceres / OpenGV to 1e-12; the bar leaves room for the float KLT gates), landmarks 1e-6."""
    g, frames = frames_and_golden()
    w, h, nf = frames.shape[2], frames.shape[1], len(frames)
    L = bind()
    L.alva_system_debug_set_initialisation.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    s = C.c_void_p(L.alva_system_create(0))
    K = g["K"]
    assert L.alva_system_configure(s, w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    Rt = np.ascontiguousarray(g["ref_init_Rt"]); outl = np.ascontiguousarray(g["ref_init_outlier"])
    assert L.alva_system_debug_set_initialisation(s, P(Rt), P(outl), len(outl)) == 0
    pose = np.zeros(16, np.float32)
    worst_T = worst_px = 0.0
    for k in range(nf):
        st = L.alva_system_find_camera_pose_ts(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(pose))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3))
        n = L.alva_system_get_tracks(s, P(ids), P(px), P(d3), P(wp), CAP)
        T = np.zeros(7); info = np.zeros(8, np.int32)
        L.alva_system_get_pose(s, P(T)); L.alva_system_get_info(s, P(info))
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k] and (info == g["ref_info"][k]).all(), (k, st, info)
        assert n == len(rids) and (ids[:n] == rids).all() and (d3[:n] == rd3).all(), k
        worst_px = max(worst_px, float(np.abs(px[:n] - rpx).max()))
        worst_T = max(worst_T, float(np.abs(T[:3] - g["ref_Twc"][k][:3]).max()) / max(1.0, float(np.linalg.norm(g["ref_Twc"][k][:3]))), quat_dist(T[3:], g["ref_Twc"][k][3:]))
        assert np.abs(wp[:n] - rwp).max() < 1e-6 * max(1.0, np.abs(rwp).max()), k
        assert np.abs(pose - g["ref_pose16"][k]).max() < 1e-6, k                    # the API's float[16]
    assert worst_T < 1e-7 and worst_px < 1e-3, (worst_T, worst_px)
    L.alva_system_destroy(s)


def test_system_wall_clock_entry_point_initialises_and_tracks():
    """findCameraPose as the reference's shim calls it (time stamps from the system clock): initialises and tracks."""
    import time
    g, frames = frames_and_golden()
    w, h = frames.shape[2], frames.shape[1]
    L = bind()
    s = C.c_void_p(L.alva_system_create(0))
    K = g["K"]
    assert L.alva_system_configure(s, w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    pose = np.zeros(16, np.float32)
    seen = []
    for k in range(24):
        seen.append(L.alva_system_find_camera_pose(s, P(np.ascontiguousarray(frames[k])), P(pose)))
        time.sleep(0.004)   # two frames inside one millisecond would give the reference's motion model dt = 0
    assert seen[0] == 3 and 1 in seen and seen[-1] == 1
    assert np.isfinite(pose).all() and abs(np.linalg.norm(pose[12:15])) > 0.1
    L.alva_system_destroy(s)


def test_system_resets_when_tracks_are_lost():
    """visual_frontend.cpp:54-58: fewer than 50 tracked keypoints before initialisation -> reset, status 2."""
    w, h = 640, 480
    frames, _ = synth.make_frames(1, w, h, seed=3, rgba=True)
    other = synth.random_rgba(w, h, 1, seed=5)[0]                                   # unrelated noise: every track fails
    K = synth.intrinsics(w, h)
    L = bind()
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_configure(s, w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    pose = np.zeros(16, np.float32)
    assert L.alva_system_find_camera_pose_ts(s, P(np.ascontiguousarray(frames[0])), 0.0, P(pose)) == 3
    assert L.alva_system_find_camera_pose_ts(s, P(np.ascontiguousarray(other)), 33.3, P(pose)) == 2
    assert L.alva_system_num_matched(s) == 0
    L.alva_system_destroy(s)


@pytest.mark.parametrize("w,h,nf,nmin", [(1280, 720, 18, 500), (1920, 1080, 16, 1200)])
def test_system_full_size_against_the_cpu_oracle_backend(oracle, w, h, nf, nmin):
    """BASELINE's frame sizes (1280x720: 784 keypoints; 1920x1080: 1621): the CUDA System against the same state machine run over
    the CPU oracle on the spot (test infrastructure; tools/compare_system_cpu.py shows that one in lockstep with the reference at
    720p): initialisation at frame 12, then tracking.  Discrete state equal; poses 1e-4 (the initialisation's refinement order)."""
    from system_util import cpu_system_lib
    K = synth.intrinsics(w, h)
    frames, _ = synth.make_frames(nf, w, h, seed=7, rgba=True)
    S = cpu_system_lib()
    c = S.cpu_system_create(w, h, K[0], K[1], K[2], K[3])
    L = bind()
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_configure(s, w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    pose = np.zeros(16, np.float32)
    seen = []
    for k in range(nf):
        f = np.ascontiguousarray(frames[k])
        Tc = np.zeros(7); T = np.zeros(7)
        st_c = S.cpu_system_process(c, P(f), k * 33.333, P(Tc))
        st = L.alva_system_find_camera_pose_ts(s, P(f), k * 33.333, P(pose))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3))
        cids = np.zeros(CAP, np.int32); cpx = np.zeros((CAP, 2), np.float32); cd3 = np.zeros(CAP, np.uint8); cwp = np.zeros((CAP, 3))
        n = L.alva_system_get_tracks(s, P(ids), P(px), P(d3), P(wp), CAP)
        m = S.cpu_system_keypoints(c, P(cids), P(cpx), P(cd3), P(cwp), CAP)
        L.alva_system_get_pose(s, P(T))
        assert st == st_c and n == m and (ids[:n] == cids[:n]).all() and (d3[:n] == cd3[:n]).all(), (k, st, st_c, n, m)
        if st == 3:
            assert (px[:n].view(np.uint32) == cpx[:n].view(np.uint32)).all(), k
        else:
            assert np.abs(px[:n] - cpx[:n]).max() < 0.02 and np.abs(T - Tc).max() < 1e-4 * max(1.0, float(np.linalg.norm(Tc[:3]))), k
        seen.append(st)
    assert seen[0] == 3 and seen[-1] == 1 and n > nmin
    S.cpu_system_destroy(c)
    L.alva_system_destroy(s)


def test_python_system_class():
    """alvaar_b200.System: the ctypes mirror of the reference's class, end to end on the golden's first frames"""
    import alvaar_b200
    g, frames = frames_and_golden()
    K = g["K"]
    s = alvaar_b200.System(frames.shape[2], frames.shape[1], K[0], K[1], K[2], K[3])
    with pytest.raises(ValueError):
        s.find_camera_pose(frames[0][:, :, :3])
    seen = []
    for k in range(20):
        st, pose = s.find_camera_pose(np.ascontiguousarray(frames[k]), k * 33.333)
        assert st == g["ref_status"][k]
        seen.append(st)
    ids, px, d3, wp = s.tracks()
    rids, rpx, rd3, rwp = frame_slice(g, "ref_", 19)
    assert (ids == rids).all() and (d3 == rd3).all() and s.info()["initialised"] == 1 and s.find_plane() is not None
    s.reset()
    assert s.info()["keypoints"] == 0
    s.close()


def test_system_batch_entry_point_equals_single_calls():
    """alva_system_find_camera_pose_batch: four independent streams (two sequences, each twice) through one call per frame step
    give, per stream, exactly what alva_system_find_camera_pose_ts gives a single System -- status and float[16] pose bits."""
    w, h, nf = 640, 480, 30
    K = synth.intrinsics(w, h)
    seqs = [synth.make_frames(nf, w, h, seed=sd, rgba=True)[0] for sd in (7, 11)]
    L = bind()
    L.alva_system_find_camera_pose_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    single = []
    for fr in seqs:
        s = C.c_void_p(L.alva_system_create(0))
        assert L.alva_system_configure(s, w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
        out = []
        for k in range(nf):
            pose = np.zeros(16, np.float32)
            st = L.alva_system_find_camera_pose_ts(s, P(np.ascontiguousarray(fr[k])), k * 33.333, P(pose))
            out.append((st, pose.copy()))
        L.alva_system_destroy(s)
        single.append(out)
    n = 4
    hs = [C.c_void_p(L.alva_system_create(0)) for _ in range(n)]
    for s in hs:
        assert L.alva_system_configure(s, w, h, K[0], K[1], K[2], K[3], 0, 0, 0, 0) == 0
    harr = (C.c_void_p * n)(*[s.value for s in hs])
    for k in range(nf):
        fr = [np.ascontiguousarray(seqs[i % 2][k]) for i in range(n)]
        parr = (C.c_void_p * n)(*[f.ctypes.data for f in fr])
        ts = np.full(n, k * 33.333)
        poses = np.zeros((n, 16), np.float32)
        status = np.zeros(n, np.int32)
        assert L.alva_system_find_camera_pose_batch(harr, parr, P(ts), n, P(poses), P(status)) == 0
        for i in range(n):
            st, pose = single[i % 2][k]
            assert status[i] == st and (poses[i].view(np.uint32) == pose.view(np.uint32)).all(), (k, i)
    assert single[0][-1][0] == 1                        # the sequences do initialise and track
    for s in hs:
        L.alva_system_destroy(s)
