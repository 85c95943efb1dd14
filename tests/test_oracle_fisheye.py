"""CPU tests of the equidistant fisheye lens (OpenCV's cv::fisheye, alva_system_set_fisheye).

The host side of alvaar_b200/csrc/camera_model.h (what the state machine and, compiled for the device, the kernels run), the
state machine's Camera dispatch, the plain-C oracle (oracle/fisheye_oracle.c) and OpenCV's own cv::fisheye agree on every case
of tests/golden/fisheye.npz -- live when oracle/_ref/libalva_ref_fisheye.so is built, else through the stored digests.  The bar
is identical float bits; a point may only differ from OpenCV where OpenCV's double lies within 4 double ulps of a float rounding
boundary (glibc's atan / tan against the header's), and the test counts those.  The host-side System state machine with the
lens (tests/host/system_cpu_fisheye.cpp) tracks a 100-frame sequence rendered through it, against the rendered ground truth."""
import ctypes as C

import numpy as np
import pytest

from camera_util import same_bits
from conftest import P, golden
from fisheye_util import (CASES, NAMES, SYSTEM_FISHEYE, case_K, case_pixels, case_points, cpu_system_lib, oracle_lib, ref_lib,
                          rounding_exempt, run_cpu_system, run_points, run_ref, system_frames, trajectory_error)
from ref_golden import digest


def opencv_results(k, hu, hp):
    """OpenCV's float results and, where they differ from the header's (hu, hp), the doubles they were rounded from: live from
    the library when it is built, else rebuilt from the golden (the header's bits with the stored differences patched in, which
    must hash to OpenCV's digest)"""
    g = golden("fisheye")
    name = NAMES[k]
    R = ref_lib()
    if R is not None:
        K, D = case_K(k)
        ru, ru64 = run_ref(R.ref_fisheye_undistort_points, case_pixels(k), K, D)
        rp, rp64 = run_ref(R.ref_fisheye_project_points, case_points(k), K, D)
        return ru, ru64, rp, rp64
    out = []
    for key, mine in (("unpx", hu), ("uv", hp)):
        r32 = mine.copy().ravel()
        r64 = np.zeros(r32.shape)
        idx = g[f"{name}/{key}_diff"]
        r32[idx] = g[f"{name}/{key}_ref32"]
        r64[idx] = g[f"{name}/{key}_ref64"]
        out += [r32.reshape(mine.shape), r64.reshape(mine.shape)]
    return out


@pytest.mark.parametrize("k", range(len(CASES)), ids=NAMES)
def test_header_oracle_and_opencv_agree(k):
    g = golden("fisheye")
    name = NAMES[k]
    K, D = case_K(k)
    px, X = case_pixels(k), case_points(k)
    assert (digest(px) == g[f"{name}/px"]).all() and (digest(X) == g[f"{name}/X"]).all(), "case generator changed: re-dump fisheye.npz"
    assert (g[f"{name}/K"] == K).all() and (g[f"{name}/D"] == D).all()
    S, O = cpu_system_lib(), oracle_lib()
    hu, hp = run_points(S.cpu_fish_undistort_points, px, K, D), run_points(S.cpu_fish_project_points, X, K, D)
    assert same_bits(hu, run_points(O.orc_fisheye_undistort_points, px, K, D))
    assert same_bits(hp, run_points(O.orc_fisheye_project_points, X, K, D))
    assert same_bits(hu, run_points(S.cpu_fish_cam_undistort_points, px, K, D))      # what the state machine calls
    assert same_bits(hp, run_points(S.cpu_fish_cam_project_points, X, K, D))
    ru, ru64, rp, rp64 = opencv_results(k, hu, hp)
    from camera_util import cdigest
    assert (cdigest(ru) == g[f"{name}/unpx"]).all() and (cdigest(rp) == g[f"{name}/uv"]).all()
    n_exempt = 0
    for what, mine, r32, r64 in (("undistort", hu, ru, ru64), ("project", hp, rp, rp64)):
        idx, ok = rounding_exempt(mine, r32, r64)
        assert ok.all(), f"{what}: {int((~ok).sum())} float results differ from OpenCV's away from a rounding boundary, e.g. flat index {idx[~ok][:4]}"
        n_exempt += len(idx)
    print(f"{name}: {2 * (len(px) + len(X))} float results, {n_exempt} exempt at a float rounding boundary")


def test_cases_cover_the_model_branches():
    g = golden("fisheye")
    assert int(g["newton_fails_640x480/n_fail"]) > 1000
    assert int(g["wide_640x480/n_fail"]) == 0 and int(g["fov180_1280x720/n_fail"]) == 0
    S = cpu_system_lib()
    k = NAMES.index("fov180_1280x720")                              # theta_d clamped to pi/2 beyond the image diagonal
    K, D = case_K(k)
    px = case_pixels(k).astype(np.float64)
    assert (np.hypot((px[:, 0] - K[2]) / K[0], (px[:, 1] - K[3]) / K[1]) > np.pi / 2).sum() > 100
    k = NAMES.index("newton_fails_640x480")
    K, D = case_K(k)
    px = case_pixels(k)
    un = run_points(S.cpu_fish_undistort_points, px, K, D)
    fail = (un[:, 0] == -1e6) & (un[:, 1] == -1e6)
    td = np.hypot((px[:, 0].astype(np.float64) - K[2]) / K[0], (px[:, 1].astype(np.float64) - K[3]) / K[1])
    assert fail.sum() == int(g["newton_fails_640x480/n_fail"]) and (td[fail] > 0.5).all() and not fail[td < 0.5].any()
    c = np.flatnonzero((px[:, 0] == np.float32(K[2])) & (px[:, 1] == np.float32(K[3])))   # |theta_d| <= 1e-8: the centre itself
    assert len(c) and (un[c] == np.float32(K[2:])).all()
    X = case_points(0)
    assert (X[:, 2] < 0).sum() >= 1000 and (X[:, 2] == 0).sum() >= 1000 and ((X[:, 0] == 0) & (X[:, 1] == 0) & (X[:, 2] != 0)).sum() >= 1000


def test_deterministic_atan_and_tan_are_within_one_ulp_of_the_c_library():
    S = cpu_system_lib()
    x = np.ascontiguousarray(np.concatenate([np.random.default_rng(0).uniform(-4, 4, 200000), np.linspace(0, np.pi / 2, 20001)[:-1],
                                             np.random.default_rng(1).uniform(-60, 60, 20000)]))
    for fn, ref in ((S.cpu_det_atan, np.arctan), (S.cpu_det_tan, np.tan)):
        y = np.zeros_like(x)
        fn(P(x), len(x), P(y))
        r = ref(x)
        assert (np.abs(y - r) <= np.spacing(np.abs(r))).all()


def test_renderer_follows_the_model():
    """synth renders a pixel with the ray whose projection through the lens (camera_model.h) is that pixel"""
    from alvaar_b200 import synth
    S = cpu_system_lib()
    w, h = 640, 480
    K = np.array(synth.intrinsics(w, h))
    u, v = np.meshgrid(np.arange(0, w, 7, dtype=np.float64), np.arange(0, h, 5, dtype=np.float64))
    xd, yd = (u.ravel() - K[2]) / K[0], (v.ravel() - K[3]) / K[1]
    td = np.hypot(xd, yd)
    th = synth.fisheye_theta(td, SYSTEM_FISHEYE)
    s = np.where(td > 0, np.tan(th) / np.where(td > 0, td, 1), 1)
    rays = np.ascontiguousarray(np.stack([xd * s, yd * s, np.ones_like(xd)], 1) * 3.0)
    uv = run_points(S.cpu_fish_project_points, rays, K, np.array(SYSTEM_FISHEYE))
    assert np.abs(uv - np.stack([u.ravel(), v.ravel()], 1)).max() < 1e-3


def test_state_machine_tracks_a_fisheye_sequence():
    """100 frames through the lens: initialisation, keyframes, local BA, and poses within 0.3 % of the path length and 0.5
    degrees of the truth after the similarity a monocular map leaves open (measured: 0.07 %, 0.14 degrees).  The same frames
    on a pinhole System keep a track whose rotation is off by degrees (measured: 24 degrees)."""
    from alvaar_b200 import synth
    frames, poses = system_frames()
    K = synth.intrinsics(640, 480)
    S = cpu_system_lib()
    tr, nba = run_cpu_system(S, frames, K)
    st = np.array([r[0] for r in tr])
    T = np.array([r[1] for r in tr])
    info = np.array([r[2] for r in tr])
    init = int(np.argmax(st == 1))
    assert 0 < init < 25 and (st[init:] == 1).all(), st
    assert info[-1][5] >= 5 and nba >= 3, (info[-1], nba)
    pos, rot = trajectory_error(T, poses, np.arange(init, len(st)))
    print(f"fisheye: init frame {init}, {info[-1][5]} keyframes, {nba} local BAs, position error {pos:.2e} of the path, rotation {rot:.3f} deg")
    assert pos < 3e-3 and rot < 0.5, (pos, rot)
    assert tr[-1][7] == 0                                          # this lens undistorts every pixel of the frame
    tr0, _ = run_cpu_system(S, frames, K, lens=None)
    st0 = np.array([r[0] for r in tr0])
    tracked = np.flatnonzero(st0 == 1)
    pos0, rot0 = trajectory_error(np.array([r[1] for r in tr0]), poses, tracked) if len(tracked) > 10 else (np.inf, np.inf)
    print(f"pinhole on the same frames: {len(tracked)} tracked, position error {pos0:.2e}, rotation {rot0:.2f} deg")
    assert len(tracked) < 50 or rot0 > 5.0 or pos0 > 0.01


def test_points_the_model_cannot_undistort_are_dropped():
    """a lens whose Newton iteration fails beyond theta_d ~0.57 on frames whose corners reach 0.69: the corner keypoints are
    dropped when detected and when tracked, counted, and never reach the frame (no (-1e6, -1e6) among its points)"""
    from alvaar_b200 import synth
    frames, _ = synth.make_frames(12, 640, 480, seed=99, rgba=True)
    K = synth.intrinsics(640, 480)
    S = cpu_system_lib()
    tr, _ = run_cpu_system(S, frames, K, lens=(-0.5, 0.05, 0.0, 0.0))
    assert tr[-1][7] > 0 and all(b >= a for a, b in zip([r[7] for r in tr], [r[7] for r in tr][1:]))
    for st, T, info, ids, px, d3, xy, drops in tr:
        assert len(ids) > 50 and not (xy == -1000000).any()
        x, y = (px[:, 0].astype(np.float64) - K[2]) / K[0], (px[:, 1].astype(np.float64) - K[3]) / K[1]
        assert (np.hypot(x, y) < 0.58).all()


def test_disabled_fisheye_is_the_pinhole():
    """set_fisheye(0, ...) on the CPU state machine is bit-identical to never calling it"""
    from alvaar_b200 import synth
    frames, _ = synth.make_frames(30, 640, 480, seed=99, rgba=True)
    K = synth.intrinsics(640, 480)
    S = cpu_system_lib()
    a, _ = run_cpu_system(S, frames, K, lens=None)
    b = []
    s = S.cpu_fish_system_create(640, 480, *K)
    S.cpu_fish_system_set_fisheye(s, 0, 0.1, 0.2, 0.3, 0.4)
    for k in range(len(frames)):
        T = np.zeros(7)
        st = S.cpu_fish_system_process(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(T))
        b.append((st, T))
    S.cpu_fish_system_destroy(s)
    for (sa, Ta, *_), (sb, Tb) in zip(a, b):
        assert sa == sb and (Ta == Tb).all()


def test_system_switch_error_codes_without_a_device():
    """alva_system_set_fisheye before configure -> ALVA_E_STATE; a null handle -> ALVA_E_INVALID"""
    from alvaar_b200 import lib
    L = lib()
    L.alva_system_create.restype = C.c_void_p
    L.alva_system_destroy.argtypes = [C.c_void_p]
    L.alva_system_set_fisheye.argtypes = [C.c_void_p, C.c_int] + [C.c_double] * 4
    L.alva_system_lens_drops.argtypes = [C.c_void_p]
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_fisheye(s, 1, *SYSTEM_FISHEYE) == -4
    assert L.alva_system_set_fisheye(s, 1, float("nan"), 0, 0, 0) == -4          # the state is checked first
    assert L.alva_system_set_fisheye(None, 1, *SYSTEM_FISHEYE) == -1
    assert L.alva_system_lens_drops(None) == -1
    L.alva_system_destroy(s)
