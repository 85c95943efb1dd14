"""CPU tests of OpenCV's whole distortion vector (k3, the rational, thin-prism and tilted models; alva_system_set_distortion_coeffs).

The host side of alvaar_b200/csrc/camera_model.h (what the kernels run, compiled for the device), the state machine's Camera
dispatch, the plain-C oracle (oracle/camera_full_oracle.c) and OpenCV's own cv::undistortPoints / cv::projectPoints agree on
every point of every lens of tests/golden/camera_full.npz -- live when oracle/_ref/libalva_ref_distortion_full.so is built,
else through the stored digests.  The bar is identical float bits, with the rounding-boundary exemption of
tests/test_oracle_fisheye.py counted (0 on every lens).  The vector (k1, k2, p1, p2, 0, ..., 0) gives the bits of the
four-coefficient functions on the inputs of tests/golden/camera.npz."""
import ctypes as C

import numpy as np
import pytest

import camera_util
from camera_full_util import (CASES, NAMES, case_K, case_pixels, case_points, host_lib, n_fold, oracle_lib, ref_lib,
                              rounding_exempt, run_cam, run_points, run_ref)
from camera_util import cdigest, same_bits
from conftest import P, golden
from ref_golden import digest


def opencv_results(k, hu, hp):
    """OpenCV's float results and the doubles of those that differ from the header's: live from the library when it is built,
    else the header's bits with the stored differences patched in (which must hash to OpenCV's digest)"""
    g = golden("camera_full")
    name = NAMES[k]
    R = ref_lib()
    if R is not None:
        K, D = case_K(k)
        ru, ru64 = run_ref(R.ref_full_undistort_points, case_pixels(k), K, D)
        rp, rp64 = run_ref(R.ref_full_project_points, case_points(k), K, D)
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
    g = golden("camera_full")
    name = NAMES[k]
    K, D = case_K(k)
    px, X = case_pixels(k), case_points(k)
    assert (digest(px) == g[f"{name}/px"]).all() and (digest(X) == g[f"{name}/X"]).all(), "case generator changed: re-dump camera_full.npz"
    assert (g[f"{name}/K"] == K).all() and (g[f"{name}/D"] == D).all()
    H, O = host_lib(), oracle_lib()
    hu, hp = run_points(H.cpu_full_undistort_points, px, K, D), run_points(H.cpu_full_project_points, X, K, D)
    assert same_bits(hu, run_points(O.orc_full_undistort_points, px, K, D))
    assert same_bits(hp, run_points(O.orc_full_project_points, X, K, D))
    lens, cu = run_cam(H, px, K, D, 0)                               # what the state machine calls
    assert lens == 3 and same_bits(hu, cu)
    lens, cp = run_cam(H, X, K, D, 1)
    assert lens == 3 and same_bits(hp, cp)
    ru, ru64, rp, rp64 = opencv_results(k, hu, hp)
    assert (cdigest(ru) == g[f"{name}/unpx"]).all() and (cdigest(rp) == g[f"{name}/uv"]).all()
    n_exempt = 0
    for what, mine, r32, r64 in (("undistort", hu, ru, ru64), ("project", hp, rp, rp64)):
        idx, ok = rounding_exempt(mine, r32, r64)
        assert ok.all(), f"{what}: {int((~ok).sum())} float results differ from OpenCV's away from a rounding boundary, e.g. flat index {idx[~ok][:4]}"
        n_exempt += len(idx)
    print(f"{name}: {2 * (len(px) + len(X))} float results, {n_exempt} exempt at a float rounding boundary")


def test_cases_cover_the_model_branches():
    g = golden("camera_full")
    assert int(g["fold_back_640x480/n_fold"]) > 100                 # icdist < 0: the pinhole fallback
    for name in NAMES[:4]:
        assert int(g[f"{name}/n_fold"]) == 0
    assert [len(c[3]) for c in CASES] == [5, 8, 12, 14, 5]
    k = NAMES.index("fold_back_640x480")
    K, D = case_K(k)
    assert n_fold(case_pixels(k), K, D) == int(g["fold_back_640x480/n_fold"])
    X = case_points(0)
    assert (X[:, 2] < 0).sum() >= 1000 and (X[:, 2] == 0).sum() >= 1000
    H = host_lib()
    t, it = np.zeros(9), np.zeros(9)
    assert H.cpu_full_tilt(P(np.ascontiguousarray(case_K(3)[1])), 14, P(t), P(it)) == 0
    assert not np.allclose(t, np.eye(3).ravel()) and np.allclose(t.reshape(3, 3) @ it.reshape(3, 3) / (t.reshape(3, 3) @ it.reshape(3, 3))[2, 2], np.eye(3))


@pytest.mark.parametrize("k", range(len(camera_util.CASES)), ids=[c[0] for c in camera_util.CASES])
def test_four_coefficients_padded_with_zeros_are_the_radial_tangential_model(k):
    """(k1, k2, p1, p2, 0, ..., 0) at every length: the bits of undistort_point / project_dist and of OpenCV's
    tests/golden/camera.npz digests, and the state machine chooses lens 1 for it"""
    g = golden("camera")
    name = camera_util.CASES[k][0]
    K, D4 = camera_util.case_K(k)
    px, X = camera_util.case_pixels(k), camera_util.case_points(k)
    S, H = camera_util.cpu_dist_system_lib(), host_lib()
    want_un = camera_util.run_points(S.cpu_radtan_undistort_points, px, K, D4)
    want_uv = camera_util.run_points(S.cpu_radtan_project_points, X, K, D4)
    assert (cdigest(want_un) == g[f"{name}/unpx"]).all() and (cdigest(want_uv) == g[f"{name}/uv"]).all()
    for n in (4, 5, 8, 12, 14):
        D = np.zeros(n)
        D[:4] = D4
        assert same_bits(run_points(H.cpu_full_undistort_points, px, K, D), want_un)
        assert same_bits(run_points(H.cpu_full_project_points, X, K, D), want_uv)
        lens, cu = run_cam(H, px, K, D, 0)
        assert lens == 1 and same_bits(cu, want_un)


def test_lens_choice_and_refusals():
    H = host_lib()
    K = np.array([500.0, 500.0, 320.0, 240.0])
    px = np.array([[10.0, 20.0]], np.float32)
    assert run_cam(H, px, K, np.zeros(14), 0)[0] == 0                # all zero: the pinhole
    assert run_cam(H, px, K, [0.1, 0, 0, 0, 0], 0)[0] == 1
    assert run_cam(H, px, K, [0, 0, 0, 0, 0.1], 0)[0] == 3           # k3 alone
    assert run_cam(H, px, K, [0] * 13 + [0.1], 0)[0] == 3            # tau_y alone
    for D in ([0.1] * 6, [0.1] * 3, [0.0, float("nan"), 0, 0, 0], [0, 0, 0, 0, float("inf")], [0] * 12 + [np.pi / 2, 0],
              [0] * 12 + [0, -1.6]):
        assert run_cam(H, px, K, np.array(D, np.float64), 0)[0] == -1, D
    assert run_cam(H, px, K, [0] * 12 + [1.5707963, -1.5707963], 0)[0] == 3


def test_system_switch_error_codes_without_a_device():
    """alva_system_set_distortion_coeffs before configure -> ALVA_E_STATE; a null handle -> ALVA_E_INVALID"""
    from alvaar_b200 import lib
    L = lib()
    L.alva_system_create.restype = C.c_void_p
    L.alva_system_destroy.argtypes = [C.c_void_p]
    L.alva_system_set_distortion_coeffs.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    D = np.array(CASES[0][3])
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_distortion_coeffs(s, P(D), len(D)) == -4
    assert L.alva_system_set_distortion_coeffs(None, P(D), len(D)) == -1
    L.alva_system_destroy(s)


def test_renderer_follows_the_model():
    """synth renders a pixel with the ray whose projection through the lens (camera_model.h) is that pixel"""
    from alvaar_b200 import synth
    from camera_full_util import SYSTEM_RATIONAL, SYSTEM_TILTED
    H = host_lib()
    w, h = 640, 480
    K = np.array(synth.intrinsics(w, h))
    u, v = np.meshgrid(np.arange(0, w, 7, dtype=np.float64), np.arange(0, h, 5, dtype=np.float64))
    for lens in (SYSTEM_RATIONAL, SYSTEM_TILTED):
        x, y = synth.undistort_normalised_full((u.ravel() - K[2]) / K[0], (v.ravel() - K[3]) / K[1], lens)
        rays = np.ascontiguousarray(np.stack([x, y, np.ones_like(x)], 1) * 3.0)
        uv = run_points(H.cpu_full_project_points, rays, K, np.array(lens))
        assert np.abs(uv - np.stack([u.ravel(), v.ravel()], 1)).max() < 1e-3


def test_matcher_and_reacquisition_oracles_reduce_to_lens_1():
    """the lens-3 oracles (oracle/match_dist_oracle.c and oracle/reacquire_oracle.c with the 14-coefficient projection) give
    their lens-1 maps on (k1, k2, p1, p2) padded with zeros -- the check that the derived sources are the same procedures"""
    import camera_util
    import localisation_util as LU
    from alvaar_b200 import synth
    from camera_full_util import oracle_lib as full_oracle
    from match_util import ORC_ARGS
    F, O = full_oracle(), camera_util.oracle_lib()
    D4 = (-0.25, 0.08, 1e-3, -5e-4)
    p = synth.make_match_problem(33, w=640, h=480, n_kf=6, n_frame_kp=150, n_local=400, dup_frac=0.3)
    order = np.ascontiguousarray(p["local_ids"], np.int32)
    maps = []
    for fn, d in ((O.orc_match_to_map_dist, D4), (F.orc_match_to_map_full, np.concatenate([D4, np.zeros(10)]))):
        fn.argtypes = ORC_ARGS + [C.c_void_p]
        mk, mm = np.zeros(len(p["kp_id"]) + 1, np.int32), np.zeros(len(p["kp_id"]) + 1, np.int32)
        d = np.ascontiguousarray(d, np.float64)
        n = fn(p["w"], p["h"], *p["K"], P(p["cur_T"]), len(p["kp_id"]), P(p["kp_id"]), P(p["kp_px"]), 200, len(p["kf_id"]), P(p["kf_id"]),
               P(p["kf_T"]), len(p["mp_id"]), P(p["mp_id"]), P(p["mp_wpt"]), P(p["mp_is3d"]), P(p["obs_start"]), P(p["obs_kf"]), P(p["obs_px"]),
               P(p["desc_start"]), P(p["desc_kf"]), P(p["desc"]), len(order), P(order), 2.0, 0.2, P(mk), P(mm), P(d))
        maps.append(dict(zip(mk[:n].tolist(), mm[:n].tolist())))
    assert maps[0] == maps[1] and len(maps[0]) > 5
    q = LU.random_problem(np.random.default_rng(3), w=1280, h=720, lens="radtan", n_mp=3000, nq=800, max_rows=6)
    want = LU.run_oracle(LU.oracle_lib(), q)
    from camera_full_util import run_reacquire_oracle
    q.lens, q.coef = 3, np.concatenate([q.coef, np.zeros(10)])
    got = run_reacquire_oracle(q)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all() and (want[0] >= 0).sum() > 10


@pytest.mark.parametrize("lens", ["rational", "tilted"])
def test_state_machine_tracks_a_sequence_through_the_lens(lens):
    """100 frames rendered through the lens: initialisation, keyframes, local BAs, and poses within 0.2 % of the path length and
    0.6 degrees of the truth after the similarity a monocular map leaves open (measured: rational 0.048 %, 0.27 degrees; tilted
    0.094 %, 0.19 degrees; both initialise at frame 14 with 8 keyframes and 6 local BAs)"""
    from alvaar_b200 import synth
    from camera_full_util import SYSTEM_RATIONAL, SYSTEM_TILTED, cpu_system_lib, run_cpu_system, system_frames
    from fisheye_util import trajectory_error
    D = SYSTEM_RATIONAL if lens == "rational" else SYSTEM_TILTED
    frames, poses = system_frames(D)
    tr, nba = run_cpu_system(cpu_system_lib(), frames, synth.intrinsics(640, 480), D)
    st = np.array([r[0] for r in tr])
    info = np.array([r[2] for r in tr])
    init = int(np.argmax(st == 1))
    assert 0 < init < 25 and (st[init:] == 1).all(), st
    assert info[-1][5] >= 5 and nba >= 3, (info[-1], nba)
    pos, rot = trajectory_error(np.array([r[1] for r in tr]), poses, np.arange(init, len(st)))
    print(f"{lens}: init frame {init}, {info[-1][5]} keyframes, {nba} local BAs, position error {pos:.2e} of the path, rotation {rot:.3f} deg")
    assert pos < 2e-3 and rot < 0.6, (pos, rot)
    assert tr[-1][7] == 0                                          # the model never drops a point
