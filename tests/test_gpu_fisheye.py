"""GPU tests (H100) of the equidistant fisheye lens: alva_k_undistort_points_fisheye / alva_k_project_points_fisheye against the
host side of camera_model.h and OpenCV's cv::fisheye (tests/golden/fisheye.npz), alva_k_match_to_map_fisheye against the C
oracle, and System with alva_system_set_fisheye against the CPU state machine with the same lens.

Exact: both kernels on every case (NaN payloads aside; against OpenCV up to the rounding-boundary exemption of
test_oracle_fisheye.py); the matcher's maps; the System's status codes, track ids in container order, 3-D flags, keyframe counters
and dropped-point counts on every frame.  Poses: within 2e-4 * max(1, |t|) of the CPU backend -- the bar test_gpu_reloc.py uses
for the same two backends: the GPU's five-point initialisation is compiled with FMA contraction and the CPU oracle's is not, so
the poses start ~1e-7 apart and every local BA carries that on."""
import ctypes as C

import numpy as np
import pytest
import torch

from camera_util import same_bits
from conftest import P
from fisheye_util import (CASES, NAMES, SYSTEM_FISHEYE, case_K, case_pixels, case_points, cpu_system_lib, oracle_lib, rounding_exempt,
                          run_cpu_system, run_points, system_frames, trajectory_error)
from match_util import ORC_ARGS
from test_oracle_fisheye import opencv_results
from alvaar_b200 import AlvaError, System, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("k", range(len(CASES)), ids=NAMES)
def test_kernels_match_the_host_and_opencv(gpu_ctx, k):
    K, D = case_K(k)
    px, X = case_pixels(k), case_points(k)
    S = cpu_system_lib()
    want_un, want_uv = run_points(S.cpu_fish_undistort_points, px, K, D), run_points(S.cpu_fish_project_points, X, K, D)
    d_un = torch.full((len(px), 2), 7.0, dtype=torch.float32, device=DEV)
    gpu_ctx.undistort_points_fisheye(dev(px), None, 1, len(px), K, D, d_un)
    d_uv = torch.full((len(X), 2), 7.0, dtype=torch.float32, device=DEV)
    gpu_ctx.project_points_fisheye(dev(X), len(X), K, D, d_uv)
    un, uv = d_un.cpu().numpy(), d_uv.cpu().numpy()
    assert same_bits(un, want_un), np.argwhere(un != want_un)[:4]
    assert same_bits(uv, want_uv), np.argwhere((uv != want_uv) & ~(np.isnan(uv) & np.isnan(want_uv)))[:4]
    ru, ru64, rp, rp64 = opencv_results(k, want_un, want_uv)
    n = 0
    for mine, r32, r64 in ((un, ru, ru64), (uv, rp, rp64)):
        idx, ok = rounding_exempt(mine, r32, r64)
        assert ok.all()
        n += len(idx)
    print(f"{NAMES[k]}: {n} results exempt at a float rounding boundary")


def test_undistort_batched_with_counts(gpu_ctx):
    """[nframes][cap] layout: each frame's first counts[f] points, the rest left alone"""
    K, D = case_K(2)
    px = case_pixels(2)[:4 * 3000].reshape(4, 3000, 2)
    counts = np.array([3000, 1234, 0, 2999], np.int32)
    out = torch.full((4, 3000, 2), -5.0, dtype=torch.float32, device=DEV)
    gpu_ctx.undistort_points_fisheye(dev(px), dev(counts), 4, 3000, K, D, out)
    got = out.cpu().numpy()
    want = run_points(cpu_system_lib().cpu_fish_undistort_points, np.ascontiguousarray(px.reshape(-1, 2)), K, D).reshape(4, 3000, 2)
    for f in range(4):
        assert (got[f, :counts[f]] == want[f, :counts[f]]).all() and (got[f, counts[f]:] == -5.0).all(), f
    assert (want == -1e6).any()


def test_kernels_reject_bad_arguments(gpu_ctx):
    K, D = case_K(0)
    px = torch.zeros((8, 2), dtype=torch.float32, device=DEV)
    X = torch.ones((8, 3), dtype=torch.float64, device=DEV)
    out = torch.zeros((8, 2), dtype=torch.float32, device=DEV)
    for KK, DD in ((K, [float("nan"), 0, 0, 0]), (K, [0, 0, 0, float("inf")]), ([0.0, K[1], K[2], K[3]], D), ([K[0], K[1], float("nan"), K[3]], D)):
        with pytest.raises(AlvaError):
            gpu_ctx.undistort_points_fisheye(px, None, 1, 8, KK, DD, out)
        with pytest.raises(AlvaError):
            gpu_ctx.project_points_fisheye(X, 8, KK, DD, out)
    for nf, cap in ((0, 8), (1, 0)):
        with pytest.raises(AlvaError):
            gpu_ctx.undistort_points_fisheye(px, None, nf, cap, K, D, out)
    with pytest.raises(AlvaError):
        gpu_ctx.project_points_fisheye(X, 0, K, D, out)
    with pytest.raises(AlvaError):
        gpu_ctx.undistort_points_fisheye(px, None, 1, 7, K, D, out.view(-1)[1:15])    # misaligned float2 output


# ------------------------------------------------------------------------------------------------ local-map matching
def fisheye_px(px, K, k4, w, h):
    """pinhole pixels -> the pixels the fisheye lens k4 shows them at (the forward model), kept inside the image"""
    x, y = (px[:, 0] - K[2]) / K[0], (px[:, 1] - K[3]) / K[1]
    r = np.hypot(x, y)
    th = np.arctan(r)
    td = th * (1 + k4[0] * th ** 2 + k4[1] * th ** 4 + k4[2] * th ** 6 + k4[3] * th ** 8)
    s = np.where(r > 1e-8, td / np.where(r > 1e-8, r, 1), 1)
    out = np.stack([np.clip(x * s * K[0] + K[2], 1.0, w - 2.0), np.clip(y * s * K[1] + K[3], 1.0, h - 2.0)], 1)
    return np.ascontiguousarray(out.astype(np.float32))


def oracle_match_fisheye(O, p, order, nkp3d, k4):
    O.orc_match_to_map_fisheye.argtypes = ORC_ARGS + [C.c_void_p]
    mk, mm = np.zeros(len(p["kp_id"]) + 1, np.int32), np.zeros(len(p["kp_id"]) + 1, np.int32)
    order = np.ascontiguousarray(order, np.int32)
    d4 = np.ascontiguousarray(k4, np.float64)
    n = O.orc_match_to_map_fisheye(p["w"], p["h"], p["K"][0], p["K"][1], p["K"][2], p["K"][3], P(p["cur_T"]), len(p["kp_id"]), P(p["kp_id"]),
                                   P(p["kp_px"]), nkp3d, len(p["kf_id"]), P(p["kf_id"]), P(p["kf_T"]), len(p["mp_id"]), P(p["mp_id"]),
                                   P(p["mp_wpt"]), P(p["mp_is3d"]), P(p["obs_start"]), P(p["obs_kf"]), P(p["obs_px"]), P(p["desc_start"]),
                                   P(p["desc_kf"]), P(p["desc"]), len(order), P(order), 2.0, 0.2, P(mk), P(mm), P(d4))
    return dict(zip(mk[:n].tolist(), mm[:n].tolist()))


def gpu_match(ctx, p, order, nkp3d, **lens):
    idx = {int(i): k for k, i in enumerate(p["mp_id"])}
    kp_mp = np.array([idx.get(int(i), -1) for i in p["kp_id"]], np.int32)
    local_mp = np.array([idx.get(int(i), -1) for i in order], np.int32)
    out = torch.full((len(kp_mp),), -7, dtype=torch.int32, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    ctx.match_to_map(p["w"], p["h"], 40, [float(v) for v in p["K"]], dev(p["cur_T"]), dev(kp_mp), dev(p["kp_px"]), nkp3d, dev(p["kf_T"]),
                     dev(p["mp_wpt"]), dev(p["mp_is3d"]), dev(p["obs_start"]), dev(p["obs_kf"]), dev(p["obs_px"]), dev(p["desc_start"]),
                     dev(p["desc"]), dev(local_mp), out, None, cnt, **lens)
    o = out.cpu().numpy()
    assert int(cnt.item()) == int((o >= 0).sum())
    return {int(p["kp_id"][k]): int(p["mp_id"][o[k]]) for k in range(len(o)) if o[k] >= 0}


@pytest.mark.parametrize("seed,nkp,nloc,w,h", [(41, 576, 5760, 1280, 720), (42, 1296, 6000, 1920, 1080), (43, 150, 400, 640, 480)])
def test_match_to_map_fisheye_vs_oracle(gpu_ctx, seed, nkp, nloc, w, h):
    """C2 / C3-sized maps seen through the lens: the keypoints' and observations' pixels are where the lens puts them; the
    pinhole matcher finds fewer of the matches"""
    O = oracle_lib()
    p = synth.make_match_problem(seed, w=w, h=h, n_kf=30 if nkp > 200 else 6, n_frame_kp=nkp, n_local=nloc, dup_frac=0.3)
    p["kp_px"] = fisheye_px(p["kp_px"].astype(np.float64), p["K"], SYSTEM_FISHEYE, w, h)
    p["obs_px"] = fisheye_px(p["obs_px"].astype(np.float64), p["K"], SYSTEM_FISHEYE, w, h)
    order = p["local_ids"][np.random.default_rng(seed).permutation(len(p["local_ids"]))]
    zero = (0.0, 0.0, 0.0, 0.0)
    for nk in (200, 7):
        want = oracle_match_fisheye(O, p, order, nk, SYSTEM_FISHEYE)
        assert gpu_match(gpu_ctx, p, order, nk, fisheye=SYSTEM_FISHEYE) == want and len(want) > min(20, nkp // 8)
        assert gpu_match(gpu_ctx, p, order, nk, fisheye=zero) == oracle_match_fisheye(O, p, order, nk, zero)
    assert len(gpu_match(gpu_ctx, p, order, 200)) < len(gpu_match(gpu_ctx, p, order, 200, fisheye=SYSTEM_FISHEYE))
    with pytest.raises(AlvaError):
        gpu_match(gpu_ctx, p, order, 200, fisheye=(float("nan"), 0.0, 0.0, 0.0))


# ------------------------------------------------------------------------------------------------ System
def gpu_run(frames, lens=SYSTEM_FISHEYE, dist=None, max_lost=None):
    s = System(640, 480, *synth.intrinsics(640, 480))
    if lens is not None:
        s.set_fisheye(True, *lens)
    if dist is not None:
        s.set_distortion(*dist)
    if max_lost is not None:
        s.set_relocalisation(max_lost)
    out = []
    for k, f in enumerate(frames):
        st, _ = s.find_camera_pose(np.ascontiguousarray(f), k * 33.333)
        ids, px, d3, _ = s.tracks()
        xy = s.frame_points()
        out.append((st, s.pose(), s.info(), ids.copy(), px.copy(), d3.copy(), xy.copy(), s.lens_drops()))
    s.close()
    return out


def test_system_with_the_lens_equals_the_cpu_backend():
    frames, poses = system_frames()
    K = synth.intrinsics(640, 480)
    cpu, _ = run_cpu_system(cpu_system_lib(), frames, K)
    gpu = gpu_run(frames)
    worst = 0.0
    keys = ("frame", "keyframe", "keypoints", "keypoints_3d", "initialised", "keyframes", "occupied_cells", "map_point_ids")
    for k, (c, g) in enumerate(zip(cpu, gpu)):
        assert c[0] == g[0], (k, c[0], g[0])
        assert (c[2] == np.array([g[2][n] for n in keys])).all(), (k, c[2], g[2])
        assert len(c[3]) == len(g[3]) and (c[3] == g[3]).all() and (c[5] == g[5]).all(), k
        assert c[7] == g[7], (k, c[7], g[7])
        d = np.abs(c[1] - g[1]).max() / max(1.0, float(np.linalg.norm(c[1][:3])))
        worst = max(worst, d)
        assert d < 2e-4, (k, d)
    st = np.array([g[0] for g in gpu])
    init = int(np.argmax(st == 1))
    pos, rot = trajectory_error(np.array([g[1] for g in gpu]), poses, np.arange(init, len(st)))
    print(f"GPU vs CPU pose |dT| / max(1, |t|) <= {worst:.2e}; GPU vs truth: position {pos:.2e} of the path, rotation {rot:.3f} deg")
    assert (st[init:] == 1).all() and pos < 3e-3 and rot < 0.5


def test_without_the_lens_the_track_drifts():
    """negative control: the same frames on a pinhole System, and on one with a radial-tangential lens, drift by degrees -- the
    lens model's run is within 0.5 degrees (test_system_with_the_lens_equals_the_cpu_backend).  Measured on an H100: 24 degrees
    without a lens, 4.2 degrees with the radial-tangential one."""
    frames, poses = system_frames()
    for kw in (dict(lens=None), dict(lens=None, dist=(-0.25, 0.08, 0.0, 0.0))):
        out = gpu_run(frames, **kw)
        st = np.array([o[0] for o in out])
        tracked = np.flatnonzero(st == 1)
        if len(tracked) < 50:
            continue
        pos, rot = trajectory_error(np.array([o[1] for o in out]), poses, tracked)
        print(kw, f"{len(tracked)} tracked, position {pos:.2e}, rotation {rot:.2f} deg")
        assert rot > 2.0 or pos > 0.01


def test_relocalisation_through_the_lens():
    """the revisit of test_gpu_reloc.py rendered through the fisheye lens: lost after the blackout, relocalised, tracking again"""
    A, poses = synth.make_frames(40, 640, 480, seed=7, rgba=True, fisheye=SYSTEM_FISHEYE)
    black = np.zeros_like(A[0]); black[..., 3] = 255
    tex = synth.make_texture()
    from reloc_util import _mid_pose
    R = [synth.gray_to_rgba(synth.render_gray(tex, _mid_pose(poses, 15 + i), 640, 480, fisheye=SYSTEM_FISHEYE)) for i in range(24)]
    frames = list(A) + [black] * 3 + R
    out = gpu_run(frames, max_lost=10)
    st = [o[0] for o in out]
    assert 4 in st and st[-1] == 1, st
    first = st.index(4)
    assert 1 in st[first:], st


def test_switch_semantics():
    frames, _ = system_frames(30)
    plain, _ = synth.make_frames(30, 640, 480, seed=99, rgba=True)
    K = synth.intrinsics(640, 480)

    def trace(setup, fr):
        s = System(640, 480, *K)
        setup(s)
        out = []
        for k, f in enumerate(fr):
            st, pose = s.find_camera_pose(np.ascontiguousarray(f), k * 33.333)
            ids, px, d3, _ = s.tracks()
            out.append((st, pose.copy(), ids.copy(), px.copy(), d3.copy(), s.frame_points().copy()))
        s.close()
        return out

    def same(a, b):
        return all(x[0] == y[0] and all(np.array_equal(u.view(np.uint8), v.view(np.uint8)) for u, v in zip(x[1:], y[1:])) for x, y in zip(a, b))

    never = trace(lambda s: None, plain)
    assert same(trace(lambda s: s.set_fisheye(False, 0.1, 0.2, 0.3, 0.4), plain), never)          # disabled = never called
    fish = trace(lambda s: s.set_fisheye(True, *SYSTEM_FISHEYE), frames)
    assert not same(trace(lambda s: None, frames), fish)
    # later calls replace each other
    assert same(trace(lambda s: (s.set_fisheye(True, 0.3, 0, 0, 0), s.set_distortion(0, 0, 0, 0), s.set_fisheye(True, *SYSTEM_FISHEYE)), frames), fish)
    assert same(trace(lambda s: (s.set_fisheye(True, *SYSTEM_FISHEYE), s.set_distortion(0, 0, 0, 0)), plain), never)
    # reset, set_preset("default"), set_clahe(False) and set_relocalisation keep it
    assert same(trace(lambda s: (s.set_fisheye(True, *SYSTEM_FISHEYE), s.reset(), s.set_preset("default"), s.set_clahe(False),
                                 s.set_relocalisation(0)), frames), fish)
    # configure clears it
    s = System(640, 480, *K)
    s.set_fisheye(True, *SYSTEM_FISHEYE)
    assert s.L.alva_system_configure(s.h, 640, 480, *K, 0.0, 0.0, 0.0, 0.0) == 0
    out = []
    for k, f in enumerate(plain):
        st, pose = s.find_camera_pose(np.ascontiguousarray(f), k * 33.333)
        ids, px, d3, _ = s.tracks()
        out.append((st, pose.copy(), ids.copy(), px.copy(), d3.copy(), s.frame_points().copy()))
    s.close()
    assert same(out, never)
    # argument checks
    s = System(640, 480, *K)
    for bad in ((float("nan"), 0, 0, 0), (0, float("inf"), 0, 0), (0, 0, float("-inf"), 0), (0, 0, 0, float("nan"))):
        with pytest.raises(AlvaError):
            s.set_fisheye(True, *bad)
    s.close()


def test_dropped_points_match_the_cpu_backend():
    """a lens that cannot undistort the frame's corners: the same keypoints are dropped on both backends"""
    frames, _ = synth.make_frames(20, 640, 480, seed=99, rgba=True)
    K = synth.intrinsics(640, 480)
    lens = (-0.5, 0.05, 0.0, 0.0)
    cpu, _ = run_cpu_system(cpu_system_lib(), frames, K, lens=lens)
    gpu = gpu_run(frames, lens=lens)
    assert cpu[-1][7] > 0
    for k, (c, g) in enumerate(zip(cpu, gpu)):
        assert c[0] == g[0] and c[7] == g[7] and (c[3] == g[3]).all(), k
