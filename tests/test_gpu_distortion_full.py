"""GPU tests (H100) of OpenCV's whole distortion vector: alva_k_undistort_points_full / alva_k_project_points_full against
OpenCV's digests (tests/golden/camera_full.npz) and the host build of camera_model.h; the lens-3 matcher and re-acquisition
against their C oracles (orc_match_to_map_full, orc_match_frame_to_map_full) on rational, thin-prism and tilted lenses, and
against lens 1 on a (k1, k2, p1, p2) vector padded with zeros; the rotated priors against the host arithmetic; the System with
alva_system_set_distortion_coeffs in lockstep with the CPU backend on sequences rendered through the rational and the tilted
lens, the padded vector giving set_distortion's trace and map blob bit for bit, and a lens-3 map round trip."""

import numpy as np
import pytest
import torch

import ctypes as C

from camera_full_util import (CASES, NAMES, SYSTEM_RATIONAL, SYSTEM_TILTED, case_K, case_pixels, case_points, cpu_system_lib, host_lib,
                              run_cpu_system, run_points, system_frames)
from camera_util import SYSTEM_DIST, cdigest, same_bits
from conftest import P, golden
from fisheye_util import trajectory_error
from alvaar_b200 import AlvaError, System, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("k", range(len(CASES)), ids=NAMES)
def test_kernels_equal_opencv(gpu_ctx, k):
    g = golden("camera_full")
    name = NAMES[k]
    K, D = case_K(k)
    px, X = case_pixels(k), case_points(k)
    d_un = torch.full((len(px), 2), 7.0, dtype=torch.float32, device=DEV)
    gpu_ctx.undistort_points_full(dev(px), None, 1, len(px), K, D, d_un)
    d_uv = torch.full((len(X), 2), 7.0, dtype=torch.float32, device=DEV)
    gpu_ctx.project_points_full(dev(X), len(X), K, D, d_uv)
    torch.cuda.synchronize()
    un, uv = d_un.cpu().numpy(), d_uv.cpu().numpy()
    assert (cdigest(un) == g[f"{name}/unpx"]).all() and len(g[f"{name}/unpx_diff"]) == 0
    assert (cdigest(uv) == g[f"{name}/uv"]).all() and len(g[f"{name}/uv_diff"]) == 0
    H = host_lib()
    assert same_bits(un, run_points(H.cpu_full_undistort_points, px, K, D))
    assert same_bits(uv, run_points(H.cpu_full_project_points, X, K, D))


def test_kernels_refuse_bad_vectors(gpu_ctx):
    K, D = case_K(3)
    px = dev(case_pixels(3)[:64])
    out = torch.zeros((64, 2), dtype=torch.float32, device=DEV)
    for bad in (list(D[:6]), [float("nan")] + list(D[1:]), list(D[:12]) + [np.pi / 2, 0.0], list(D[:13]) + [-2.0]):
        with pytest.raises(AlvaError):
            gpu_ctx.undistort_points_full(px, None, 1, 64, K, bad, out)
        with pytest.raises(AlvaError):
            gpu_ctx.project_points_full(dev(case_points(3)[:64]), 64, K, bad, out)


def test_undistort_batched_with_counts(gpu_ctx):
    K, D = case_K(1)
    px = case_pixels(1)[:3 * 500].reshape(3, 500, 2)
    counts = dev(np.array([500, 17, 0], np.int32))
    out = torch.full((3, 500, 2), 7.0, dtype=torch.float32, device=DEV)
    gpu_ctx.undistort_points_full(dev(px), counts, 3, 500, K, D, out)
    o = out.cpu().numpy()
    want = run_points(host_lib().cpu_full_undistort_points, np.ascontiguousarray(px.reshape(-1, 2)), K, D).reshape(3, 500, 2)
    assert same_bits(o[0], want[0]) and same_bits(o[1, :17], want[1, :17]) and (o[1, 17:] == 7).all() and (o[2] == 7).all()


def padded(d4, n=14):
    D = np.zeros(n)
    D[:4] = d4
    return D


def distort_full_px(px, K, D, w, h):
    """pinhole pixels -> the pixels the lens D shows them at (camera_model.h's projection of the ray), kept inside the image"""
    rays = np.ascontiguousarray(np.stack([(px[:, 0] - K[2]) / K[0], (px[:, 1] - K[3]) / K[1], np.ones(len(px))], 1))
    uv = run_points(host_lib().cpu_full_project_points, rays, K, D).astype(np.float64)
    return np.ascontiguousarray(np.stack([np.clip(uv[:, 0], 1.0, w - 2.0), np.clip(uv[:, 1], 1.0, h - 2.0)], 1).astype(np.float32))


def oracle_match_full(p, order, nkp3d, D):
    from camera_full_util import oracle_lib
    from match_util import ORC_ARGS
    O = oracle_lib()
    O.orc_match_to_map_full.argtypes = ORC_ARGS + [C.c_void_p]
    mk, mm = np.zeros(len(p["kp_id"]) + 1, np.int32), np.zeros(len(p["kp_id"]) + 1, np.int32)
    order = np.ascontiguousarray(order, np.int32)
    d = np.zeros(14)
    d[:len(D)] = D
    n = O.orc_match_to_map_full(p["w"], p["h"], p["K"][0], p["K"][1], p["K"][2], p["K"][3], P(p["cur_T"]), len(p["kp_id"]), P(p["kp_id"]),
                                P(p["kp_px"]), nkp3d, len(p["kf_id"]), P(p["kf_id"]), P(p["kf_T"]), len(p["mp_id"]), P(p["mp_id"]),
                                P(p["mp_wpt"]), P(p["mp_is3d"]), P(p["obs_start"]), P(p["obs_kf"]), P(p["obs_px"]), P(p["desc_start"]),
                                P(p["desc_kf"]), P(p["desc"]), len(order), P(order), 2.0, 0.2, P(mk), P(mm), P(d))
    return dict(zip(mk[:n].tolist(), mm[:n].tolist())), n


def gpu_match_full(ctx, p, order, nkp3d, coeffs):
    idx = {int(i): k for k, i in enumerate(p["mp_id"])}
    kp_mp = np.array([idx.get(int(i), -1) for i in p["kp_id"]], np.int32)
    local_mp = np.array([idx.get(int(i), -1) for i in order], np.int32)
    out = torch.full((len(kp_mp),), -7, dtype=torch.int32, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    ctx.match_to_map(p["w"], p["h"], 40, [float(v) for v in p["K"]], dev(p["cur_T"]), dev(kp_mp), dev(p["kp_px"]), nkp3d, dev(p["kf_T"]),
                     dev(p["mp_wpt"]), dev(p["mp_is3d"]), dev(p["obs_start"]), dev(p["obs_kf"]), dev(p["obs_px"]), dev(p["desc_start"]),
                     dev(p["desc"]), dev(local_mp), out, None, cnt, coeffs=coeffs)
    o = out.cpu().numpy()
    return {int(p["kp_id"][k]): int(p["mp_id"][o[k]]) for k in range(len(o)) if o[k] >= 0}, int(cnt.item())


MATCH_LENSES = {"rational": SYSTEM_RATIONAL, "thin_prism": CASES[2][3], "tilted": CASES[3][3]}


@pytest.mark.parametrize("lens", list(MATCH_LENSES))
@pytest.mark.parametrize("seed,nkp,nloc,w,h", [(31, 576, 5760, 1280, 720), (32, 1296, 6000, 1920, 1080), (33, 150, 400, 640, 480)])
def test_match_to_map_full_vs_oracle(gpu_ctx, lens, seed, nkp, nloc, w, h):
    """C2 / C3-sized maps seen through the lens (keypoints and observations where the lens puts them): the lens-3 matcher's
    kp_match and n_match equal orc_match_to_map_full's exactly; the padded (k1, k2, p1, p2) vector gives lens 1's map"""
    from test_gpu_distortion import gpu_match_dist
    D = np.array(MATCH_LENSES[lens])
    p = synth.make_match_problem(seed, w=w, h=h, n_kf=30 if nkp > 200 else 6, n_frame_kp=nkp, n_local=nloc, dup_frac=0.3)
    K = np.array(p["K"], np.float64)
    p["kp_px"] = distort_full_px(p["kp_px"].astype(np.float64), K, D, w, h)
    p["obs_px"] = distort_full_px(p["obs_px"].astype(np.float64), K, D, w, h)
    order = p["local_ids"][np.random.default_rng(seed).permutation(len(p["local_ids"]))]
    for nk in (200, 7):
        want, n_want = oracle_match_full(p, order, nk, D)
        got, n_got = gpu_match_full(gpu_ctx, p, order, nk, D)
        assert got == want and n_got == n_want and len(want) > min(20, nkp // 8), (len(got), len(want))
        # the four-coefficient part alone, through lens 3 and lens 1: the same map
        assert gpu_match_full(gpu_ctx, p, order, nk, padded(D[:4]))[0] == gpu_match_dist(gpu_ctx, p, order, nk, tuple(D[:4]))
    with pytest.raises(AlvaError):
        gpu_match_full(gpu_ctx, p, order, 200, list(D[:6]))


def test_rotate_priors_lens_3(gpu_ctx):
    """the gyro prior of lens 3: the host arithmetic on every test lens, and lens 1's bits on a padded vector"""
    rng = np.random.default_rng(7)
    n = 4000
    ang = 0.03
    R = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]]).ravel()
    bv = rng.normal(size=(n, 3))
    bv[:, 2] = np.abs(bv[:, 2]) * 3
    bv /= np.linalg.norm(bv, axis=1, keepdims=True)
    flag = (rng.uniform(size=n) < 0.8).astype(np.uint8)

    def run(K, D, lens, w, h):
        prior = torch.full((n, 2), -3.0, dtype=torch.float32, device=DEV)
        rot = torch.zeros(n, dtype=torch.uint8, device=DEV)
        gpu_ctx.rotate_priors(dev(bv), dev(flag), n, w, h, K, D, lens, R, prior, rot)
        return prior.cpu().numpy(), rot.cpu().numpy()

    H = host_lib()
    for k, (name, w, h, _) in enumerate(CASES):
        K, D = case_K(k)
        pr, rot = run(K, np.concatenate([D, np.zeros(14 - len(D))]), 3, w, h)
        c = np.ascontiguousarray(bv @ R.reshape(3, 3))                 # R^T bv, per row
        uv = run_points(H.cpu_full_project_points, c, K, D)
        ok = flag.astype(bool) & (c[:, 2] > 0) & (uv[:, 0] >= 0) & (uv[:, 1] >= 0) & (uv[:, 0] < w) & (uv[:, 1] < h)
        assert (rot.astype(bool) == ok).all() and ok.sum() > 100, name
        assert np.allclose(pr[ok], uv[ok], atol=1e-3) and (pr[~ok] == -3.0).all(), name
    K, _ = case_K(0)
    a, ra = run(K, SYSTEM_DIST, 1, 640, 480)
    b, rb = run(K, padded(SYSTEM_DIST), 3, 640, 480)
    assert same_bits(a, b) and (ra == rb).all()


@pytest.mark.parametrize("lens", list(MATCH_LENSES))
@pytest.mark.parametrize("cell", [40, 50])
def test_match_frame_to_map_lens_3_vs_oracle(gpu_ctx, monkeypatch, lens, cell):
    """re-acquisition with lens 3: the queries are planted at the lens-3 projections of the table's points, and q_row / q_dist
    equal orc_match_frame_to_map_full's exactly; the padded (k1, k2, p1, p2) vector gives lens 1's result"""
    import localisation_util as LU
    from camera_full_util import oracle_lib, run_reacquire_oracle
    from test_gpu_localisation import run_gpu
    D14 = np.zeros(14)
    D = MATCH_LENSES[lens]
    D14[:len(D)] = D
    F = oracle_lib()

    class Shim:   # random_problem plants its queries at the projections of lens 2's slot: point that slot at the full model
        orc_fisheye_project_points = F.orc_full14_project_points
    for k, ((w, h), n_mp, nq, rows) in enumerate([((1280, 720), 10000, 2000, 30), ((1920, 1080), 100000, 8192, 32)]):
        with monkeypatch.context() as m:
            m.setitem(LU.LENSES, "full", (2, tuple(D14)))
            m.setattr(LU, "oracle_lib", lambda: Shim)
            p = LU.random_problem(np.random.default_rng(77 * cell + k), w=w, h=h, cell=cell, lens="full", n_mp=n_mp, nq=nq,
                                  max_rows=rows, radius=2.0)
        p.lens, p.coef = 3, np.array(D14)
        want = run_reacquire_oracle(p)
        got = run_gpu(gpu_ctx, p)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all() and (want[0] >= 0).sum() > 50, ((got[0] != want[0]).sum(), (want[0] >= 0).sum())
        p.lens, p.coef = 1, np.array(D14[:4])
        want1 = run_gpu(gpu_ctx, p)
        p.lens, p.coef = 3, padded(D14[:4])
        got1 = run_gpu(gpu_ctx, p)
        assert (got1[0] == want1[0]).all() and (got1[1] == want1[1]).all()


# ------------------------------------------------------------------------------------------------ System
def frames(n):
    f, _ = synth.make_frames(n, 640, 480, seed=99, rgba=True, dist=SYSTEM_DIST)
    return f


def trace(s, fr):
    out = []
    for k in range(len(fr)):
        st, pose = s.find_camera_pose(np.ascontiguousarray(fr[k]), k * 33.333)
        ids, px, d3, _ = s.tracks()
        out.append((st, pose.copy(), ids.copy(), px.copy(), d3.copy(), tuple(s.info().values())))
    return out


def new_system():
    return System(640, 480, *synth.intrinsics(640, 480))


def test_padded_vector_is_set_distortion_bit_for_bit():
    fr = frames(60)
    a, b = new_system(), new_system()
    for s in (a, b):
        s.set_relocalisation(5)
    a.set_distortion(*SYSTEM_DIST)
    b.set_distortion_coeffs(padded(SYSTEM_DIST, 5))
    ta, tb = trace(a, fr), trace(b, fr)
    for x, y in zip(ta, tb):
        assert x[0] == y[0] and (x[1] == y[1]).all() and (x[2] == y[2]).all() and (x[3] == y[3]).all() and (x[4] == y[4]).all() and x[5] == y[5]
    assert ta[-1][0] == 1 and a.save_map() == b.save_map()
    a.close(); b.close()


def gpu_run(frames, lens):
    s = new_system()
    s.set_distortion_coeffs(lens)
    out = []
    for k, f in enumerate(frames):
        st, _ = s.find_camera_pose(np.ascontiguousarray(f), k * 33.333)
        ids, px, d3, _ = s.tracks()
        out.append((st, s.pose(), s.info(), ids.copy(), px.copy(), d3.copy(), s.frame_points().copy(), s.lens_drops()))
    s.close()
    return out


@pytest.mark.parametrize("lens", ["rational", "tilted"])
def test_system_with_the_lens_equals_the_cpu_backend(lens):
    """100 frames rendered through the lens: the GPU System and the CPU backend agree in statuses and lens drops on every
    frame, poses within 2e-4 (the fisheye lockstep's tolerance), and in ids, 3-D flags and counters on at least 80 frames; the
    GPU track is within the CPU test's bounds of the truth.

    The two backends' poses are not bit-identical (measured up to 1.6e-4), and the pose sets the KLT priors of 3-D keypoints, so
    a tracked pixel can differ by ~1e-3 px and a keypoint that sits on a gate can be kept by one backend and dropped by the
    other.  On the tilted sequence this happens once: keypoint 236 lands on x = 400.0 at frame 84 on the CPU (398.0497 vs
    398.0486 at frame 83) and is dropped on the GPU; the two keypoint sets differ by that one point until the map replaces it,
    and agree again from frame 98 (14 frames).  Such a frame is allowed only as a difference of at most two keypoints, with the frame,
    keyframe and map point counters equal."""
    D = SYSTEM_RATIONAL if lens == "rational" else SYSTEM_TILTED
    fr, poses = system_frames(D)
    cpu, _ = run_cpu_system(cpu_system_lib(), fr, synth.intrinsics(640, 480), D)
    gpu = gpu_run(fr, D)
    keys = ("frame", "keyframe", "keypoints", "keypoints_3d", "initialised", "keyframes", "occupied_cells", "map_point_ids")
    worst, near = 0.0, []
    for k, (c, g) in enumerate(zip(cpu, gpu)):
        assert c[0] == g[0], (k, c[0], g[0])
        assert c[7] == g[7] == 0, (k, c[7], g[7])
        d = np.abs(c[1] - g[1]).max() / max(1.0, float(np.linalg.norm(c[1][:3])))
        worst = max(worst, d)
        assert d < 2e-4, (k, d)
        gi = np.array([g[2][n] for n in keys])
        if (c[2] == gi).all() and len(c[3]) == len(g[3]) and (c[3] == g[3]).all() and (c[5] == g[5]).all():
            continue
        near.append(k)
        sym = set(c[3].tolist()) ^ set(g[3].tolist())
        diff = np.abs(c[2] - gi)
        assert len(sym) <= 2 and (diff[[0, 1, 4, 5, 7]] == 0).all() and (diff <= 2).all(), (k, sym, c[2], gi)
    st = np.array([g[0] for g in gpu])
    init = int(np.argmax(st == 1))
    pos, rot = trajectory_error(np.array([g[1] for g in gpu]), poses, np.arange(init, len(st)))
    print(f"{lens}: GPU vs CPU pose |dT| / max(1, |t|) <= {worst:.2e}, frames one keypoint apart: {near}; "
          f"GPU vs truth: position {pos:.2e} of the path, rotation {rot:.3f} deg")
    assert len(near) <= 20 and 0 < init < 25 and (st[init:] == 1).all() and pos < 2e-3 and rot < 0.6


def test_lens_3_system_round_trips_its_map():
    """a System tracking the tilted sequence: its blob (lens 3, 14 coefficients) loads back into a System with the same lens and
    saves byte for byte, and is refused under set_distortion's lens and under another 14-entry vector"""
    D = np.array(SYSTEM_TILTED)
    fr, _ = system_frames(SYSTEM_TILTED, n=60)
    s = new_system()
    s.set_relocalisation(5)
    s.set_distortion_coeffs(D)
    tr = trace(s, fr)
    st = np.array([t[0] for t in tr])
    init = int(np.argmax(st == 1))
    assert 0 < init < 25 and (st[init:] == 1).all() and s.info()["keyframes"] >= 4 and s.lens_drops() == 0, st
    blob = s.save_map()
    t = new_system()
    t.set_relocalisation(5)
    t.set_distortion_coeffs(D)
    t.load_map(blob)
    assert t.save_map() == blob
    u = new_system()
    u.set_relocalisation(5)
    u.set_distortion(*D[:4])
    with pytest.raises(AlvaError):
        u.load_map(blob)
    D2 = D.copy()
    D2[13] = 0.0
    u.set_distortion_coeffs(D2)
    with pytest.raises(AlvaError):
        u.load_map(blob)
    with pytest.raises(AlvaError):
        u.set_distortion_coeffs(D[:6])
    for x in (s, t, u):
        x.close()
