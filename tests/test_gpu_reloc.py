"""GPU tests (H100) of System's relocalisation (alva_system_set_relocalisation): alva_k_hamming_knn2_grouped exact against the
oracle at its structural limits, alva_k_p3p_ransac against the oracle at the bar of the LMedS tests (same hypothesis, same inlier
set, pose 1e-9), and System on the GPU through the sequences of test_system_reloc_cpu.py against the CPU backend (status, ids in
order and 3-D flags exact, poses at test_gpu_system.py's CPU-vs-GPU bar through the relocalisation: see compare_with_cpu)."""
import ctypes as C

import numpy as np
import pytest
import torch

import reloc_util as U
from alvaar_b200 import System, lib, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.fixture(scope="module")
def L():
    return U.reloc_oracle_lib()


# ------------------------------------------------------------------------------------------------ grouped 2-NN
def _table(name):
    rng = np.random.default_rng(["tiny", "c2", "max_nq", "empty", "single", "chunk_inside", "chunk_between"].index(name) + 101)
    if name == "tiny":
        return U.random_table(rng, 5, 3, 7)
    if name == "c2":       # 30 keyframes x 600 map points, up to 30 descriptors each
        return U.random_table(rng, 18000, 30, 256)
    if name == "max_nq":   # the frame capacity at 1920x1080 under ACCURATE (35-px cells)
        return U.random_table(rng, 3000, 8, 6884)
    if name == "empty":
        return rng.integers(0, 256, (100, 32), dtype=np.uint8), np.zeros(1, np.int32), np.zeros((0, 32), np.uint8)
    if name == "single":
        return U.random_table(rng, 1, 30, 300, min_rows=30)
    if name == "chunk_inside":   # 30-row groups: the 2048-row chunk boundaries fall inside groups
        return U.random_table(rng, 300, 30, 500, min_rows=30)
    # groups of 2048 / 1024 rows: the chunk boundaries fall between groups
    rows = np.array([2048, 1024, 1024, 2048, 1, 2047], np.int32)
    ds = np.concatenate([[0], np.cumsum(rows)]).astype(np.int32)
    d = rng.integers(0, 256, (int(ds[-1]), 32), dtype=np.uint8)
    q = d[rng.integers(0, len(d), 200)] ^ np.packbits(rng.random((200, 256)) < 0.1, axis=1)
    return q, ds, d


@pytest.mark.parametrize("name", ["tiny", "c2", "max_nq", "empty", "single", "chunk_inside", "chunk_between"])
def test_knn2_grouped_exact(gpu_ctx, L, name):
    q, ds, d = _table(name)
    nq, ng, nr = len(q), len(ds) - 1, len(d)
    out = torch.full((nq, 4), 7, dtype=torch.int32, device=DEV)
    dd = dev(d) if nr else torch.zeros((1, 32), dtype=torch.uint8, device=DEV)
    gpu_ctx.hamming_knn2_grouped(dev(q), nq, dev(ds), ng, dd, nr, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = U.knn2_grouped_oracle(L, q, ds, d)
    assert (got == want).all(), np.argwhere((got != want).any(1))[:5]
    if name == "empty":
        assert (got == -1).all()
    if name in ("c2", "max_nq", "chunk_inside", "chunk_between"):
        assert (got[:, 1] <= 51).sum() > nq // 4    # the planted queries found their groups


# ------------------------------------------------------------------------------------------------ P3P-RANSAC
def _problems(nprob, n, shares, seeds, w=1280, h=720):
    prs = [synth.make_pose_problem(n=n, seed=s, w=w, h=h, noise_px=0.0 if k == 0 else 0.5, outlier_frac=f)
           for k, (s, f) in enumerate(zip(seeds, shares))]
    return prs[:nprob]


def test_p3p_ransac_matches_the_oracle_batched(gpu_ctx, L):
    """three problems in one launch (80 %, 60 % and 40 % outliers, noise 0 / 0.5 / 0.5 px): the selected hypothesis, the inlier
    set and the pose (1e-9) equal the oracle's"""
    n = 400
    prs = _problems(3, n, (0.8, 0.6, 0.4), (4, 9, 12))
    fx = float(prs[0]["K"][0])
    bv = np.stack([p["bv"] for p in prs]); X = np.stack([p["X"] for p in prs])
    counts = np.array([n, n - 37, n - 100], np.int32)
    T = torch.zeros((3, 12), dtype=torch.float64, device=DEV); o = torch.zeros((3, n), dtype=torch.uint8, device=DEV)
    info = torch.zeros((3, 4), dtype=torch.float64, device=DEV)
    gpu_ctx.p3p_ransac(3, n, dev(bv), dev(X), dev(counts), T, o, info, max_iter=512, fx=fx, fy=fx)
    torch.cuda.synchronize()
    T, o, info = T.cpu().numpy(), o.cpu().numpy(), info.cpu().numpy()
    for p in range(3):
        m = int(counts[p])
        To = np.zeros(12); oo = np.zeros(m, np.uint8); io = np.zeros(3)
        ok = L.orc_p3p_ransac(U.P(np.ascontiguousarray(bv[p, :m])), U.P(np.ascontiguousarray(X[p, :m])), m, 512, 3.0, fx, fx, 12345,
                              U.P(To), U.P(oo), U.P(io))
        assert int(info[p, 0]) == ok == 1, p
        assert int(info[p, 2]) == int(io[1]) and int(info[p, 1]) == int(io[0]) and int(info[p, 3]) == int(io[2]), (p, info[p], io)
        assert (o[p, :m] == oo).all() and (o[p, m:] == 1).all(), p
        assert np.abs(T[p] - To).max() < 1e-9, p


def test_p3p_lmeds_unchanged_beside_ransac(gpu_ctx, oracle):
    """LMedS before and after a RANSAC call on the same context (they share the sampler table): bit-identical, and equal to
    the LMedS oracle"""
    import ctypes
    n = 300
    pr = synth.make_pose_problem(n=n, seed=21, w=1280, h=720, outlier_frac=0.2)
    fx = float(pr["K"][0])
    bv, X = dev(pr["bv"]), dev(pr["X"])

    def lmeds():
        T = torch.zeros(12, dtype=torch.float64, device=DEV); o = torch.zeros(n, dtype=torch.uint8, device=DEV)
        info = torch.zeros(4, dtype=torch.float64, device=DEV)
        gpu_ctx.p3p_lmeds(1, n, bv, X, None, T, o, info, max_iter=100, fx=fx, fy=fx)
        torch.cuda.synchronize()
        return T.cpu().numpy(), o.cpu().numpy(), info.cpu().numpy()
    a = lmeds()
    T = torch.zeros(12, dtype=torch.float64, device=DEV); o = torch.zeros(n, dtype=torch.uint8, device=DEV)
    gpu_ctx.p3p_ransac(1, n, bv, X, None, T, o, None, max_iter=1024, fx=fx, fy=fx)
    b = lmeds()
    assert all((x == y).all() for x, y in zip(a, b))
    oracle.orc_p3p_lmeds.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                                             ctypes.c_uint32] + [ctypes.c_void_p] * 3
    To = np.zeros(12); oo = np.zeros(n, np.uint8); io = np.zeros(3)
    ok = oracle.orc_p3p_lmeds(U.P(pr["bv"]), U.P(pr["X"]), n, 100, 3.0, fx, fx, 12345, U.P(To), U.P(oo), U.P(io))
    assert ok == int(a[2][0]) and (oo == a[1]).all() and np.abs(To - a[0]).max() < 1e-9


# ------------------------------------------------------------------------------------------------ System
class GpuRun:
    def __init__(self, max_lost=None, preset=None, dist=None):
        K = synth.intrinsics(U.W, U.H)
        self.s = System(U.W, U.H, *K)
        if preset is not None:
            self.s.set_preset(["default", "fast", "average", "accurate"][preset])
        if dist is not None:
            self.s.set_distortion(*dist)
        if max_lost is not None:
            self.s.set_relocalisation(max_lost)

    def frame(self, rgba, t_ms):
        st, _ = self.s.find_camera_pose(np.ascontiguousarray(rgba), t_ms)
        ids, px, d3, _ = self.s.tracks()
        return st, self.s.pose(), ids.copy(), px.copy(), d3.copy()


# Poses, relative to max(1, |t|).  The two backends' poses start 1e-7 apart at the initialisation (the order of its refinement's
# sums), and every later local BA, and a re-initialisation after a reset, carries the difference on.  Observed on an H100: before
# the loss 5.5e-5 (plain), 1.04e-4 (through the lens, frame 21: just above test_gpu_system.py's 1e-4); after it 2.7e-4
# (revisit) and 5.3e-4 (unrelated scene, after the reset and a new initialisation).  Bars: 2e-4 until the track is lost, 1e-2
# from then on.  Status, ids and 3-D flags are exact on every frame.
def compare_with_cpu(frames, **kw):
    S = U.cpu_reloc_system_lib()
    c = U.CpuRelocRun(S, **kw)
    g = GpuRun(**kw)
    sts, worst = [], [0.0, 0.0]
    for k, f in enumerate(frames):
        st_c, T_c, _, ids_c, _, d3_c = c.frame(f, k * 33.333)
        st_g, T_g, ids_g, _, d3_g = g.frame(f, k * 33.333)
        assert st_c == st_g, (k, st_c, st_g)
        assert len(ids_c) == len(ids_g) and (ids_c == ids_g).all() and (d3_c == d3_g).all(), k
        after = 4 in sts or st_g == 4
        d = np.abs(T_c - T_g).max() / max(1.0, float(np.linalg.norm(T_c[:3])))
        worst[after] = max(worst[after], d)
        assert d < (1e-2 if after else 2e-4), (k, d)
        sts.append(st_g)
    c.close()
    g.s.close()
    print("pose |CPU - GPU| / max(1, |t|): %.2e before the loss, %.2e after it" % tuple(worst))
    return sts


def test_system_revisit_equals_the_cpu_backend():
    frames, _ = U.revisit_sequence()
    sts = compare_with_cpu(frames, max_lost=10)
    assert 4 in sts and sts[-1] == 1 and 2 not in sts[13:]


def test_system_revisit_through_a_lens_equals_the_cpu_backend():
    frames, _ = U.revisit_sequence(dist=U.DIST)
    sts = compare_with_cpu(frames, max_lost=10, dist=U.DIST)
    assert 4 in sts and sts[-1] == 1


def test_system_revisit_under_accurate_equals_the_cpu_backend():
    frames, _ = U.revisit_sequence()
    sts = compare_with_cpu(frames, max_lost=10, preset=3)
    assert 4 in sts and sts[-1] == 1


def test_system_unrelated_scene_equals_the_cpu_backend():
    sts = compare_with_cpu(U.unrelated_sequence(), max_lost=10)
    k = sts.index(4)
    assert sts[k:k + 10] == [4] * 10 and sts[k + 10] == 2


def test_off_is_bit_identical_to_never_calling_it():
    seq = U.failure_paths_sequence()
    a, b = GpuRun(), GpuRun(max_lost=0)
    for k, f in enumerate(seq):
        x, y = a.frame(f, k * 33.333), b.frame(f, k * 33.333)
        assert x[0] == y[0] and (x[1] == y[1]).all(), k
        assert len(x[2]) == len(y[2]) and (x[2] == y[2]).all() and (x[3].view(np.uint32) == y[3].view(np.uint32)).all() and (x[4] == y[4]).all(), k


def test_batch_entry_point_passes_the_lost_status_through():
    frames, _ = U.revisit_sequence()
    L = lib()
    L.alva_system_find_camera_pose_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    one = GpuRun(max_lost=10)
    pair = [GpuRun(max_lost=10), GpuRun(max_lost=10)]
    handles = (C.c_void_p * 2)(pair[0].s.h.value, pair[1].s.h.value)
    seen = set()
    for k, f in enumerate(frames):
        f = np.ascontiguousarray(f)
        st1, T1, ids1, _, _ = one.frame(f, k * 33.333)
        ptrs = (C.c_void_p * 2)(f.ctypes.data, f.ctypes.data)
        t = np.array([k * 33.333] * 2)
        poses = np.zeros((2, 16), np.float32); status = np.zeros(2, np.int32)
        assert L.alva_system_find_camera_pose_batch(handles, ptrs, U.P(t), 2, U.P(poses), U.P(status)) == 0
        assert status.tolist() == [st1, st1], k
        for g in pair:
            assert (g.s.pose() == T1).all() and (g.s.tracks()[0] == ids1).all(), k
        seen.add(st1)
    assert 4 in seen


def test_argument_and_state_errors():
    L = lib()
    System(64, 64, 50.0, 50.0, 32.0, 32.0).close()   # binds the System entry points
    h = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_relocalisation(h, 5) == -4    # ALVA_E_STATE: not configured
    L.alva_system_destroy(h)
    assert L.alva_system_set_relocalisation(None, 5) == -1
    K = synth.intrinsics(U.W, U.H)
    s = System(U.W, U.H, *K)
    assert L.alva_system_set_relocalisation(s.h, -1) == -1
    s.set_relocalisation(0)
    s.set_relocalisation(3)
    s.close()
