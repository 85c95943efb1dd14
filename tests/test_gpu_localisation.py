"""H100: the localisation-only mode of the CUDA System (alva_system_set_localisation_only) and its re-acquisition kernel
(alva_k_match_frame_to_map).  The kernel equals oracle/reacquire_oracle.c exactly at and beyond the sizes System produces, for
every lens and cell size and on the boundary cases; from the same blob the GPU System and the CPU backend run a frozen
session in lockstep; a frozen GPU session leaves the loaded map records unchanged; the batch entry point and the Python errors
behave as documented."""
import ctypes as C

import numpy as np
import pytest
import torch

import localisation_util as LU
import reloc_util as U
from alvaar_b200 import AlvaError, Context, System, lib, synth

pytestmark = pytest.mark.gpu

MAX_LOST = 10
N_A = 320
DT = 33.333


@pytest.fixture(scope="module")
def L():
    return LU.oracle_lib()


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, torch.cuda.current_stream().cuda_stream)
    yield c
    c.close()


def run_gpu(ctx, p):
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()  # noqa: E731
    nq = len(p.q_px)
    row = torch.full((max(nq, 1),), -7, dtype=torch.int32, device="cuda"); dist = torch.full_like(row, -7)
    wpt = d(p.wpt if len(p.wpt) else np.zeros((0, 3)), np.float64)
    desc = d(p.desc if len(p.desc) else np.zeros((1, 32)), np.uint8)
    ctx.match_frame_to_map(p.w, p.h, p.cell, p.K, d(p.Twc, np.float64), wpt, d(p.desc_start, np.int32), desc,
                           d(p.q_px.reshape(-1, 2), np.float32), d(p.q_desc.reshape(-1, 32), np.uint8), d(p.q_kept, np.uint8), row, dist,
                           radius=p.radius, skip=None if p.skip is None else d(p.skip, np.uint8), lens=p.lens, coef=p.coef)
    torch.cuda.synchronize()
    return row.cpu().numpy()[:nq], dist.cpu().numpy()[:nq]


def check(ctx, L, p):
    want = LU.run_oracle(L, p)
    got = run_gpu(ctx, p)
    bad = np.nonzero((got[0] != want[0]) | (got[1] != want[1]))[0]
    assert len(bad) == 0, (len(bad), bad[:8], got[0][bad[:8]], want[0][bad[:8]])
    return want


SIZES = [((640, 480), 500, 800, 6), ((1280, 720), 10000, 2000, 30), ((1920, 1080), 100000, 8192, 32), ((1920, 1080), 30000, 8192, 1)]


@pytest.mark.parametrize("lens", ["pinhole", "radtan", "fisheye"])
@pytest.mark.parametrize("cell", [35, 40, 45, 50])
def test_kernel_equals_oracle(ctx, L, lens, cell):
    for k, ((w, h), n_mp, nq, rows) in enumerate(SIZES):
        for radius in (2.0, 4.0):
            p = LU.random_problem(np.random.default_rng(1000 * cell + 10 * k + int(radius)), w=w, h=h, cell=cell, lens=lens, n_mp=n_mp,
                                  nq=nq, max_rows=rows, radius=radius)
            row, _ = check(ctx, L, p)
            assert (row >= 0).sum() > 0


def test_kernel_boundaries(ctx, L):
    import test_system_localisation_cpu as T
    rng = np.random.default_rng(5)
    D = rng.integers(0, 256, (8, 32), dtype=np.uint8)
    probs = []
    base = T.hand_problem([T.at_px(100.3, 200.7)], [[D[0]]], [[0, 0]], [D[0]])
    pr = T.proj_of(L, base)[0]
    for r in (2.0, 4.0):
        q_in = np.float32(pr[0] + np.float32(r))
        for qx in (q_in, np.nextafter(q_in, np.float32(1e9))):
            probs.append(T.hand_problem([T.at_px(100.3, 200.7)], [[D[0]]], [[qx, pr[1]]], [D[0]], radius=r))
    for nb in (51, 52):
        probs.append(T.hand_problem([T.at_px(300, 300)], [[D[0], D[1]]], [[300, 300]], [T.flip(D[0], nb)]))
    for b in range(0, 52):
        for s in range(b, 52, 3):
            probs.append(T.hand_problem([T.at_px(200, 150)], [[D[2]]], [[200, 150], [200.5, 150]], [T.flip(D[2], b), T.flip(D[2], s, 100)]))
    probs.append(T.hand_problem([T.at_px(400, 100), T.at_px(400.5, 100)], [[D[3]], [D[3]]], [[400.2, 100]], [D[3]]))
    for z in (0.1, np.nextafter(0.1, 0), -1.0):
        probs.append(T.hand_problem([[0.0, 0.0, z]], [[D[4]]], [[320, 240]], [D[4]]))
    for ang in np.linspace(30, 50, 41):
        x = np.tan(np.radians(ang))
        probs.append(T.hand_problem([[x, 0.0, 1.0]], [[D[5]]], [[500 * x + 320, 240]], [D[5]], w=2000))
    probs.append(T.hand_problem([T.at_px(-0.5, 100), T.at_px(640.2, 100)], [[D[6]], [D[6]]], [[0.5, 100], [639.5, 100]], [D[6], D[6]]))
    for cell in (35, 40, 45, 50):
        c = float(cell)
        probs.append(T.hand_problem([T.at_px(3 * c - 0.6, 2 * c - 0.6)], [[D[7]]], [[3 * c + 0.6, 2 * c + 0.6]], [D[7]], cell=cell))
    probs.append(T.hand_problem([T.at_px(300, 300)], [[D[0]]], [[300, 300]], [D[0]], skip=[1]))
    probs.append(T.hand_problem([T.at_px(300, 300)], [[D[0]]], [[300, 300]], [D[0]], kept=[0]))
    probs.append(T.hand_problem(np.zeros((0, 3)), [], [[300, 300]], [D[0]]))
    probs.append(T.hand_problem([T.at_px(300, 300)], [[D[0]]], np.zeros((0, 2)), np.zeros((0, 32))))
    for p in probs:
        check(ctx, L, p)


# ------------------------------------------------------------------------------------------------ System
class GpuRun:
    def __init__(self, max_lost=MAX_LOST):
        self.s = System(U.W, U.H, *synth.intrinsics(U.W, U.H))
        if max_lost:
            self.s.set_relocalisation(max_lost)

    def frame(self, rgba, t_ms):
        st, _ = self.s.find_camera_pose(np.ascontiguousarray(rgba), t_ms)
        ids, px, d3, _ = self.s.tracks()
        return st, self.s.pose(), ids.copy(), px.copy(), d3.copy()


@pytest.fixture(scope="module")
def S():
    return LU.bind(LU.cpu_loc_system_lib())


@pytest.fixture(scope="module")
def session(S):
    """session A (make_frames(320, seed 99)) on each backend -> frames, CPU blob, GPU blob, revisit views"""
    A, poses = synth.make_frames(N_A, U.W, U.H, seed=99, rgba=True)
    tex = synth.make_texture()
    R = [synth.gray_to_rgba(synth.render_gray(tex, U._mid_pose(poses, 15 + i), U.W, U.H)) for i in range(24)]
    c, g = LU.CpuLocRun(S, max_lost=MAX_LOST), GpuRun()
    for k in range(N_A):
        c.frame(A[k], k * DT)
        g.frame(A[k], k * DT)
    bc, bg = c.save(), g.s.save_map()
    c.close(); g.s.close()
    return A, bc, bg, R


def test_frozen_lockstep(S, session):
    """from the CPU blob: the frozen revisit views and a replay of A's path, statuses, track ids in order and 3-D flags exact,
    poses within 2e-4 max(1, |t|)"""
    A, bc, _, R = session
    c, g = LU.CpuLocRun(S, max_lost=MAX_LOST), GpuRun()
    assert c.load(bc) == 0, c.error()
    g.s.load_map(bc)
    assert c.freeze(True) == 0
    g.s.set_localisation_only(True)
    frames = list(R) + list(A)
    worst, sts = 0.0, []
    for j, f in enumerate(frames):
        st_c, T_c, _, ids_c, _, d3_c = c.frame(f, j * DT)
        st_g, T_g, ids_g, _, d3_g = g.frame(f, j * DT)
        assert st_c == st_g, (j, st_c, st_g)
        assert len(ids_c) == len(ids_g) and (ids_c == ids_g).all() and (d3_c == d3_g).all(), j
        d = np.abs(T_c - T_g).max() / max(1.0, float(np.linalg.norm(T_c[:3])))
        worst = max(worst, d)
        assert d < 2e-4, (j, d)
        sts.append(st_g)
    cc, gs = c.counters(), g.s.localisation_stats()
    assert (cc["reacq_runs"], cc["reacq_points"]) == (gs["runs"], gs["points"]) and gs["points"] > 100
    assert 2 not in sts and 1 in sts
    assert LU.map_records(g.s.save_map()) == LU.map_records(bc)
    c.close(); g.s.close()
    print("frozen lockstep: %d frames, re-acquisition on %d frames, %d points; pose |CPU - GPU| / max(1, |t|) %.2e" %
          (len(frames), gs["runs"], gs["points"], worst))


def test_gpu_blob_records_unchanged(session):
    A, _, bg, R = session
    g = GpuRun()
    g.s.load_map(bg)
    g.s.set_localisation_only(True)
    other, _ = synth.make_frames(MAX_LOST + 5, U.W, U.H, seed=33, rgba=True, texture_seed=4321)
    sts = [g.frame(f, j * DT)[0] for j, f in enumerate(list(R) + list(A[:120]) + list(other) + list(A[:40]))]
    assert 2 not in sts and sts[-1] == 1
    assert LU.map_records(g.s.save_map()) == LU.map_records(bg)
    g.s.close()


def test_batch_entry_point(session):
    A, _, bg, R = session
    Lb = lib()
    Lb.alva_system_find_camera_pose_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    single = GpuRun()
    single.s.load_map(bg); single.s.set_localisation_only(True)
    pair = [GpuRun(), GpuRun()]
    pair[0].s.load_map(bg); pair[0].s.set_localisation_only(True)
    pair[1].s.load_map(bg)
    other = GpuRun()
    other.s.load_map(bg)
    handles = (C.c_void_p * 2)(pair[0].s.h.value, pair[1].s.h.value)
    seen = []
    for j, f in enumerate(list(R) + list(A[:60])):
        f = np.ascontiguousarray(f)
        t = j * DT
        st1, T1, ids1, _, _ = single.frame(f, t)
        st2, T2, ids2, _, _ = other.frame(f, t)
        ptrs = (C.c_void_p * 2)(f.ctypes.data, f.ctypes.data)
        poses = np.zeros((2, 16), np.float32); status = np.zeros(2, np.int32)
        assert Lb.alva_system_find_camera_pose_batch(handles, ptrs, U.P(np.array([t, t])), 2, U.P(poses), U.P(status)) == 0
        assert status.tolist() == [st1, st2], j
        assert (pair[0].s.pose() == T1).all() and (pair[0].s.tracks()[0] == ids1).all(), j
        assert (pair[1].s.pose() == T2).all() and (pair[1].s.tracks()[0] == ids2).all(), j
        seen.append(st1)
    assert 1 in seen and 2 not in seen


def test_python_errors(session):
    _, _, bg, _ = session
    g = GpuRun(max_lost=0)
    with pytest.raises(AlvaError, match="-4"):
        g.s.set_localisation_only(True)          # relocalisation off (and no map)
    g.s.set_relocalisation(MAX_LOST)
    with pytest.raises(AlvaError, match="-4"):
        g.s.set_localisation_only(True)          # no map
    g.s.set_localisation_only(False)             # disabling is always allowed
    g.s.load_map(bg)
    g.s.set_localisation_only(True)
    assert g.s.localisation_stats()["on"] == 1
    with pytest.raises(AlvaError, match="-4"):
        g.s.set_relocalisation(0)
    g.s.set_clahe(True)
    g.s.load_map(bg)
    assert g.s.localisation_stats()["on"] == 1   # load_map and set_clahe keep it
    g.s.set_preset("fast")
    assert g.s.localisation_stats()["on"] == 0   # set_preset ends it with the map
    Lb = lib()
    assert Lb.alva_system_set_localisation_only(None, 1) == -1
    assert Lb.alva_system_set_localisation_only(g.s.h, 2) == -1
    g.s.close()
    h = C.c_void_p(Lb.alva_system_create(0))
    assert Lb.alva_system_set_localisation_only(h, 1) == -4    # not configured
    assert Lb.alva_system_set_localisation_only(h, 0) == -4
    Lb.alva_system_destroy(h)
