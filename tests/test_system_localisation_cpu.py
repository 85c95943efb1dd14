"""CPU: the localisation-only mode of System (system_core.h setLocalisationOnly / reacquireFrame, alva_system_set_localisation_only)
and its re-acquisition match (oracle/reacquire_oracle.c, the restatement of alva_k_match_frame_to_map).  The oracle equals a
brute-force numpy model on random problems and on every boundary; over the CPU oracle backend (tests/host/system_cpu_localisation.cpp)
a loaded map stays exactly as saved while the frozen session tracks, relocalises and re-acquires, a loss never resets it,
unfreezing resumes mapping, and every refusal changes nothing."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

import localisation_util as LU
import map_util as M
import reloc_util as U
from alvaar_b200 import synth

MAX_LOST = 10
N_A = 320                         # session A: make_frames(320, seed 99)
TOL_T, TOL_DEG = 0.05, 0.5        # the relocalisation bars of test_system_reloc_cpu.py
DT = 33.333


# ------------------------------------------------------------------------------------------------ the oracle
@pytest.fixture(scope="module")
def L():
    return LU.oracle_lib()


def same(L, p):
    a, b = LU.run_oracle(L, p), LU.run_numpy(L, p)
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all(), (np.nonzero(a[0] != b[0])[0][:10], a[0][a[0] != b[0]][:10], b[0][a[0] != b[0]][:10])
    return a


@pytest.mark.parametrize("lens", ["pinhole", "radtan", "fisheye"])
@pytest.mark.parametrize("cell", [35, 40, 45, 50])
def test_oracle_equals_numpy_on_random_problems(L, lens, cell):
    for seed, radius, rows in ((cell, 2.0, 6), (cell + 1, 4.0, 30), (cell + 2, 2.0, 1)):
        rng = np.random.default_rng(seed)
        p = LU.random_problem(rng, lens=lens, cell=cell, radius=radius, max_rows=rows, n_mp=500, nq=400)
        row, _ = same(L, p)
        assert (row >= 0).sum() > 20
        # one-to-one
        assert len(set(row[row >= 0].tolist())) == (row >= 0).sum()


def hand_problem(points, rows, queries, q_desc, kept=None, skip=None, radius=2.0, w=640, h=480, cell=40, K=(500.0, 500.0, 320.0, 240.0),
                 Twc=(0, 0, 0, 0, 0, 0, 1)):
    """identity pose (world = camera frame); rows: per point a list of descriptors"""
    desc_start = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    desc = np.array([d for r in rows for d in r], np.uint8).reshape(-1, 32)
    nq = len(queries)
    return LU.Problem(w, h, cell, K, 0, None, np.array(Twc, np.float64), np.array(points, np.float64).reshape(-1, 3), desc_start, desc,
                      None if skip is None else np.array(skip, np.uint8), np.array(queries, np.float32).reshape(-1, 2),
                      np.array(q_desc, np.uint8).reshape(-1, 32), np.ones(nq, np.uint8) if kept is None else np.array(kept, np.uint8), radius)


def flip(d, nbits, start=0):
    bits = np.unpackbits(np.asarray(d, np.uint8))
    bits[start:start + nbits] ^= 1
    return np.packbits(bits)


def at_px(u, v, z=2.0, K=(500.0, 500.0, 320.0, 240.0)):
    """a camera-frame point projecting to (u, v) (up to the float rounding of the projection)"""
    return [(u - K[2]) / K[0] * z, (v - K[3]) / K[1] * z, z]


def proj_of(L, p):
    return LU.project(L, p, LU.world_to_cam(p.Twc, p.wpt))


def test_oracle_boundaries(L):
    rng = np.random.default_rng(5)
    D = rng.integers(0, 256, (8, 32), dtype=np.uint8)
    # a candidate exactly at the radius (in), one float step beyond (out), at 2 and 4 px
    for r in (2.0, 4.0):
        base = hand_problem([at_px(100.3, 200.7)], [[D[0]]], [[0, 0]], [D[0]], radius=r)
        pr = proj_of(L, base)[0]
        q_in = np.float32(pr[0] + np.float32(r))
        for qx, want in ((q_in, 0), (np.nextafter(q_in, np.float32(1e9)), -1)):
            p = hand_problem([at_px(100.3, 200.7)], [[D[0]]], [[qx, pr[1]]], [D[0]], radius=r)
            assert (np.float32(qx - pr[0]) == np.float32(r)) == (want == 0)
            assert same(L, p)[0][0] == want, (r, qx)
    # distances 51 (a match) and 52 (none)
    for nb, want in ((51, 0), (52, -1)):
        p = hand_problem([at_px(300, 300)], [[D[0], D[1]]], [[300, 300]], [flip(D[0], nb)])
        row, dist = same(L, p)
        assert row[0] == want and (want < 0 or dist[0] == 51)
    # the ratio test over two candidates of one map point: kept iff 0.9 * second >= best, exhaustively over 0..51
    for b in range(0, 52, 3):
        for s in range(b, 52, 4):
            p = hand_problem([at_px(200, 150)], [[D[2]]], [[200, 150], [200.5, 150]], [flip(D[2], b), flip(D[2], s, 100)])
            row, _ = same(L, p)
            ok = not (0.9 * s < b)
            assert (row >= 0).sum() == (1 if ok else 0), (b, s)
            if ok:
                assert row[1 if s == b else 0] == 0        # equal distances: the later query is the best
    # ties between map points: two points at the same distance to one query -> the higher row
    p = hand_problem([at_px(400, 100), at_px(400.5, 100)], [[D[3]], [D[3]]], [[400.2, 100]], [D[3]])
    assert same(L, p)[0][0] == 1
    # c_z at 0.1 (kept) and just below (dropped); a point behind the camera
    for z, want in ((0.1, 0), (np.nextafter(0.1, 0), -1), (-1.0, -1)):
        p = hand_problem([[0.0, 0.0, z]], [[D[4]]], [[320, 240]], [D[4]])
        assert same(L, p)[0][0] == want, z
    # the view gate: rays on both sides of view_th, which here lie outside the image (so both gates are exercised)
    for ang in np.linspace(30, 50, 21):
        x = np.tan(np.radians(ang))
        p = hand_problem([[x, 0.0, 1.0]], [[D[5]]], [[500 * x + 320, 240]], [D[5]], w=2000, h=480, K=(500.0, 500.0, 320.0, 240.0))
        same(L, p)
    # outside the image
    p = hand_problem([at_px(-0.5, 100), at_px(640.2, 100)], [[D[6]], [D[6]]], [[0.5, 100], [639.5, 100]], [D[6], D[6]], radius=2.0)
    assert (same(L, p)[0] == -1).all()
    # a projection near a cell's lower-right corner, its query across the corner: found (the reference's 2 x 2 upper-left
    # neighbourhood of getSurroundingKeypoints would miss it)
    p = hand_problem([at_px(119.4, 79.4)], [[D[7]]], [[120.6, 80.6]], [D[7]], cell=40)
    assert same(L, p)[0][0] == 0
    # masked rows, not-kept queries, an empty table, no queries
    p = hand_problem([at_px(300, 300)], [[D[0]]], [[300, 300]], [D[0]], skip=[1])
    assert same(L, p)[0][0] == -1
    p = hand_problem([at_px(300, 300)], [[D[0]]], [[300, 300]], [D[0]], kept=[0])
    assert same(L, p)[0][0] == -1
    p = hand_problem(np.zeros((0, 3)), [], [[300, 300]], [D[0]])
    assert same(L, p)[0][0] == -1
    p = hand_problem([at_px(300, 300)], [[D[0]]], np.zeros((0, 2)), np.zeros((0, 32)))
    assert len(same(L, p)[0]) == 0


# ------------------------------------------------------------------------------------------------ the state machine
@pytest.fixture(scope="module")
def S():
    return LU.bind(LU.cpu_loc_system_lib())


@pytest.fixture(scope="module")
def session_a(S):
    """session A over make_frames(320, seed 99) and 24 revisit views (halfway poses from frame 15 on, turned 1 degree): frames,
    true poses, A's outputs, counters and blob"""
    A, poses = synth.make_frames(N_A, U.W, U.H, seed=99, rgba=True)
    tex = synth.make_texture()
    rv = [U._mid_pose(poses, 15 + i) for i in range(24)]
    R = [synth.gray_to_rgba(synth.render_gray(tex, p, U.W, U.H)) for p in rv]
    a = LU.CpuLocRun(S, max_lost=MAX_LOST)
    out = [a.frame(A[k], k * DT) for k in range(N_A)]
    blob, c = a.save(), a.counters()
    a.close()
    assert isinstance(blob, bytes)
    return dict(A=A, poses=poses, R=R, rv=rv, out=out, counters=c, blob=blob)


def frozen_run(S, sa, frames, freeze=True):
    b = LU.CpuLocRun(S, max_lost=MAX_LOST)
    assert b.load(sa["blob"]) == 0, b.error()
    if freeze:
        assert b.freeze(True) == 0
    out, cs = [], []
    for j, f in enumerate(frames):
        out.append(b.frame(f, j * DT))
        cs.append(b.counters())
    return b, out, cs


def test_frozen_resume(S, session_a):
    sa = session_a
    ca = sa["counters"]
    frames = list(sa["R"]) + list(sa["A"])
    truth = list(sa["rv"]) + list(sa["poses"])
    b, out, cs = frozen_run(S, sa, frames)
    st = [o[0] for o in out]
    assert st[0] == 1 or st[:2] == [4, 1], st[:5]
    assert 2 not in st and set(st) <= {1, 4}
    for c, o in zip(cs, out):
        assert (c["n_kf_ids"], c["n_mp_ids"], c["keyframes"], c["mappoints"]) == (ca["n_kf_ids"], ca["n_mp_ids"], ca["keyframes"], ca["mappoints"])
        assert o[2][5] == ca["keyframes"] and o[2][7] == ca["n_mp_ids"]
    assert cs[-1]["table_version"] == cs[0]["table_version"]      # never rebuilt
    # the map records saved at the end are those loaded
    assert LU.map_records(b.save()) == LU.map_records(sa["blob"])
    # poses: the similarity from the synthetic frame to A's, then every tracked frame within the relocalisation bars
    tracked = {k: sa["out"][k][1] for k in range(N_A) if sa["out"][k][0] == 1}
    fit = U.fit_from_track(sa["poses"], tracked)
    worst = (0.0, 0.0)
    for j, o in enumerate(out):
        if o[0] == 1:
            dt, dr = U.pose_error(o[1], U.true_in_map(fit, truth[j]))
            worst = (max(worst[0], dt), max(worst[1], dr))
    assert worst[0] < TOL_T and worst[1] < TOL_DEG, worst
    # the last relocalisation's keypoints all leave the frame, and the track carries on with re-acquired ids
    last = max(j for j in range(len(out)) if cs[j]["relocalised"] != (cs[j - 1]["relocalised"] if j else 0))
    reloc_ids = set(out[last][3].tolist())
    assert all(s == 1 for s in st[last:]), st[last:]
    gone = [j for j in range(last, len(out)) if not (set(out[j][3].tolist()) & reloc_ids)]
    assert gone and len(out) - gone[0] >= 50, (last, gone[:3])
    c = cs[-1]
    assert c["reacq_points"] > 100 and c["reacq_runs"] >= 5
    b.close()
    print("frozen resume: %d frames, %d relocalisations, re-acquisition ran on %d frames and supplied %d points; the relocalised "
          "points had all left by frame %d; worst pose error %.4f, %.3f deg" % (len(out), c["relocalised"], c["reacq_runs"], c["reacq_points"],
                                                                            gone[0], worst[0], worst[1]))


def test_lost_while_frozen(S, session_a):
    sa = session_a
    other, _ = synth.make_frames(2 * MAX_LOST + 5, U.W, U.H, seed=33, rgba=True, texture_seed=4321)
    b, out, cs = frozen_run(S, sa, list(other) + list(sa["R"][:6]))
    st = [o[0] for o in out]
    assert st[:len(other)] == [4] * len(other), st
    assert 1 in st[len(other):] and 2 not in st, st
    assert cs[len(other) - 1]["lost_frames"] == len(other)
    assert LU.map_records(b.save()) == LU.map_records(sa["blob"])
    b.close()


def test_unfreeze_resumes_mapping(S, session_a):
    sa = session_a
    ca = sa["counters"]
    b, out, cs = frozen_run(S, sa, list(sa["A"][:40]))
    assert [o[0] for o in out].count(1) >= 35
    assert b.freeze(False) == 0 and b.counters()["frozen"] == 0
    st, new_kf = [], None
    for k in range(40, N_A):
        o = b.frame(sa["A"][k], (k + 40) * DT)
        st.append(o[0])
        if new_kf is None and b.counters()["n_kf_ids"] > ca["n_kf_ids"]:
            new_kf = int(o[2][1])
    c = b.counters()
    assert new_kf == ca["n_kf_ids"], (new_kf, ca)
    assert c["n_mp_ids"] > ca["n_mp_ids"] and c["n_kf_ids"] > 31, c
    # the 30-keyframe window applies again: keyframe k - 30 left when keyframe k > 30 was made (keyframe 0 is never removed)
    blob = b.save()
    secs, _ = M.sections(blob)
    kfs = [struct.unpack_from("<i", blob, off)[0] for n, off in secs if n.startswith("keyframe")]
    assert not [k for k in kfs if 1 <= k <= c["n_kf_ids"] - 1 - 30], (kfs, c)
    b.close()


def run_frames(S, frames, calls, max_lost=MAX_LOST):
    """a session with calls {frame index: [(name, args)]} made before that frame -> outputs and the calls' return codes"""
    r = LU.CpuLocRun(S, max_lost=max_lost)
    out, rcs = [], []
    for k, f in enumerate(frames):
        for name, args in calls.get(k, []):
            rcs.append(getattr(r.S, "cpu_loc_system_" + name)(r.s, *args))
        out.append(r.frame(f, k * DT))
    r.close()
    return out, rcs


def test_refusals_change_nothing(S, session_a):
    frames = list(session_a["A"][:40])
    ref, _ = run_frames(S, frames, {})
    cases = [({3: [("set_localisation_only", (1,))]}, [-4]),            # before the initialisation
             ({20: [("set_localisation_only", (2,))]}, [-1]),           # enabled other than 0 / 1
             ({20: [("set_localisation_only", (-1,))]}, [-1]),
             ({20: [("set_localisation_only", (0,))]}, [0])]            # disabling is always allowed
    for calls, want in cases:
        out, rcs = run_frames(S, frames, calls)
        assert rcs == want, (calls, rcs)
        assert all(M.same_frame(x, y) for x, y in zip(ref, out)), calls
    # relocalisation off: enabling is refused
    ref0, _ = run_frames(S, frames, {}, max_lost=0)
    out, rcs = run_frames(S, frames, {20: [("set_localisation_only", (1,))]}, max_lost=0)
    assert rcs == [-4] and all(M.same_frame(x, y) for x, y in zip(ref0, out))
    # set_relocalisation(0) while frozen: refused, the frozen run goes on as without the call
    fz, rcs0 = run_frames(S, frames, {20: [("set_localisation_only", (1,))]})
    out, rcs = run_frames(S, frames, {20: [("set_localisation_only", (1,))], 25: [("set_relocalisation", (0,))]})
    assert rcs0 == [0] and rcs == [0, -4] and all(M.same_frame(x, y) for x, y in zip(fz, out))


def test_what_keeps_and_ends_the_mode(S, session_a):
    blob = session_a["blob"]
    r = LU.CpuLocRun(S, max_lost=MAX_LOST)
    assert r.load(blob) == 0 and r.freeze(True) == 0
    assert r.load(blob) == 0 and r.counters()["frozen"] == 1          # load_map keeps it
    r.S.cpu_loc_system_set_clahe(r.s, 1)
    assert r.counters()["frozen"] == 1                                  # so does CLAHE
    for name, args in (("reset", ()), ("set_preset", (0,)), ("set_distortion", (0.0, 0.0, 0.0, 0.0)), ("set_fisheye", (0, 0.0, 0.0, 0.0, 0.0))):
        assert r.load(blob) == 0 and r.freeze(True) == 0
        getattr(r.S, "cpu_loc_system_" + name)(r.s, *args)
        assert r.counters()["frozen"] == 0, name
    r.close()


def test_freeze_a_live_session(S, session_a):
    """a live, initialised session freezes its own map: the 2-D keypoints go, the counters stop"""
    A = session_a["A"]
    r = LU.CpuLocRun(S, max_lost=MAX_LOST)
    for k in range(60):
        r.frame(A[k], k * DT)
    c0 = r.counters()
    assert r.freeze(True) == 0
    o = r.frame(A[60], 60 * DT)
    assert (o[5] == 1).all()
    st = [r.frame(A[k], k * DT)[0] for k in range(61, 160)]
    c = r.counters()
    assert set(st) <= {1, 4} and (c["n_kf_ids"], c["n_mp_ids"], c["keyframes"]) == (c0["n_kf_ids"], c0["n_mp_ids"], c0["keyframes"])
    r.close()


FROZEN = r"""
import sys
sys.path[:0] = [{tests!r}, {root!r}]
import numpy as np
import localisation_util as LU
S = LU.bind({so!r})
blob = open({blob!r}, "rb").read()
frames = np.load({frames!r})
r = LU.CpuLocRun(S, max_lost=3)
assert r.load(blob) == 0
assert r.freeze(True) == 0
st = [r.frame(f, k * 33.333)[0] for k, f in enumerate(frames)]
assert r.freeze(False) == 0
st += [r.frame(f, (k + len(frames)) * 33.333)[0] for k, f in enumerate(frames[-20:])]
r.close()
print(" ".join(map(str, st)))
"""


def test_frozen_run_under_sanitizers(S, session_a, tmp_path):
    """the shim built with -fsanitize=address,undefined: a frozen run (relocalisation, re-acquisition, a loss longer than
    max_lost_frames, unfreezing) without a sanitizer report"""
    so = LU.cpu_loc_system_lib(sanitize=True)
    asan = subprocess.check_output(["g++", "-print-file-name=libasan.so"], text=True).strip()
    ubsan = subprocess.check_output(["g++", "-print-file-name=libubsan.so"], text=True).strip()
    bp = tmp_path / "map.bin"
    bp.write_bytes(session_a["blob"])
    black = np.zeros_like(session_a["A"][0]); black[..., 3] = 255
    fp = tmp_path / "frames.npy"
    np.save(fp, np.stack(list(session_a["R"][:8]) + list(session_a["A"][:40]) + [black] * 6 + list(session_a["A"][40:80])))
    code = FROZEN.format(tests=os.path.dirname(os.path.abspath(__file__)), root=U.ROOT, so=so, blob=str(bp), frames=str(fp))
    env = dict(os.environ, LD_PRELOAD=asan + " " + ubsan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1",
               UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0, p.stderr[-4000:]
    assert "runtime error" not in p.stderr and "AddressSanitizer" not in p.stderr, p.stderr[-4000:]
    st = list(map(int, p.stdout.split()))
    assert 1 in st and 4 in st and 2 not in st[:94], st
