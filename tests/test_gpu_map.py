"""H100: the map blob of the CUDA System (alva_system_save_map / alva_system_load_map).  A blob saved by either backend loads into
the other, and from the same blob both run the revisit views in lockstep; the GPU round trip is byte-exact; saving on every
frame changes nothing; a loaded handle relocalises through the batch entry point; the Python binding raises AlvaError for every
refusal."""
import ctypes as C
import struct

import numpy as np
import pytest

import map_util as M
import reloc_util as U
from alvaar_b200 import AlvaError, System, lib, synth

pytestmark = pytest.mark.gpu

MAX_LOST = 10
N_BEFORE = 40
DT = 33.333


class GpuRun:
    def __init__(self, max_lost=MAX_LOST, preset=None, dist=None):
        K = synth.intrinsics(U.W, U.H)
        self.s = System(U.W, U.H, *K)
        if preset is not None:
            self.s.set_preset(["default", "fast", "average", "accurate"][preset])
        if dist is not None:
            self.s.set_distortion(*dist)
        if max_lost:
            self.s.set_relocalisation(max_lost)

    def frame(self, rgba, t_ms):
        st, _ = self.s.find_camera_pose(np.ascontiguousarray(rgba), t_ms)
        ids, px, d3, _ = self.s.tracks()
        return st, self.s.pose(), ids.copy(), px.copy(), d3.copy()


@pytest.fixture(scope="module")
def S():
    return M.bind(M.cpu_map_system_lib())


def _blobs(S, **kw):
    """session A over make_frames(40, seed 7) on each backend -> (frames, CPU blob, GPU blob)"""
    frames, _ = U.revisit_sequence(dist=kw.get("dist"))
    c = M.CpuMapRun(S, max_lost=MAX_LOST, **kw)
    g = GpuRun(**kw)
    for k in range(N_BEFORE):
        c.frame(frames[k], k * DT)
        g.frame(frames[k], k * DT)
    bc, bg = c.save(), g.s.save_map()
    c.close(); g.s.close()
    assert isinstance(bc, bytes) and isinstance(bg, bytes)
    return frames, bc, bg


# Both backends load the same bits, so the gap comes from their own arithmetic after the load (the relocalised PnP, KLT and the
# local BAs of the new keyframes), as test_gpu_reloc.py's 2e-4 before the loss.
def lockstep(S, frames, blob, **kw):
    c = M.CpuMapRun(S, max_lost=MAX_LOST, **kw)
    g = GpuRun(**kw)
    assert c.load(blob) == 0, c.error()
    g.s.load_map(blob)
    worst, sts = 0.0, []
    for k in range(N_BEFORE, len(frames)):
        st_c, T_c, _, ids_c, _, d3_c = c.frame(frames[k], (k - N_BEFORE) * DT)
        st_g, T_g, ids_g, _, d3_g = g.frame(frames[k], (k - N_BEFORE) * DT)
        assert st_c == st_g, (k, st_c, st_g)
        assert len(ids_c) == len(ids_g) and (ids_c == ids_g).all() and (d3_c == d3_g).all(), k
        d = np.abs(T_c - T_g).max() / max(1.0, float(np.linalg.norm(T_c[:3])))
        worst = max(worst, d)
        assert d < 2e-4, (k, d)
        sts.append(st_g)
    c.close(); g.s.close()
    return sts, worst


@pytest.mark.parametrize("case", ["plain", "lens", "accurate"])
def test_cross_backend_lockstep(S, case):
    kw = {"plain": {}, "lens": dict(dist=U.DIST), "accurate": dict(preset=3)}[case]
    frames, bc, bg = _blobs(S, **kw)
    for name, blob in (("CPU blob", bc), ("GPU blob", bg)):
        sts, worst = lockstep(S, frames, blob, **kw)
        assert sts[:3] == [4, 4, 4] and sts[-1] == 1 and 2 not in sts, sts
        print("%s, %s: pose |CPU - GPU| / max(1, |t|) %.2e" % (case, name, worst))


def test_long_session(S):
    """470 frames of make_frames(500, seed 99): keyframe filtering and the 30-keyframe window have removed keyframes the map
    still names.  The GPU blob round-trips byte for byte, and from the CPU session's blob both backends resume on the last 30
    frames in lockstep."""
    frames, _ = synth.make_frames(500, U.W, U.H, seed=99, rgba=True)
    c = M.CpuMapRun(S, max_lost=MAX_LOST)
    g = GpuRun()
    for k in range(470):
        c.frame(frames[k], k * DT)
        g.frame(frames[k], k * DT)
    bc, bg = c.save(), g.s.save_map()
    cc = c.counters()
    c.close(); g.s.close()
    assert cc["n_kf_ids"] > 30 and cc["keyframes"] < cc["n_kf_ids"] - 5, cc
    h = GpuRun()
    h.s.load_map(bg)
    assert h.s.save_map() == bg
    h.s.close()
    c = M.CpuMapRun(S, max_lost=MAX_LOST)
    g = GpuRun()
    assert c.load(bc) == 0, c.error()
    g.s.load_map(bc)
    worst, sts = 0.0, []
    for k in range(470, 500):
        st_c, T_c, _, ids_c, _, d3_c = c.frame(frames[k], (k - 470) * DT)
        st_g, T_g, ids_g, _, d3_g = g.frame(frames[k], (k - 470) * DT)
        assert st_c == st_g, (k, st_c, st_g)
        assert len(ids_c) == len(ids_g) and (ids_c == ids_g).all() and (d3_c == d3_g).all(), k
        d = np.abs(T_c - T_g).max() / max(1.0, float(np.linalg.norm(T_c[:3])))
        worst = max(worst, d)
        assert d < 2e-4, (k, d)
        sts.append(st_g)
    c.close(); g.s.close()
    assert sts[0] in (1, 4) and 1 in sts[:2] and all(s == 1 for s in sts[sts.index(1):]), sts
    print("long session: pose |CPU - GPU| / max(1, |t|) %.2e" % worst)


def test_gpu_round_trip_is_byte_identical(S):
    _, _, bg = _blobs(S)
    g = GpuRun()
    g.s.load_map(bg)
    assert g.s.save_map() == bg
    g.s.close()


def test_save_has_no_side_effects_on_the_gpu():
    frames, _ = U.revisit_sequence()
    a, b = GpuRun(), GpuRun()
    seen = set()
    for k, f in enumerate(frames):
        x = a.frame(f, k * DT)
        y = b.frame(f, k * DT)
        if x[0] in (1, 4):
            b.s.save_map()
        assert x[0] == y[0] and (x[1].view(np.uint64) == y[1].view(np.uint64)).all(), k
        assert len(x[2]) == len(y[2]) and (x[2] == y[2]).all() and (x[3].view(np.uint32) == y[3].view(np.uint32)).all() and (x[4] == y[4]).all(), k
        seen.add(x[0])
    assert {1, 4} <= seen
    assert a.s.save_map() == b.s.save_map()


def test_batch_entry_point_with_a_loaded_handle(S):
    frames, _, bg = _blobs(S)
    L = lib()
    L.alva_system_find_camera_pose_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    single = GpuRun()
    single.s.load_map(bg)
    pair = [GpuRun(), GpuRun()]
    pair[0].s.load_map(bg)            # pair[1] never loads a map
    never = GpuRun()
    handles = (C.c_void_p * 2)(pair[0].s.h.value, pair[1].s.h.value)
    seen = []
    for k in range(N_BEFORE, len(frames)):
        f = np.ascontiguousarray(frames[k])
        t = (k - N_BEFORE) * DT
        st1, T1, ids1, _, _ = single.frame(f, t)
        st2, T2, ids2, _, _ = never.frame(f, t)
        ptrs = (C.c_void_p * 2)(f.ctypes.data, f.ctypes.data)
        poses = np.zeros((2, 16), np.float32); status = np.zeros(2, np.int32)
        assert L.alva_system_find_camera_pose_batch(handles, ptrs, U.P(np.array([t, t])), 2, U.P(poses), U.P(status)) == 0
        assert status.tolist() == [st1, st2], k
        assert (pair[0].s.pose() == T1).all() and (pair[0].s.tracks()[0] == ids1).all(), k
        assert (pair[1].s.pose() == T2).all() and (pair[1].s.tracks()[0] == ids2).all(), k
        seen.append(st1)
    assert seen[:3] == [4, 4, 4] and seen[3] == 1, seen


def test_python_errors(S):
    frames, _, bg = _blobs(S)
    g = GpuRun(max_lost=0)
    with pytest.raises(AlvaError, match="-4"):
        g.s.save_map()                            # not initialised
    with pytest.raises(AlvaError, match="-4"):
        g.s.load_map(bg)                          # relocalisation off
    g.s.set_relocalisation(MAX_LOST)
    secs, _ = M.sections(bg)
    off = dict(secs)
    rec = M.mappoint_records(bg)
    bad = [b"XLMP" + bg[4:], bg[:4] + struct.pack("<I", 2) + bg[8:], bg[:off["pose"]], bg[:-1],
           bg[:8] + struct.pack("<Q", len(bg) + 1) + bg[16:]]
    b = bytearray(bg); struct.pack_into("<d", b, off["camera"] + 8, 401.0); bad.append(bytes(b))
    b = bytearray(bg); struct.pack_into("<i", b, off["grid"], 35); bad.append(bytes(b))
    b = bytearray(bg); struct.pack_into("<d", b, off["pose"], float("nan")); bad.append(bytes(b))
    b = bytearray(bg); struct.pack_into("<i", b, rec[1][0], rec[0][1]); bad.append(bytes(b))
    b = bytearray(bg); struct.pack_into("<i", b, rec[3][0] + 4, 10 ** 6); bad.append(bytes(b))
    for k, blob in enumerate(bad):
        with pytest.raises(AlvaError, match="-1"):
            g.s.load_map(blob)
    # a refused load leaves the handle as it was: it still initialises on the frames that follow
    sts = [g.frame(frames[k], k * DT)[0] for k in range(20)]
    assert 1 in sts
    # the C ABI: size query, a short buffer, null arguments
    L = lib()
    n = C.c_size_t(0)
    assert L.alva_system_save_map(g.s.h, None, 0, C.byref(n)) == 0 and n.value > 0
    short = C.create_string_buffer(n.value - 1)
    m = C.c_size_t(0)
    assert L.alva_system_save_map(g.s.h, short, n.value - 1, C.byref(m)) == -3 and m.value == n.value
    assert L.alva_system_save_map(None, None, 0, C.byref(m)) == -1
    assert L.alva_system_load_map(None, bg, len(bg)) == -1
    assert L.alva_system_load_map(g.s.h, None, 0) == -1
    g.s.close()
    h = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_load_map(h, bg, len(bg)) == -4    # not configured
    assert L.alva_system_save_map(h, None, 0, C.byref(m)) == -4
    L.alva_system_destroy(h)
