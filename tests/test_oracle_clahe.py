"""CPU tests of the CLAHE pre-processing (the reference's optional cv::CLAHE before the KLT pyramid, visual_frontend.cpp:672-698).

orc_clahe (oracle/clahe_oracle.c) is bit-identical to cv::createCLAHE(...)->apply of the reference's own OpenCV on every case of
tests/golden/clahe.npz (live when oracle/_ref/libalva_ref_clahe.so is built, else through the stored SHA-256 digests).  The host-side System state
machine over the CPU oracle with CLAHE on (tests/host/system_cpu_clahe.cpp), given the reference's own initialisation through
the five-point hook, follows the reference System's 100-frame trace (tests/golden/system_clahe.npz, tools/make_golden_clahe.py):
status, track ids in the reference's order, 3-D flags and counters exact on every frame, pixel positions bit for bit before the
initialisation, poses and world points 1e-9."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from clahe_util import CASES, case_input, clahe_oracle_lib, compress_contrast, cpu_clahe_system_lib, ref_clahe_lib
from conftest import P, golden
from ref_golden import digest
from system_util import CAP, frame_slice

NAMES = [c[0] for c in CASES]


def run_orc(k):
    name, w, h, n, clip, tx, ty, kind = CASES[k]
    x = case_input(k)
    y = np.empty_like(x)
    assert clahe_oracle_lib().orc_clahe(P(x), P(y), w, h, n, clip, tx, ty) == 0
    return x, y


@pytest.mark.parametrize("k", range(len(CASES)), ids=NAMES)
def test_orc_clahe_matches_the_reference(ref, k):
    g = golden("clahe")
    name, w, h, n, clip, tx, ty, kind = CASES[k]
    x, y = run_orc(k)
    assert (digest(x) == g[f"{name}/in"]).all(), "case input generator changed: re-dump tests/golden/clahe.npz"
    refc = ref_clahe_lib(ref)
    if refc is not None:
        want = np.empty_like(x)
        for f in range(n):
            refc.ref_clahe(P(np.ascontiguousarray(x[f])), w, h, clip, tx, ty, P(want[f]))
        bad = np.argwhere(want != y)
        assert len(bad) == 0, f"{len(bad)} pixels differ, first {bad[:4].tolist()}"
    assert (digest(y) == g[f"{name}/out"]).all()


def test_orc_clahe_in_place_and_argument_checks():
    orc = clahe_oracle_lib()
    x, y = run_orc(NAMES.index("neither_divisible"))
    name, w, h, n, clip, tx, ty, kind = CASES[NAMES.index("neither_divisible")]
    z = x.copy()
    assert orc.orc_clahe(P(z), P(z), w, h, n, clip, tx, ty) == 0 and (z == y).all()
    for args in ((clip, 0, 4), (clip, 4, 0), (clip, w + 1, 4), (clip, 4, h + 1), (-1.0, 4, 4), (float("nan"), 4, 4)):
        assert orc.orc_clahe(P(z), P(z), w, h, n, args[0], args[1], args[2]) == -1, args


def frames_and_golden():
    from alvaar_b200 import synth
    g = golden("system_clahe")
    w, h, nf = int(g["w"]), int(g["h"]), int(g["nframes"])
    frames = compress_contrast(synth.make_frames(nf, w, h, seed=int(g["seed"]), rgba=True)[0])
    assert hashlib.sha256(frames.tobytes()).hexdigest() == str(g["sha256"]), "synthetic frames changed: re-dump the golden"
    return g, frames


def test_golden_trace_initialises_and_runs_a_local_ba():
    g, frames = frames_and_golden()
    init = int(np.argmax(g["ref_status"] == 1))
    assert (g["ref_status"] == 1).any() and 0 < init
    kf_init = int(g["ref_info"][init][1])
    assert int(g["ref_info"][:, 1].max()) >= kf_init + 2                       # at least two keyframes after the initialisation
    assert init < int(g["first_ba_frame"]) < len(frames)                        # and a local BA
    assert (g["ref_status"][init:] == 1).all()


class ReplayHook:
    """The reference's compute5ptEssentialMatrix as the CPU state machine's initialisation hook: live when the reference is
    built, else replaying its calls recorded in system_clahe.npz (their inputs' digests are checked)."""
    PROTO = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p)

    def __init__(self, ref, g):
        self.ref, self.g, self.n, self.errors = ref, g, 0, []
        if ref is not None:
            ref.ref_essential_5pt.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
        self.cb = self.PROTO(self._call)
        self.ptr = C.cast(self.cb, C.c_void_p)

    def _call(self, b1, b2, n, it, err, opt, fx, fy, Rt, outl):
        try:
            i = self.n
            self.n += 1
            if self.ref is not None:
                return self.ref.ref_essential_5pt(b1, b2, n, it, err, opt, fx, fy, Rt, outl)
            ins = digest(np.concatenate([np.ctypeslib.as_array((C.c_double * (3 * n)).from_address(b1)),
                                         np.ctypeslib.as_array((C.c_double * (3 * n)).from_address(b2)),
                                         np.array([it, err, opt, fx, fy], np.float64)]))
            if not (self.g[f"ess_c{i}_in"] == ins).all() or len(self.g[f"ess_c{i}_outl"]) != n:
                self.errors.append(f"call {i}: inputs differ from the recorded ones")
                return 0
            C.memmove(Rt, np.ascontiguousarray(self.g[f"ess_c{i}_Rt"]).ctypes.data, 96)
            C.memmove(outl, np.ascontiguousarray(self.g[f"ess_c{i}_outl"]).ctypes.data, n)
            return int(self.g[f"ess_c{i}_ok"])
        except Exception as e:   # an exception cannot cross the C frame
            self.errors.append(repr(e))
            return 0

    def finish(self):
        assert not self.errors, self.errors
        if self.ref is None:
            assert self.n == int(self.g["ess_ncalls"]), (self.n, int(self.g["ess_ncalls"]))


def run(S, frames, K, clahe=True, hook=None, nframes=None):
    s = S.cpu_clahe_system_create(frames.shape[2], frames.shape[1], K[0], K[1], K[2], K[3])
    if clahe:
        assert S.cpu_system_set_clahe(s, 1, 3.0, 50) == 0
    if hook is not None:
        S.cpu_clahe_system_set_essential_hook(s, hook)
    out = []
    for k in range(nframes or len(frames)):
        T = np.zeros(7)
        st = S.cpu_clahe_system_process(s, P(np.ascontiguousarray(frames[k])), k * 33.333, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3)); info = np.zeros(8, np.int32)
        n = S.cpu_clahe_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP)
        S.cpu_clahe_system_info(s, P(info))
        out.append((st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy(), wp[:n].copy()))
    S.cpu_clahe_system_destroy(s)
    return out


def test_state_machine_with_clahe_given_the_reference_initialisation(oracle, ref):
    g, frames = frames_and_golden()
    hook = ReplayHook(ref, g)
    tr = run(cpu_clahe_system_lib(), frames, g["K"], hook=hook.ptr)
    hook.finish()
    init = int(np.argmax(g["ref_status"] == 1))
    for k, (st, T, info, ids, px, d3, wp) in enumerate(tr):
        rids, rpx, rd3, rwp = frame_slice(g, "ref_", k)
        assert st == g["ref_status"][k] and (info == g["ref_info"][k]).all(), (k, st, info, g["ref_info"][k])
        assert len(ids) == len(rids) and (ids == rids).all() and (d3 == rd3).all(), k
        if k < init:
            assert (px.view(np.uint32) == rpx.view(np.uint32)).all(), k
        assert np.abs(T - g["ref_Twc"][k]).max() < 1e-9, k
        assert np.abs(wp - rwp).max(initial=0) < 1e-9 * max(1.0, np.abs(rwp).max(initial=0)), k


def test_committed_cpu_trace_is_this_state_machine(oracle):
    """the `cpu_*` trace (what the GPU build is compared with, its own initialisation) is this very state machine"""
    g, frames = frames_and_golden()
    tr = run(cpu_clahe_system_lib(), frames, g["K"])
    for k, (st, T, info, ids, px, d3, wp) in enumerate(tr):
        cids, cpx, cd3, cwp = frame_slice(g, "cpu_", k)
        assert st == g["cpu_status"][k] and (info == g["cpu_info"][k]).all(), k
        assert (ids == cids).all() and (d3 == cd3).all() and (px.view(np.uint32) == cpx.view(np.uint32)).all(), k
        assert np.abs(T - g["cpu_Twc"][k]).max() < 1e-12, k


def test_clahe_off_is_the_plain_backend(oracle):
    """with CLAHE off the CLAHE backend is the plain one: the first 20 frames of system.npz's `cpu_*` trace, bit for bit"""
    g = golden("system")
    from alvaar_b200 import synth
    frames, _ = synth.make_frames(20, int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True)
    tr = run(cpu_clahe_system_lib(), frames, g["K"], clahe=False)
    for k, (st, T, info, ids, px, d3, wp) in enumerate(tr):
        cids, cpx, cd3, cwp = frame_slice(g, "cpu_", k)
        assert st == g["cpu_status"][k] and (ids == cids).all() and (px.view(np.uint32) == cpx.view(np.uint32)).all(), k
        assert (T == g["cpu_Twc"][k]).all(), k


def test_cpu_switch_rejects_an_empty_grid(oracle):
    S = cpu_clahe_system_lib()
    s = S.cpu_clahe_system_create(640, 480, 500.0, 500.0, 320.0, 240.0)
    assert S.cpu_system_set_clahe(s, 1, 3.0, 481) == -1 and S.cpu_system_set_clahe(s, 1, 3.0, 0) == -1
    assert S.cpu_system_set_clahe(s, 1, 3.0, 480) == 0
    S.cpu_clahe_system_destroy(s)


def test_system_switch_needs_a_configured_system():
    """alva_system_set_clahe before configure -> ALVA_E_STATE; a null handle -> ALVA_E_INVALID (no device needed)"""
    from alvaar_b200 import lib
    L = lib()
    L.alva_system_create.restype = C.c_void_p
    L.alva_system_destroy.argtypes = [C.c_void_p]
    L.alva_system_set_clahe.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int]
    s = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_clahe(s, 1, 3.0, 50) == -4
    assert L.alva_system_set_clahe(None, 1, 3.0, 50) == -1
    L.alva_system_destroy(s)
