"""Shared by the relocalisation tests: the oracle of the matching and RANSAC stages (oracle/reloc_oracle.c), the CPU oracle build
of the System state machine with relocalisation (tests/host/system_cpu_reloc.cpp), a numpy grouped 2-NN, the synthetic
sequences (a loss, then a revisit or an unrelated scene) and the similarity fit between the synthetic and the tracked frames."""
import ctypes as C
import os
import subprocess

import numpy as np

from alvaar_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
CAP = 8192
W, H = 640, 480
DIST = (-0.12, 0.03, 0.001, -0.0005)


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def _oracle_so():
    orc = os.path.join(ROOT, "oracle", "_build", "libalva_oracle.so")
    if not os.path.exists(orc):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL)
    return orc


def reloc_oracle_lib():
    """oracle/reloc_oracle.c (with libalva_oracle.so for the sampler and the P3P hypotheses) -- test infrastructure"""
    so = os.path.join(ROOT, "tests", "_build", "libreloc_oracle.so")
    orc = _oracle_so()
    src = os.path.join(ROOT, "oracle", "reloc_oracle.c")
    if _stale(so, [src, orc]):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-std=gnu11", "-Wall", "-shared", "-o", so, src, orc, "-lm",
                               "-Wl,-rpath," + os.path.dirname(orc)])
    L = C.CDLL(so)
    L.orc_hamming_knn2_grouped.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_reloc_select.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_p3p_ransac.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_uint32, C.c_void_p, C.c_void_p,
                                 C.c_void_p]
    O = C.CDLL(orc)
    O.orc_p3p_lmeds.argtypes = L.orc_p3p_ransac.argtypes
    L.lmeds = O.orc_p3p_lmeds
    return L


def knn2_grouped_oracle(L, q, desc_start, desc):
    nq, ng = len(q), len(desc_start) - 1
    out = np.zeros((max(nq, 1), 4), np.int32)
    L.orc_hamming_knn2_grouped(P(np.ascontiguousarray(q)), nq, P(np.ascontiguousarray(desc_start, dtype=np.int32)), ng,
                               P(np.ascontiguousarray(desc) if len(desc) else np.zeros((1, 32), np.uint8)), P(out))
    return out[:nq]


def knn2_grouped_numpy(q, desc_start, desc):
    """brute force: per query the distance to every row, the minimum per group, a stable sort by (distance, group)"""
    nq, ng = len(q), len(desc_start) - 1
    out = np.full((nq, 4), -1, np.int32)
    if nq == 0 or ng == 0 or len(desc) == 0:
        return out
    qb = np.unpackbits(q, axis=1).astype(np.int32)
    tb = np.unpackbits(desc, axis=1).astype(np.int32)
    d = (qb[:, None, :] != tb[None, :, :]).sum(-1)
    big = 1 << 20
    gd = np.full((nq, ng), big, np.int64)
    for g in range(ng):
        a, b = desc_start[g], desc_start[g + 1]
        if b > a:
            gd[:, g] = d[:, a:b].min(1)
    for i in range(nq):
        order = np.lexsort((np.arange(ng), gd[i]))
        for k in range(2):
            if k < ng and gd[i, order[k]] < big:
                out[i, 2 * k] = order[k]
                out[i, 2 * k + 1] = gd[i, order[k]]
    return out


def random_table(rng, n_grp, max_rows, nq, planted=0.5, flip=0.05, min_rows=1):
    """a CSR table of n_grp groups with min_rows..max_rows random descriptors, and nq queries of which a share are a few bits
    from a row of a random group"""
    rows = rng.integers(min_rows, max_rows + 1, n_grp)
    desc_start = np.concatenate([[0], np.cumsum(rows)]).astype(np.int32)
    desc = rng.integers(0, 256, (int(desc_start[-1]), 32), dtype=np.uint8)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    npl = int(nq * planted)
    if len(desc) and npl:
        src = rng.integers(0, len(desc), npl)
        q[:npl] = desc[src] ^ np.packbits(rng.random((npl, 256)) < flip, axis=1)
    return q, desc_start, desc


# ------------------------------------------------------------------------------------------------ the CPU state machine
def cpu_reloc_system_lib():
    """alvaar_b200/csrc/system_core.h over the CPU oracle with relocalisation (tests/host/system_cpu_reloc.cpp)"""
    from preset_util import cpu_preset_system_lib
    cpu_preset_system_lib()   # builds the CLAHE and cell-size matcher oracles it links
    reloc_oracle_lib()
    so = os.path.join(ROOT, "tests", "_build", "libsystem_cpu_reloc.so")
    orc = _oracle_so()
    b = os.path.join(ROOT, "tests", "_build")
    corc, morc, rorc = (os.path.join(b, n) for n in ("libclahe_oracle.so", "libmatch_cell_oracle.so", "libreloc_oracle.so"))
    host = os.path.join(ROOT, "tests", "host")
    srcs = [os.path.join(host, f) for f in ("system_cpu_reloc.cpp", "system_cpu_preset.cpp", "system_cpu_clahe.cpp", "system_cpu_backend.cpp")]
    srcs += [os.path.join(ROOT, "alvaar_b200", "csrc", "system_core.h"), orc, corc, morc, rorc]
    if _stale(so, srcs):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0], orc, corc, morc, rorc,
                               "-Wl,-rpath," + os.path.dirname(orc), "-Wl,-rpath," + b])
    S = C.CDLL(so)
    S.cpu_reloc_system_create.restype = C.c_void_p
    S.cpu_reloc_system_create.argtypes = [C.c_int, C.c_int] + [C.c_double] * 4
    S.cpu_reloc_system_set_relocalisation.argtypes = [C.c_void_p, C.c_int]
    S.cpu_reloc_system_set_preset.argtypes = [C.c_void_p, C.c_int]
    S.cpu_reloc_system_set_distortion.argtypes = [C.c_void_p] + [C.c_double] * 4
    S.cpu_reloc_system_process.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    S.cpu_reloc_system_keypoints.argtypes = [C.c_void_p] * 5 + [C.c_int]
    S.cpu_reloc_system_info.argtypes = [C.c_void_p, C.c_void_p]
    S.cpu_reloc_system_counters.argtypes = [C.c_void_p, C.c_void_p]
    S.cpu_reloc_system_reset.argtypes = [C.c_void_p]
    S.cpu_reloc_system_destroy.argtypes = [C.c_void_p]
    return S


class CpuRelocRun:
    """the CPU state machine, frame by frame: (status, Twc7, info8, ids, px, is3d)"""

    def __init__(self, S, max_lost=None, preset=None, dist=None):
        K = synth.intrinsics(W, H)
        self.S, self.s = S, S.cpu_reloc_system_create(W, H, *K)
        if preset is not None:
            assert S.cpu_reloc_system_set_preset(self.s, preset) == 0
        if dist is not None:
            S.cpu_reloc_system_set_distortion(self.s, *dist)
        if max_lost is not None:
            assert S.cpu_reloc_system_set_relocalisation(self.s, max_lost) == 0

    def frame(self, rgba, t_ms):
        S, s = self.S, self.s
        T = np.zeros(7)
        st = S.cpu_reloc_system_process(s, P(np.ascontiguousarray(rgba)), t_ms, P(T))
        ids = np.zeros(CAP, np.int32); px = np.zeros((CAP, 2), np.float32); d3 = np.zeros(CAP, np.uint8); wp = np.zeros((CAP, 3))
        info = np.zeros(8, np.int32)
        n = S.cpu_reloc_system_keypoints(s, P(ids), P(px), P(d3), P(wp), CAP)
        S.cpu_reloc_system_info(s, P(info))
        return st, T, info, ids[:n].copy(), px[:n].copy(), d3[:n].copy()

    def counters(self):
        o = np.zeros(8, np.int32)
        self.S.cpu_reloc_system_counters(self.s, P(o))
        return dict(zip(("lost", "relocalised", "matches", "inliers", "is_lost", "lost_frames", "table_points", "table_rows"), o.tolist()))

    def close(self):
        self.S.cpu_reloc_system_destroy(self.s)


# ------------------------------------------------------------------------------------------------ sequences
def _mid_pose(poses, k, yaw_deg=1.0):
    """halfway between trajectory poses k and k + 1, turned by yaw_deg about the camera's vertical axis: a view never rendered"""
    from scipy.spatial.transform import Rotation, Slerp
    (R0, t0), (R1, t1) = poses[k], poses[k + 1]
    Rm = Slerp([0, 1], Rotation.from_matrix([R0, R1]))(0.5).as_matrix()
    return Rm @ Rotation.from_euler("y", yaw_deg, degrees=True).as_matrix(), 0.5 * (t0 + t1)


def revisit_sequence(dist=None, n_revisit=24):
    """make_frames(40, seed 7), three black frames, then n_revisit views at new poses from frame 15 on, and the true
    camera-to-world poses of every rendered frame (None for the black ones)"""
    A, poses = synth.make_frames(40, W, H, seed=7, rgba=True, dist=dist)
    black = np.zeros_like(A[0]); black[..., 3] = 255
    tex = synth.make_texture()
    # halfway poses from frame 15 on, turned by 1 degree: the first ten lie among frames 15-25, the rest continue the path
    rv = [_mid_pose(poses, 15 + i) for i in range(n_revisit)]
    R = [synth.gray_to_rgba(synth.render_gray(tex, p, W, H, dist=dist)) for p in rv]
    frames = list(A) + [black] * 3 + R
    truth = list(poses) + [None] * 3 + rv
    return frames, truth


def unrelated_sequence(n_after=24):
    """make_frames(40, seed 7), three black frames, then frames of another scene (texture seed 4321)"""
    A, poses = synth.make_frames(40, W, H, seed=7, rgba=True)
    B, _ = synth.make_frames(n_after, W, H, seed=33, rgba=True, texture_seed=4321)
    black = np.zeros_like(A[0]); black[..., 3] = 255
    return list(A) + [black] * 3 + list(B)


def failure_paths_sequence():
    """the sequence of test_system_core_cpu.py's failure-path lockstep: a blackout, a jump to another path, a jump back"""
    A, _ = synth.make_frames(40, W, H, seed=7, rgba=True)
    B, _ = synth.make_frames(26, W, H, seed=33, rgba=True)
    black = np.zeros_like(A[0]); black[..., 3] = 255
    return [A[k] for k in range(24)] + [black] + [B[k] for k in range(26)] + [A[k] for k in range(20, 40)]


def _Twc_of(T7):
    return synth.quat_to_R(T7[3:]), T7[:3]


def true_in_map(fit, pose):
    """a synthetic camera-to-world pose (R_wc, t_wc) mapped into the system's frame by the similarity fit"""
    s, R, t = fit
    return R @ pose[0], s * R @ pose[1] + t


def pose_error(T7, want):
    """(|dt|, rotation angle in degrees) between a tracked [t, q] and a (R, t) pose in the same frame"""
    Rg, tg = _Twc_of(T7)
    dR = Rg.T @ want[0]
    ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
    return float(np.linalg.norm(tg - want[1])), float(ang)


def fit_from_track(truth, tracked):
    """the similarity (s, R, t) from the synthetic frame to the system's, fitted over the frames tracked with status 1
    ({frame: Twc7}).  The camera path of a short sequence is close to a line, which leaves the rotation of a centres-only
    (Umeyama) fit loose about it: the rotation is the chordal mean of R_sys R_true^T over the frames, and scale and
    translation are then Umeyama's least-squares solution given that rotation."""
    M = sum(_Twc_of(tracked[k])[0] @ truth[k][0].T for k in tracked)
    U, _, Vt = np.linalg.svd(M)
    R = U @ np.diag([1, 1, np.linalg.det(U @ Vt)]) @ Vt
    y = np.array([R @ truth[k][1] for k in tracked])
    c = np.array([tracked[k][:3] for k in tracked])
    yc, cc = y - y.mean(0), c - c.mean(0)
    s = float((yc * cc).sum() / (yc * yc).sum())
    return s, R, c.mean(0) - s * y.mean(0)
