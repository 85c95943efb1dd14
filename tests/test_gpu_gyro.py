"""H100: gyro-aided tracking in the CUDA System (alva_system_set_gyro / alva_system_find_camera_pose_gyro) and its kernel
(alva_k_rotate_priors).  The kernel equals the host build of the same arithmetic (camera_model.h, through the CPU gyro shim) bit
for bit on every lens, from 1 to 100 000 points and on the boundary cases; from the same frames and samples the GPU System and
the CPU backend track the pan sequence in lockstep; with the mode off the GPU outputs are those of a run that never calls it;
the Python facade reports its errors."""
import ctypes as C

import numpy as np
import pytest
import torch

import gyro_util as G
import reloc_util as U
from alvaar_b200 import AlvaError, Context, System, synth
from alvaar_b200.system import _bind

pytestmark = pytest.mark.gpu

PEAK = 240.0


@pytest.fixture(scope="module")
def S():
    return G.lib()


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, torch.cuda.current_stream().cuda_stream)
    yield c
    c.close()


LENS = {"pinhole": (0, None), "radtan": (1, U.DIST), "fisheye": (2, G.FISHEYE)}


def _rot(rng, deg):
    from scipy.spatial.transform import Rotation
    v = rng.normal(size=3)
    return Rotation.from_rotvec(v / np.linalg.norm(v) * np.radians(deg)).as_matrix()


def _check(ctx, S, bv, flag, w, h, lens, R, prior0):
    code, D = LENS[lens]
    K = synth.intrinsics(w, h)
    want, wrot = G.rotate_priors_host(S, bv, flag, w, h, K, D, code, R.reshape(9), prior0)
    n = len(flag)
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()  # noqa: E731
    pr = d(prior0, np.float32)
    rot = torch.full((max(n, 1),), 7, dtype=torch.uint8, device="cuda")
    ctx.rotate_priors(d(bv, np.float64), d(flag, np.uint8), n, w, h, K, D, code, R.reshape(9), pr, rot)
    torch.cuda.synchronize()
    got, grot = pr.cpu().numpy(), rot.cpu().numpy()[:n]
    assert got.view(np.uint32).tobytes() == want.view(np.uint32).tobytes()
    assert np.array_equal(grot, wrot)
    return wrot


@pytest.mark.parametrize("lens", ["pinhole", "radtan", "fisheye"])
@pytest.mark.parametrize("n", [1, 7, 1000, 100000])
def test_kernel_equals_the_host_build(ctx, S, lens, n):
    rng = np.random.default_rng(n)
    w, h = (1920, 1080) if n > 1000 else (640, 480)
    K = synth.intrinsics(w, h)
    # bearings of pixels over (and beyond) the image, a share behind the camera; rotations up to 20 degrees
    u, v = rng.uniform(-0.2, 1.2, n) * w, rng.uniform(-0.2, 1.2, n) * h
    bv = np.stack([(u - K[2]) / K[0], (v - K[3]) / K[1], np.ones(n)], 1)
    bv[rng.random(n) < 0.05] *= -1
    bv /= np.linalg.norm(bv, axis=1, keepdims=True)
    flag = (rng.random(n) < 0.8).astype(np.uint8)
    prior0 = rng.uniform(0, w, (n, 2)).astype(np.float32)
    rot = _check(ctx, S, bv, flag, w, h, lens, _rot(rng, rng.uniform(0, 20)), prior0)
    if n >= 1000:
        assert 0 < rot.sum() < flag.sum()


def test_kernel_boundaries(ctx, S):
    """z = 0, z < 0 and z a hair above 0; projections straddling every image edge by a few float steps; fisheye rays at and
    beyond the lens's limit (incidence near and past 90 degrees)"""
    w, h = 640, 480
    K = synth.intrinsics(w, h)
    R = np.eye(3)
    rays = [[0.1, 0.1, 0.0], [0.1, 0.1, -0.0], [0.1, 0.1, -1e-300], [0.1, 0.1, 1e-300], [0.0, 0.0, 1.0], [0.0, 0.0, -1.0]]
    for edge_u in (0.0, w):
        for du in np.arange(-40, 41) * 2e-6 * (1 + edge_u):   # a few float steps either side of the edge
            x = (edge_u + du - K[2]) / K[0]
            rays.append([x, 0.0, 1.0])
    for edge_v in (0.0, h):
        for dv in np.arange(-40, 41) * 2e-6 * (1 + edge_v):
            rays.append([0.0, (edge_v + dv - K[3]) / K[1], 1.0])
    for ang in np.radians([80, 88, 89.9, 89.999999, 90.0, 90.0001, 100, 179.9]):
        for az in np.radians([0, 37, 90, 200]):
            rays.append([np.sin(ang) * np.cos(az), np.sin(ang) * np.sin(az), np.cos(ang)])
    bv = np.array(rays, np.float64)
    flag = np.ones(len(bv), np.uint8)
    prior0 = np.full((len(bv), 2), 12.5, np.float32)
    for lens in ("pinhole", "radtan", "fisheye"):
        rot = _check(ctx, S, bv, flag, w, h, lens, R, prior0)
        assert rot[0] == rot[1] == rot[2] == 0 and rot[4] == 1 and rot[5] == 0
    # the edge sweeps land on both sides of the image border (pinhole: one float step decides)
    _, r = G.rotate_priors_host(S, bv, flag, w, h, K, None, 0, R.reshape(9), prior0)
    edges = r[6:6 + 4 * 81].reshape(4, 81)
    assert all(0 < e.sum() < 81 for e in edges)
    # a turned frame: rotations move the same rays across the edges
    rng = np.random.default_rng(9)
    for lens in ("pinhole", "radtan", "fisheye"):
        _check(ctx, S, bv, flag, w, h, lens, _rot(rng, 3.0), prior0)


# ------------------------------------------------------------------------------------------------ the System
class GpuRun:
    def __init__(self, fisheye=None, max_lost=30, gyro=True):
        K = synth.intrinsics(G.W, G.H)
        self.s = System(G.W, G.H, *K)
        if fisheye is not None:
            self.s.set_fisheye(True, *fisheye)
        self.s.set_relocalisation(max_lost)
        if gyro:
            self.s.set_gyro(True, G.R_CI, G.BIAS)

    def frame(self, rgba, t, smp):
        st, pose = self.s.find_camera_pose_gyro(np.ascontiguousarray(rgba), t, smp)
        ids, px, d3, _ = self.s.tracks()
        return st, self.s.pose(), ids.copy(), px.copy(), d3.copy(), pose


# Poses relative to max(1, |t|).  Statuses, ids, 3-D flags and counters are identical frame by frame; the poses drift apart
# slowly because the two backends' P3P / PnP / local-BA solves agree to ~1e-9 .. 1e-4 relative per solve and the pan makes a
# keyframe (and a local BA) every few frames.  Observed on an H100 over the 90 frames: worst 5.2e-4 (pinhole) and 3.9e-4
# (fisheye), above test_gpu_reloc.py's 2e-4 from frame 37 / 57 on.  Bar: 2e-3 over the whole sequence.
@pytest.mark.parametrize("lens", ["pinhole", "fisheye"])
def test_system_equals_the_cpu_backend(S, lens):
    kw = {"fisheye": G.FISHEYE} if lens == "fisheye" else {}
    frames, times, smp, _ = G.pan_sequence(90, peak_dps=PEAK, **kw)
    cpu = G.CpuGyroRun(S, max_lost=30, gyro=(G.R_CI, G.BIAS), **kw)
    gpu = GpuRun(**kw)
    worst = 0.0
    for k in range(len(frames)):
        st_c, T_c, _, ids_c, _, d3_c = cpu.frame(frames[k], times[k], smp[k])
        st_g, T_g, ids_g, _, d3_g, _ = gpu.frame(frames[k], times[k], smp[k])
        assert st_c == st_g, k
        oc, og = np.argsort(ids_c), np.argsort(ids_g)
        assert np.array_equal(ids_c[oc], ids_g[og]) and np.array_equal(d3_c[oc], d3_g[og]), k
        worst = max(worst, np.abs(T_c - T_g).max() / max(1.0, float(np.linalg.norm(T_c[:3]))))
    print(f"{lens}: pose |CPU - GPU| / max(1, |t|) <= {worst:.2e}")
    sc, dRc = cpu.stats()
    sg, dRg = gpu.s.gyro_stats()
    assert all(sc[k] == sg[k] for k in sg), (sc, sg)
    assert np.abs(dRc - dRg).max() <= 1e-15
    assert sg["predicted"] == len(frames) - 1 and sg["rotated"] > 0
    assert worst < 2e-3, worst
    cpu.close()
    gpu.s.close()


def test_mode_off_is_bit_identical(S):
    frames, times, smp, _ = G.pan_sequence(60, peak_dps=PEAK)
    runs = []
    for mode in ("never", "off", "samples_mode_never_on"):
        K = synth.intrinsics(G.W, G.H)
        s = System(G.W, G.H, *K)
        s.set_relocalisation(30)
        if mode == "off":
            s.set_gyro(False)
        out = []
        for k in range(len(frames)):
            f = np.ascontiguousarray(frames[k])
            st, pose = s.find_camera_pose(f, times[k]) if mode == "never" else s.find_camera_pose_gyro(f, times[k], smp[k])
            ids, px, d3, _ = s.tracks()
            out.append((st, pose.tobytes(), s.pose().tobytes(), ids.tobytes(), px.tobytes(), d3.tobytes()))
        assert s.gyro_stats()[0]["predicted"] == 0
        s.close()
        runs.append(out)
    assert runs[0] == runs[1] == runs[2]


def test_python_facade_errors():
    K = synth.intrinsics(G.W, G.H)
    L = _bind()
    raw = C.c_void_p(L.alva_system_create(0))
    assert L.alva_system_set_gyro(raw, 1, None, None) == -4          # before configure
    assert L.alva_system_set_gyro(None, 1, None, None) == -1
    assert L.alva_system_find_camera_pose_gyro(raw, None, 0.0, None, 0, None) == -1
    L.alva_system_destroy(raw)
    s = System(G.W, G.H, *K)
    with pytest.raises(AlvaError):
        s.set_gyro(True, np.diag([1.0, 1.0, -1.0]))                 # a reflection
    with pytest.raises(AlvaError):
        s.set_gyro(True, 1.001 * np.eye(3))
    with pytest.raises(AlvaError):
        s.set_gyro(True, None, [0.0, np.nan, 0.0])
    assert L.alva_system_set_gyro(s.h, 2, None, None) == -1
    s.set_gyro(True, G.R_CI, G.BIAS)
    frame = synth.gray_to_rgba(synth.crop(G.W, G.H))
    s.find_camera_pose_gyro(frame, 10.0, [[5.0, 0, 0, 0, 0, 0, 0], [9.0, 0, 0, 0, 0, 0, 0]])
    for bad in ([[8.0, 0, 0, 0, 0, 0, 0]], [[12.0, 0, 0, 0, 0, 0, 0], [11.0, 0, 0, 0, 0, 0, 0]], [[12.0, np.inf, 0, 0, 0, 0, 0]]):
        with pytest.raises(AlvaError):
            s.find_camera_pose_gyro(frame, 20.0, bad)
    assert s.info()["frame"] == 0                                    # no refused call processed a frame
    pose = np.zeros(16, np.float32)
    assert L.alva_system_find_camera_pose_gyro(s.h, frame.ctypes.data_as(C.c_void_p), 20.0, None, 3, pose.ctypes.data_as(C.c_void_p)) == -1
    assert L.alva_system_gyro_stats(s.h, None, None) == -1
    s.find_camera_pose_gyro(frame, 33.0, np.zeros((0, 7)))
    assert s.info()["frame"] == 1
    s.close()
