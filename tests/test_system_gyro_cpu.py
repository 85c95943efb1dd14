"""Gyro-aided tracking (alva_system_set_gyro / alva_system_find_camera_pose_gyro) on the CPU oracle build of the System state
machine (tests/host/system_cpu_gyro.cpp): the mode off changes nothing, the integration equals a numpy model of the rule in
system_core.h, a fast pan that the camera-only tracker loses keeps tracking with the gyro on all three lenses, the reported
rotation follows the camera through a blackout, refusals change nothing, and a gyro run is clean under AddressSanitizer and
UBSan."""
import os
import subprocess
import sys

import numpy as np
import pytest

import gyro_util as G
import reloc_util as U
from alvaar_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "system.npz")
PEAK = 240.0   # deg/s at the sweeps' peak (24 deg raised-cosine yaw, half that in pitch): the camera-only tracker loses it


@pytest.fixture(scope="module")
def S():
    return G.lib()


@pytest.fixture(scope="module")
def pan():
    return G.pan_sequence(90, peak_dps=PEAK)


def _same(a, b):
    """two runs' outputs are bit-identical: statuses, ids, 3-D flags, positions and pose bits"""
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert x[0] == y[0], (k, x[0], y[0])
        assert x[1].tobytes() == y[1].tobytes(), k
        for i in (2, 3, 4, 5):
            assert np.array_equal(x[i], y[i]), (k, i)


def _run(S, frames, times, smp=None, setup=None, **kw):
    r = G.CpuGyroRun(S, **kw)
    if setup:
        setup(r)
    out = [r.frame(frames[k], times[k], None if smp is None else smp[k]) for k in range(len(frames))]
    stats = r.stats()
    r.close()
    return out, stats


# ------------------------------------------------------------------------------------------------ the mode off
def _golden_frames():
    g = np.load(GOLDEN)
    frames, _ = synth.make_frames(int(g["nframes"]), int(g["w"]), int(g["h"]), seed=int(g["seed"]), rgba=True)
    return list(frames), [k * 33.333 for k in range(len(frames))]


@pytest.mark.parametrize("seq", ["system_npz", "pan"])
def test_mode_off_equals_no_call(S, pan, seq):
    """mode off, mode on without samples (every frame falls back) and samples with the mode off: bit-identical to a run that
    never calls the API"""
    if seq == "pan":
        frames, times, smp, _ = pan
    else:
        frames, times = _golden_frames()
        rng = np.random.default_rng(3)
        smp = [np.concatenate([(t - np.array([25.0, 17.0, 9.0, 1.0]))[:, None], rng.normal(0, 2, (4, 6))], 1) for t in times]
    base, _ = _run(S, frames, times, max_lost=0 if seq == "system_npz" else 30)
    ml = 0 if seq == "system_npz" else 30
    off, st_off = _run(S, frames, times, setup=lambda r: r.set_gyro(0), max_lost=ml)
    _same(base, off)
    nosmp, st_ns = _run(S, frames, times, gyro=(G.R_CI, G.BIAS), max_lost=ml)
    _same(base, nosmp)
    assert st_ns[0]["predicted"] == 0 and st_ns[0]["fallback"] == len(frames) - 1 and st_ns[0]["rotated"] == 0
    ignored, st_ig = _run(S, frames, times, smp, max_lost=ml)
    _same(base, ignored)
    assert st_ig[0]["held"] == 0 and st_off[0]["held"] == 0


# ------------------------------------------------------------------------------------------------ the integration rule
def _random_stream(rng, nframes):
    """per frame: its time stamp and the samples passed with it -- 100-200 Hz jittered, duplicate time stamps, samples
    running past the frame time, gaps of more than 50 ms, bursts of fast rotation"""
    t, tf, out, pending = 0.0, 0.0, [], []
    rate = 0.0
    for k in range(nframes):
        tf += rng.choice([33.0, 33.0, 34.0, 16.0, 66.0, 0.0])   # equal frame times too
        smp = list(pending)
        pending = []
        while t <= tf + rng.uniform(-5, 20):
            step = rng.choice([5.0, 7.5, 10.0, 0.0, 1.0, 60.0, 120.0], p=[0.3, 0.2, 0.2, 0.1, 0.1, 0.05, 0.05])
            t += step
            rate += rng.normal(0, 0.5)
            s = [t] + list(rng.normal(0, 1.0, 3) * (1 + abs(rate))) + list(rng.normal(0, 9.8, 3))
            if t <= tf or (not pending and rng.random() < 0.3):   # (the second: a sample past the frame time handed over early)
                smp.append(s)
            else:
                pending.append(s)
        out.append((tf, np.array(smp, np.float64).reshape(-1, 7)))
    return out


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_integration_equals_numpy_model(S, seed):
    """dR9 after every frame equals the numpy model of the rule within 1e-12; uncovered frames count as fallbacks"""
    rng = np.random.default_rng(seed)
    from scipy.spatial.transform import Rotation
    R_ci = Rotation.from_rotvec(rng.normal(size=3)).as_matrix() if seed % 2 else G.R_CI
    bias = rng.normal(0, 0.05, 3)
    w, h = 640, 480
    img = synth.gray_to_rgba(synth.crop(w, h))    # a static scene (the random rotations still make KLT lose it at times)
    r = G.CpuGyroRun(S, gyro=(R_ci, bias), w=w, h=h)
    model = G.GyroModel(R_ci, bias)
    fallbacks, covered, prev_id = 0, 0, -1
    info = np.zeros(8, np.int32)
    for k, (tf, smp) in enumerate(_random_stream(rng, 120)):
        st, _ = r.process(img, tf, smp)
        assert st in (1, 2, 3), st
        want = model.frame(tf, smp)
        stats, dR = r.stats()
        on_path = prev_id >= 0              # the frame after a reset starts the track: nothing to predict, nothing counted
        S.cpu_gyro_system_info(r.s, G.P(info))
        prev_id = int(info[0])
        if want is None:
            fallbacks += on_path
            assert np.array_equal(dR, np.eye(3)), k
        else:
            covered += 1
            assert np.abs(dR - want).max() <= 1e-12, (k, np.abs(dR - want).max())
        assert stats["fallback"] == fallbacks, k
        assert stats["held"] == len(model.buf), k
    assert covered > 40 and fallbacks > 5
    r.close()


# ------------------------------------------------------------------------------------------------ the pan sequence
# Observed on this sequence (90 frames at 30 Hz, initialisation at frame 13, peak 240 deg/s), after the similarity fit over the
# tracked frames: max |dt| 0.026 / 0.058 / 0.038 and max rotation error 0.12 / 0.23 / 0.20 deg (pinhole / radial-tangential /
# fisheye; |t| reaches ~0.8 in the fitted frame).  Bars: about twice those.
BARS = {"pinhole": (0.06, 0.3), "radtan": (0.12, 0.5), "fisheye": (0.08, 0.4)}


def _lens_kw(lens):
    return {"pinhole": {}, "radtan": {"dist": U.DIST}, "fisheye": {"fisheye": G.FISHEYE}}[lens]


@pytest.mark.parametrize("lens", ["pinhole", "radtan", "fisheye"])
def test_pan_tracks_with_the_gyro(S, pan, lens):
    kw = _lens_kw(lens)
    frames, times, smp, poses = pan if lens == "pinhole" else G.pan_sequence(90, peak_dps=PEAK, **kw)
    # the camera-only tracker loses the pan: status 4 with relocalisation on, a reset (status 2) with it off
    lost, _ = _run(S, frames, times, smp, max_lost=30, **kw)
    reset, _ = _run(S, frames, times, smp, max_lost=0, **kw)
    assert 4 in [o[0] for o in lost]
    assert 2 in [o[0] for o in reset]
    out, (stats, _) = _run(S, frames, times, smp, max_lost=30, gyro=(G.R_CI, G.BIAS), **kw)
    st = [o[0] for o in out]
    first = st.index(1)
    assert set(st[first:]) == {1}, "".join(map(str, st))
    assert stats["predicted"] == len(frames) - 1 and stats["fallback"] == 0 and stats["carried"] == 0
    assert stats["rotated"] > 5 * stats["kept"] > 0
    tracked = {k: out[k][1] for k in range(first, len(out))}
    fit = U.fit_from_track(poses, tracked)
    err = [U.pose_error(tracked[k], U.true_in_map(fit, poses[k])) for k in tracked]
    bt, ba = BARS[lens]
    assert max(e[0] for e in err) <= bt and max(e[1] for e in err) <= ba, (max(e[0] for e in err), max(e[1] for e in err))


# Observed: through a 5-frame blackout at frame 40 (mid-sweep) the reported rotation stays within 0.16 deg of the truth over
# the 16 lost frames, and the track relocalises at frame 56.  Bar: 0.5 deg.
def test_blackout_rotation_follows_the_camera(S):
    frames, times, smp, poses = G.pan_sequence(90, peak_dps=PEAK, blackout=(40, 5))
    out, (stats, _) = _run(S, frames, times, smp, max_lost=30, gyro=(G.R_CI, G.BIAS))
    st = [o[0] for o in out]
    lost = [k for k in range(40, len(st)) if st[k] == 4]
    assert lost[0] == 40 and len(lost) >= 5, "".join(map(str, st))
    assert st[lost[-1] + 1:] == [1] * (len(st) - lost[-1] - 1), "".join(map(str, st))   # relocalised, then tracking
    assert stats["carried"] == len(lost)
    tracked = {k: out[k][1] for k in range(len(out)) if st[k] == 1}
    fit = U.fit_from_track(poses, tracked)
    rot = [U.pose_error(out[k][1], U.true_in_map(fit, poses[k]))[1] for k in lost]
    assert max(rot) <= 0.5, rot
    # without the gyro the lost frames hold the last tracked rotation: far off by the end of the loss
    out0, _ = _run(S, frames, times, smp, max_lost=30)
    held = [U.pose_error(out0[k][1], U.true_in_map(fit, poses[k]))[1] for k in range(40, 45) if out0[k][0] == 4]
    assert held and max(held) > 5.0, held


def test_map_saved_while_lost_carries_the_rotation(S):
    frames, times, smp, _ = G.pan_sequence(46, peak_dps=PEAK, blackout=(40, 5))
    r = G.CpuGyroRun(S, max_lost=30, gyro=(G.R_CI, G.BIAS))
    for k in range(44):
        st, T = r.frame(frames[k], times[k], smp[k])[:2]
    assert st == 4
    blob = r.save()
    assert isinstance(blob, bytes)
    # the pose of the blob (after header 24 + camera 76 + grid 4 + counters 12 bytes): t [3], q [4] f64
    pose = np.frombuffer(blob[116:172], np.float64)
    assert pose.tobytes() == T.tobytes()
    r.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_change_nothing(S, pan):
    frames, times, smp, _ = pan
    n = 40
    ref, ref_stats = _run(S, frames[:n], times[:n], smp[:n], max_lost=30, gyro=(G.R_CI, G.BIAS))
    r = G.CpuGyroRun(S, max_lost=30, gyro=(G.R_CI, G.BIAS))
    out = []
    nan = np.nan
    for k in range(n):
        if k == 25:
            bad_R = [np.diag([1.0, 1.0, 1.0 + 1e-8]), np.diag([1.0, -1.0, 1.0]), np.where(np.eye(3) > 0, nan, 0.0)]
            for R in bad_R:
                assert r.set_gyro(1, R, G.BIAS) == -1, R
            assert r.set_gyro(1, G.R_CI, [0.0, np.inf, 0.0]) == -1
            assert r.set_gyro(2, G.R_CI, G.BIAS) == -1
            held = r.stats()[0]["held"]
            assert held >= 1
            last = smp[k - 1][-1, 0]
            s1 = np.array([[last + 1, 0, 0, 0, 0, 0, 0]], np.float64)
            for bad, cnt in [(s1, -1), (None, 1), (np.array([[last + 1, nan, 0, 0, 0, 0, 0]]), 1),
                             (np.array([[last + 1, 0, 0, 0, 0, 0, np.inf]]), 1),
                             (np.array([[last + 3, 0, 0, 0, 0, 0, 0], [last + 2, 0, 0, 0, 0, 0, 0]]), 2),
                             (np.array([[last - 1, 0, 0, 0, 0, 0, 0]]), 1)]:
                st, _ = r.process(frames[k], times[k], bad, cnt)
                assert st == -1, (bad, cnt)
            assert r.stats()[0]["held"] == held
        out.append(r.frame(frames[k], times[k], smp[k]))
    _same(ref, out)
    assert r.stats()[0] == ref_stats[0] and np.array_equal(r.stats()[1], ref_stats[1])
    r.close()


def test_what_keeps_and_ends_the_mode(S, pan):
    frames, times, smp, _ = pan
    r = G.CpuGyroRun(S, max_lost=30, gyro=(G.R_CI, G.BIAS))
    for k in range(3):
        r.frame(frames[k], times[k], smp[k])
    assert r.stats()[0]["predicted"] == 2
    S.cpu_gyro_system_reset(r.s)
    S.cpu_gyro_system_set_distortion(r.s, *U.DIST)
    S.cpu_gyro_system_set_fisheye(r.s, 1, *G.FISHEYE)
    S.cpu_gyro_system_set_relocalisation(r.s, 5)
    r.frame(frames[3], times[3], smp[3])
    r.frame(frames[4], times[4], smp[4])
    assert r.stats()[0]["predicted"] == 3          # still on: frame 4 (frame 3 starts the track after the resets)
    S.cpu_gyro_system_configure(r.s)               # configure ends it and clears the counters
    r.frame(frames[5], times[5], smp[5])
    r.frame(frames[6], times[6], smp[6])
    st, dR = r.stats()
    assert st["predicted"] == 0 and st["held"] == 0 and np.array_equal(dR, np.eye(3))
    assert r.set_gyro(1, G.R_CI, G.BIAS) == 0 and r.set_gyro(0) == 0 and r.stats()[0]["held"] == 0
    r.close()


# ------------------------------------------------------------------------------------------------ sanitizers
GYRO_RUN = r"""
import sys
sys.path[:0] = [{tests!r}, {root!r}]
import numpy as np
import gyro_util as G
S = G.bind({so!r})
d = np.load({data!r}, allow_pickle=True)
frames, times, smp = d["frames"], d["times"], list(d["smp"])
r = G.CpuGyroRun(S, max_lost=30, gyro=(G.R_CI, G.BIAS))
st = [r.frame(frames[k], times[k], smp[k])[0] for k in range(len(frames))]
assert r.process(frames[0], times[-1], np.zeros((1, 7)), 1)[0] == -1
r.set_gyro(0)
st += [r.frame(frames[k], times[-1] + 33 * k)[0] for k in range(3)]
print(" ".join(map(str, st)), r.stats()[0])
r.close()
"""


def test_gyro_run_under_sanitizers(tmp_path):
    """the shim built with -fsanitize=address,undefined: a pan with a blackout (prediction, rotated priors, lost frames the
    gyro carries, relocalisation), a refusal and the mode switched off, without a sanitizer report"""
    so = G.cpu_gyro_system_lib(sanitize=True)
    asan = subprocess.check_output(["g++", "-print-file-name=libasan.so"], text=True).strip()
    ubsan = subprocess.check_output(["g++", "-print-file-name=libubsan.so"], text=True).strip()
    frames, times, smp, _ = G.pan_sequence(64, peak_dps=PEAK, blackout=(40, 4))
    dp = tmp_path / "seq.npz"
    sm = np.empty(len(smp), object)
    sm[:] = smp
    np.savez(dp, frames=np.stack(frames), times=np.array(times), smp=sm)
    code = GYRO_RUN.format(tests=os.path.dirname(os.path.abspath(__file__)), root=U.ROOT, so=so, data=str(dp))
    env = dict(os.environ, LD_PRELOAD=asan + " " + ubsan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1",
               UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0, p.stderr[-4000:]
    assert "runtime error" not in p.stderr and "AddressSanitizer" not in p.stderr, p.stderr[-4000:]
    st = list(map(int, p.stdout.split("{")[0].split()))
    assert 1 in st and 4 in st, st
