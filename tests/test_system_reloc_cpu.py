"""CPU: System's relocalisation mode (system_core.h, alva_system_set_relocalisation) over the CPU oracle backend
(tests/host/system_cpu_reloc.cpp): off is the reference's behaviour bit for bit; on, a revisit after a blackout relocalises
against the kept map, an unrelated scene falls back to the reference's reset after max_lost_frames."""
import numpy as np
import pytest

import reloc_util as U

MAX_LOST = 10
N_BEFORE = 40        # frames tracked before the blackout (make_frames(40, seed 7))
# The relocalised pose against the true pose of the rendered view, mapped into the system's frame by the similarity fitted over
# the frames tracked before the loss.  Map units: the initial baseline is 1, and this map has ~3.6 map units per world unit.
# The fit itself is good to 1e-3 and 0.01 degrees on those frames.  The relocalised pose was observed 0.029 (plain), 0.032
# (lens) and 0.034 (ACCURATE) off, with 0.11-0.17 degrees of rotation.  The offset stays the same on the frames tracked after
# it, so it belongs to the map points the relocalised frame is matched to, not to the relocalisation.  The translation bar is
# therefore 0.05, not 0.02.
TOL_T, TOL_DEG = 0.05, 0.5


@pytest.fixture(scope="module")
def S():
    return U.cpu_reloc_system_lib()


def run(S, frames, **kw):
    r = U.CpuRelocRun(S, **kw)
    out = [r.frame(f, k * 33.333) for k, f in enumerate(frames)]
    c = r.counters()
    r.close()
    return out, c


def test_off_equals_never_calling_it(S):
    """the failure-path sequence (blackout, jump to another path, jump back: resets and re-initialisations) with
    set_relocalisation(0) is bit-identical to a run without the call"""
    seq = U.failure_paths_sequence()
    a, _ = run(S, seq)
    b, cb = run(S, seq, max_lost=0)
    assert {x[0] for x in a} == {1, 2, 3}
    for k, (x, y) in enumerate(zip(a, b)):
        assert x[0] == y[0] and (x[2] == y[2]).all(), k
        assert (x[1] == y[1]).all(), k
        assert len(x[3]) == len(y[3]) and (x[3] == y[3]).all() and (x[4].view(np.uint32) == y[4].view(np.uint32)).all() and (x[5] == y[5]).all(), k
    assert cb["lost"] == 0


def check_revisit(S, **kw):
    frames, truth = U.revisit_sequence(dist=kw.get("dist"))
    out, c = run(S, frames, max_lost=MAX_LOST, **kw)
    st = [x[0] for x in out]
    first_fail = next(k for k in range(N_BEFORE) if st[k] == 4) if 4 in st[:N_BEFORE] else N_BEFORE
    assert 1 in st[:N_BEFORE] and 2 not in st[:first_fail]
    # lost from the first failure through the blackout; back on the first revisit frame, or at the latest the second
    back = next(k for k in range(first_fail, len(st)) if st[k] == 1)
    assert all(s == 4 for s in st[first_fail:back]) and back - first_fail <= MAX_LOST
    assert back in (N_BEFORE + 3, N_BEFORE + 4), st[N_BEFORE:]
    assert 2 not in st[first_fail:] and 3 not in st[first_fail:]
    # keyframe ids continue: no reset
    kf_ids = [int(x[2][1]) for x in out]
    assert all(b >= a for a, b in zip(kf_ids[first_fail:], kf_ids[first_fail + 1:]))
    assert kf_ids[-1] > kf_ids[first_fail - 1]
    # while lost: the last tracked pose, an empty frame
    for k in range(first_fail, back):
        assert (out[k][1] == out[first_fail - 1][1]).all() and len(out[k][3]) == 0
    # the relocalised pose against the rendered view's true pose in the system's frame
    tracked = {k: out[k][1] for k in range(first_fail) if st[k] == 1}
    fit = U.fit_from_track(truth, tracked)
    dt, dr = U.pose_error(out[back][1], U.true_in_map(fit, truth[back]))
    assert dt < TOL_T and dr < TOL_DEG, (dt, dr)
    # tracking continues: 20 frames with status 1, at least one new keyframe; >= 30 3-D keypoints on the relocalised frame
    assert all(s == 1 for s in st[back:back + 20]) and len(st) >= back + 20
    assert kf_ids[back + 19] > kf_ids[first_fail - 1]
    assert int(out[back][5].sum()) >= 30
    assert c["lost"] == 1 and c["relocalised"] == 1
    return dt, dr


def test_revisit_relocalises(S):
    print("revisit: |dt| %.4f, %.3f deg" % check_revisit(S))


def test_revisit_relocalises_through_a_lens(S):
    print("revisit, lens: |dt| %.4f, %.3f deg" % check_revisit(S, dist=U.DIST))


def test_revisit_relocalises_under_accurate(S):
    print("revisit, ACCURATE: |dt| %.4f, %.3f deg" % check_revisit(S, preset=3))


def test_unrelated_scene_falls_back_to_the_reset(S):
    frames = U.unrelated_sequence()
    out, c = run(S, frames, max_lost=MAX_LOST)
    st = [x[0] for x in out]
    first_fail = st.index(4)
    assert first_fail <= N_BEFORE
    # exactly MAX_LOST lost frames, then the reference's reset, never relocalised
    assert st[first_fail:first_fail + MAX_LOST] == [4] * MAX_LOST and st[first_fail + MAX_LOST] == 2
    assert c["relocalised"] == 0
    # then it re-initialises as after any reset: not initialised, then tracking on a new map from keyframe 0
    after = st[first_fail + MAX_LOST + 1:]
    assert after[0] == 3 and 1 in after and 4 not in after[:after.index(1)]
    k1 = first_fail + MAX_LOST + 1 + after.index(1)
    assert out[first_fail + MAX_LOST][2][0] == -1 or out[first_fail + MAX_LOST][2][5] == 0   # the map was discarded
    assert out[k1][2][1] <= 1
