"""CPU tests: the feature-selection oracle (orc_fast9, orc_orb_detect) against the reference's own cv::FAST and
ORB::detectAndCompute on the structural-limit scenes that tests/test_gpu_feature_limits.py drives the kernels through
(tests/feature_limits_util.py): the dense dot lattice near the NMS bound, identical-dot lattices where every FAST score and
Harris response ties, a scene whose n-th Harris response is negative, noise with more corners than 1024 candidates, and a
clamped threshold.  The reference's outputs are stored in tests/golden/ref_live_feature_limits.npz, so this runs without it.
Bit-exact, floats included.

The reference keeps every tie at the n-th best response, and so does the oracle (these tests show both keep more than n).
Truncating a tied selection at a fixed number of slots (the pipeline's fcap, in row-major order) is this project's rule, not
the reference's: it is tested on the GPU side only."""
import ctypes as C

import numpy as np
import pytest

from conftest import P
from feature_limits_util import (nms_bound, oracle_fast, oracle_orb_detect, ref_fast, ref_orb_detect, ref_outputs, scene)
from ref_golden import digest

BIG = 4096   # outputs with more rows than this are stored as their count and digest


def stored(a):
    return {"n": np.int64(len(a)), "d": digest(a)} if len(a) > BIG else {"n": np.int64(len(a)), "a": a}


def same(a, want):
    if "a" in want:
        return len(a) == len(want["a"]) and np.array_equal(a, want["a"])
    return len(a) == int(want["n"]) and (digest(a) == want["d"]).all()


FAST_SCENES = [("texture", 241, 63, 20), ("texture", 241, 63, 0), ("texture", 241, 63, 255), ("texture", 4095, 200, 12),
               ("dense", 640, 480, 20), ("ties", 320, 240, 20), ("edges", 336, 240, 20), ("noise", 1280, 720, 20)]


@pytest.mark.parametrize("kind,w,h,thr", FAST_SCENES)
def test_fast_vs_reference(oracle, ref, kind, w, h, thr):
    img = scene(kind, w, h, 1)
    got = oracle_fast(oracle, img, thr)
    want = ref_outputs(ref, f"feature_limits_fast_{kind}_{w}x{h}_{thr}", lambda R: stored(ref_fast(R, img, thr)))
    assert same(got, want), (kind, w, h, thr, len(got), int(want["n"]))
    if kind == "dense":
        assert len(got) > 0.9 * nms_bound(w, h)
    if kind == "ties":
        assert len(np.unique(got[:, 2])) == 1
    if thr == 255:
        assert len(got) == 0


def test_clamped_threshold_is_the_reference_behaviour(oracle):
    """the oracle clamps the threshold to 0..255 as cv::FAST does (fast.cpp:78: threshold = std::min(std::max(threshold, 0),
    255)): -5 is 0 and 300 is 255"""
    img = scene("texture", 241, 63, 1)
    assert np.array_equal(oracle_fast(oracle, img, -5), oracle_fast(oracle, img, 0))
    assert np.array_equal(oracle_fast(oracle, img, 300), oracle_fast(oracle, img, 255))


ORB_SCENES = [("edges", 336, 240, 300), ("ties", 320, 240, 100), ("dense", 640, 480, 500), ("noise", 640, 480, 600),
              ("texture", 320, 240, 5000)]


@pytest.mark.parametrize("kind,w,h,nf", ORB_SCENES)
def test_orb_detect_vs_reference(oracle, ref, kind, w, h, nf):
    """orc_orb_detect == ORB::detectAndCompute as a SET (sorted row-major: the reference's order comes from nth_element) of
    {x, y, response, angle} and descriptors"""
    for seed in (1, 2):
        img = scene(kind, w, h, seed)
        kp, d = oracle_orb_detect(oracle, img, nf, 20)

        def run(R):
            rk, rd = ref_orb_detect(R, img, nf, 20)
            out = {("k" + k): v for k, v in stored(rk.view(np.uint32)).items()}
            out.update({("d" + k): v for k, v in stored(rd).items()})
            return out
        want = ref_outputs(ref, f"feature_limits_orb_{kind}_{w}x{h}_{nf}_{seed}", run)
        assert same(kp.view(np.uint32), {k[1:]: v for k, v in want.items() if k[0] == "k"}), (kind, seed, len(kp))
        assert same(d, {k[1:]: v for k, v in want.items() if k[0] == "d"}), (kind, seed)
        if kind in ("ties", "dense"):
            assert len(kp) > nf            # every tie at the n-th response is kept, by the reference too
        if kind == "edges":
            assert kp[:, 2].min() < 0 and len(kp) == nf
        if kind == "texture":
            assert len(kp) < nf


@pytest.mark.parametrize("kind,w,h,nf", [s for s in ORB_SCENES if s[0] != "dense"])
def test_composition_equals_orc_orb_detect(oracle, kind, w, h, nf):
    """the stage-by-stage composition these tests use (feature_limits_util.oracle_orb_detect) is orc_orb_detect, bit for bit,
    wherever orc_orb_detect's own FAST list (w * h / 8 corners) holds the frame's corners; the dense scene has more"""
    img = np.ascontiguousarray(scene(kind, w, h, 1))
    assert len(oracle_fast(oracle, img, 20)) <= w * h // 8
    kp, d = oracle_orb_detect(oracle, img, nf, 20)
    cap = nms_bound(w, h)
    ok, od = np.zeros((cap, 4), np.float32), np.zeros((cap, 32), np.uint8)
    n = oracle.orc_orb_detect(P(img), w, h, nf, 20, 0, P(ok), P(od), C.c_int(cap))
    assert n == len(kp) and (ok[:n].view(np.uint32) == kp.view(np.uint32)).all() and (od[:n] == d).all()
    assert len(oracle_fast(oracle, scene("dense", 640, 480, 1), 20)) > 640 * 480 // 8
