"""CPU tests of the detector at the reference's preset cell sizes (state.hpp:9-17: 35, 45, 50 px).  The widths reach the three
other `cell & 3` tails of OpenCV's 3x3 blur (3, 1, 2; DESIGN section 2: its SIMD body and its scalar tail round differently).
orc_detect_points (oracle/detect_oracle.c) is bit-identical to the reference's FeatureExtractor::detectFeaturePoints on every
case of tests/golden/detect_presets.npz (tools/make_golden_presets.py): points as float bit patterns, their count and order,
and the blur and minimum-eigenvalue intermediate of one cell; live against the reference where it is built."""
import ctypes as C

import numpy as np
import pytest

from conftest import P, golden
from detect_util import oracle_detect

TAGS = ["c35", "c45", "c50", "c35b"]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_cases_cover_the_three_blur_tails():
    g = golden("detect_presets")
    assert sorted({int(g[f"{t}_cell"]) & 3 for t in TAGS}) == [1, 2, 3]
    assert sorted({int(g[f"{t}_cell"]) for t in TAGS}) == [35, 45, 50]


@pytest.mark.parametrize("tag", TAGS)
def test_detector_oracle_matches_the_reference(oracle, ref, tag):
    g = golden("detect_presets")
    img, cs, cur, roi = np.ascontiguousarray(g[f"{tag}_img"]), int(g[f"{tag}_cell"]), g[f"{tag}_cur"], g[f"{tag}_roi"]
    pts, ints, q = oracle_detect(oracle, img, cs, cur, roi, 0.001)
    want = g[f"{tag}_pts"]
    assert len(pts) == len(want) > 0
    assert (bits(pts) == bits(want)).all()
    if ref is not None:
        h, w = img.shape
        ref.ref_detect_points.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_int]
        out = np.zeros((4096, 2), np.float32)
        n = ref.ref_detect_points(P(img), w, h, cs, P(np.ascontiguousarray(cur, np.float32)), len(cur), P(np.ascontiguousarray(roi, np.int32)),
                                  0.001, P(out), 4096)
        assert n == len(pts) and (bits(out[:n]) == bits(pts)).all()


@pytest.mark.parametrize("tag", TAGS)
def test_cell_intermediates_match_the_reference(oracle, tag):
    """the blurred cell and its minimum-eigenvalue map (cell (1, 1)), through the oracle's own cell routine"""
    g = golden("detect_presets")
    img, cs = np.ascontiguousarray(g[f"{tag}_img"]), int(g[f"{tag}_cell"])
    h, w = img.shape
    hm = np.zeros((cs, cs), np.float32)
    bl = np.zeros((cs, cs), np.uint8)
    oracle.orc_blur3_cell(P(img), w, h, cs, cs, cs, P(bl))
    oracle.orc_min_eig_cell(P(img), w, h, cs, cs, cs, P(hm))
    assert (bl == g[f"{tag}_blur11"]).all()
    assert (bits(hm) == bits(g[f"{tag}_hmap11"])).all()
