"""CPU tests: the detector oracle (orc_detect_points, orc_corner_subpix) against the reference's own FeatureExtractor /
cv::cornerSubPix at the structural limits that tests/test_gpu_detect_limits.py drives the kernels through, on the same scenes
(tests/detect_limits_util.py): small and odd cell sizes, where OpenCV's vector / scalar-tail split of the 3 x 3 blur moves; frames
0..3 px past the last full cell; degenerate frame shapes; keypoints in (-cell, 0) and on cell boundaries; the re-scan
scenes; exact ties; the quality-adaptation boundaries; grids past 8 191 cells.  The reference's outputs are stored in
tests/golden/ref_live_detect_limits.npz (detect_limits_util.ref_outputs), so this runs without it.  Bit-exact, floats included."""
import ctypes as C

import numpy as np
import pytest

from conftest import P
from detect_limits_util import (REF_CELLS, dot_frame, edge_cur, ref_detect, ref_outputs, rescan_scene, subpix_scene, sweep_case,
                                texture, tie_scenes)
from detect_util import oracle_detect, random_cur
from ref_golden import digest

BIG = 4096   # outputs larger than this many points are stored as digests


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check_runs(oracle, ref, key, runs):
    """runs: [(img, cs, cur, roi, q0)], each run through the oracle and the reference; returns the oracle's (pts, ints, q)"""
    def compute(R):
        out = {}
        for i, (img, cs, cur, roi, q0) in enumerate(runs):
            p = ref_detect(R, img, cs, cur, roi, q0, (img.shape[0] // cs) * (img.shape[1] // cs) + 1)
            if len(p) > BIG:
                out[f"n{i}"], out[f"d{i}"] = np.int64(len(p)), digest(p)
            else:
                out[f"p{i}"] = p
        return out
    want = ref_outputs(ref, key, compute)
    res = []
    for i, (img, cs, cur, roi, q0) in enumerate(runs):
        pts, ints, q = oracle_detect(oracle, img, cs, cur, roi, q0, cap=(img.shape[0] // cs) * (img.shape[1] // cs) + 1)
        if f"p{i}" in want:
            assert len(pts) == len(want[f"p{i}"]), (key, i, len(pts), len(want[f"p{i}"]))
            assert (bits(pts) == bits(want[f"p{i}"])).all(), (key, i)
        else:
            assert len(pts) == int(want[f"n{i}"]) and (digest(pts) == want[f"d{i}"]).all(), (key, i)
        res.append((pts, ints, q))
    return res


@pytest.mark.parametrize("cs", REF_CELLS)
def test_cell_sizes_and_remainders_vs_reference(oracle, ref, cs):
    for g in range(4):
        imgs, curs, qs, roi = sweep_case(cs, g)
        res = check_runs(oracle, ref, f"detect_limits_sweep_{cs}_{g}", [(imgs[f], cs, curs[f], roi, qs[f]) for f in range(4)])
        c = [len(r[0]) for r in res]
        assert c[2] > c[0] and c[3] < c[2] and c[1] > 0, c   # the strict quality rejects maxima; keypoints occupy cells


def test_frame_geometry_vs_reference(oracle, ref):
    runs = []
    for cs in (8, 33, 64):
        runs += [(texture(cs, cs, cs), cs, np.zeros((0, 2), np.float32), [0, 0, cs, cs], 0.001)]
    # strips one cell wide and high; cv::cornerSubPix refuses frames under 11 px (win * 2 + 5, cornersubpix.cpp:65), so at
    # cell 8 the reference's narrowest strip with points is 11 px, not cell + 2
    for cs, d in ((8, 11), (40, 42)):
        for w, h in ((d, 4000), (4000, d)):
            runs += [(texture(w, h, 5 + cs), cs, np.zeros((0, 2), np.float32), [0, 0, w, h], 0.0003),
                     (texture(w, h, 6 + cs), cs, random_cur(w, h, 40, cs), [0, 0, w, h], 0.0003)]
    for cs in (35, 64):
        runs += [(texture(4095, 4095, 11), cs, random_cur(4095, 4095, 500, 3), [20, 20, 4055, 4055], 0.001),
                 (texture(4095, 4095, 12), cs, np.zeros((0, 2), np.float32), [20, 20, 4055, 4055], 0.0003)]
    res = check_runs(oracle, ref, "detect_limits_geometry", runs)
    for k in range(3):                                   # one unsearched cell: no point, the quality halves
        assert len(res[k][0]) == 0 and res[k][2] == 0.0005


def test_edge_keypoints_vs_reference(oracle, ref):
    runs = []
    for cs in (8, 13, 16, 20, 40):
        w, h = 7 * cs + 3, 6 * cs + 2
        cur = edge_cur(w, h, cs)
        runs += [(texture(w, h, 40 + cs + k), cs, cur, [1, 1, w - 2, h - 2], 0.0003) for k in range(2)]
    check_runs(oracle, ref, "detect_limits_edge_keypoints", runs)


def test_negative_keypoint_marks_first_cell_occupied_in_the_reference(oracle, ref):
    """the reference indexes occupiedCells[px.y / cellSize][px.x / cellSize]: a coordinate in (-cell, 0) truncates to
    row / column 0, which is then skipped.  Without those two keypoints both cells yield points."""
    cs, w, h = 16, 160, 112
    img = texture(w, h, 3)
    cur = np.array([[-0.5, 2.5 * cs], [3.5 * cs, -cs + 0.5]], np.float32)
    res = check_runs(oracle, ref, "detect_limits_negative_keypoints",
                     [(img, cs, cur, [0, 0, w, h], 0.0001), (img, cs, cur[:0], [0, 0, w, h], 0.0001)])
    cells = [{(int(y) // cs, int(x) // cs) for x, y in r[1]} for r in res]
    assert not cells[0] & {(2, 0), (0, 3)}
    assert {(2, 0), (0, 3)} <= cells[1]


@pytest.mark.parametrize("cs", [32, 40, 48])
def test_rescan_scene_vs_reference(oracle, ref, cs):
    """the scene does what it claims: the pre-computed (static-mask) maximum of each target cell lies inside the disc of the
    detection of the neighbour that precedes it, so the kernel must re-scan it; and the oracle matches the reference"""
    img, roi = rescan_scene(cs)
    h, w = img.shape
    res = check_runs(oracle, ref, f"detect_limits_rescan_{cs}",
                     [(img, cs, np.zeros((0, 2), np.float32), roi, 2e-6),
                      (np.ascontiguousarray(img[::-1]), cs, np.zeros((0, 2), np.float32), roi, 0.0),
                      (np.ascontiguousarray(img[:, ::-1]), cs, random_cur(w, h, 12, cs), roi, 2e-6)])
    ints = res[0][1]
    rad = cs // 4
    hw = np.zeros(rad + 1, np.int32)
    oracle.orc_circle_halfwidths(rad, P(hw))
    ncw = w // cs
    hm = np.zeros((cs, cs), np.float32)
    by_cell = {}
    for x, y in ints:
        by_cell.setdefault((y // cs) * ncw + x // cs, []).append((x, y))
    n_cov = {"W": 0, "N": 0, "NW": 0, "NE": 0}
    for r in range(1, h // cs):
        for c in range(ncw):
            oracle.orc_min_eig_cell(P(img), w, h, c * cs, r * cs, cs, P(hm))
            i = int(np.argmax(hm))
            X, Y = c * cs + i % cs, r * cs + i // cs
            for name, (dr, dc) in {"W": (0, -1), "N": (-1, 0), "NW": (-1, -1), "NE": (-1, 1)}.items():
                if not 0 <= c + dc < ncw:
                    continue
                for x, y in by_cell.get((r + dr) * ncw + c + dc, []):
                    if abs(Y - y) <= rad and abs(X - x) <= hw[abs(Y - y)]:
                        n_cov[name] += 1
    assert min(n_cov.values()) > 0, n_cov
    flat = [(8, 5), (9, 5), (8, 6), (9, 6)]
    for c, r in flat:
        oracle.orc_min_eig_cell(P(img), w, h, c * cs, r * cs, cs, P(hm))
        assert (hm == 0).all()


@pytest.mark.parametrize("cs", [8, 16, 24, 32, 40, 64])
def test_ties_vs_reference(oracle, ref, cs):
    frames, cur, roi = tie_scenes(cs)
    none = np.zeros((0, 2), np.float32)
    flat = np.full((4 * cs + 2, 5 * cs + 2), 128, np.uint8)
    runs = [(frames[0], cs, none, roi, 1e-7), (frames[1], cs, none, roi, 0.0), (frames[0], cs, cur, roi, 1e-7),
            (frames[1], cs, cur, roi, 0.0), (flat, cs, none, [0, 0, 5 * cs + 2, 3 * cs], 0.0),
            (flat, cs, cur[:3], [0, 0, 5 * cs + 2, 3 * cs], 0.0)]
    res = check_runs(oracle, ref, f"detect_limits_ties_{cs}", runs)
    assert len(res[4][0]) == 20                          # 15 zero-valued primaries (first pixel), then 5 secondaries
    hm = np.zeros((cs, cs), np.float32)
    h, w = frames[0].shape
    oracle.orc_min_eig_cell(P(frames[0]), w, h, cs, cs, cs, P(hm))
    assert (hm == hm.max()).sum() > 1                    # the cell maximum is tied


def test_dot_boundary_scene_vs_reference(oracle, ref):
    """an isolated dot leaves no secondary from some cell size on; the oracle and the reference agree on where"""
    runs = []
    for cs in range(8, 41):
        img, cur, roi = dot_frame(cs, 3, 3, [4], [])
        runs.append((img, cs, cur, roi, 1e-9))
    res = check_runs(oracle, ref, "detect_limits_dot", runs)
    c = [len(r[0]) for r in res]
    first = c.index(1)
    assert first > 0 and all(n == 1 for n in c[first:]) and all(n == 2 for n in c[:first]), c
    # the quality-boundary frames of the GPU test: the count is the number of dots, whatever the occupied cells
    cs = 8 + first
    rng = np.random.default_rng(5)
    runs = []
    for nocc, ndots in [(3, 32), (3, 88), (0, 33), (0, 91), (9, 30), (9, 82)]:
        cells = rng.permutation(100)
        img, cur, roi = dot_frame(cs, 10, 10, list(cells[nocc:nocc + ndots]), list(cells[:nocc]))
        runs.append((img, cs, cur, roi, 1e-3))
    res = check_runs(oracle, ref, "detect_limits_dot_counts", runs)
    assert [len(r[0]) for r in res] == [32, 88, 33, 91, 30, 82]


@pytest.mark.parametrize("w,h", [(731, 722), (1027, 514), (4095, 4095)])
def test_largest_grids_vs_reference(oracle, ref, w, h):
    img = texture(w, h, 60)
    res = check_runs(oracle, ref, f"detect_limits_grid_{w}x{h}", [(img, 8, random_cur(w, h, 300, 9), [4, 4, w - 8, h - 8], 0.0003)])
    assert len(res[0][0]) > (w // 8) * (h // 8) // 2


def test_corner_subpix_sampler_edges_vs_reference(oracle, ref):
    w, h = 211, 157
    argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double]
    scenes = [subpix_scene(w, h, s) for s in (1, 2, 3)]

    def run_ref(R):
        R.ref_corner_subpix.argtypes = argtypes
        out = {}
        for s, (img, p) in enumerate(scenes):
            a = p.copy()
            R.ref_corner_subpix(P(img), w, h, P(a), len(a), 3, 30, 0.01)
            out[f"pts{s}"] = a
        return out
    want = ref_outputs(ref, "detect_limits_subpix", run_ref)
    oracle.orc_corner_subpix.argtypes = argtypes
    for s, (img, p) in enumerate(scenes):
        a = p.copy()
        oracle.orc_corner_subpix(P(img), w, h, P(a), len(a), 3, 30, 0.01)
        assert (bits(a) == bits(want[f"pts{s}"])).all()
        moved = (a != p).any(1)
        assert 0 < moved.sum() < len(p)
