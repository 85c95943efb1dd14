"""GPU tests (H100): the keyframe corner detector (alva_k_detect_grid) and cornerSubPix (alva_k_corner_subpix) at their
structural limits, bit-exact against the CPU oracle (orc_detect_points run per frame): integer maxima, the float bit patterns
of the refined points, the count and the adapted quality.  Every cell size 8..64 at every grid remainder, degenerate frame
shapes, current keypoints on the edges of the occupancy / disc arithmetic, the select kernel's re-scan path (proven to run),
exact ties, the quality-adaptation and capacity boundaries, and grids past the 8 191 cells that fit in shared memory.
The inputs are the scenes of tests/detect_limits_util.py, whose oracle outputs tests/test_oracle_detect_limits.py checks
against the reference."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from detect_limits_util import dot_frame, edge_cur, rescan_scene, subpix_scene, sweep_case, texture, tie_scenes
from detect_util import oracle_detect, random_cur

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def gpu_detect(ctx, imgs, cs, curs, roi, qs, cap=4096, ncur=None, null_cur=False):
    """one batched alva_k_detect_grid call: frame f has the keypoints curs[f] (ncur[f] of them are passed, default all) and
    the start quality qs[f]"""
    nf, h, w = imgs.shape
    ccap = max(1, max(len(c) for c in curs))
    cur = np.zeros((nf, ccap, 2), np.float32)
    for i, c in enumerate(curs):
        cur[i, :len(c)] = c
    n = np.array([len(c) for c in curs] if ncur is None else ncur, np.int32)
    q = dev(np.asarray(qs, np.float64))
    out = torch.zeros((nf, cap, 2), dtype=torch.float32, device=DEV)
    oi = torch.full((nf, cap, 2), -7, dtype=torch.int32, device=DEV)
    cnt = torch.full((nf,), -1, dtype=torch.int32, device=DEV)
    ctx.detect_grid(dev(imgs), w, h, nf, cs, None if null_cur else dev(cur), None if null_cur else dev(n), ccap, roi, q, out, oi,
                    cnt, cap)
    torch.cuda.synchronize()
    return out.cpu().numpy(), oi.cpu().numpy(), cnt.cpu().numpy(), q.cpu().numpy()


def check_vs_oracle(oracle, got, imgs, cs, curs, roi, qs, cap):
    """frame by frame against the oracle run uncapped: the true count, the first `cap` points (integer and refined, bit for bit)
    and the quality adapted by the true count"""
    out, oi, cnt, q = got
    h, w = imgs.shape[1:]
    counts = []
    for f in range(len(imgs)):
        pts, ints, qo = oracle_detect(oracle, imgs[f], cs, curs[f], roi, qs[f], cap=(h // cs) * (w // cs) + 1)
        n = min(len(pts), cap)
        assert cnt[f] == len(pts), (cs, w, h, f, cnt[f], len(pts))
        assert (oi[f, :n] == ints[:n]).all(), (cs, w, h, f)
        assert (bits(out[f, :n]) == bits(pts[:n])).all(), (cs, w, h, f)
        assert q[f] == qo, (cs, w, h, f, q[f], qo)
        counts.append(len(pts))
    return counts


def run_and_check(ctx, oracle, imgs, cs, curs, roi, qs, cap=4096, **kw):
    imgs = np.ascontiguousarray(imgs)
    return check_vs_oracle(oracle, gpu_detect(ctx, imgs, cs, curs, roi, qs, cap, **kw), imgs, cs, curs, roi, qs, cap)


# ---- 1. every cell size 8..64, the frame 0..3 px past the last full cell in each direction --------------------------------

@pytest.mark.parametrize("cs", range(8, 65))
def test_every_cell_size_and_remainder(gpu_ctx, oracle, cs):
    for g in range(4):
        imgs, curs, qs, roi = sweep_case(cs, g)
        c = run_and_check(gpu_ctx, oracle, imgs, cs, curs, roi, qs)
        assert c[2] > c[0] and c[3] < c[2] and c[1] > 0    # the strict quality rejects maxima; keypoints occupy cells


# ---- 2. frame geometry -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cs", [8, 33, 64])
def test_frame_of_one_unsearched_cell(gpu_ctx, oracle, cs):
    imgs = np.stack([texture(cs, cs, cs), texture(cs, cs, cs + 1)])
    out, oi, cnt, q = gpu_detect(gpu_ctx, imgs, cs, [np.zeros((0, 2), np.float32)] * 2, [0, 0, cs, cs], [0.001, 0.0])
    assert (cnt == 0).all() and (q == [0.0005, 0.0]).all()
    check_vs_oracle(oracle, (out, oi, cnt, q), imgs, cs, [np.zeros((0, 2))] * 2, [0, 0, cs, cs], [0.001, 0.0], 4096)


@pytest.mark.parametrize("cs", [8, 40])
def test_strips(gpu_ctx, oracle, cs):
    """one cell wide / high, searched (cell + 2) and one pixel wider; at cell 8 the 10-px strip is below what cv::cornerSubPix
    accepts (11 px), so there only the oracle defines the result"""
    for w, h in ((cs + 2, 4000), (4000, cs + 2), (cs + 3, 4000), (4000, cs + 3)):
        imgs = np.stack([texture(w, h, 5 + cs), texture(w, h, 6 + cs)])
        curs = [np.zeros((0, 2), np.float32), random_cur(w, h, 40, cs)]
        c = run_and_check(gpu_ctx, oracle, imgs, cs, curs, [0, 0, w, h], [0.0003, 0.0003])
        assert c[0] >= 4000 // cs


@pytest.mark.parametrize("cs", [35, 64])
def test_largest_frame(gpu_ctx, oracle, cs):
    """4095 x 4095: 117 x 117 = 13 689 cells at cell 35 (past shared memory), 63 x 63 at cell 64"""
    imgs = np.stack([texture(4095, 4095, 11), texture(4095, 4095, 12)])
    curs = [random_cur(4095, 4095, 500, 3), np.zeros((0, 2), np.float32)]
    c = run_and_check(gpu_ctx, oracle, imgs, cs, curs, [20, 20, 4055, 4055], [0.001, 0.0003], cap=2 * (4095 // cs) ** 2)
    assert min(c) > (4095 // cs) ** 2 // 2


# ---- 3. current keypoints at the edges ------------------------------------------------------------------------------------

@pytest.mark.parametrize("cs", [8, 13, 16, 20, 40])
def test_keypoints_on_the_edges(gpu_ctx, oracle, cs):
    w, h = 7 * cs + 3, 6 * cs + 2
    cur = edge_cur(w, h, cs)
    imgs = np.stack([texture(w, h, 40 + cs + k) for k in range(3)])
    roi = [1, 1, w - 2, h - 2]
    # frame 1 passes more keypoints than its rows hold: clamped to cur_cap
    ccap = len(cur)
    got = gpu_detect(gpu_ctx, imgs, cs, [cur, cur, cur[:0]], roi, [0.0003] * 3, ncur=[ccap, ccap + 9, 0])
    check_vs_oracle(oracle, got, imgs, cs, [cur, cur, cur[:0]], roi, [0.0003] * 3, 4096)
    # no keypoint array at all
    got = gpu_detect(gpu_ctx, imgs, cs, [cur] * 3, roi, [0.0003] * 3, null_cur=True)
    check_vs_oracle(oracle, got, imgs, cs, [cur[:0]] * 3, roi, [0.0003] * 3, 4096)


def test_negative_keypoint_marks_first_cell_occupied(gpu_ctx, oracle):
    """a keypoint in (-cell, 0) marks row / column 0 occupied, as the reference's float -> size_t cell index does"""
    cs, w, h = 16, 160, 112
    img = texture(w, h, 3)[None]
    cur = np.array([[-0.5, 2.5 * cs], [3.5 * cs, -cs + 0.5]], np.float32)   # in cells (2, 0) and (0, 3)
    _, oi, cnt, _ = gpu_detect(gpu_ctx, img, cs, [cur], [0, 0, w, h], [0.0001])
    cells = {(int(y) // cs, int(x) // cs) for x, y in oi[0, :cnt[0]]}
    assert not cells & {(2, 0), (0, 3)}
    run_and_check(gpu_ctx, oracle, img, cs, [cur], [0, 0, w, h], [0.0001])


# ---- 4. the re-scan path, proven to run -----------------------------------------------------------------------------------

_DEBUG_RUN = r"""
import sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import alvaar_b200
d = np.load(sys.argv[2])
ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
imgs, cur, ncur, cs, roi, q0 = d["imgs"], d["cur"], d["ncur"], int(d["cs"]), [int(v) for v in d["roi"]], d["q"]
nf, h, w = imgs.shape
cap = 4096
q = torch.from_numpy(q0).cuda()
out = torch.zeros((nf, cap, 2), dtype=torch.float32, device="cuda")
oi = torch.zeros((nf, cap, 2), dtype=torch.int32, device="cuda")
cnt = torch.zeros(nf, dtype=torch.int32, device="cuda")
ctx.detect_grid(torch.from_numpy(imgs).cuda(), w, h, nf, cs, torch.from_numpy(cur).cuda(), torch.from_numpy(ncur).cuda(), cur.shape[1],
                roi, q, out, oi, cnt, cap)
torch.cuda.synchronize()
np.savez(sys.argv[3], out=out.cpu().numpy(), oi=oi.cpu().numpy(), cnt=cnt.cpu().numpy(), q=q.cpu().numpy())
ctx.close()
"""


@pytest.mark.parametrize("cs", [32, 40, 48])
def test_rescan_paths_run_and_agree(oracle, tmp_path, cs):
    """the select kernel's counters (ALVA_DETECT_DEBUG, read once per process: one child process) show every re-scan reason --
    a pre-computed maximum <= 0, a primary that differs from the pre-computed one, a maximum covered by a neighbour's disc --
    and the result is still the oracle's"""
    if not torch.cuda.is_available():
        pytest.skip("gpu tests need a CUDA device")
    img, roi = rescan_scene(cs)
    h, w = img.shape
    imgs = np.stack([img, np.ascontiguousarray(img[:, ::-1])])
    curs = [np.zeros((0, 2), np.float32), random_cur(w, h, 12, cs)]
    cur = np.zeros((2, 12, 2), np.float32)
    cur[1] = curs[1]
    qs = np.array([2e-6, 2e-6])
    np.savez(tmp_path / "in.npz", imgs=imgs, cur=cur, ncur=np.array([0, 12], np.int32), cs=cs, roi=np.array(roi), q=qs)
    env = dict(os.environ, ALVA_DETECT_DEBUG="1")
    r = subprocess.run([sys.executable, "-c", _DEBUG_RUN, ROOT, str(tmp_path / "in.npz"), str(tmp_path / "out.npz")], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [ln for ln in r.stderr.splitlines() if ln.startswith("[detect]")][-1]
    nums = [int(t.strip(",")) for t in line.split() if t.strip(",").lstrip("-").isdigit()]
    searches, le0, differs, covered = nums
    assert searches > 0 and le0 > 0 and differs > 0 and covered > 0, line
    o = np.load(tmp_path / "out.npz")
    check_vs_oracle(oracle, (o["out"], o["oi"], o["cnt"], o["q"]), imgs, cs, curs, roi, list(qs), 4096)


def test_rescan_scene_direct(gpu_ctx, oracle):
    """the same scenes through the in-process context (no debug counters), three cell sizes in one pass"""
    for cs in (32, 40, 48):
        img, roi = rescan_scene(cs)
        imgs = np.stack([img, np.ascontiguousarray(img[::-1])])
        run_and_check(gpu_ctx, oracle, imgs, cs, [np.zeros((0, 2), np.float32)] * 2, roi, [2e-6, 0.0])


# ---- 5. exact ties ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cs", [8, 16, 24, 32, 40, 64])
def test_exact_ties(gpu_ctx, oracle, cs):
    frames, cur, roi = tie_scenes(cs)
    imgs = np.stack(frames + frames)
    none = np.zeros((0, 2), np.float32)
    # without and with keypoints whose discs cover the first tied maxima, and quality 0: flat and fully covered cells then
    # accept their zero-valued first pixel
    run_and_check(gpu_ctx, oracle, imgs, cs, [none, none, cur, cur], roi, [1e-7, 0.0, 1e-7, 0.0])
    # a flat frame whose last cell row lies outside the roi: 15 zero-valued primaries (each cell's first pixel), then 5
    # secondaries (the first pixel outside that disc)
    flat = np.full((1, 4 * cs + 2, 5 * cs + 2), 128, np.uint8)
    c = run_and_check(gpu_ctx, oracle, np.concatenate([flat, flat]), cs, [none, cur[:3]], [0, 0, 5 * cs + 2, 3 * cs], [0.0, 0.0])
    assert c[0] == 20


# ---- 6. quality adaptation and capacity at their boundaries ----------------------------------------------------------------

@pytest.fixture(scope="module")
def dot_cell(oracle):
    """the smallest cell size at which an isolated dot on a flat frame yields exactly one point: its disc covers every
    non-zero minimum eigenvalue around it, so the cell has no secondary (found, not assumed)"""
    for cs in range(8, 65):
        img, cur, roi = dot_frame(cs, 3, 3, [4], [])
        pts, _, _ = oracle_detect(oracle, img, cs, cur, roi, 1e-9)
        if len(pts) == 1:
            return cs
    pytest.fail("no cell size isolates a dot")


def test_quality_and_capacity_boundaries(gpu_ctx, oracle, dot_cell):
    cs, ncw, nch = dot_cell, 10, 10
    rng = np.random.default_rng(5)
    imgs, curs, qs, want = [], [], [], []
    for f, (nocc, ndots) in enumerate([(3, 32), (3, 33), (3, 87), (3, 88), (0, 32), (0, 33), (0, 90), (0, 91), (9, 30), (9, 31),
                                       (9, 81), (9, 82)]):
        cells = rng.permutation(ncw * nch)
        img, cur, roi = dot_frame(cs, ncw, nch, list(cells[nocc:nocc + ndots]), list(cells[:nocc]))
        free = ncw * nch - nocc
        q0 = 1e-4 * (1 + f)
        imgs.append(img); curs.append(cur); qs.append(q0)
        want.append(q0 * (0.5 if ndots < 0.33 * free else 1.5 if ndots > 0.9 * free else 1.0))
    imgs = np.stack(imgs)
    for cap in (4096, 60):
        got = gpu_detect(gpu_ctx, imgs, cs, curs, roi, qs, cap=cap)
        counts = check_vs_oracle(oracle, got, imgs, cs, curs, roi, qs, cap)
        assert counts == [32, 33, 87, 88, 32, 33, 90, 91, 30, 31, 81, 82]
        assert list(got[3]) == want                     # the quality follows the true count, capped or not


# ---- 7. the largest grids ---------------------------------------------------------------------------------------------------

# 91 x 90 = 8 190 cells: the largest grid (8 191 is prime) whose select state fits in shared memory
@pytest.mark.parametrize("w,h,nf", [(731, 722, 2),
                                    (1027, 514, 2),     # 128 x 64 = 8 192 cells: past it
                                    (4095, 4095, 2)])   # 511 x 511 = 261 121 cells
def test_largest_grids(gpu_ctx, oracle, w, h, nf):
    cs = 8
    imgs = np.stack([texture(w, h, 60 + k) for k in range(nf)])
    curs = [random_cur(w, h, 300, 9), np.zeros((0, 2), np.float32)][:nf]
    ncells = (w // cs) * (h // cs)
    c = run_and_check(gpu_ctx, oracle, imgs, cs, curs, [4, 4, w - 8, h - 8], [0.0003, 0.0003][:nf], cap=ncells)
    assert min(c) > ncells // 2


def test_system_on_the_largest_frame_with_the_accurate_preset():
    """a System at 4095 x 4095 on ACCURATE's 35-px grid (13 689 detector cells) detects and tracks"""
    if not torch.cuda.is_available():
        pytest.skip("gpu tests need a CUDA device")
    from alvaar_b200 import synth
    from alvaar_b200.system import System
    w = h = 4095
    s = System(w, h, *synth.intrinsics(w, h))
    try:
        s.set_preset("accurate")
        base = texture(w + 16, h + 16, 2)
        n = []
        for k in range(4):
            g = np.ascontiguousarray(base[2 * k:2 * k + h, 3 * k:3 * k + w])
            st, _ = s.find_camera_pose(np.ascontiguousarray(synth.gray_to_rgba(g[None])[0]), 33.0 * k)
            assert st in (1, 2, 3), st
            n.append(s.info()["keypoints"])
        assert n[0] > 8191 and min(n[1:]) > n[0] // 2, n
    finally:
        s.close()


# ---- 8. cornerSubPix alone ---------------------------------------------------------------------------------------------------

def test_corner_subpix_on_the_sampler_edges(gpu_ctx, oracle):
    import ctypes as C
    from conftest import P
    w, h = 211, 157
    scenes = [subpix_scene(w, h, s) for s in (1, 2, 3)]
    counts = [len(scenes[0][1]), len(scenes[1][1]) // 2, 7]
    cap = max(len(p) for _, p in scenes)
    pts = np.zeros((3, cap, 2), np.float32)
    for f, (_, p) in enumerate(scenes):
        pts[f, :len(p)] = p
    want = pts.copy()
    oracle.orc_corner_subpix.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double]
    for f, (img, _) in enumerate(scenes):
        a = np.ascontiguousarray(want[f])
        oracle.orc_corner_subpix(P(img), w, h, P(a), counts[f], 3, 30, 0.01)
        want[f] = a
    d = dev(pts)
    gpu_ctx.corner_subpix(dev(np.stack([img for img, _ in scenes])), w, h, 3, d, dev(np.array(counts, np.int32)), cap)
    torch.cuda.synchronize()
    got = d.cpu().numpy()
    assert (bits(got) == bits(want)).all()                    # points past each frame's count are left alone
    moved = (got[0, :counts[0]] != scenes[0][1]).any(1)
    assert 0 < moved.sum() < counts[0]
