"""GPU tests (H100): the per-frame feature selection at its structural limits, bit for bit against the CPU oracle -- the fused
front end (both kernels, at tile boundaries, under every run-time switch), FAST capacity and threshold clamping,
alva_k_retain_best (counts around the 1024-thread CTA, the border, ties, truncation at out_cap), Harris and the float
selection (alva_k_orb_detect), and the pipeline's two selection modes on tie scenes and on frames with more corners than its
old key capacity.  Keys, counts, order, scores, levels, responses, angles and descriptors are all exact.  The scenes are those
of tests/feature_limits_util.py, whose oracle outputs tests/test_oracle_feature_limits.py checks against the reference."""
import functools

import numpy as np
import pytest
import torch

from conftest import P
from alvaar_b200 import ORB_HARRIS, ORB_IC_ANGLE
from alvaar_b200.pipeline import Pipeline
from feature_limits_util import (dense_dots, nms_bound, oracle_fast, oracle_harris, oracle_orb_detect, oracle_retain_best, pack,
                                 random_keys, scene, tie_dots, to_rgba)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def oracle_gray(oracle, rgba):
    h, w = rgba.shape[:2]
    g = np.empty((h, w), np.uint8)
    oracle.orc_gray(P(np.ascontiguousarray(rgba)), w, h, P(g))
    return g


def oracle_pyrdown(oracle, img):
    h, w = img.shape
    out = np.empty(((h + 1) // 2, (w + 1) // 2), np.uint8)
    oracle.orc_pyrdown(P(np.ascontiguousarray(img)), w, h, P(out))
    return out


_want = {}


def oracle_frame(oracle, rgba, thr, tag):
    """gray, L1 and FAST corners of one RGBA frame by the oracle, cached by tag (the option sets and source offsets repeat them)"""
    key = (tag, thr)
    if key not in _want:
        g = oracle_gray(oracle, rgba)
        _want[key] = (g, oracle_pyrdown(oracle, g), oracle_fast(oracle, g, thr))
    return _want[key]


# ---- the front end's run-time switches, restored after each test (options are process-wide) ------------------------------------

OPTION_SETS = {"default": {}, "ctas4": {"frontend_ctas": 4}, "prefetch": {"frontend_prefetch": 1}, "variant0": {"frontend_variant": 0}}
OPTION_DEFAULTS = {"frontend_ctas": 5, "frontend_prefetch": 0, "frontend_variant": 2}


@pytest.fixture(params=list(OPTION_SETS))
def frontend_options(request, gpu_ctx):
    L = gpu_ctx.L

    def restore():
        for k, v in OPTION_DEFAULTS.items():
            L.alva_set_option(k.encode(), v)
    request.addfinalizer(restore)
    for k, v in OPTION_SETS[request.param].items():
        assert L.alva_set_option(k.encode(), v) == 0
    return request.param


@functools.lru_cache(maxsize=None)
def frames_for(w, h, n, seed=0):
    """frame 2k: the texture with mixed channels; frame 2k + 1: the dense dot lattice with R = G = B (gray = the lattice)"""
    out = []
    for f in range(n):
        if f % 2 == 0:
            out.append(to_rgba(scene("texture", w, h, seed + f), f))
        else:
            g = dense_dots(w, h, f // 2)
            out.append(np.ascontiguousarray(np.stack([g, g, g, np.full_like(g, 7)], -1)))
    return np.stack(out)


def run_frontend(ctx, rgba, thr, shift=0, cap=None, sorted_=True, api="frontend"):
    """alva_k_frontend (L0, L1, keys) on a device copy of rgba that starts `shift` bytes into its allocation (4: not 16-byte
    aligned, the round-1 kernel), or alva_k_fast9 on its gray frames"""
    n, h, w = rgba.shape[:3]
    cap = cap or nms_bound(w, h)
    keys = torch.full((n, cap), -1, dtype=torch.int32, device=DEV)
    counts = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    if api == "frontend":
        flat = torch.zeros(rgba.size + 16, dtype=torch.uint8, device=DEV)
        src = flat[shift:shift + rgba.size]
        src.copy_(torch.from_numpy(rgba.reshape(-1)))
        l0 = torch.zeros((n, h, w), dtype=torch.uint8, device=DEV)
        l1 = torch.zeros((n, (h + 1) // 2, (w + 1) // 2), dtype=torch.uint8, device=DEV)
        ctx.frontend(src, w, h, n, l0, l1, None, None, thr, keys, counts, cap, sorted_)
    else:
        flat = torch.zeros(n * w * h + 16, dtype=torch.uint8, device=DEV)
        src = flat[shift:shift + n * w * h]
        src.copy_(torch.from_numpy(np.ascontiguousarray(rgba[..., 0]).reshape(-1)))
        l0 = l1 = None
        ctx.fast9(src, w, h, n, thr, keys, counts, cap, sorted_)
    torch.cuda.synchronize()
    lv = (l0.cpu().numpy(), l1.cpu().numpy()) if l0 is not None else None
    return keys.cpu().numpy().view(np.uint32), counts.cpu().numpy(), lv


def check_frontend(oracle, rgba, thr, got, tag):
    keys, counts, lv = got
    w = rgba.shape[2]
    for f in range(len(rgba)):
        g, g1, want = oracle_frame(oracle, rgba[f], thr, (tag, f))
        if lv is not None:
            assert (lv[0][f] == g).all() and (lv[1][f] == g1).all(), (tag, f)
        assert counts[f] == len(want), (tag, f, counts[f], len(want))
        assert (keys[f, :len(want)] == pack(want)).all(), (tag, f)   # same corners, scores and (unsigned) row-major order
    return w


# ---- 1. front-end geometry: both kernels at tile boundaries ---------------------------------------------------------------------

# variant 2 (w % 4 == 0, 16-B aligned source) tiles 120 x 60; the round-1 kernel (w % 4 != 0 or a shifted source) 120 x 62
GEOMS = [(w, h) for w in (16, 120, 124, 239, 241) for h in (16, 60, 61, 62, 63)] + [(4092, 63), (124, 4095), (4092, 4095),
                                                                                     (4095, 4095)]


@pytest.mark.parametrize("shift", [0, 4])
def test_frontend_geometry(gpu_ctx, oracle, frontend_options, shift):
    big = 0
    for w, h in GEOMS:
        rgba = frames_for(w, h, 2, seed=w + h)
        check_frontend(oracle, rgba, 12, run_frontend(gpu_ctx, rgba, 12, shift), ("geom", w, h))
        if h > 2048:   # keys with y >= 2048 have bit 31 set: they still sort (and count) as unsigned
            want = oracle_frame(oracle, rgba[0], 12, (("geom", w, h), 0))[2]
            big += int((want[:, 1] >= 2048).sum())
    assert big > 1000


def test_fast9_geometry(gpu_ctx, oracle):
    """alva_k_fast9 on gray frames (its own TMA rule: w % 16 == 0 and a 16-B aligned source), sorted and unsorted"""
    for w, h in [(16, 16), (128, 61), (240, 62), (241, 63), (4096 - 16, 4095)]:
        rgba = frames_for(w, h, 2, seed=3 * w + h)
        grays = np.stack([oracle_gray(oracle, f) for f in rgba])
        rg = np.ascontiguousarray(np.repeat(grays[..., None], 4, -1))
        for shift in (0, 8):
            check_frontend(oracle, rgba, 12, run_frontend(gpu_ctx, rg, 12, shift, api="fast9"), ("fast9", w, h))
            keys, counts, _ = run_frontend(gpu_ctx, rg, 12, shift, sorted_=False, api="fast9")
            for f in range(2):
                want = pack(oracle_frame(oracle, rgba[f], 12, (("fast9", w, h), f))[2])
                assert counts[f] == len(want) and (np.sort(keys[f, :counts[f]]) == want).all()


def test_frontend_batches(gpu_ctx, oracle, frontend_options):
    """300 small frames in one call (fewer than variant 2's prefetch distance: one tile per frame), and 8 frames of 1280 x 720,
    more than that distance, whose dense frames come within 10 % of the NMS bound"""
    for w, h, n in ((64, 48, 300), (66, 50, 300), (1280, 720, 8)):
        rgba = frames_for(w, h, n, seed=n)
        check_frontend(oracle, rgba, 20, run_frontend(gpu_ctx, rgba, 20), ("batch", w, h))
    want = oracle_frame(oracle, rgba[1], 20, (("batch", 1280, 720), 1))[2]
    assert len(want) > 0.9 * nms_bound(1280, 720)


# ---- 2. capacity and threshold ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("api", ["frontend", "fast9"])
def test_corners_past_cap(gpu_ctx, oracle, api):
    """a frame with more corners than cap: the call succeeds, counts[f] is the true count, and the stored keys are cap distinct
    corners of the frame (which ones is unspecified)"""
    w, h = 640, 480
    rgba = frames_for(w, h, 2, seed=11)
    wants = [pack(oracle_frame(oracle, rgba[f], 20, (("cap", w, h), f))[2]) for f in range(2)]
    n = len(wants[1])
    assert n > 0.9 * nms_bound(w, h)
    src = rgba if api == "frontend" else np.repeat(np.stack([oracle_gray(oracle, f) for f in rgba])[..., None], 4, -1)
    for cap in (1000, n - 1, n):
        for sorted_ in (False, True):
            keys, counts, _ = run_frontend(gpu_ctx, np.ascontiguousarray(src), 20, cap=cap, sorted_=sorted_, api=api)
            for f in range(2):
                assert counts[f] == len(wants[f])
                m = min(cap, len(wants[f]))
                got = keys[f, :m]
                assert len(np.unique(got)) == m and np.isin(got, wants[f]).all()
                if sorted_:
                    assert (np.diff(got.astype(np.int64)) > 0).all()
                if m == len(wants[f]) and sorted_:
                    assert (got == wants[f]).all()


def test_threshold_is_clamped(gpu_ctx, oracle):
    w, h = 244, 124
    rgba = frames_for(w, h, 2, seed=5)
    got = {}
    for thr in (-5, 0, 255, 300):
        for api in ("frontend", "fast9"):
            src = rgba if api == "frontend" else np.repeat(np.stack([oracle_gray(oracle, f) for f in rgba])[..., None], 4, -1)
            r = run_frontend(gpu_ctx, np.ascontiguousarray(src), thr, api=api)
            check_frontend(oracle, rgba, thr, r, ("thr", w, h))
            got[thr, api] = r[1]
    assert (got[-5, "frontend"] == got[0, "frontend"]).all() and (got[300, "fast9"] == got[255, "fast9"]).all()
    assert got[0, "frontend"].min() > 0


# ---- 3. alva_k_retain_best -------------------------------------------------------------------------------------------------------

def rowmajor(xys):
    xys = np.asarray(xys, np.int32).reshape(-1, 3)
    return xys[np.lexsort((xys[:, 0], xys[:, 1]))]


def gpu_retain_best(ctx, lists, w, h, n, edge, out_cap, cap=None):
    nf = len(lists)
    cap = cap or max(1, max(len(k) for k in lists))
    keys = np.zeros((nf, cap), np.uint32)
    for f, k in enumerate(lists):
        keys[f, :len(k)] = pack(k)
    okeys = torch.full((nf, out_cap), -1, dtype=torch.int32, device=DEV)
    ocounts = torch.full((nf,), -1, dtype=torch.int32, device=DEV)
    ctx.retain_best(dev(keys.view(np.int32)), dev(np.array([len(k) for k in lists], np.int32)), cap, nf, w, h, n, edge, okeys,
                    ocounts, out_cap)
    torch.cuda.synchronize()
    return okeys.cpu().numpy().view(np.uint32), ocounts.cpu().numpy()


def check_retain_best(ctx, oracle, lists, w, h, n, edge, out_cap, cap=None):
    okeys, ocounts = gpu_retain_best(ctx, lists, w, h, n, edge, out_cap, cap)
    kept = []
    for f, k in enumerate(lists):
        want = oracle_retain_best(oracle, rowmajor(k), w, h, n, edge)
        m = min(len(want), out_cap)
        assert ocounts[f] == m, (f, n, edge, out_cap, ocounts[f], len(want))
        assert (okeys[f, :m] == pack(want[:m])).all(), (f, n, edge, out_cap)
        kept.append(len(want))
    return okeys, ocounts, kept


@pytest.mark.parametrize("count", [1023, 1024, 1025, 5000])
def test_retain_best_counts_and_n(gpu_ctx, oracle, count):
    """counts around the kernel's 1024 threads, n at 0, 1 and around the count, keys over the whole 4095 x 4095 frame (bit 31
    set where y >= 2048), scores with few and with many ties, out_cap above and below the kept count"""
    w = h = 4095
    lists = [random_keys(count, w, h, count), random_keys(count, w, h, count + 1, score_hi=4)]
    for edge in (0, 31):
        c = len(oracle_retain_best(oracle, lists[0], w, h, -1, edge))
        for n in (0, 1, c - 1, c, c + 1):
            for out_cap in (count, count + 100, 700):   # the key capacity itself, more, and fewer than kept
                check_retain_best(gpu_ctx, oracle, lists, w, h, n, edge, out_cap)


@pytest.mark.parametrize("w,h", [(62, 62), (63, 63), (200, 150)])
def test_retain_best_border(gpu_ctx, oracle, w, h):
    """corners on the border's edge and one pixel outside it, on all four sides"""
    pts = set()
    for edge in (31, 1):
        for v in (edge - 1, edge, w - edge - 1, w - edge):
            for u in (edge - 1, edge, h // 2, h - edge - 1, h - edge):
                if 0 <= v < w and 0 <= u < h:
                    pts.add((v, u))
        for u in (edge - 1, edge, h - edge - 1, h - edge):
            if 0 <= u < h:
                pts.add((w // 2, u))
    rng = np.random.default_rng(w)
    xys = np.array([(x, y, int(rng.integers(0, 256))) for x, y in sorted(pts)], np.int32)
    lists = [xys[rng.permutation(len(xys))], xys[::-1].copy()]
    for edge in (0, 1, 31):
        for n in (3, len(xys)):
            _, counts, kept = check_retain_best(gpu_ctx, oracle, lists, w, h, n, edge, len(xys))
    if w <= 62:
        assert kept == [0, 0]   # edge 31 leaves no pixel of a 62-px frame (the last check ran with edge 31)


def test_retain_best_ties_truncate_in_row_major_order(gpu_ctx, oracle):
    """every corner tied at one score: all are kept, more than out_cap; the call keeps the first out_cap in row-major order
    and reports out_cap, the same on every call"""
    w, h = 640, 480
    base = rowmajor(oracle_fast(oracle, tie_dots(w, h), 20))
    assert len(np.unique(base[:, 2])) == 1 and len(base) > 4096
    rng = np.random.default_rng(1)
    lists = [base[rng.permutation(len(base))], base[rng.permutation(len(base))][: len(base) // 2]]
    runs = []
    for _ in range(3):
        okeys, ocounts, kept = check_retain_best(gpu_ctx, oracle, lists, w, h, 10, 31, 192, cap=nms_bound(w, h))
        assert (ocounts == 192).all() and min(kept) > 1000
        runs.append(okeys)
    assert all((r == runs[0]).all() for r in runs)


# ---- 4. Harris and the float selection ---------------------------------------------------------------------------------------------

def test_harris_at_its_border(gpu_ctx, oracle):
    """points where the 7 x 7 block (+ the Sobel ring) meets the frame's edge -- x0 = 3, 4, w - 5, w - 4 -- and on .5
    coordinates (round half to even)"""
    for w, h in ((64, 48), (201, 99)):
        img = scene("texture", w, h, w)
        xs = [3.0, 3.5, 4.0, 4.5, 5.5, w / 2 + 0.5, w - 5.5, w - 5.0, w - 4.5, w - 4.0, 2.5, w - 3.5]
        ys = [3.0, 3.5, 4.0, 4.5, h / 2 - 0.5, h - 5.5, h - 5.0, h - 4.5, h - 4.0]
        pts = np.array([(x, y) for x in xs for y in ys], np.float32)
        resp = torch.full((len(pts),), 7.0, dtype=torch.float32, device=DEV)
        gpu_ctx.harris(dev(img), w, h, 1, dev(pts), None, len(pts), resp)
        torch.cuda.synchronize()
        want = oracle_harris(oracle, img, pts)
        assert (bits(resp.cpu().numpy()) == bits(want)).all()
        assert (want == 0).sum() > 0 and (want != 0).sum() > 0


def gpu_orb_detect(ctx, imgs, nfeatures, thr, out_cap):
    n, h, w = imgs.shape
    kp = torch.zeros((n, out_cap, 4), dtype=torch.float32, device=DEV)
    desc = torch.zeros((n, out_cap, 32), dtype=torch.uint8, device=DEV)
    counts = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    ctx.orb_detect(dev(imgs), w, h, n, nfeatures, thr, 0, kp, desc, counts, out_cap)
    torch.cuda.synchronize()
    return kp.cpu().numpy(), desc.cpu().numpy(), counts.cpu().numpy()


ORB_SCENES = {   # kind, w, h, nfeatures
    "negative_nth": ("edges", 336, 240, 300),
    "harris_ties": ("ties", 320, 240, 100),
    "dense": ("dense", 640, 480, 500),           # more corners than the old key capacity max(8192, w h / 24)
    "many_candidates": ("noise", 640, 480, 600),  # 2n = 1200 > 1024 candidates in the float selection
    "n_above_candidates": ("texture", 320, 240, 5000),
}


@pytest.mark.parametrize("name", list(ORB_SCENES))
def test_orb_detect_vs_oracle(gpu_ctx, oracle, name):
    kind, w, h, nf = ORB_SCENES[name]
    imgs = np.stack([scene(kind, w, h, s) for s in (1, 2)])
    wants = [oracle_orb_detect(oracle, imgs[f], nf, 20) for f in range(2)]
    if name == "negative_nth":
        assert all(k[:, 2].min() < 0 for k, _ in wants)       # the n-th best response is negative
    if name == "harris_ties":
        assert all(len(k) > nf and len(np.unique(k[:, 2])) <= 2 for k, _ in wants)
    if name == "dense":
        assert all(len(oracle_fast(oracle, im, 20)) > max(8192, w * h // 24) for im in imgs)
    if name == "n_above_candidates":
        assert all(len(k) < nf for k, _ in wants)
    for out_cap in (max(len(k) for k, _ in wants), 256):
        kp, desc, counts = gpu_orb_detect(gpu_ctx, imgs, nf, 20, out_cap)
        for f, (wk, wd) in enumerate(wants):
            m = min(len(wk), out_cap)
            assert counts[f] == len(wk), (name, f, counts[f], len(wk))   # the true count; the first out_cap are stored
            assert (bits(kp[f, :m]) == bits(wk[:m])).all(), (name, f)
            assert (desc[f, :m] == wd[:m]).all(), (name, f)


# ---- 5. the pipeline ------------------------------------------------------------------------------------------------------------------

def pipeline_outputs(pipe, batch):
    fcap = pipe.fcap
    torch.cuda.synchronize()
    return {"sel": pipe.buffer("sel", (batch, fcap), torch.int32).cpu().numpy().view(np.uint32).copy(),
            "selcounts": pipe.buffer("selcounts", (batch,), torch.int32).cpu().numpy().copy(),
            "pts": pipe.buffer("pts", (batch, fcap, 2), torch.float32).cpu().numpy().copy(),
            "angles": pipe.buffer("angles", (batch, fcap), torch.float32).cpu().numpy().copy(),
            "desc": pipe.buffer("desc", (batch, fcap, 32), torch.uint8).cpu().numpy().copy(),
            "kept": pipe.buffer("kept", (batch, fcap), torch.uint8).cpu().numpy().copy()}


def run_pipeline_twice(gpu_ctx, frames, nfeat, flags):
    batch, h, w = frames.shape[:3]
    pipe = Pipeline(gpu_ctx, w, h, batch, fast_thr=20, nfeatures=nfeat, orb_flags=flags, map_size=0)
    try:
        assert pipe.kcap == nms_bound(w, h)
        d_in = dev(frames)
        outs = []
        for _ in range(2):
            pipe.step_dev(d_in)
            outs.append(pipeline_outputs(pipe, batch))
        for k in outs[0]:
            assert (outs[0][k] == outs[1][k]).all(), k
        return outs[0], pipe.fcap
    finally:
        pipe.close()


def check_pipeline(oracle, frames, out, fcap, nfeat, harris):
    """the oracle composition (as in test_pipeline_vs_oracle), truncated at fcap in row-major order: this project's rule -- the
    reference keeps every tie"""
    for f in range(len(frames)):
        h, w = frames.shape[1:3]
        g = oracle_gray(oracle, frames[f])
        if harris:
            wk, wd = oracle_orb_detect(oracle, g, nfeat, 20)
            m = min(len(wk), fcap)
            pts, ang = np.ascontiguousarray(wk[:m, :2]), wk[:m, 3]
        else:
            want = oracle_retain_best(oracle, oracle_fast(oracle, g, 20), w, h, nfeat, 31)
            m = min(len(want), fcap)
            pts = np.ascontiguousarray(want[:m, :2].astype(np.float32))
            ang = np.zeros(m, np.float32)
            oracle.orc_ic_angles(P(g), w, h, P(pts), m, P(ang))
            blur = np.empty_like(g)
            oracle.orc_orb_blur(P(g), w, h, 0, P(blur))
            wd, wkept = np.zeros((m, 32), np.uint8), np.zeros(m, np.uint8)
            oracle.orc_orb_describe(P(blur), w, h, P(pts), P(ang), m, P(wd), P(wkept))
            assert wkept.all()
            assert (out["sel"][f, :m] == pack(want[:m])).all(), f
        assert out["selcounts"][f] == m, (f, out["selcounts"][f], m)
        k = out["sel"][f, :m].astype(np.int64)
        assert ((k >> 8) & 0xFFF == pts[:, 0]).all() and ((k >> 20) & 0xFFF == pts[:, 1]).all(), f
        assert (bits(out["pts"][f, :m]) == bits(pts)).all(), f
        assert (bits(out["angles"][f, :m]) == bits(ang)).all(), f
        assert (out["desc"][f, :m] == wd[:m]).all(), f
        assert (out["kept"][f, :m] == 1).all() and (out["kept"][f, m:] == 0).all(), f


def rgba_of(grays):
    return np.ascontiguousarray(np.stack([np.stack([g, g, g, np.full_like(g, 255)], -1) for g in grays]))


@pytest.mark.parametrize("harris", [False, True], ids=["fast_score", "harris"])
def test_pipeline_tie_scene_past_fcap(gpu_ctx, oracle, harris):
    """every corner tied (FAST score, and Harris response away from the edge): far more than fcap survive the selection"""
    w, h, nfeat = 640, 480, 100
    frames = rgba_of([tie_dots(w, h, 4, 1, 2), tie_dots(w, h, 4, 3, 0)])
    flags = ORB_IC_ANGLE | (ORB_HARRIS if harris else 0)
    out, fcap = run_pipeline_twice(gpu_ctx, frames, nfeat, flags)
    assert fcap == 192
    check_pipeline(oracle, frames, out, fcap, nfeat, harris)
    assert (out["selcounts"] == fcap).all()


@pytest.mark.parametrize("harris", [False, True], ids=["fast_score", "harris"])
@pytest.mark.parametrize("w,h,nfeat", [(1280, 720, 1000), (256, 4095, 300)])
def test_pipeline_more_corners_than_the_old_key_capacity(gpu_ctx, oracle, harris, w, h, nfeat):
    """noise and the dense dot lattice: more corners than max(w h / 16, 32768), the parent's key capacity; at 256 x 4095 half
    the selected keys lie at y >= 2048 (bit 31 set)"""
    grays = [scene("noise", w, h, 3), dense_dots(w, h, 1)]
    assert all(len(oracle_fast(oracle, g, 20)) > max(w * h // 16, 32768) for g in grays)
    frames = rgba_of(grays)
    out, fcap = run_pipeline_twice(gpu_ctx, frames, nfeat, ORB_IC_ANGLE | (ORB_HARRIS if harris else 0))
    check_pipeline(oracle, frames, out, fcap, nfeat, harris)
    if h > 2048:
        assert (out["pts"][0, :out["selcounts"][0], 1] >= 2048).sum() > 10
