"""GPU parity tests (H100): gray / pyramid / FAST-9 through the C ABI vs the CPU oracle and the golden vectors.
Integer stages: bit-exact."""
import numpy as np
import pytest
import torch

from conftest import P, golden
from alvaar_b200 import synth, unpack_keys

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def oracle_fast(oracle, img, thr=20, nms=1):
    h, w = img.shape
    out = np.zeros((w * h, 3), np.int32)
    n = oracle.orc_fast9(P(img), w, h, thr, nms, P(out), w * h)
    return out[:n].copy()


def oracle_pyrdown(oracle, img):
    h, w = img.shape
    out = np.empty(((h + 1) // 2, (w + 1) // 2), np.uint8)
    oracle.orc_pyrdown(P(img), w, h, P(out))
    return out


@pytest.mark.parametrize("w,h,n", [(64, 48, 1), (641, 479, 2), (1280, 720, 2), (17, 33, 3)])
def test_gray(gpu_ctx, oracle, w, h, n):
    rgba = synth.random_rgba(w, h, n, seed=w)
    d_in, d_out = dev(rgba), torch.zeros((n, h, w), dtype=torch.uint8, device=DEV)
    gpu_ctx.gray(d_in, d_out, w, h, n)
    got = d_out.cpu().numpy()
    for f in range(n):
        want = np.empty((h, w), np.uint8)
        oracle.orc_gray(P(rgba[f]), w, h, P(want))
        assert (got[f] == want).all()


def test_gray_golden(gpu_ctx):
    g = golden("gray")
    d_out = torch.zeros((48, 64), dtype=torch.uint8, device=DEV)
    gpu_ctx.gray(dev(g["rgba"]), d_out, 64, 48, 1)
    assert (d_out.cpu().numpy() == g["gray"]).all()


@pytest.mark.parametrize("w,h,n", [(1280, 720, 2), (161, 91, 1), (45, 37, 3), (16, 16, 1), (2, 3, 1), (1, 1, 1)])
def test_pyrdown(gpu_ctx, oracle, w, h, n):
    imgs = np.stack([synth.crop(w, h, 31 * f, 17 * f) for f in range(n)])
    dw, dh = (w + 1) // 2, (h + 1) // 2
    d_out = torch.zeros((n, dh, dw), dtype=torch.uint8, device=DEV)
    gpu_ctx.pyrdown(dev(imgs), d_out, w, h, n)
    got = d_out.cpu().numpy()
    for f in range(n):
        assert (got[f] == oracle_pyrdown(oracle, imgs[f])).all()


def test_pyramid_golden(gpu_ctx):
    g = golden("pyramid")
    cur = dev(g["img"])
    h, w = g["img"].shape
    for k in (1, 2, 3):
        dw, dh = (w + 1) // 2, (h + 1) // 2
        nxt = torch.zeros((dh, dw), dtype=torch.uint8, device=DEV)
        gpu_ctx.pyrdown(cur, nxt, w, h, 1)
        assert (nxt.cpu().numpy() == g[f"l{k}"]).all()
        cur, w, h = nxt, dw, dh


def run_fast(gpu_ctx, imgs, thr, sorted_=True, cap=None):
    n, h, w = imgs.shape
    cap = cap or w * h // 4
    keys = torch.zeros((n, cap), dtype=torch.int32, device=DEV)
    counts = torch.zeros(n, dtype=torch.int32, device=DEV)
    gpu_ctx.fast9(dev(imgs), w, h, n, thr, keys, counts, cap, sorted_)
    torch.cuda.synchronize()
    c = counts.cpu().numpy()
    k = keys.cpu().numpy().view(np.uint32)
    return [unpack_keys(k[f, :c[f]]) for f in range(n)], c


# TMA path (w % 16 == 0), generic path (odd sizes), partial tiles, tiny images, multi-frame batches
@pytest.mark.parametrize("w,h,n,thr", [(640, 480, 2, 20), (1280, 720, 1, 20), (333, 217, 2, 20), (120, 62, 1, 20),
                                       (121, 63, 1, 10), (16, 16, 1, 5), (1920, 1080, 1, 35), (320, 240, 3, 7)])
def test_fast9_vs_oracle(gpu_ctx, oracle, w, h, n, thr):
    imgs = np.stack([synth.crop(w, h, 100 + 37 * f, 50 + 91 * f) for f in range(n)])
    got, counts = run_fast(gpu_ctx, imgs, thr)
    for f in range(n):
        want = oracle_fast(oracle, imgs[f], thr)
        assert counts[f] == len(want), (f, counts[f], len(want))
        assert (got[f] == want).all()          # same corners, same scores, same (row-major) order


def test_fast9_golden(gpu_ctx):
    g = golden("fast")
    for thr in (20, 7):
        got, _ = run_fast(gpu_ctx, g["img"][None], thr)
        want = g[f"kp_t{thr}_n1"]
        assert len(got[0]) == len(want) and (got[0] == want).all()


def test_fast9_flat_and_saturated(gpu_ctx, oracle):
    """Edge cases: constant image (no corners), 0/255 checkerboard blocks (saturating c+-t), isolated dots."""
    w, h = 256, 128
    imgs = np.zeros((4, h, w), np.uint8)
    imgs[0] = 77
    yy, xx = np.mgrid[0:h, 0:w]
    imgs[1] = (((yy // 5) + (xx // 5)) % 2) * 255
    imgs[2] = 250
    imgs[2, 10::9, 10::11] = 255
    imgs[3] = 3
    imgs[3, 8::7, 8::13] = 0
    for thr in (1, 20, 254):
        got, counts = run_fast(gpu_ctx, imgs, thr)
        for f in range(4):
            want = oracle_fast(oracle, imgs[f], thr)
            assert counts[f] == len(want) and (got[f] == want).all(), (thr, f)


def test_fast9_capacity_reported(gpu_ctx):
    img = synth.crop(640, 480)[None]
    cap = 64
    keys = torch.zeros((1, cap), dtype=torch.int32, device=DEV)
    counts = torch.zeros(1, dtype=torch.int32, device=DEV)
    gpu_ctx.fast9(dev(img), 640, 480, 1, 20, keys, counts, cap, False)
    assert counts.item() > cap          # the true count is reported; the caller detects the overflow


@pytest.mark.parametrize("w,h,n", [(1280, 720, 2), (641, 479, 1), (644, 478, 2), (160, 90, 1), (1920, 1080, 1)])
def test_frontend_fused(gpu_ctx, oracle, w, h, n):
    """RGBA -> L0..L3 + FAST in one call == cvtColor + 3x pyrDown + FAST of the oracle."""
    rng = np.random.default_rng(w + h)
    gray = np.stack([synth.crop(w, h, 10 + 50 * f, 20 + 30 * f) for f in range(n)])
    rgba = np.stack([gray, np.roll(gray, 1, 2), rng.integers(0, 256, gray.shape, dtype=np.uint8),
                     np.full_like(gray, 255)], -1)
    sizes = [(w, h)]
    for _ in range(3):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    lv = [torch.zeros((n, s[1], s[0]), dtype=torch.uint8, device=DEV) for s in sizes]
    cap = w * h // 4
    keys = torch.zeros((n, cap), dtype=torch.int32, device=DEV)
    counts = torch.zeros(n, dtype=torch.int32, device=DEV)
    gpu_ctx.frontend(dev(rgba), w, h, n, lv[0], lv[1], lv[2], lv[3], 20, keys, counts, cap, True)
    torch.cuda.synchronize()
    c = counts.cpu().numpy()
    k = keys.cpu().numpy().view(np.uint32)
    for f in range(n):
        g0 = np.empty((h, w), np.uint8)
        oracle.orc_gray(P(np.ascontiguousarray(rgba[f])), w, h, P(g0))
        assert (lv[0][f].cpu().numpy() == g0).all()
        cur = g0
        for lvl in (1, 2, 3):
            cur = oracle_pyrdown(oracle, cur)
            assert (lv[lvl][f].cpu().numpy() == cur).all(), lvl
        want = oracle_fast(oracle, g0, 20)
        assert c[f] == len(want) and (unpack_keys(k[f, :c[f]]) == want).all()


def test_frontend_full_size_properties(gpu_ctx):
    """BASELINE config size (1280x720, batch of frames): size-independent properties -- the unsorted and the
    sorted outputs are the same SET, sorted output is strictly increasing in (y, x), and two runs agree."""
    n, w, h = 8, 1280, 720
    frames, _ = synth.make_frames(n, w, h)
    d_in = dev(frames)
    cap = 32768
    outs = []
    for sorted_ in (False, True, True):
        keys = torch.zeros((n, cap), dtype=torch.int32, device=DEV)
        counts = torch.zeros(n, dtype=torch.int32, device=DEV)
        l0 = torch.zeros((n, h, w), dtype=torch.uint8, device=DEV)
        gpu_ctx.frontend(d_in, w, h, n, l0, None, None, None, 20, keys, counts, cap, sorted_)
        torch.cuda.synchronize()
        outs.append((keys.cpu().numpy().view(np.uint32), counts.cpu().numpy()))
        assert (l0.cpu().numpy() == frames[..., 0]).all()      # R = G = B input: gray == R
    for f in range(n):
        c = outs[0][1][f]
        assert c == outs[1][1][f] == outs[2][1][f] and 5000 < c < cap
        a, b, b2 = outs[0][0][f, :c], outs[1][0][f, :c], outs[2][0][f, :c]
        assert (np.sort(a) == b).all() and (b == b2).all()
        assert (np.diff((b >> 8).astype(np.int64)) > 0).all()


def test_retain_best(gpu_ctx, oracle):
    w, h, n = 640, 480, 2
    imgs = np.stack([synth.crop(w, h, 5, 7), synth.crop(w, h, 900, 1200)])
    cap = w * h // 4
    keys = torch.zeros((n, cap), dtype=torch.int32, device=DEV)
    counts = torch.zeros(n, dtype=torch.int32, device=DEV)
    gpu_ctx.fast9(dev(imgs), w, h, n, 20, keys, counts, cap, False)
    ocap = 4096
    okeys = torch.zeros((n, ocap), dtype=torch.int32, device=DEV)
    ocounts = torch.zeros(n, dtype=torch.int32, device=DEV)
    gpu_ctx.retain_best(keys, counts, cap, n, w, h, 500, 31, okeys, ocounts, ocap)
    torch.cuda.synchronize()
    for f in range(n):
        allk = oracle_fast(oracle, imgs[f], 20)
        inb = allk[(allk[:, 0] >= 31) & (allk[:, 0] < w - 31) & (allk[:, 1] >= 31) & (allk[:, 1] < h - 31)]
        thr = oracle.orc_retain_best_threshold(P(np.ascontiguousarray(inb)), len(inb), 500)
        want = inb[inb[:, 2] >= thr]
        c = ocounts[f].item()
        got = unpack_keys(okeys[f, :c].cpu().numpy().view(np.uint32))
        assert c == len(want) >= 500 and (got == want).all()


@pytest.mark.parametrize("w,h,n", [(1280, 720, 2), (640, 360, 1), (161, 91, 2), (45, 37, 3), (6, 5, 1), (1, 9, 1), (9, 1, 1),
                                   (2, 2, 1)])
def test_scharr_vs_oracle(gpu_ctx, oracle, w, h, n):
    """Derivative image of buildOpticalFlowPyramid(withDerivatives): int16 (dx, dy), bit-exact, incl. odd widths
    (byte path) and degenerate 1-pixel-wide / -high levels."""
    imgs = np.stack([np.ascontiguousarray(synth.crop(max(w, 16), max(h, 16), 10 + 37 * f, 20 + 11 * f)[:h, :w]) for f in range(n)])
    out = torch.full((n, h, w, 2), -7, dtype=torch.int16, device=DEV)
    gpu_ctx.scharr(dev(imgs), out, w, h, n)
    got = out.cpu().numpy()
    for f in range(n):
        want = np.zeros((h, w, 2), np.int16)
        oracle.orc_scharr(P(np.ascontiguousarray(imgs[f])), w, h, P(want))
        assert (got[f] == want).all()


def test_scharr_golden(gpu_ctx):
    g = golden("scharr")
    for k in range(4):
        lv = g[f"l{k}"]
        h, w = lv.shape
        out = torch.zeros((h, w, 2), dtype=torch.int16, device=DEV)
        gpu_ctx.scharr(dev(lv), out, w, h, 1)
        assert (out.cpu().numpy() == g[f"d{k}"]).all()
