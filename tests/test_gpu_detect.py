"""GPU parity tests (H100): the reference's grid Shi-Tomasi detector + cornerSubPix through the C ABI vs the CPU oracle and
the golden vectors dumped from the reference's own FeatureExtractor.  Bit-exact: integer maxima, order, count, adapted
quality, and sub-pixel positions as float bit patterns."""
import numpy as np
import pytest
import torch

from conftest import golden
from alvaar_b200 import synth
from detect_util import oracle_detect, random_cur

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def gpu_detect(ctx, imgs, cs, curs, roi, q0, cap=4096):
    nf, h, w = imgs.shape
    ccap = max(1, max(len(c) for c in curs))
    cur = np.zeros((nf, ccap, 2), np.float32)
    ncur = np.zeros(nf, np.int32)
    for i, c in enumerate(curs):
        cur[i, :len(c)] = c
        ncur[i] = len(c)
    q = dev(np.full(nf, q0, np.float64))
    out = torch.zeros((nf, cap, 2), dtype=torch.float32, device=DEV)
    oi = torch.zeros((nf, cap, 2), dtype=torch.int32, device=DEV)
    cnt = torch.zeros(nf, dtype=torch.int32, device=DEV)
    ctx.detect_grid(dev(imgs), w, h, nf, cs, dev(cur), dev(ncur), ccap, roi, q, out, oi, cnt, cap)
    torch.cuda.synchronize()
    return out.cpu().numpy(), oi.cpu().numpy(), cnt.cpu().numpy(), q.cpu().numpy()


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_detect_golden(gpu_ctx, tag):
    g = golden("detect")
    img, cs = np.ascontiguousarray(g[f"{tag}_img"]), int(g[f"{tag}_cell"])
    out, _, cnt, _ = gpu_detect(gpu_ctx, img[None], cs, [g[f"{tag}_cur"]], g[f"{tag}_roi"], 0.001)
    want = g[f"{tag}_pts"]
    assert cnt[0] == len(want)
    assert (bits(out[0, :cnt[0]]) == bits(want)).all()


@pytest.mark.parametrize("w,h,cs,nf,ncur", [(640, 480, 40, 3, 60), (1280, 720, 40, 2, 300), (1280, 720, 30, 2, 0), (1920, 1080, 32, 1, 500),
                                            (333, 251, 24, 2, 7)])
def test_detect_vs_oracle(gpu_ctx, oracle, w, h, cs, nf, ncur):
    fr, _ = synth.make_frames(nf, w, h, seed=w + cs, rgba=False)
    imgs = np.ascontiguousarray(fr)
    curs = [random_cur(w, h, max(0, ncur - 17 * f), 100 + f) for f in range(nf)]
    roi = [20, 20, w - 40, h - 40]
    for q0 in (0.001, 0.00003):
        out, oi, cnt, q = gpu_detect(gpu_ctx, imgs, cs, curs, roi, q0)
        for f in range(nf):
            pts, ints, qo = oracle_detect(oracle, imgs[f], cs, curs[f], roi, q0)
            assert cnt[f] == len(pts) > 0
            assert (oi[f, :cnt[f]] == ints).all()
            assert (bits(out[f, :cnt[f]]) == bits(pts)).all()
            assert q[f] == qo


def test_detect_flat_and_capacity(gpu_ctx, oracle):
    flat = np.full((1, 240, 320), 90, np.uint8)
    out, _, cnt, q = gpu_detect(gpu_ctx, flat, 40, [np.zeros((0, 2), np.float32)], [20, 20, 280, 200], 0.001)
    assert cnt[0] == 0 and q[0] == 0.0005
    fr, _ = synth.make_frames(1, 640, 480, seed=3, rgba=False)
    out, _, cnt, _ = gpu_detect(gpu_ctx, np.ascontiguousarray(fr), 40, [np.zeros((0, 2), np.float32)], [20, 20, 600, 440], 0.001, cap=16)
    pts, _, _ = oracle_detect(oracle, np.ascontiguousarray(fr[0]), 40, np.zeros((0, 2)), [20, 20, 600, 440])
    assert cnt[0] == len(pts) > 16                       # true count is reported, only `cap` are stored
    assert (bits(out[0]) == bits(pts[:16])).all()


def test_corner_subpix_alone(gpu_ctx, oracle):
    import ctypes as C
    from conftest import P
    w, h, n = 640, 480, 500
    fr, _ = synth.make_frames(1, w, h, seed=9, rgba=False)
    img = np.ascontiguousarray(fr[0])
    rng = np.random.default_rng(1)
    pts = np.stack([rng.uniform(0, w - 1, n), rng.uniform(0, h - 1, n)], 1).astype(np.float32)   # border points included
    want = pts.copy()
    oracle.orc_corner_subpix.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double]
    oracle.orc_corner_subpix(P(img), w, h, P(want), n, 3, 30, 0.01)
    d = dev(pts[None])
    gpu_ctx.corner_subpix(dev(img[None]), w, h, 1, d, dev(np.array([n], np.int32)), n)
    torch.cuda.synchronize()
    assert (bits(d.cpu().numpy()[0]) == bits(want)).all()
