"""GPU parity tests (H100): ORB blur / rBRIEF descriptors / IC angle / Hamming 2-NN vs the oracle and goldens.
Descriptors and match indices are bit-exact; the blur is float arithmetic rounded to u8 and is checked bit-exact
too (the kernel pins evaluation order and fusion exactly like the reference build it mirrors)."""
import numpy as np
import pytest
import torch

from conftest import P, golden
from alvaar_b200 import synth, ORB_FMA, ORB_IC_ANGLE

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("w,h", [(1280, 720), (641, 479), (64, 64), (130, 35), (256, 100), (176, 64), (1296, 130), (160, 8)])
@pytest.mark.parametrize("fma", [0, 1])
def test_orb_blur(gpu_ctx, oracle, w, h, fma):
    img = synth.crop(w, h, 11, 13)
    want = np.empty_like(img)
    oracle.orc_orb_blur(P(img), w, h, fma, P(want))
    out = torch.zeros((h, w), dtype=torch.uint8, device=DEV)
    gpu_ctx.orb_blur(dev(img), out, w, h, 1, ORB_FMA if fma else 0)
    assert (out.cpu().numpy() == want).all()


def test_orb_blur_golden(gpu_ctx):
    g = golden("orb")
    h, w = g["img"].shape
    for flags, key in ((0, "blur"), (ORB_FMA, "blur_fma")):
        out = torch.zeros((h, w), dtype=torch.uint8, device=DEV)
        gpu_ctx.orb_blur(dev(g["img"]), out, w, h, 1, flags)
        assert (out.cpu().numpy() == g[key]).all()


def gpu_describe(gpu_ctx, img, blur, pts, flags, nframes=1, npf=None):
    h, w = img.shape[-2:]
    n = pts.shape[-2]
    desc = torch.zeros((nframes, n, 32), dtype=torch.uint8, device=DEV)
    kept = torch.zeros((nframes, n), dtype=torch.uint8, device=DEV)
    ang = torch.zeros((nframes, n), dtype=torch.float32, device=DEV)
    gpu_ctx.orb_describe(dev(img), dev(blur), w, h, nframes, dev(pts), None if npf is None else dev(npf), n, flags,
                         desc, kept, ang)
    torch.cuda.synchronize()
    return desc.cpu().numpy(), kept.cpu().numpy(), ang.cpu().numpy()


def test_orb_describe_constant_angle(gpu_ctx, oracle):
    """AlvaAR mode: every keypoint steered by -1 degree (feature_extractor.cpp:179-182)."""
    w, h = 1280, 720
    img = synth.crop(w, h, 40, 60)
    blur = np.empty_like(img)
    oracle.orc_orb_blur(P(img), w, h, 0, P(blur))
    rng = np.random.default_rng(1)
    n = 100000                                   # >= 1e5 keypoints (SURVEY 7 "hard parts")
    pts = np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], 1).astype(np.float32)
    pts[:5000] = np.floor(pts[:5000]) + 0.5      # round-half-even cases
    want_d, want_k = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
    oracle.orc_orb_describe(P(blur), w, h, P(pts), None, n, P(want_d), P(want_k))
    d, k, a = gpu_describe(gpu_ctx, img, blur, pts, 0)
    assert (k[0] == want_k).all() and (d[0] == want_d).all()
    assert (a[0][want_k == 1] == -1).all()


def test_orb_describe_ic_angle(gpu_ctx, oracle):
    """ORB detect mode: intensity-centroid angle (exact integer moments + fastAtan2) then steered BRIEF."""
    w, h = 1280, 720
    img = synth.crop(w, h, 400, 300)
    blur = np.empty_like(img)
    oracle.orc_orb_blur(P(img), w, h, 0, P(blur))
    rng = np.random.default_rng(2)
    n = 50000
    pts = np.stack([rng.integers(0, w, n), rng.integers(0, h, n)], 1).astype(np.float32)
    ang = np.zeros(n, np.float32)
    oracle.orc_ic_angles(P(img), w, h, P(pts), n, P(ang))
    want_d, want_k = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
    oracle.orc_orb_describe(P(blur), w, h, P(pts), P(ang), n, P(want_d), P(want_k))
    d, k, a = gpu_describe(gpu_ctx, img, blur, pts, ORB_IC_ANGLE)
    m = want_k == 1
    assert (k[0] == want_k).all()
    assert (a[0][m].view(np.uint32) == ang[m].view(np.uint32)).all()      # angles bit-identical
    assert (d[0][m] == want_d[m]).all()



def test_orb_golden(gpu_ctx):
    g = golden("orb")
    img, blur = g["img"], g["blur"]
    d, k, _ = gpu_describe(gpu_ctx, img, blur, g["pts"], 0)
    m = g["kept"] == 1
    assert (k[0] == g["kept"]).all() and (d[0][m] == g["desc"][m]).all()
    # reference ORB::detectAndCompute keypoints: angle + descriptor straight from the reference
    kp = g["det_kp"]
    d, k, a = gpu_describe(gpu_ctx, img, blur, np.ascontiguousarray(kp[:, :2]), ORB_IC_ANGLE)
    assert k[0].all()
    assert (a[0].view(np.uint32) == kp[:, 3].copy().view(np.uint32)).all()
    assert (d[0] == g["det_desc"]).all()


def test_orb_describe_ragged_batch(gpu_ctx, oracle):
    """Several frames with different point counts in one call; slots past the count come back empty."""
    w, h, nf, n = 320, 240, 3, 64
    imgs = np.stack([synth.crop(w, h, 50 * f, 80 * f) for f in range(nf)])
    blurs = np.stack([np.empty_like(imgs[0]) for _ in range(nf)])
    for f in range(nf):
        oracle.orc_orb_blur(P(imgs[f]), w, h, 0, P(blurs[f]))
    rng = np.random.default_rng(4)
    pts = np.stack([rng.uniform(0, w, (nf, n)), rng.uniform(0, h, (nf, n))], -1).astype(np.float32)
    npf = np.array([64, 0, 17], np.int32)
    d, k, _ = gpu_describe(gpu_ctx, imgs, blurs, pts, 0, nf, npf)
    for f in range(nf):
        want_d, want_k = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
        c = int(npf[f])
        if c:
            oracle.orc_orb_describe(P(blurs[f]), w, h, P(np.ascontiguousarray(pts[f, :c])), None, c, P(want_d), P(want_k))
        assert (k[f] == want_k).all() and (d[f] == want_d).all()


@pytest.mark.parametrize("nq,nt", [(1000, 10000), (1000, 1000), (7, 1), (1, 2), (33, 1025), (1000, 20000)])
def test_knn2_vs_oracle(gpu_ctx, oracle, nq, nt):
    q, t = synth.make_descriptors(nq, nt, seed=nq + nt, planted=0.3 if nt >= nq else 0.0)
    if nt > 100:
        t[nt // 2:nt // 2 + 20] = t[:20]          # exact duplicates -> tie rule (lowest index first)
    want = np.zeros((nq, 4), np.int32)
    oracle.orc_knn2(P(q), nq, P(t), nt, P(want))
    out = torch.zeros((nq, 4), dtype=torch.int32, device=DEV)
    gpu_ctx.hamming_knn2(dev(q), nq, dev(t), nt, out)
    assert (out.cpu().numpy() == want).all()


def test_knn2_golden(gpu_ctx):
    g = golden("knn")
    out = torch.zeros((len(g["q"]), 4), dtype=torch.int32, device=DEV)
    gpu_ctx.hamming_knn2(dev(g["q"]), len(g["q"]), dev(g["t"]), len(g["t"]), out)
    assert (out.cpu().numpy() == g["out"]).all()


def test_knn2_self_match_property(gpu_ctx):
    """Size-independent property at the largest size: matching a set against itself gives (i, 0) first."""
    _, t = synth.make_descriptors(8, 20000, seed=5, planted=0.0)
    d_t = dev(t)
    out = torch.zeros((20000, 4), dtype=torch.int32, device=DEV)
    gpu_ctx.hamming_knn2(d_t, 20000, d_t, 20000, out)
    o = out.cpu().numpy()
    assert (o[:, 0] == np.arange(20000)).all() and (o[:, 1] == 0).all() and (o[:, 3] > 0).all()


@pytest.fixture
def knn_mma(gpu_ctx):
    """force the tensor-core formulation (hamming_mma.cu) for every size; restored to automatic afterwards"""
    assert gpu_ctx.L.alva_set_option(b"knn_mma", 2) == 0
    yield gpu_ctx
    gpu_ctx.L.alva_set_option(b"knn_mma", 1)
    gpu_ctx.L.alva_set_option(b"knn_mma_mode", 0)
    gpu_ctx.L.alva_set_option(b"knn_mma_kind", 0)


@pytest.mark.parametrize("kind,mode", [(1, 0), (1, 1), (0, 0), (0, 1)])
@pytest.mark.parametrize("nq,nt", [(1000, 10000), (1000, 1000), (7, 1), (1, 2), (33, 1025), (1000, 20000), (257, 129), (4100, 300)])
def test_knn2_mma_vs_oracle(knn_mma, oracle, nq, nt, kind, mode):
    """tensor-core (wgmma) formulation (dot = 256 - 2 * distance; E4M3 / fp32 and int8 / int32 operand kinds, both shared-memory operand
    layouts): bit-identical 2-NN lists incl. the tie rule"""
    assert knn_mma.L.alva_set_option(b"knn_mma_mode", mode) == 0
    assert knn_mma.L.alva_set_option(b"knn_mma_kind", kind) == 0
    q, t = synth.make_descriptors(nq, nt, seed=nq + nt, planted=0.3 if nt >= nq else 0.0)
    if nt > 100:
        t[nt // 2:nt // 2 + 20] = t[:20]
    want = np.zeros((nq, 4), np.int32)
    oracle.orc_knn2(P(q), nq, P(t), nt, P(want))
    out = torch.full((nq, 4), -7, dtype=torch.int32, device=DEV)
    knn_mma.hamming_knn2(dev(q), nq, dev(t), nt, out)
    assert (out.cpu().numpy() == want).all()


def test_knn2_mma_golden(knn_mma):
    g = golden("knn")
    out = torch.zeros((len(g["q"]), 4), dtype=torch.int32, device=DEV)
    knn_mma.hamming_knn2(dev(g["q"]), len(g["q"]), dev(g["t"]), len(g["t"]), out)
    assert (out.cpu().numpy() == g["out"]).all()


@pytest.mark.parametrize("kind", [1, 0])
def test_knn2_mma_ragged_batch(knn_mma, oracle, kind):
    """[nbatch][qcap] query slots with per-batch live counts (incl. an empty and a full batch): live slots equal the oracle's
    lists, dead slots come back as -1 -- the compaction of the live rows must not leak between batches."""
    nb, qcap, nt = 9, 256, 3000
    counts = np.array([256, 0, 1, 255, 17, 128, 129, 200, 64], np.int32)
    q, t = synth.make_descriptors(nb * qcap, nt, seed=11, planted=0.3)
    assert knn_mma.L.alva_set_option(b"knn_mma_kind", kind) == 0
    out = torch.full((nb * qcap, 4), -7, dtype=torch.int32, device=DEV)
    knn_mma.hamming_knn2_batch(dev(q), torch.from_numpy(counts).to(DEV), nb, qcap, dev(t), nt, out)
    got = out.cpu().numpy().reshape(nb, qcap, 4)
    for b in range(nb):
        c = int(counts[b])
        if c:
            want = np.zeros((c, 4), np.int32)
            qb = np.ascontiguousarray(q[b * qcap:b * qcap + c])
            oracle.orc_knn2(P(qb), c, P(t), nt, P(want))
            assert (got[b, :c] == want).all(), b
        assert (got[b, c:] == -1).all(), b


def test_knn2_mma_equals_lop3_on_bench_shape(gpu_ctx):
    """the bench's matcher problem (64 x 1536 slots, ~1100 live, 10 000-descriptor map): automatic dispatch (tensor cores)
    against the LOP3 / POPC kernel"""
    nb, qcap, nt = 64, 1536, 10000
    rng = np.random.default_rng(3)
    q, t = synth.make_descriptors(nb * qcap, nt, seed=21, planted=0.05)
    counts = torch.from_numpy(rng.integers(900, 1300, nb).astype(np.int32)).to(DEV)
    outs = []
    for opt in (0, 1):
        assert gpu_ctx.L.alva_set_option(b"knn_mma", opt) == 0
        out = torch.full((nb * qcap, 4), -7, dtype=torch.int32, device=DEV)
        gpu_ctx.hamming_knn2_batch(dev(q), counts, nb, qcap, dev(t), nt, out)
        outs.append(out.cpu().numpy())
    gpu_ctx.L.alva_set_option(b"knn_mma", 1)
    assert (outs[0] == outs[1]).all()


@pytest.mark.parametrize("w,h,n", [(640, 480, 700), (130, 100, 40)])
def test_harris_vs_oracle(gpu_ctx, oracle, w, h, n):
    """HarrisResponses: integer block sums + float formula in the reference's order -> bit-identical floats."""
    img = synth.crop(w, h, 31, 77)
    rng = np.random.default_rng(w)
    pts = np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], -1).astype(np.float32)
    want = np.zeros(n, np.float32)
    oracle.orc_harris(P(img), w, h, P(pts), n, P(want))
    out = torch.full((n,), -1.0, dtype=torch.float32, device=DEV)
    gpu_ctx.harris(dev(img), w, h, 1, dev(pts), None, n, out)
    assert (out.cpu().numpy().view(np.uint32) == want.view(np.uint32)).all()
    assert (want != 0).sum() > n // 2


def gpu_detect(gpu_ctx, imgs, nfeat, thr, flags=0, cap=4096):
    nf, h, w = imgs.shape
    kp = torch.zeros((nf, cap, 4), dtype=torch.float32, device=DEV)
    desc = torch.zeros((nf, cap, 32), dtype=torch.uint8, device=DEV)
    cnt = torch.zeros(nf, dtype=torch.int32, device=DEV)
    gpu_ctx.orb_detect(dev(imgs), w, h, nf, nfeat, thr, flags, kp, desc, cnt, cap)
    torch.cuda.synchronize()
    return kp.cpu().numpy(), desc.cpu().numpy(), cnt.cpu().numpy()


def test_orb_detect_golden(gpu_ctx):
    """alva_k_orb_detect == the reference's ORB::detectAndCompute keypoint set (x, y, Harris response, IC angle, rBRIEF)."""
    g = golden("orb")
    kp, d, c = gpu_detect(gpu_ctx, g["img"][None], 300, 20)
    gk, gd = g["det_kp"], g["det_desc"]
    o = np.lexsort((gk[:, 0], gk[:, 1]))
    n = int(c[0])
    assert n == len(gk)
    assert (kp[0, :n].view(np.uint32) == np.ascontiguousarray(gk[o][:, :4]).view(np.uint32)).all()
    assert (d[0, :n] == gd[o]).all()


@pytest.mark.parametrize("w,h,nfeat,thr,fma", [(1280, 720, 1000, 20, 0), (640, 480, 500, 20, 1), (200, 150, 1000, 10, 0),
                                               (320, 240, 0 + 1, 30, 0)])
def test_orb_detect_vs_oracle(gpu_ctx, oracle, w, h, nfeat, thr, fma):
    imgs = np.stack([synth.crop(w, h, 40 + 97 * f, 10 + 53 * f) for f in range(3)])
    kp, d, c = gpu_detect(gpu_ctx, imgs, nfeat, thr, ORB_FMA if fma else 0)
    for f in range(3):
        wk, wd = np.zeros((4096, 4), np.float32), np.zeros((4096, 32), np.uint8)
        n = oracle.orc_orb_detect(P(imgs[f]), w, h, nfeat, thr, fma, P(wk), P(wd), 4096)
        assert n == c[f] and n >= min(nfeat, 1)
        assert (kp[f, :n].view(np.uint32) == wk[:n].view(np.uint32)).all()
        assert (d[f, :n] == wd[:n]).all()
