"""GPU parity tests (H100): pyramidal LK / forward-backward KLT through the C ABI vs the CPU oracle and the golden vectors
dumped from the reference's own FeatureTracker.  Bit-exact: tracked positions are compared as float bit patterns."""
import numpy as np
import pytest
import torch

from conftest import golden
from alvaar_b200 import synth
from klt_util import build_pyramid, klt_points, oracle_fb_klt, oracle_klt_lk

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def gpu_fb(ctx, pa, da, pb, db, w, h, levels, pts, pri, nframes=1, npf=None):
    n = pts.shape[-2]
    d_pts, d_pri = dev(pts), dev(pri)
    good = torch.zeros((nframes, n), dtype=torch.uint8, device=DEV)
    ctx.klt_fb([dev(x) for x in pa], [dev(x) for x in da], [dev(x) for x in pb], [dev(x) for x in db], w, h, nframes, levels,
               d_pts, d_pri, n, good, npts_per_frame=None if npf is None else dev(npf))
    torch.cuda.synchronize()
    return d_pri.cpu().numpy(), good.cpu().numpy()


@pytest.mark.parametrize("levels", [1, 3])
def test_fb_klt_golden(gpu_ctx, oracle, levels):
    g = golden("klt")
    a, b = g["prev"], g["cur"]
    h, w = a.shape
    L = int(g["pyr_levels"])
    pa, da = build_pyramid(oracle, a, L)
    pb, db = build_pyramid(oracle, b, L)
    q, good = gpu_fb(gpu_ctx, pa, da, pb, db, w, h, levels, g["pts"], g["priors"])
    assert (good[0] == g[f"fb{levels}_good"]).all()
    assert (bits(q) == bits(g[f"fb{levels}_pos"])).all()


@pytest.mark.parametrize("levels,ui", [(1, 0), (1, 1), (3, 0), (3, 1)])
def test_klt_lk_golden(gpu_ctx, oracle, levels, ui):
    g = golden("klt")
    a, b = g["prev"], g["cur"]
    h, w = a.shape
    L = int(g["pyr_levels"])
    pa, da = build_pyramid(oracle, a, L)
    pb, _ = build_pyramid(oracle, b, L)
    n = len(g["pts"])
    d_next = dev(g["priors"])
    st = torch.zeros(n, dtype=torch.uint8, device=DEV)
    er = torch.zeros(n, dtype=torch.float32, device=DEV)
    gpu_ctx.klt_lk([dev(x) for x in pa], [dev(x) for x in da], [dev(x) for x in pb], w, h, 1, levels, dev(g["pts"]), d_next, n,
                   st, er, use_initial=bool(ui))
    torch.cuda.synchronize()
    assert (st.cpu().numpy() == g[f"lk{levels}_{ui}_status"]).all()
    assert (bits(d_next.cpu().numpy()) == bits(g[f"lk{levels}_{ui}_pos"])).all()
    assert (bits(er.cpu().numpy()) == bits(g[f"lk{levels}_{ui}_err"])).all()


@pytest.mark.parametrize("w,h,n,seed", [(161, 91, 300, 2), (640, 480, 800, 9), (1280, 720, 1000, 4)])
def test_fb_klt_vs_oracle(gpu_ctx, oracle, w, h, n, seed):
    """Seeded frames (points outside the image, large prior noise included) -- batch of 2 frame pairs, ragged counts."""
    fr, _ = synth.make_frames(3, w, h, seed=seed, rgba=False)
    pyr = [build_pyramid(oracle, np.ascontiguousarray(f), 3) for f in fr]
    pts = np.stack([klt_points(w, h, n, seed + k)[0] for k in range(2)])
    pri = np.stack([klt_points(w, h, n, seed + k, sigma=3.0)[1] for k in range(2)])
    npf = np.array([n, n - 37], np.int32)
    for levels in (1, 3):
        pa = [np.stack([pyr[0][0][k], pyr[1][0][k]]) for k in range(4)]
        da = [np.stack([pyr[0][1][k], pyr[1][1][k]]) for k in range(4)]
        pb = [np.stack([pyr[1][0][k], pyr[2][0][k]]) for k in range(4)]
        db = [np.stack([pyr[1][1][k], pyr[2][1][k]]) for k in range(4)]
        q, good = gpu_fb(gpu_ctx, pa, da, pb, db, w, h, levels, pts, pri, nframes=2, npf=npf)
        for f in range(2):
            m = int(npf[f])
            qo, go = oracle_fb_klt(oracle, pyr[f][0], pyr[f][1], pyr[f + 1][0], pyr[f + 1][1], w, h, levels, pts[f, :m], pri[f, :m])
            assert go.sum() > m // 3
            assert (good[f, :m] == go).all()
            assert (good[f, m:] == 0).all()
            assert (bits(q[f, :m]) == bits(qo)).all()
            assert (bits(q[f, m:]) == bits(pri[f, m:])).all()   # dead slots are left untouched


def test_klt_lk_vs_oracle_720p(gpu_ctx, oracle):
    w, h, n = 1280, 720, 1000
    fr, _ = synth.make_frames(2, w, h, seed=21, rgba=False)
    pa, da = build_pyramid(oracle, np.ascontiguousarray(fr[0]), 3)
    pb, _ = build_pyramid(oracle, np.ascontiguousarray(fr[1]), 3)
    pts, pri = klt_points(w, h, n, 21)
    qo, so, eo = oracle_klt_lk(oracle, pa, da, pb, w, h, 3, pts, pri, use_initial=0)
    d_next = dev(pri)
    st = torch.zeros(n, dtype=torch.uint8, device=DEV)
    er = torch.zeros(n, dtype=torch.float32, device=DEV)
    gpu_ctx.klt_lk([dev(x) for x in pa], [dev(x) for x in da], [dev(x) for x in pb], w, h, 1, 3, dev(pts), d_next, n, st, er,
                   use_initial=False)
    torch.cuda.synchronize()
    assert (st.cpu().numpy() == so).all() and so.sum() > 800
    assert (bits(d_next.cpu().numpy()) == bits(qo)).all()
    assert (bits(er.cpu().numpy()) == bits(eo)).all()


def test_klt_identity_property(gpu_ctx, oracle):
    """Size-independent property at full size: a frame tracked onto itself from exact priors does not move."""
    w, h = 1280, 720
    fr, _ = synth.make_frames(1, w, h, seed=1, rgba=False)
    pa, da = build_pyramid(oracle, np.ascontiguousarray(fr[0]), 3)
    rng = np.random.default_rng(0)
    pts = np.stack([rng.uniform(12, w - 12, 2000), rng.uniform(12, h - 12, 2000)], 1).astype(np.float32)
    q, good = gpu_fb(gpu_ctx, pa, da, pa, da, w, h, 3, pts[None], pts[None].copy())
    assert good.sum() > 1800
    assert np.abs(q[0][good[0] == 1] - pts[good[0] == 1]).max() <= 2e-5


def test_klt_rejects_other_windows(gpu_ctx):
    import alvaar_b200
    t = torch.zeros((1, 32, 32), dtype=torch.uint8, device=DEV)
    d = torch.zeros((1, 32, 32, 2), dtype=torch.int16, device=DEV)
    p = torch.zeros((1, 4, 2), dtype=torch.float32, device=DEV)
    g = torch.zeros((1, 4), dtype=torch.uint8, device=DEV)
    with pytest.raises(alvaar_b200.AlvaError):
        gpu_ctx.klt_fb([t], [d], [t], [d], 32, 32, 1, 0, p, p.clone(), 4, g, win=21)
