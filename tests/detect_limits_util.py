"""Input scenes of the detector's structural-limit tests (tests/test_oracle_detect_limits.py checks the oracle against the
reference on them, tests/test_gpu_detect_limits.py runs them through the kernels), the reference's detector behind a C call,
and the store of the reference's outputs on these scenes (tests/golden/ref_live_detect_limits.npz)."""
import ctypes as C
import os

import numpy as np

from conftest import P

STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_live_detect_limits.npz")
_stored = {}


def ref_outputs(ref, key, compute):
    """compute(ref) -> {name: array} from the live reference (oracle/_ref/libalva_ref.so built in the tree), else the stored
    arrays of `key`; with the reference built, ALVA_RECORD_REF=1 rewrites the stored entries of `key`.  The same rule as
    ref_golden.ref_outputs, over this file's own store."""
    if not _stored and os.path.exists(STORE):
        _stored.update(dict(np.load(STORE)))
    if ref is not None:
        out = {k: np.asarray(v) for k, v in compute(ref).items()}
        if os.environ.get("ALVA_RECORD_REF") == "1":
            for k in [k for k in _stored if k.startswith(key + "/")]:
                del _stored[k]
            _stored.update({f"{key}/{k}": v for k, v in out.items()})
            np.savez_compressed(STORE, **_stored)
        return out
    out = {k[len(key) + 1:]: v for k, v in _stored.items() if k.startswith(key + "/")}
    assert out, f"no stored reference outputs for {key}: build oracle/_ref and record them (ALVA_RECORD_REF=1)"
    return out


def ref_detect(R, img, cs, cur, roi, q0, cap):
    """the reference's FeatureExtractor::detectFeaturePoints (ref_detect_points): its sub-pixel points"""
    R.ref_detect_points.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p,
                                    C.c_int]
    h, w = img.shape
    cur = np.ascontiguousarray(cur, np.float32)
    out = np.zeros((cap, 2), np.float32)
    n = R.ref_detect_points(P(np.ascontiguousarray(img)), w, h, cs, P(cur), len(cur), P(np.ascontiguousarray(roi, np.int32)), q0,
                            P(out), cap)
    assert n <= cap
    return out[:n].copy()


# ---- input scenes of the structural-limit tests (tests/test_oracle_detect_limits.py, tests/test_gpu_detect_limits.py) --------

SWEEP_GEOM = ((0, 2), (1, 3), (2, 0), (3, 1))   # (w, h) = (10, 7) cells + these: every remainder 0..3 in both directions
REF_CELLS = (8, 9, 10, 11, 12, 13, 15, 16, 17, 20, 63, 64)


def texture(w, h, seed, contrast=1.0, mean=128.0):
    """a w x h crop of the synthetic scene texture (wrapped, so any size), optionally with its contrast scaled about `mean`"""
    from alvaar_b200 import synth
    tex = synth.make_texture()
    rng = np.random.default_rng(seed)
    oy, ox = (int(v) for v in rng.integers(0, tex.shape[0], 2))
    t = np.roll(tex, (-oy, -ox), (0, 1))
    img = np.tile(t, ((h + t.shape[0] - 1) // t.shape[0], (w + t.shape[1] - 1) // t.shape[1]))[:h, :w]
    if contrast != 1.0:
        img = np.clip(np.rint(mean + (img.astype(np.float64) - 128.0) * contrast), 0, 255)
    return np.ascontiguousarray(img, np.uint8)


def sweep_cur(w, h, cs, seed):
    """a few hundred current keypoints: most in the left three cell columns (those cells occupied, their discs reaching into
    the free ones), the rest in the last partial cell column / row and the last full cells, where the grid ends"""
    rng = np.random.default_rng(seed)
    a = np.stack([rng.uniform(0, 3 * cs, 160), rng.uniform(0, h - 1, 160)], 1)
    ncw, nch = w // cs, h // cs
    b = np.stack([rng.uniform((ncw - 1) * cs + cs / 2, w - 0.25, 24), rng.uniform(0, h - 1, 24)], 1)
    c = np.stack([rng.uniform(3 * cs, w - 1, 16), rng.uniform((nch - 1) * cs + cs / 2, h - 0.25, 16)], 1)
    return np.concatenate([a, b, c]).astype(np.float32)


def sweep_q(cs):
    """a strict start quality (about half the cells' maxima of the texture reach it; they grow with the cell) and a lenient one"""
    return 0.0025 + 5e-5 * cs, 0.0003


def sweep_case(cs, g):
    """case g (0..3) of cell size cs: frames (no keypoints, keypoints) x the two start qualities, roi 2 px inside the frame"""
    dw, dh = SWEEP_GEOM[g]
    w, h = 10 * cs + dw, 7 * cs + dh
    imgs = np.stack([texture(w, h, 1000 * cs + 10 * g + k) for k in range(4)])
    cur = sweep_cur(w, h, cs, 7 * cs + g)
    none = np.zeros((0, 2), np.float32)
    qs = sweep_q(cs)
    return imgs, [none, cur, none, cur], [qs[0], qs[0], qs[1], qs[1]], [2, 2, w - 4, h - 4]


def edge_cur(w, h, cs):
    """current keypoints at the edges of the occupancy / disc arithmetic: half-integer centres (cvRound's ties to even),
    coordinates on cell boundaries and one float ulp either side, coordinates in (-cell, 0) (truncation of the cell index
    to 0), and coordinates in [size - 0.5, size)"""
    up, dn = (lambda v: np.nextafter(np.float32(v), np.float32(np.inf))), (lambda v: np.nextafter(np.float32(v), np.float32(-np.inf)))
    p = [(2.5 * cs + 0.5, 1.5 * cs + 0.5), (3 * cs + 1.5, 4.5), (10.5, 3 * cs + 11.5), (5 * cs + 2.5, 2 * cs - 0.5)]
    for k, (x, y) in enumerate([(2 * cs, 3 * cs), (4 * cs, cs), (cs, 4 * cs)]):
        p += [(x, y + 5), (up(x), y + 7 + k), (dn(x), y + 9), (x + 6, y), (x + 3, up(y)), (x + 9, dn(y))]
    p += [(-0.5, 2.3 * cs), (-0.49, 3.3 * cs), (-1.5, 1.2 * cs), (-cs + 0.25, 4.6 * cs), (dn(0.0), 3.9 * cs),
          (4.4 * cs, -0.5), (2.2 * cs, -cs + 0.5), (1.1 * cs, -3.25), (-2.5, -1.5),
          (w - 0.5, 2.5 * cs), (dn(w), 1.3 * cs), (w - 0.25, 3.1 * cs), (2.7 * cs, h - 0.5), (3.6 * cs, dn(h)), (dn(w), dn(h))]
    return np.array(p, np.float32)


def square(img, x, y, v, n=3):
    img[y:y + n, x:x + n] = v


def rescan_scene(cs):
    """a low-contrast texture with strong isolated squares planted near cell borders in W, N, NW and NE arrangements: the
    neighbour's square is the stronger, so its detection's disc covers the pre-computed maximum of the cell that follows it
    in the serial order (re-scan: covered, then primary differs), plus a flat 2 x 2 block of cells (maximum 0: re-scan)"""
    ncw, nch = 12, 9
    w, h = ncw * cs + 3, nch * cs + 3
    img = texture(w, h, 77 + cs, contrast=0.12, mean=110.0)
    img[5 * cs - 2:7 * cs + 2, 8 * cs - 2:10 * cs + 2] = 110   # flat with the pixel ring the cells' blur reads

    def pair(rs, cs_, rt, ct, dx, dy):
        # strong square in cell (rs, cs_) against the border towards (rt, ct), weaker one in (rt, ct) just across it: centres
        # 4 px apart in each direction the pair spans
        xs, ys = cs_ * cs + cs // 2 - 1, rs * cs + cs // 2 - 1
        xt, yt = ct * cs + cs // 2 - 1, rt * cs + cs // 2 - 1
        if dx > 0: xs, xt = (cs_ + 1) * cs - 3, ct * cs + 1
        if dx < 0: xs, xt = cs_ * cs + 1, (ct + 1) * cs - 3
        if dy > 0: ys, yt = (rs + 1) * cs - 3, rt * cs + 1
        square(img, xs, ys, 250)
        square(img, xt, yt, 200)

    for r, c in ((1, 2), (4, 5), (7, 9)):
        pair(r, c - 1, r, c, 1, 0)            # W
        pair(r - 1, c + 1, r, c + 1, 0, 1)    # N
    for r, c in ((2, 6), (6, 2), (7, 6)):
        pair(r - 1, c - 1, r, c, 1, 1)        # NW
    for r, c in ((2, 9), (5, 2), (8, 4)):
        pair(r - 1, c + 1, r, c, -1, 1)       # NE
    return img, [2, 2, w - 4, h - 4]


def tie_scenes(cs):
    """exact ties of the cell maximum: a checkerboard and a lattice of identical blobs, both with a period dividing the cell
    (every cell is the same and each holds many equal maxima), with current keypoints whose discs cover the first ties"""
    w, h = 8 * cs + 2, 6 * cs + 2
    yy, xx = np.mgrid[0:h, 0:w]
    per = 4 if cs % 4 == 0 else cs
    board = np.where(((xx // (per // 2)) + (yy // (per // 2))) % 2 == 0, 90, 160).astype(np.uint8)
    blobs = np.full((h, w), 100, np.uint8)
    pb = 8 if cs % 8 == 0 else cs
    m = ((xx % pb) < 2) & ((yy % pb) < 2)
    blobs[m] = 220
    cur = np.array([[c * cs + 1.0, r * cs + 1.0] for r in range(1, 5) for c in range(1, 7, 2)] +
                   [[c * cs - 2.0, r * cs + 3.0] for r in range(2, 5, 2) for c in range(2, 8, 3)], np.float32)
    return [np.ascontiguousarray(board), np.ascontiguousarray(blobs)], cur, [0, 0, w, h]


def dot_frame(cs, ncw, nch, dots, occupied):
    """a flat frame of ncw x nch full cells (+ 2 px) with an isolated bright dot at the centre of the cells `dots` and a current
    keypoint at the centre of the cells `occupied` (lists of cell indices)"""
    w, h = ncw * cs + 2, nch * cs + 2
    img = np.full((h, w), 60, np.uint8)
    for i in dots:
        r, c = divmod(i, ncw)
        square(img, c * cs + cs // 2 - 1, r * cs + cs // 2 - 1, 230, 2)
    cur = np.array([[(i % ncw) * cs + cs / 2 + 0.25, (i // ncw) * cs + cs / 2 + 0.25] for i in occupied], np.float32).reshape(-1, 2)
    return img, cur, [0, 0, w, h]


def subpix_scene(w, h, seed):
    """points for cv::cornerSubPix alone on a textured frame with a flat band: on both sides of the interior / border switch of
    the 9 x 9 sampler (ipx = 0, ipx + 9 = w and the same in y), at the frame's edge, on the flat band (det ~ 0) and on the
    texture (some converge, some run more than 3 px away or out of the frame and are reverted / stopped)"""
    img = texture(w, h, seed)
    img[:, w // 2:w // 2 + 40] = 97
    def up(v):
        return float(np.nextafter(np.float32(v), np.float32(np.inf)))

    def dn(v):
        return float(np.nextafter(np.float32(v), np.float32(-np.inf)))
    rng = np.random.default_rng(seed)
    ys = rng.uniform(12, h - 12, 64)
    xs = rng.uniform(12, w // 2 - 12, 64)
    p = []
    for k in range(16):
        for x in (4.0, dn(4.0), up(4.0), w - 5.0, dn(w - 5.0), up(w - 5.0), 0.0, 0.4, w - 1.0, w - 1.3):
            p.append((x, ys[k]))
        for y in (4.0, dn(4.0), up(4.0), h - 5.0, dn(h - 5.0), up(h - 5.0), 0.0, 0.6, h - 1.0, h - 1.2):
            p.append((xs[k], y))
    p += [(w // 2 + 20.0 + rng.uniform(-5, 5), y) for y in ys[:32]]
    p += list(zip(rng.uniform(0, w - 1, 200), rng.uniform(0, h - 1, 200)))
    return img, np.array(p, np.float32)
