"""Input scenes of the feature-selection structural-limit tests (tests/test_gpu_feature_limits.py runs them through the front end,
retainBest, Harris and the pipeline; tests/test_oracle_feature_limits.py checks the oracle against the reference on them), the
oracle's FAST / retainBest / ORB-detect behind plain calls, and the store of the reference's outputs on these scenes
(tests/golden/ref_live_feature_limits.npz)."""
import ctypes as C
import os

import numpy as np

from conftest import P
from detect_limits_util import texture

STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_live_feature_limits.npz")
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


def nms_bound(w, h):
    """FAST's 3x3 non-maximum suppression is strict, so no two corners are neighbours: at most one per 2 x 2 block"""
    return ((w + 1) // 2) * ((h + 1) // 2)


# ---- the oracle ---------------------------------------------------------------------------------------------------------------

def oracle_fast(oracle, img, thr):
    """orc_fast9 with NMS: (n, 3) int32 (x, y, score), row-major"""
    h, w = img.shape
    out = np.zeros((nms_bound(w, h) + 16, 3), np.int32)
    n = oracle.orc_fast9(P(np.ascontiguousarray(img)), w, h, thr, 1, P(out), len(out))
    assert n <= len(out)
    return out[:n].copy()


def pack(xys):
    """(n, 3) (x, y, score) -> packed uint32 keys (y << 20 | x << 8 | score)"""
    a = np.asarray(xys, np.int64).reshape(-1, 3)
    return ((a[:, 1] << 20) | (a[:, 0] << 8) | a[:, 2]).astype(np.uint32)


def oracle_retain_best(oracle, xys, w, h, n, edge):
    """KeyPointsFilter::retainBest(n) after the border filter, in the input's (row-major) order: every key scoring at least the
    n-th best score"""
    xys = np.asarray(xys, np.int32).reshape(-1, 3)
    if edge > 0:
        x, y = xys[:, 0], xys[:, 1]
        xys = xys[(x >= edge) & (x < w - edge) & (y >= edge) & (y < h - edge)]
    xys = np.ascontiguousarray(xys)
    thr = oracle.orc_retain_best_threshold(P(xys), len(xys), n)
    return xys[xys[:, 2] >= thr]


def oracle_orb_detect(oracle, img, nfeatures, thr):
    """ORB::detectAndCompute (nlevels 1, HARRIS_SCORE) composed from the oracle's stages exactly as orc_orb_detect composes
    them -- FAST -> border 31 -> retainBest(2n) on the FAST score -> Harris -> retainBest(n) on the response -> IC angle ->
    blur -> rBRIEF -- with FAST's list sized by the NMS bound (orc_orb_detect keeps w * h / 8 corners, fewer than a dense frame
    has).  The full keypoint list (row-major) {x, y, Harris response, angle} and descriptors."""
    h, w = img.shape
    img = np.ascontiguousarray(img)
    xys = oracle_fast(oracle, img, thr)
    if h <= 62 or w <= 62:
        xys = xys[:0]
    xys = oracle_retain_best(oracle, xys, w, h, 2 * nfeatures, 31)
    pts = np.ascontiguousarray(xys[:, :2].astype(np.float32))
    resp = oracle_harris(oracle, img, pts)
    if len(resp) > nfeatures:   # every response >= the n-th largest (qsort's threshold in orc_orb_detect)
        keep = resp >= np.sort(resp)[::-1][nfeatures - 1]
        pts, resp = np.ascontiguousarray(pts[keep]), resp[keep]
    n = len(pts)
    ang = np.zeros(n, np.float32)
    oracle.orc_ic_angles(P(img), w, h, P(pts), n, P(ang))
    blur = np.empty_like(img)
    oracle.orc_orb_blur(P(img), w, h, 0, P(blur))
    d, kept = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
    oracle.orc_orb_describe(P(blur), w, h, P(pts), P(ang), n, P(d), P(kept))
    return np.ascontiguousarray(np.column_stack([pts, resp, ang]).astype(np.float32)), d


def oracle_harris(oracle, img, pts):
    h, w = img.shape
    pts = np.ascontiguousarray(pts, np.float32)
    r = np.zeros(len(pts), np.float32)
    oracle.orc_harris(P(np.ascontiguousarray(img)), w, h, P(pts), len(pts), P(r))
    return r


# ---- scenes ---------------------------------------------------------------------------------------------------------------------

def dense_dots(w, h, phase=0):
    """single bright pixels on black, every other pixel of every other row, the rows alternately shifted by one: nearly every dot
    is a corner (over 90 % of the NMS bound), so each tile's keypoint list comes close to its structural limit"""
    img = np.zeros((h, w), np.uint8)
    for y in range(phase % 2, h, 2):
        img[y, ((y // 2) + phase // 2) % 2::2] = 255
    return img


def tie_dots(w, h, period=4, x0=0, y0=0):
    """identical isolated dots on a period x period lattice: every dot is a corner of the same FAST score, and (away from the
    frame's edge) of the same Harris response"""
    img = np.full((h, w), 40, np.uint8)
    img[y0::period, x0::period] = 230
    return img


def edge_dots(w, h, seed):
    """vertical bright bands with dots on their dark side 3 or 4 px from the band's edge: FAST fires at the dots, and the
    7 x 7 Harris window there is dominated by the straight edge, so their responses are negative (and varied: the dots'
    brightness and distance vary).  Every fourth dot is bright and 5 px away, with a positive response."""
    rng = np.random.default_rng(seed)
    img = np.zeros((h, w), np.uint8)
    for x0 in range(0, w - 23, 24):
        img[:, x0 + 12:x0 + 24] = 200
    k = 0
    for y in range(6, h - 6, 6):
        for x0 in range(0, w - 23, 24):
            if k % 4 == 3:
                img[y, x0 + 7] = 255
            else:
                img[y, x0 + 12 - int(rng.integers(3, 5))] = int(rng.integers(100, 141))
            k += 1
    return img


def noise(w, h, seed):
    """uniform noise: about 40 % of the NMS bound are corners, with every FAST score"""
    return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)


def scene(kind, w, h, seed=0):
    if kind == "texture":
        return texture(w, h, seed)
    if kind == "dense":
        return dense_dots(w, h, seed)
    if kind == "ties":
        return tie_dots(w, h, 4, seed % 4, (seed // 4) % 4)
    if kind == "edges":
        return edge_dots(w, h, seed)
    if kind == "noise":
        return noise(w, h, seed)
    raise ValueError(kind)


def to_rgba(gray, seed=0):
    """an RGBA frame whose gray conversion is not simply one channel (the front end's cvtColor is checked too)"""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(np.stack([gray, np.roll(gray, 1, -1), rng.integers(0, 256, gray.shape, dtype=np.uint8),
                                          np.full_like(gray, 255)], -1))


def random_keys(n, w, h, seed, score_hi=256):
    """n distinct corner positions (in a w x h frame) with random scores, in a random order -- a front end's raw list"""
    rng = np.random.default_rng(seed)
    flat = rng.choice(w * h, n, replace=False)
    return np.stack([flat % w, flat // w, rng.integers(0, score_hi, n)], 1).astype(np.int32)


# ---- the reference ------------------------------------------------------------------------------------------------------------

def ref_fast(R, img, thr):
    h, w = img.shape
    out = np.zeros((nms_bound(w, h) + 16, 3), np.int32)
    n = R.ref_fast(P(np.ascontiguousarray(img)), w, h, thr, 1, P(out), len(out))
    return out[:n].copy()


def ref_orb_detect(R, img, nfeatures, thr):
    """ORB::detectAndCompute (nlevels 1, HARRIS_SCORE): {x, y, response, angle} and descriptors, sorted row-major (the
    reference's own order is whatever nth_element leaves)"""
    h, w = img.shape
    cap = nms_bound(w, h)
    kp, d = np.zeros((cap, 5), np.float32), np.zeros((cap, 32), np.uint8)
    R.ref_orb_detect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    n = R.ref_orb_detect(P(np.ascontiguousarray(img)), w, h, nfeatures, thr, P(kp), P(d), cap)
    assert n <= cap
    kp, d = kp[:n, :4], d[:n]
    o = np.lexsort((kp[:, 0], kp[:, 1]))
    return np.ascontiguousarray(kp[o]), np.ascontiguousarray(d[o])
