"""Host model of the cross-stream loop-closure detector (alva_lc_*, csrc/loopclosure.cu), written from its contract
(include/alva_b200.h, DESIGN.md §5) rather than from the kernels: the keyframe-block wire format, the Hamming 2-NN of every live
local descriptor among the live remote ones (the oracle's orc_knn2: ties keep the lowest index), the ratio test and the absolute
gate, ordered compaction of the survivors in local-index order truncated to ALVA_LC_PAIR_CAP, float64 bearing vectors with each
block's own intrinsics, the relative match gate, the five-point RANSAC on the step's newest keyframe (the oracle's
orc_essential_5pt, one round of 32 hypotheses, no refinement) and the temporal rule of alva_lc_poll.  Plus a two-view scene that
plants a chosen number of true matches in a remote keyframe."""
import numpy as np

from conftest import P
from init_util import orc_essential

MAGIC, VERSION, HDR, PAIR_CAP = 0x464B4C41, 1, 64, 512
DEFAULTS = dict(min_matches=30, max_dist=64, ratio_num=4, ratio_den=5, min_consecutive=3, min_inliers=20, err_px=3.0, fx_hint=500.0,
                fy_hint=500.0)


def block_bytes(n_max):
    return HDR + 40 * n_max


def config(n_max, K, world, rank, **kw):
    """the configuration alva_lc_create works with: a field <= 0 (or left out) takes its documented default; the ratio is replaced
    as a whole when either of its two terms is <= 0"""
    c = dict(n_max=n_max, K=K, world=world, rank=rank)
    for k, v in DEFAULTS.items():
        c[k] = kw[k] if kw.get(k, 0) > 0 else v
    if kw.get("ratio_num", 0) <= 0 or kw.get("ratio_den", 0) <= 0:
        c["ratio_num"], c["ratio_den"] = DEFAULTS["ratio_num"], DEFAULTS["ratio_den"]
    return c


def header(stream, seq, count, n_max, K4, magic=MAGIC, version=VERSION):
    h = np.zeros(16, np.int32)
    h[:6] = magic, version, stream, seq, count, n_max
    h.view(np.float32)[6:10] = np.asarray(K4, np.float32)
    return h.view(np.uint8)


def make_block(n_max, px, desc, K4, stream, seq, count=None, magic=MAGIC, version=VERSION):
    """one keyframe block built on the host: len(px) live entries, zero past them; `count` overrides the header's count"""
    n = len(px)
    b = np.zeros(block_bytes(n_max), np.uint8)
    b[:HDR] = header(stream, seq, n if count is None else count, n_max, K4, magic, version)
    b[HDR:HDR + 8 * n_max].view(np.float32).reshape(n_max, 2)[:n] = px
    b[HDR + 8 * n_max:].reshape(n_max, 32)[:n] = desc
    return b


def pack_model(desc, pts, counts, cap, kf_frames, seq0, K4, n_max, rank):
    """alva_lc_pack: frames kf_frames[e] of desc [nframes][cap][32] / pts [nframes][cap][2] -> the bytes of len(kf_frames) blocks;
    the live count is min(counts[f], cap, n_max), never below 0"""
    out = []
    for e, f in enumerate(kf_frames):
        n = int(np.clip(min(int(counts[f]), cap), 0, n_max))
        out.append(make_block(n_max, pts[f, :n], desc[f, :n], K4, rank, seq0 + e))
    return np.concatenate(out)


def parse(blk, n_max):
    h = blk[:HDR].view(np.int32)
    return dict(magic=int(h[0]), version=int(h[1]), seq=int(h[3]), live=int(np.clip(h[4], 0, n_max)),
                K4=blk[:HDR].view(np.float32)[6:10].astype(np.float64),
                px=blk[HDR:HDR + 8 * n_max].view(np.float32).reshape(n_max, 2),
                desc=np.ascontiguousarray(blk[HDR + 8 * n_max:].reshape(n_max, 32)))


def bearings(px, K4):
    """unit bearing vectors of float32 pixels in float64 with the block's float32 intrinsics {fx, fy, cx, cy}"""
    x = (px[:, 0].astype(np.float64) - K4[2]) / K4[0]
    y = (px[:, 1].astype(np.float64) - K4[3]) / K4[1]
    n = np.sqrt(x * x + y * y + 1.0)
    return np.stack([x / n, y / n, 1.0 / n], 1)


def detect_model(oracle, gathered, cfg):
    """every keyframe pair (e, r) of one alva_lc_detect on the gathered [world][K] blocks.  Arrays [K][world]: nmatch, npair,
    verdict (0 too few matches or check failed / 1 check passed / 2 enough matches, not the newest keyframe), inliers, remote_kf;
    lists [K][world]: nn (2-NN rows of the live local descriptors), bvl / bvr (bearings of the first min(nmatch, PAIR_CAP)
    putative matches), Rt (3x4 RANSAC model where the verdict is 1)"""
    n_max, K, world, rank = cfg["n_max"], cfg["K"], cfg["world"], cfg["rank"]
    bb = block_bytes(n_max)
    z = lambda dt: np.zeros((K, world), dt)  # noqa: E731
    m = dict(nmatch=z(np.int64), npair=z(np.int64), verdict=z(np.int64), inliers=z(np.int64), remote_kf=z(np.int64),
             nn=[[None] * world for _ in range(K)], bvl=[[None] * world for _ in range(K)], bvr=[[None] * world for _ in range(K)],
             Rt=[[None] * world for _ in range(K)])
    for e in range(K):
        loc = parse(gathered[(rank * K + e) * bb:(rank * K + e + 1) * bb], n_max)
        for r in range(world):
            rem = parse(gathered[(r * K + e) * bb:(r * K + e + 1) * bb], n_max)
            m["remote_kf"][e, r] = rem["seq"]
            if r == rank:
                continue
            nq, nt = loc["live"], rem["live"]
            nn = np.full((nq, 4), -1, np.int32)
            if nq:
                oracle.orc_knn2(P(np.ascontiguousarray(loc["desc"][:nq])), nq, P(np.ascontiguousarray(rem["desc"][:nt])), nt, P(nn))
            m["nn"][e][r] = nn
            valid = all(b["magic"] == MAGIC and b["version"] == VERSION for b in (loc, rem))
            if not valid:
                continue
            keep = (nn[:, 0] >= 0) & (nn[:, 1] <= cfg["max_dist"]) & \
                   ((nn[:, 2] < 0) | (nn[:, 1].astype(np.int64) * cfg["ratio_den"] < nn[:, 3].astype(np.int64) * cfg["ratio_num"]))
            qi = np.nonzero(keep)[0]
            n = len(qi)
            m["nmatch"][e, r] = n
            qi = qi[:PAIR_CAP]
            m["bvl"][e][r] = bearings(loc["px"][qi], loc["K4"])
            m["bvr"][e][r] = bearings(rem["px"][nn[qi, 0]], rem["K4"])
            enough = n >= max(cfg["min_matches"], nq // 8)
            if e < K - 1:
                m["verdict"][e, r] = 2 if enough else 0
            elif enough:
                m["npair"][e, r] = len(qi)
                ok, Rt, _, info = orc_essential(oracle, m["bvl"][e][r], m["bvr"][e][r], (cfg["fx_hint"], cfg["fy_hint"]), 0,
                                                seed=12345, max_iter=32, err=cfg["err_px"])
                m["verdict"][e, r] = ok
                m["inliers"][e, r] = int(info[0])
                if ok:
                    m["Rt"][e][r] = Rt.reshape(3, 4)
    return m


def poll_model(steps, cfg):
    """alva_lc_poll's temporal rule over [(local_seq0, detect_model result), ...] in step order -> the events"""
    consecutive = [0] * cfg["world"]
    events = []
    K = cfg["K"]
    for seq0, m in steps:
        for e in range(K):
            for r in range(cfg["world"]):
                if r == cfg["rank"]:
                    continue
                checked = e == K - 1
                ok = (m["verdict"][e, r] == 1 and m["inliers"][e, r] >= cfg["min_inliers"]) if checked else m["verdict"][e, r] == 2
                consecutive[r] = consecutive[r] + 1 if ok else 0
                if ok and checked and consecutive[r] >= cfg["min_consecutive"]:
                    events.append(dict(local_kf=seq0 + e, remote_rank=r, remote_kf=int(m["remote_kf"][e, r]), n_matches=int(m["nmatch"][e, r]),
                                       n_inliers=int(m["inliers"][e, r]), consecutive=consecutive[r], Rt=m["Rt"][e][r]))
    return events


def random_desc(rng, n):
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


def flip_bits(rng, d, k):
    """d with k distinct bits flipped (Hamming distance exactly k)"""
    out = d.copy()
    for b in rng.choice(256, k, replace=False):
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def local_keyframe(rng, n, K4):
    """n keypoints inside the image of K4 = {fx, fy, cx, cy} (size 2 cx x 2 cy) with random descriptors and depths 2..8"""
    f = np.asarray(K4, np.float64)
    px = np.stack([rng.uniform(10, 2 * f[2] - 10, n), rng.uniform(10, 2 * f[3] - 10, n)], 1).astype(np.float32)
    z = rng.uniform(2, 8, n)
    X = np.stack([(px[:, 0] - f[2]) / f[0] * z, (px[:, 1] - f[3]) / f[1] * z, z], 1)
    return dict(px=px, desc=random_desc(rng, n), X=X)


def remote_view(rng, loc, n_remote, planted, K4r, max_bits=6, noise_px=0.3, shifted=0.0, dups=0, rot_deg=2.0, baseline=0.3):
    """A remote keyframe of n_remote entries of which `planted` are keypoints of the local keyframe `loc` seen from a second
    camera (intrinsics K4r, rotated by up to rot_deg, moved by `baseline`): projected pixels with Gaussian noise, descriptors at
    most max_bits away, at shuffled positions.  A fraction `shifted` of the planted pixels is moved a further 15..40 px: outliers
    of the geometric check, as every true match is an inlier, each by a wide margin.  The device's five-point RANSAC is compiled
    with FMA contraction, so a correspondence within ulps of the threshold could score a hypothesis differently from the oracle
    and change which of two equally scored models is kept.  `dups` of the planted remote descriptors are copied, exactly, to
    unplanted positions.  The other entries are random.  -> (px, desc, (local indices, remote positions) of the planted pairs)"""
    f = np.asarray(K4r, np.float64)
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(rot_deg) * rng.uniform(0.3, 1.0)
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx
    t = rng.normal(size=3)
    t *= baseline / np.linalg.norm(t)
    X2 = (loc["X"] - t) @ R
    uv2 = np.stack([f[0] * X2[:, 0] / X2[:, 2] + f[2], f[1] * X2[:, 1] / X2[:, 2] + f[3]], 1)
    li = rng.choice(len(loc["X"]), planted, replace=False)
    ri = rng.permutation(n_remote)[:planted]
    px = np.stack([rng.uniform(0, 2 * f[2], n_remote), rng.uniform(0, 2 * f[3], n_remote)], 1)
    desc = random_desc(rng, n_remote)
    px[ri] = uv2[li] + rng.normal(0, noise_px, (planted, 2))
    sh = rng.random(planted) < shifted
    ang = rng.uniform(0, 2 * np.pi, int(sh.sum()))
    px[ri[sh]] += rng.uniform(15, 40, len(ang))[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1)
    for i, j in zip(li, ri):
        desc[j] = flip_bits(rng, loc["desc"][i], int(rng.integers(0, max_bits + 1)))
    perm = rng.permutation(n_remote)
    free = perm[~np.isin(perm, ri)][:min(dups, planted)]
    desc[free] = desc[ri[:len(free)]]          # exact duplicates: the 2-NN tie rule, then a failed ratio test
    return px.astype(np.float32), desc, (li, ri)
