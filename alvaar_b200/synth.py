"""Seeded synthetic inputs shared by the oracle, the GPU tests and bench.py (SURVEY.md section 8d).

* texture : 3 octaves of uniform noise, Gaussian-blurred (sigma 1.5 / 3 / 6, weights proportional to sigma),
            contrast-normalised to mean 128 / std 60 and clipped -- about 15 k FAST-9 (thr 20, NMS) corners per
            1280x720 view, so 1000 features/frame is always reachable.
* frames  : a pinhole camera on a smooth seeded SE(3) trajectory (about 3 px/frame lateral motion, +-0.2 deg/frame
            rotation) looking at the texture plane z = 4; bilinear sampling; RGBA with R = G = B, A = 255.  Optionally
            through OpenCV's radial-tangential lens (k1, k2, p1, p2).
* descriptors / BA problems for the matcher and bundle-adjustment stages.
Pure numpy (+ scipy.ndimage for the blur); nothing here is on the product path.
"""
import numpy as np

_TEX_CACHE = {}


def make_texture(size=2048, seed=1234):
    key = (size, seed)
    if key not in _TEX_CACHE:
        from scipy.ndimage import gaussian_filter
        rng = np.random.default_rng(seed)
        acc = np.zeros((size, size), np.float32)
        for sigma in (1.5, 3.0, 6.0):
            n = rng.random((size, size), dtype=np.float32)
            b = gaussian_filter(n, sigma, mode="wrap")
            b = (b - b.mean()) / b.std()
            acc += sigma * b
        acc = (acc - acc.mean()) / acc.std() * 60.0 + 128.0
        _TEX_CACHE[key] = np.clip(np.rint(acc), 0, 255).astype(np.uint8)
    return _TEX_CACHE[key]


def intrinsics(w, h):
    """AlvaAR's JS shim: f = min(w/2 / tan(fovH/2), h/2 / tan(fovV/2)), fovV = 45 deg, fovH = 45 deg * aspect
    (reference: src/system.js:101-123)."""
    fov_v = np.deg2rad(45.0)
    fov_h = fov_v * (w / h)
    f = min(w / 2 / np.tan(fov_h / 2), h / 2 / np.tan(fov_v / 2))
    return float(f), float(f), w / 2.0, h / 2.0


def _rot(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def trajectory(nframes, w, h, seed=99, plane_z=4.0):
    """Camera-to-world poses (R_wc, t_wc): smooth random walk, ~3 px/frame lateral, +-0.2 deg/frame."""
    rng = np.random.default_rng(seed)
    fx = intrinsics(w, h)[0]
    step = 3.0 * plane_z / fx
    poses = []
    ang = np.zeros(3)
    pos = np.zeros(3)
    dirn = rng.uniform(0, 2 * np.pi)
    for k in range(nframes):
        poses.append((_rot(*ang), pos.copy()))
        dirn += rng.normal(0, 0.05)
        pos = pos + np.array([np.cos(dirn) * step, np.sin(dirn) * step, rng.normal(0, 0.002)])
        ang = np.clip(ang + np.deg2rad(rng.uniform(-0.2, 0.2, 3)), -0.15, 0.15)
    return poses


def undistort_normalised(xd, yd, dist, tol=1e-12, max_iter=500):
    """The normalised point (x, y) that OpenCV's radial-tangential model (k1, k2, p1, p2) maps to (xd, yd): fixed-point
    iteration run to convergence (scene generation, not the reference's 5-iteration cv::undistortPoints)."""
    k1, k2, p1, p2 = dist
    x, y = xd.copy(), yd.copy()
    for _ in range(max_iter):
        r2 = x * x + y * y
        radial = 1 + k1 * r2 + k2 * r2 * r2
        nx = (xd - (2 * p1 * x * y + p2 * (r2 + 2 * x * x))) / radial
        ny = (yd - (p1 * (r2 + 2 * y * y) + 2 * p2 * x * y)) / radial
        done = max(np.abs(nx - x).max(), np.abs(ny - y).max()) < tol
        x, y = nx, ny
        if done:
            return x, y
    raise ValueError(f"lens model {dist} does not invert over this image")


def render_gray(tex, pose, w, h, plane_z=4.0, tex_scale=None, dist=None):
    """Bilinear render of the texture plane z = plane_z seen from pose (R_wc, t_wc); dist = (k1, k2, p1, p2): through that lens."""
    fx, fy, cx, cy = intrinsics(w, h)
    if tex_scale is None:
        tex_scale = fx / plane_z          # texture pixels per world unit: ~1 texel per image pixel
    R, t = pose
    u, v = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    if dist is None:
        rays = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], -1) @ R.T
    else:
        x, y = undistort_normalised((u - cx) / fx, (v - cy) / fy, dist)
        rays = np.stack([x, y, np.ones_like(u)], -1) @ R.T
    s = (plane_z - t[2]) / rays[..., 2]
    X = t[0] + s * rays[..., 0]
    Y = t[1] + s * rays[..., 1]
    S = tex.shape[0]
    tu = (X * tex_scale + S / 2.0) % S
    tv = (Y * tex_scale + S / 2.0) % S
    x0 = np.floor(tu).astype(np.int64)
    y0 = np.floor(tv).astype(np.int64)
    ax = (tu - x0).astype(np.float32)
    ay = (tv - y0).astype(np.float32)
    x1 = (x0 + 1) % S
    y1 = (y0 + 1) % S
    T = tex.astype(np.float32)
    val = (T[y0, x0] * (1 - ax) * (1 - ay) + T[y0, x1] * ax * (1 - ay) + T[y1, x0] * (1 - ax) * ay + T[y1, x1] * ax * ay)
    return np.clip(np.rint(val), 0, 255).astype(np.uint8)


def gray_to_rgba(g):
    out = np.empty(g.shape + (4,), np.uint8)
    out[..., 0] = g
    out[..., 1] = g
    out[..., 2] = g
    out[..., 3] = 255
    return out


def make_frames(nframes, w, h, seed=99, rgba=True, texture_seed=1234, dist=None):
    """`seed` picks the camera path, `texture_seed` the scene (two calls with the same texture_seed look at the same plane);
    dist = (k1, k2, p1, p2) renders through OpenCV's radial-tangential lens with the intrinsics() camera (None: a pinhole)."""
    tex = make_texture(seed=texture_seed)
    poses = trajectory(nframes, w, h, seed)
    frames = [render_gray(tex, p, w, h, dist=dist) for p in poses]
    g = np.stack(frames)
    return (gray_to_rgba(g) if rgba else g), poses


def crop(w, h, ox=300, oy=200):
    """A plain crop of the texture (cheap test input with the same statistics)."""
    return np.ascontiguousarray(make_texture()[oy:oy + h, ox:ox + w])


def random_rgba(w, h, n=1, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 4), dtype=np.uint8)


def make_descriptors(nq=1000, nt=10000, seed=7, planted=0.3, flip=0.08):
    """Random 256-bit strings with `planted` fraction of true matches at Hamming ~ Binomial(256, flip)."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    npl = int(nq * planted)
    idx = rng.choice(nt, npl, replace=False)
    noise = np.packbits(rng.random((npl, 256)) < flip, axis=1)
    q[:npl] = t[idx] ^ noise
    return q, t


def _quat_from_R(R):
    """(x, y, z, w) unit quaternion of a rotation matrix."""
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = [(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s]
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k]) * 2
        q = [0, 0, 0, 0]
        q[i] = 0.25 * s
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
        q[3] = (R[k, j] - R[j, k]) / s
    q = np.array(q)
    return q / np.linalg.norm(q)


def make_ba_problem(nkf=20, nlm=3000, obs_per_lm=4, seed=42, w=1280, h=720, noise_px=0.5, outlier_frac=0.05,
                    outlier_px=20.0, pose_noise_t=0.01, pose_noise_r_deg=0.2, nconst=2):
    """Local-BA problem in the reference's parametrisation (SURVEY 8d, config C4): nkf cameras on a circle arc looking
    at a point cloud (depth 2-8 m), every landmark observed by `obs_per_lm` of its 6 nearest cameras; the first
    observer is the ANCHOR (inverse depth, no residual) -> nlm*(obs_per_lm-1) residuals; pixel noise, 5 % gross
    outliers, perturbed initial poses, the `nconst` oldest keyframes fixed.
    Returns a dict of flat arrays in the layout of include/alva_b200.h (poses = [t, q(x,y,z,w)] camera-to-world)."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = intrinsics(w, h)
    # cameras on an arc, looking along +z with a slight toe-in
    poses_gt = []
    for k in range(nkf):
        a = (k - (nkf - 1) / 2) * 0.03
        t = np.array([3.0 * np.sin(a) + 0.08 * k, 0.02 * np.sin(0.7 * k), 0.3 * (1 - np.cos(a))])
        R = _rot(0.01 * np.sin(k), -a * 0.8, 0.005 * k)
        poses_gt.append((R, t))
    # landmarks: sample a pixel + depth in a random camera, keep if visible in >= obs_per_lm cameras
    pts, obs_list = [], []
    while len(pts) < nlm:
        k0 = rng.integers(0, nkf)
        u, v, z = rng.uniform(40, w - 40), rng.uniform(40, h - 40), rng.uniform(2.0, 8.0)
        R, t = poses_gt[k0]
        X = R @ np.array([(u - cx) / fx * z, (v - cy) / fy * z, z]) + t
        vis = []
        for k, (Rk, tk) in enumerate(poses_gt):
            pc = Rk.T @ (X - tk)
            if pc[2] > 0.5:
                uu, vv = fx * pc[0] / pc[2] + cx, fy * pc[1] / pc[2] + cy
                if 20 <= uu < w - 20 and 20 <= vv < h - 20:
                    vis.append((abs(k - k0), k, uu, vv))
        if len(vis) < obs_per_lm:
            continue
        vis.sort()
        near = vis[:6]
        sel = sorted(rng.choice(len(near), obs_per_lm, replace=False))
        chosen = sorted([near[i] for i in sel], key=lambda e: e[1])
        pts.append(X)
        obs_list.append([(k, uu, vv) for _, k, uu, vv in chosen])
    # perturbed initial poses
    poses = np.zeros((nkf, 7))
    for k, (R, t) in enumerate(poses_gt):
        if k >= nconst:
            dr = np.deg2rad(rng.normal(0, pose_noise_r_deg, 3))
            R = _rot(*dr) @ R
            t = t + rng.normal(0, pose_noise_t, 3)
        poses[k, :3] = t
        poses[k, 3:] = _quat_from_R(R)
    pose_const = np.zeros(nkf, np.uint8)
    pose_const[:nconst] = 1
    anch_kf = np.zeros(nlm, np.int32)
    anch_uv = np.zeros((nlm, 2))
    invd = np.zeros(nlm)
    okf, olm, ouv = [], [], []
    for l, (X, ob) in enumerate(zip(pts, obs_list)):
        ka, ua, va = ob[0]
        anch_kf[l] = ka
        anch_uv[l] = (ua + rng.normal(0, noise_px), va + rng.normal(0, noise_px))
        Ra, ta = poses_gt[ka]
        za = (Ra.T @ (X - ta))[2]
        invd[l] = 1.0 / (za * (1 + rng.normal(0, 0.02)))
        for k, uu, vv in ob[1:]:
            sig = outlier_px if rng.random() < outlier_frac else noise_px
            okf.append(k)
            olm.append(l)
            ouv.append((uu + rng.normal(0, sig), vv + rng.normal(0, sig)))
    return dict(calib=np.array([fx, fy, cx, cy]), poses=poses, pose_const=pose_const, invd=invd, anch_kf=anch_kf,
                anch_uv=np.ascontiguousarray(anch_uv), obs_kf=np.array(okf, np.int32), obs_lm=np.array(olm, np.int32),
                obs_uv=np.ascontiguousarray(np.array(ouv)), huber=float(np.sqrt(5.9915)))


def quat_to_R(q):
    """rotation matrix of a unit quaternion (x, y, z, w)"""
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def make_pose_problem(n=300, seed=0, w=1280, h=720, noise_px=0.5, outlier_frac=0.1, pose_noise=(0.05, 0.02)):
    """n world points seen by a camera T_wc = [t, q(x,y,z,w)]: pixels (noise + gross outliers), unit bearing vectors
    (Frame::computeKeypoint: normalised K^-1 [u v 1]), an initial pose guess perturbed by pose_noise (m, rad)."""
    rng = np.random.default_rng(seed)
    K = np.array(intrinsics(w, h))
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    ang = rng.uniform(0.05, 0.4)
    q = np.concatenate([np.sin(ang / 2) * ax, [np.cos(ang / 2)]])
    t = rng.normal(0, 0.5, 3)
    R = quat_to_R(q)
    uv = np.stack([rng.uniform(30, w - 30, n), rng.uniform(30, h - 30, n)], 1)
    z = rng.uniform(2, 8, n)
    Xc = np.stack([(uv[:, 0] - K[2]) / K[0] * z, (uv[:, 1] - K[3]) / K[1] * z, z], 1)
    X = Xc @ R.T + t
    obs = uv + rng.normal(0, noise_px, uv.shape)
    out = rng.random(n) < outlier_frac
    obs[out] += rng.normal(0, 25, (int(out.sum()), 2))
    bv = np.stack([(obs[:, 0] - K[2]) / K[0], (obs[:, 1] - K[3]) / K[1], np.ones(n)], 1)
    bv /= np.linalg.norm(bv, axis=1, keepdims=True)
    dq_ax = rng.normal(size=3); dq_ax /= np.linalg.norm(dq_ax)
    da = pose_noise[1]
    dq = np.concatenate([np.sin(da / 2) * dq_ax, [np.cos(da / 2)]])
    x1, y1, z1, w1 = dq; x2, y2, z2, w2 = q
    q0 = np.array([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                   w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2])
    pose0 = np.concatenate([t + rng.normal(0, pose_noise[0], 3), q0 / np.linalg.norm(q0)])
    return dict(K=K, pose_true=np.concatenate([t, q]), pose0=pose0, X=np.ascontiguousarray(X), uv=np.ascontiguousarray(obs),
                bv=np.ascontiguousarray(bv), outlier_true=out)


def make_twoview_problem(n=150, seed=0, w=640, h=480, noise_px=0.3, outlier_frac=0.1, baseline=0.4, rot_deg=3.0):
    """n scene points seen by two cameras (camera 1 = the keyframe at the origin, camera 2 at [R12 | t12]): unit bearing
    vectors of both views (Frame::computeKeypoint: normalised K^-1 [u v 1]) with pixel noise and gross outliers -- the
    input of VisualFrontend::checkReadyForInit's 5-point initialisation."""
    rng = np.random.default_rng(seed)
    K = np.array(intrinsics(w, h))
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    ang = np.deg2rad(rot_deg) * rng.uniform(0.3, 1.0)
    q = np.concatenate([np.sin(ang / 2) * ax, [np.cos(ang / 2)]])
    R12 = quat_to_R(q)
    t12 = rng.normal(size=3); t12[2] *= 0.3; t12 *= baseline / np.linalg.norm(t12)
    uv1 = np.stack([rng.uniform(25, w - 25, n), rng.uniform(25, h - 25, n)], 1)
    z = rng.uniform(2, 8, n)
    X1 = np.stack([(uv1[:, 0] - K[2]) / K[0] * z, (uv1[:, 1] - K[3]) / K[1] * z, z], 1)
    X2 = (X1 - t12) @ R12                      # R12^T (X1 - t12)
    uv2 = np.stack([K[0] * X2[:, 0] / X2[:, 2] + K[2], K[1] * X2[:, 1] / X2[:, 2] + K[3]], 1)
    uv1n = uv1 + rng.normal(0, noise_px, uv1.shape)
    uv2n = uv2 + rng.normal(0, noise_px, uv2.shape)
    out = rng.random(n) < outlier_frac
    uv2n[out] += rng.normal(0, 25, (int(out.sum()), 2))

    def bearing(uv):
        b = np.stack([(uv[:, 0] - K[2]) / K[0], (uv[:, 1] - K[3]) / K[1], np.ones(len(uv))], 1)
        return np.ascontiguousarray(b / np.linalg.norm(b, axis=1, keepdims=True))
    return dict(K=K, R12=R12, t12=t12, bv1=bearing(uv1n), bv2=bearing(uv2n), uv1=uv1n, uv2=uv2n, outlier_true=out, X1=X1)

def make_match_problem(seed=0, w=640, h=480, n_kf=6, n_frame_kp=150, n_local=400, dup_frac=0.4, cell=40):
    """A consistent little map for Mapper::matchToMap (mapper.cpp:354-587), in flat arrays:
    keyframes with poses; a current frame observing n_frame_kp map points (its keypoints); n_local further map points of the
    local map that the frame does not observe -- a fraction dup_frac of them are re-detections of frame keypoints (same
    world point up to noise, seen from DISJOINT keyframes, descriptors a few bits apart), the rest are unrelated.
    Poses are T_wc = [t, q(x,y,z,w)]; pixels are projections + noise; descriptors 256-bit."""
    rng = np.random.default_rng(seed)
    K = np.array(intrinsics(w, h))

    def rand_pose(scale):
        ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
        ang = rng.uniform(0, 0.08)
        return np.concatenate([rng.normal(0, scale, 3), np.sin(ang / 2) * ax, [np.cos(ang / 2)]])

    def project(pose, X):
        R = quat_to_R(pose[3:])
        c = (X - pose[:3]) @ R
        return np.stack([K[0] * c[:, 0] / c[:, 2] + K[2], K[1] * c[:, 1] / c[:, 2] + K[3]], 1), c[:, 2]

    kf_T = np.stack([rand_pose(0.15) for _ in range(n_kf)])
    cur_T = rand_pose(0.15)
    # world points seen by the current frame
    uv = np.stack([rng.uniform(10, w - 10, n_frame_kp), rng.uniform(10, h - 10, n_frame_kp)], 1)
    z = rng.uniform(2, 8, n_frame_kp)
    Rc = quat_to_R(cur_T[3:])
    Xc = np.stack([(uv[:, 0] - K[2]) / K[0] * z, (uv[:, 1] - K[3]) / K[1] * z, z], 1)
    Xa = Xc @ Rc.T + cur_T[:3]
    base_desc = rng.integers(0, 256, (n_frame_kp, 32), dtype=np.uint8)

    def flip(d, nbits):
        d = d.copy()
        for b in rng.integers(0, 256, nbits):
            d[b >> 3] ^= np.uint8(1 << (b & 7))
        return d

    mp_id, mp_wpt, mp_is3d, obs_start, obs_kf, obs_px, desc_start, desc_kf, desc = [], [], [], [0], [], [], [0], [], []

    def add_mp(pid, X, kfs, dbase, is3d=True, flips=6):
        mp_id.append(pid); mp_wpt.append(X); mp_is3d.append(1 if is3d else 0)
        for k in kfs:
            p, _ = project(kf_T[k], X[None])
            q = p[0] + rng.normal(0, 0.4, 2)   # keyframe keypoints live on the keyframe's grid: keep them inside the image
            obs_kf.append(k); obs_px.append(np.array([min(max(q[0], 1.0), w - 2.0), min(max(q[1], 1.0), h - 2.0)]))
            desc_kf.append(k); desc.append(flip(dbase, int(rng.integers(0, flips + 1))))
        obs_start.append(len(obs_kf)); desc_start.append(len(desc_kf))

    half = n_kf // 2
    kp_id, kp_px = [], []
    for i in range(n_frame_kp):       # the frame's keypoints: observed in keyframes of the FIRST half
        pid = 1000 + i
        kfs = sorted(rng.choice(half, size=int(rng.integers(1, half + 1)), replace=False).tolist())
        add_mp(pid, Xa[i], kfs, base_desc[i], is3d=bool(rng.random() < 0.8))
        kp_id.append(pid); kp_px.append(uv[i] + rng.normal(0, 0.3, 2))
    local_ids = []
    for j in range(n_local):          # local map points not observed by the frame
        pid = 5000 + j
        if rng.random() < dup_frac:   # a re-detection of frame keypoint i, seen from the SECOND half (disjoint keyframe sets)
            i = int(rng.integers(0, n_frame_kp))
            X = Xa[i] + rng.normal(0, 0.002, 3)
            kfs = sorted((half + rng.choice(n_kf - half, size=int(rng.integers(1, n_kf - half + 1)), replace=False)).tolist())
            if rng.random() < 0.15:   # some share a keyframe with the keypoint's map point: not a candidate
                kfs = sorted(set(kfs) | {0})
            add_mp(pid, X, kfs, base_desc[i], is3d=bool(rng.random() < 0.9), flips=10)
        else:
            u = np.array([rng.uniform(-50, w + 50), rng.uniform(-50, h + 50)]); zz = rng.uniform(-1, 8)
            X = np.array([(u[0] - K[2]) / K[0] * zz, (u[1] - K[3]) / K[1] * zz, zz]) @ Rc.T + cur_T[:3]
            kfs = sorted(rng.choice(n_kf, size=int(rng.integers(1, 4)), replace=False).tolist())
            add_mp(pid, X, kfs, rng.integers(0, 256, 32, dtype=np.uint8), is3d=bool(rng.random() < 0.9))
        local_ids.append(pid)
    local_ids += kp_id[:10]           # a few ids the frame already observes: skipped (mapper.cpp:404-407)
    f32, i32 = np.float32, np.int32
    return dict(w=w, h=h, K=K, cell=cell, cur_T=cur_T, kp_id=np.array(kp_id, i32), kp_px=np.array(kp_px, f32),
                kf_id=np.arange(n_kf, dtype=i32) + 3, kf_T=np.ascontiguousarray(kf_T), mp_id=np.array(mp_id, i32),
                mp_wpt=np.ascontiguousarray(np.array(mp_wpt)), mp_is3d=np.array(mp_is3d, np.uint8),
                obs_start=np.array(obs_start, i32), obs_kf=np.array(obs_kf, i32), obs_px=np.array(obs_px, f32),
                desc_start=np.array(desc_start, i32), desc_kf=np.array(desc_kf, i32), desc=np.ascontiguousarray(np.array(desc, np.uint8)),
                local_ids=np.array(local_ids, i32))
