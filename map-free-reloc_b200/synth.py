"""Seeded synthetic inputs for the feature-matching + scale-from-depth path (SURVEY.md §8(d)).

Nothing here is pinned by the reference (it ships no data); the shapes and conventions are:
image 3x720x540 float32 in [0,1], depth 720x540 float32 metres quantised to millimetres like
``read_depth_image`` (reference lib/datasets/utils.py:77-81), intrinsics fx=fy=600,
cx=269.5, cy=359.5, pose convention X_1 = R X_0 + t (reference README.md:104-108).
Pure numpy/scipy: used by tests, bench.py and the golden-vector script alike.
"""
import numpy as np

H, W = 720, 540
K_DEFAULT = np.array([[600.0, 0.0, 269.5], [0.0, 600.0, 359.5], [0.0, 0.0, 1.0]], dtype=np.float64)


def rodrigues(rvec):
    """Axis-angle (3,) -> rotation matrix (3,3), float64."""
    rvec = np.asarray(rvec, dtype=np.float64)
    th = np.linalg.norm(rvec)
    if th < 1e-12:
        return np.eye(3)
    k = rvec / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)


def random_pose(rng, max_rot=0.25, max_t=0.5, min_t=0.1):
    rvec = rng.uniform(-max_rot, max_rot, 3)
    while True:
        t = rng.uniform(-max_t, max_t, 3)
        if np.linalg.norm(t) >= min_t:
            break
    return rodrigues(rvec), t


def make_depth(rng, h=H, w=W, invalid_frac=0.02):
    """Smooth depth field in [1,8] m, millimetre-quantised, a fraction of pixels zeroed."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    d = np.full((h, w), 3.0)
    for _ in range(4):
        a = rng.uniform(0.2, 0.8)
        om, nu = rng.uniform(0.004, 0.02, 2)
        ph, ps = rng.uniform(0, 2 * np.pi, 2)
        d += a * np.sin(om * x + ph) * np.cos(nu * y + ps)
    d = np.clip(d, 1.0, 8.0)
    d = np.round(d * 1000.0).astype(np.uint16).astype(np.float32) / 1000.0
    if invalid_frac > 0:
        d[rng.random((h, w)) < invalid_frac] = 0.0
    return d.astype(np.float32)


def make_texture(rng, h=H, w=W):
    """Band-limited RGB noise, uint8 [h,w,3]."""
    from scipy.ndimage import gaussian_filter
    img = rng.random((h, w, 3))
    img = gaussian_filter(img, sigma=(2, 2, 0))
    lo, hi = img.min(), img.max()
    img = (img - lo) / (hi - lo)
    return np.clip(np.round(img * 255.0), 0, 255).astype(np.uint8)


def warp_forward(tex0, depth0, R, t, K):
    """Forward-splat (texture0, depth0) into camera 1 with a z-buffer and 3x3 dilation."""
    h, w = depth0.shape
    v, u = np.mgrid[0:h, 0:w]
    valid = depth0 > 0
    u0, v0, d0 = u[valid].astype(np.float64), v[valid].astype(np.float64), depth0[valid].astype(np.float64)
    Kinv = np.linalg.inv(K)
    X0 = d0[None] * (Kinv @ np.stack([u0, v0, np.ones_like(u0)]))
    X1 = R @ X0 + t[:, None]
    z1 = X1[2]
    ok = z1 > 0.05
    p = K @ X1[:, ok]
    u1 = np.round(p[0] / p[2]).astype(np.int64)
    v1 = np.round(p[1] / p[2]).astype(np.int64)
    z1 = z1[ok]
    col = tex0[valid][ok]
    order = np.argsort(-z1, kind="stable")  # far first, near overwrites
    u1, v1, z1, col = u1[order], v1[order], z1[order], col[order]
    tex1 = np.zeros_like(tex0)
    dep1 = np.zeros((h, w), dtype=np.float32)
    zbuf = np.full((h, w), np.inf)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            uu, vv = u1 + dx, v1 + dy
            m = (uu >= 0) & (uu < w) & (vv >= 0) & (vv < h)
            uu, vv, zz, cc = uu[m], vv[m], z1[m], col[m]
            # later entries are nearer; keep only where nearer than what is there
            closer = zz < zbuf[vv, uu]
            # resolve duplicates inside this pass: last (nearest) write wins
            zbuf[vv[closer], uu[closer]] = zz[closer]
            tex1[vv[closer], uu[closer]] = cc[closer]
    filled = np.isfinite(zbuf)
    dep1[filled] = (np.round(zbuf[filled] * 1000.0).astype(np.uint16).astype(np.float32) / 1000.0)
    return tex1, dep1


def make_pair(i, h=H, w=W, K=None):
    """Pair ``i`` (seed 1000+i): dict shaped like the reference sample (lib/datasets/mapfree.py:250-268)
    without the batch axis, plus ground truth ``R_gt``, ``t_gt``."""
    rng = np.random.default_rng(1000 + i)
    K = (K_DEFAULT if K is None else np.asarray(K, dtype=np.float64)).copy()
    depth0 = make_depth(rng, h, w)
    tex0 = make_texture(rng, h, w)
    R, t = random_pose(rng)
    tex1, depth1 = warp_forward(tex0, depth0, R, t, K)
    return {
        "image0": np.ascontiguousarray(tex0.transpose(2, 0, 1)).astype(np.float32) / 255.0,
        "image1": np.ascontiguousarray(tex1.transpose(2, 0, 1)).astype(np.float32) / 255.0,
        "depth0": depth0, "depth1": depth1,
        "K_color0": K.astype(np.float32), "K_color1": K.astype(np.float32),
        "R_gt": R, "t_gt": t, "pair_id": i,
    }


def make_scene(seed, n_queries, h=H, w=W, K=None):
    """A Map-free-style scene (lib/datasets/mapfree.py:148-165: every pair of a scene shares its first frame): one map
    frame and ``n_queries`` query frames rendered from it with ``warp_forward``, each with its own ground-truth pose.
    Drawn from ``np.random.default_rng(seed)`` in ``make_pair``'s order (depth, texture, then one pose per query), so
    ``make_scene(1000 + i, 1)`` holds ``make_pair(i)``. Returns {"image0" [3,h,w], "gray0" [h,w] float32 in [0,1] (the
    BT.601 gray the matchers read), "depth0", "K_color0", "queries": [{"image1", "gray1", "depth1", "K_color1", "R_gt",
    "t_gt"}, ...]}."""
    rng = np.random.default_rng(seed)
    K = (K_DEFAULT if K is None else np.asarray(K, dtype=np.float64)).copy()
    depth0 = make_depth(rng, h, w)
    tex0 = make_texture(rng, h, w)
    image0 = np.ascontiguousarray(tex0.transpose(2, 0, 1)).astype(np.float32) / 255.0
    queries = []
    for _ in range(n_queries):
        R, t = random_pose(rng)
        tex1, depth1 = warp_forward(tex0, depth0, R, t, K)
        image1 = np.ascontiguousarray(tex1.transpose(2, 0, 1)).astype(np.float32) / 255.0
        queries.append({"image1": image1, "gray1": rgb_to_gray_u8(image1).astype(np.float32) / 255.0, "depth1": depth1,
                        "K_color1": K.astype(np.float32), "R_gt": R, "t_gt": t})
    return {"image0": image0, "gray0": rgb_to_gray_u8(image0).astype(np.float32) / 255.0, "depth0": depth0,
            "K_color0": K.astype(np.float32), "queries": queries}


def rgb_to_gray_u8(img_chw):
    """OpenCV COLOR_RGB2GRAY (BT.601 fixed point) of a float [3,H,W] image in [0,1] -> uint8 [H,W]
    (reference lib/models/matching/feature_matching.py:61-65)."""
    rgb = (255 * np.asarray(img_chw).transpose(1, 2, 0)).astype(np.uint8).astype(np.int64)
    g = (rgb[..., 0] * 4899 + rgb[..., 1] * 9617 + rgb[..., 2] * 1868 + 8192) >> 14
    return g.astype(np.uint8)


def make_correspondences(seed, n=2000, inlier_ratio=0.5, noise_px=0.5, h=H, w=W, K=None,
                         with_depth=True):
    """Correspondence set without images (BASELINE config C5): ``n`` matches, a fraction of them
    true projections of random 3-D points (+ Gaussian pixel noise), the rest uniform outliers.
    Returns dict with kpts0/kpts1 float32 [n,2], depth maps consistent with the inliers, K, R_gt,
    t_gt and the ground-truth inlier flags."""
    rng = np.random.default_rng(seed)
    K = (K_DEFAULT if K is None else np.asarray(K, dtype=np.float64)).copy()
    R, t = random_pose(rng)
    depth0 = make_depth(rng, h, w, invalid_frac=0.0)
    n_in = int(round(n * inlier_ratio))
    Kinv = np.linalg.inv(K)
    k0 = np.zeros((0, 2))
    k1 = np.zeros((0, 2))
    z1s = np.zeros((0,))
    # rejection-sample inliers that land inside image 1
    while len(k0) < n_in:
        m = 2 * (n_in - len(k0)) + 16
        u = rng.uniform(2, w - 3, m)
        v = rng.uniform(2, h - 3, m)
        d = depth0[v.astype(np.int64), u.astype(np.int64)].astype(np.float64)
        X0 = d[None] * (Kinv @ np.stack([u, v, np.ones(m)]))
        X1 = R @ X0 + t[:, None]
        p = K @ X1
        u1, v1 = p[0] / p[2], p[1] / p[2]
        ok = (X1[2] > 0.1) & (u1 >= 2) & (u1 < w - 3) & (v1 >= 2) & (v1 < h - 3)
        k0 = np.concatenate([k0, np.stack([u, v], 1)[ok]])
        k1 = np.concatenate([k1, np.stack([u1, v1], 1)[ok]])
        z1s = np.concatenate([z1s, X1[2][ok]])
    k0, k1, z1s = k0[:n_in], k1[:n_in], z1s[:n_in]
    k1 = k1 + rng.normal(0, noise_px, k1.shape)
    k1[:, 0] = np.clip(k1[:, 0], 0, w - 1.001)
    k1[:, 1] = np.clip(k1[:, 1], 0, h - 1.001)
    n_out = n - n_in
    o0 = np.stack([rng.uniform(0, w - 1, n_out), rng.uniform(0, h - 1, n_out)], 1)
    o1 = np.stack([rng.uniform(0, w - 1, n_out), rng.uniform(0, h - 1, n_out)], 1)
    kpts0 = np.concatenate([k0, o0]).astype(np.float32)
    kpts1 = np.concatenate([k1, o1]).astype(np.float32)
    gt = np.concatenate([np.ones(n_in, bool), np.zeros(n_out, bool)])
    perm = rng.permutation(n)
    kpts0, kpts1, gt = kpts0[perm], kpts1[perm], gt[perm]
    out = {"kpts0": kpts0, "kpts1": kpts1, "inlier_gt": gt, "R_gt": R, "t_gt": t,
           "K_color0": K.astype(np.float32), "K_color1": K.astype(np.float32), "depth0": depth0}
    if with_depth:
        # depth1: a smooth field, overwritten at the inlier pixels so that the lift is consistent
        depth1 = make_depth(rng, h, w, invalid_frac=0.0)
        kk1 = np.int32(kpts1)
        zq = np.round(z1s * 1000.0).astype(np.uint16).astype(np.float32) / 1000.0
        inl_idx = np.where(gt)[0]
        inv = np.empty(n, dtype=np.int64)
        inv[perm] = np.arange(n)
        # perm maps new->old; z1s is in old (pre-permutation) inlier order
        old_of_new = perm
        for new_i in inl_idx:
            old_i = old_of_new[new_i]
            depth1[kk1[new_i, 1], kk1[new_i, 0]] = zq[old_i]
        out["depth1"] = depth1
    return out


def make_correspondence_points(seed, n=2000, inlier_ratio=0.5, noise_px=0.5, h=H, w=W, K=None):
    """Correspondence set without images AND without depth maps (BASELINE config C5, essential-matrix cells): the same
    construction as ``make_correspondences`` — inliers are projections of 3-D points at a smooth depth field, Gaussian
    pixel noise in image 1, outliers uniform in both images — but the depth field is evaluated only at the sampled
    pixels, so a cell of 256 sets costs milliseconds. Returns kpts0/kpts1 float32 [n,2], inlier_gt, R_gt, t_gt, K."""
    rng = np.random.default_rng(seed)
    K = (K_DEFAULT if K is None else np.asarray(K, dtype=np.float64)).copy()
    R, t = random_pose(rng)
    amp = rng.uniform(0.2, 0.8, 4); om = rng.uniform(0.004, 0.02, 4); nu = rng.uniform(0.004, 0.02, 4)
    ph = rng.uniform(0, 2 * np.pi, 4); ps = rng.uniform(0, 2 * np.pi, 4)

    def depth_at(u, v):
        d = np.full(u.shape, 3.0)
        for k in range(4):
            d += amp[k] * np.sin(om[k] * np.floor(u) + ph[k]) * np.cos(nu[k] * np.floor(v) + ps[k])
        return np.round(np.clip(d, 1.0, 8.0) * 1000.0) / 1000.0

    n_in = int(round(n * inlier_ratio))
    Kinv = np.linalg.inv(K)
    k0 = np.zeros((0, 2)); k1 = np.zeros((0, 2))
    while len(k0) < n_in:
        m = 2 * (n_in - len(k0)) + 16
        u = rng.uniform(2, w - 3, m); v = rng.uniform(2, h - 3, m)
        X0 = depth_at(u, v)[None] * (Kinv @ np.stack([u, v, np.ones(m)]))
        X1 = R @ X0 + t[:, None]
        p = K @ X1
        u1, v1 = p[0] / p[2], p[1] / p[2]
        ok = (X1[2] > 0.1) & (u1 >= 2) & (u1 < w - 3) & (v1 >= 2) & (v1 < h - 3)
        k0 = np.concatenate([k0, np.stack([u, v], 1)[ok]]); k1 = np.concatenate([k1, np.stack([u1, v1], 1)[ok]])
    k0, k1 = k0[:n_in], k1[:n_in]
    k1 = k1 + rng.normal(0, noise_px, k1.shape)
    n_out = n - n_in
    o0 = np.stack([rng.uniform(0, w - 1, n_out), rng.uniform(0, h - 1, n_out)], 1)
    o1 = np.stack([rng.uniform(0, w - 1, n_out), rng.uniform(0, h - 1, n_out)], 1)
    perm = rng.permutation(n)
    gt = np.concatenate([np.ones(n_in, bool), np.zeros(n_out, bool)])[perm]
    return {"kpts0": np.concatenate([k0, o0]).astype(np.float32)[perm], "kpts1": np.concatenate([k1, o1]).astype(np.float32)[perm],
            "inlier_gt": gt, "R_gt": R, "t_gt": t, "K_color0": K.astype(np.float32), "K_color1": K.astype(np.float32)}
