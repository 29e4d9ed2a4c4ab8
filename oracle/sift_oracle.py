"""ORACLE (test infrastructure only — never imported by the product path).

numpy float32 restatement of OpenCV 4.x SIFT (``cv2.SIFT_create(nfeatures).detectAndCompute``) at the default
settings: 3 layers per octave, contrast threshold 0.04, edge threshold 10, sigma 1.6, first octave -1 (doubled
input), CV_32F descriptors. The reference's SIFT plugins call exactly this (lib/models/matching/
feature_matching.py:53-118, etc/feature_matching_baselines/matchers.py:123-188).

The pyramid is built from cv2's own primitives (``cv2.resize``, ``cv2.GaussianBlur``), so it IS OpenCV's pyramid.
Everything after it (extrema, refinement, orientation, duplicate removal, retainBest, descriptors) is written here,
stage by stage, and each stage starts from given arrays, so the GPU tests can feed it the engine's own pyramid.

Arithmetic follows OpenCV's float order; the few fused multiply-adds of OpenCV's SIMD paths (fastAtan2's
polynomial, magnitude, the orientation smoothing) are rounded once, as a fused operation does. OpenCV's exp32f
and the compiler's own contractions are not emulated: they move values by a few ulp, which the tests bound.

Keypoints travel as a dict of equal-length arrays: x, y, size, angle, response (float32), octave (int32, OpenCV's
packed field) and, before the final rescale, the internal o (octave index from the doubled image), layer, r, c.
"""
import numpy as np

F32 = np.float32
N_LAYERS = 3
CONTRAST = F32(0.04)
EDGE = F32(10.0)
SIGMA = F32(1.6)
BORDER = 5
MAX_STEPS = 5
ORI_BINS = 36
DESC_D, DESC_N = 4, 8
FLT_EPS = F32(np.finfo(np.float32).eps)
IMG_SCALE = F32(1.0) / F32(255.0)
DERIV_SCALE = IMG_SCALE * F32(0.5)
CROSS_SCALE = IMG_SCALE * F32(0.25)
THRESHOLD = int(np.floor(0.5 * 0.04 / N_LAYERS * 255))       # = 1 on the 0..255 scale


def _fma(a, b, c):
    """float32 fused multiply-add (one rounding): the float32 product is exact in float64."""
    return (np.float64(a) * np.float64(b) + np.float64(c)).astype(np.float32)


def n_octaves(h, w):
    """cvRound(log2(min side of the doubled base) - 2) - firstOctave."""
    return int(np.rint(np.log(min(2 * h, 2 * w)) / np.log(2.0) - 2)) + 1


def level_sigmas():
    """sig[0] = the base blur, sig[i] the incremental blur of level i (buildGaussianPyramid)."""
    sig = [float(np.sqrt(max(F32(SIGMA * SIGMA) - F32(1.0), F32(0.01))).astype(np.float32))]
    k = 2.0 ** (1.0 / N_LAYERS)
    for i in range(1, N_LAYERS + 3):
        prev = k ** (i - 1) * 1.6
        sig.append(float(np.sqrt((prev * k) ** 2 - prev ** 2)))
    return sig


def build_pyramid(gray_u8):
    """-> (gauss[o][0..5], dog[o][0..4]) float32, o = 0 the doubled image (OpenCV octave -1)."""
    import cv2
    h, w = gray_u8.shape
    sig = level_sigmas()
    dbl = cv2.resize(gray_u8.astype(np.float32), (2 * w, 2 * h), interpolation=cv2.INTER_LINEAR)
    base = cv2.GaussianBlur(dbl, (0, 0), sig[0], sigmaY=sig[0])
    gauss, dog = [], []
    for o in range(n_octaves(h, w)):
        lv = [base if o == 0 else np.ascontiguousarray(gauss[o - 1][N_LAYERS][::2, ::2][:gauss[o - 1][N_LAYERS].shape[0] // 2,
                                                                                     :gauss[o - 1][N_LAYERS].shape[1] // 2])]
        for i in range(1, N_LAYERS + 3):
            lv.append(cv2.GaussianBlur(lv[-1], (0, 0), sig[i], sigmaY=sig[i]))
        gauss.append(lv)
        dog.append([lv[i + 1] - lv[i] for i in range(N_LAYERS + 2)])
    return gauss, dog


# ------------------------------------------------------------------------------ extrema + refinement
def find_extrema(dog_o):
    """Candidates of one octave: (layer, r, c) int arrays, raster order per layer (findScaleSpaceExtrema)."""
    D = np.stack(dog_o)
    rows, cols = D.shape[1:]
    out = []
    for i in range(1, N_LAYERS + 1):
        if rows - 2 * BORDER <= 0 or cols - 2 * BORDER <= 0:
            break
        sl = lambda a, dr, dc: a[BORDER + dr:rows - BORDER + dr, BORDER + dc:cols - BORDER + dc]
        v = sl(D[i], 0, 0)
        mx = np.full(v.shape, -np.inf, np.float32); mn = np.full(v.shape, np.inf, np.float32)
        for l in (i - 1, i, i + 1):
            for dr in (-1, 0, 1):
                for dc in (-1, 0, 1):
                    if l == i and dr == 0 and dc == 0:
                        continue
                    n = sl(D[l], dr, dc)
                    mx = np.maximum(mx, n); mn = np.minimum(mn, n)
        keep = (np.abs(v) > THRESHOLD) & (((v > 0) & (v >= mx)) | ((v < 0) & (v <= mn)))
        r, c = np.nonzero(keep)
        out.append((np.full(r.shape, i), r + BORDER, c + BORDER))
    if not out:
        z = np.zeros(0, np.int64)
        return z, z, z
    return tuple(np.concatenate([o[k] for o in out]) for k in range(3))


def _derivs(D, l, r, c):
    g = lambda dl, dr, dc: D[l + dl, r + dr, c + dc]
    dD = np.stack([(g(0, 0, 1) - g(0, 0, -1)) * DERIV_SCALE,
                   (g(0, 1, 0) - g(0, -1, 0)) * DERIV_SCALE,
                   (g(1, 0, 0) - g(-1, 0, 0)) * DERIV_SCALE], -1)
    v2 = g(0, 0, 0) * F32(2)
    dxx = (g(0, 0, 1) + g(0, 0, -1) - v2) * IMG_SCALE
    dyy = (g(0, 1, 0) + g(0, -1, 0) - v2) * IMG_SCALE
    dss = (g(1, 0, 0) + g(-1, 0, 0) - v2) * IMG_SCALE
    dxy = (g(0, 1, 1) - g(0, 1, -1) - g(0, -1, 1) + g(0, -1, -1)) * CROSS_SCALE
    dxs = (g(1, 0, 1) - g(1, 0, -1) - g(-1, 0, 1) + g(-1, 0, -1)) * CROSS_SCALE
    dys = (g(1, 1, 0) - g(1, -1, 0) - g(-1, 1, 0) + g(-1, -1, 0)) * CROSS_SCALE
    H = np.stack([np.stack([dxx, dxy, dxs], -1), np.stack([dxy, dyy, dys], -1), np.stack([dxs, dys, dss], -1)], -2)
    return dD, H, dxx, dyy, dxy


def solve3(H, b):
    """Matx33f::solve(DECOMP_LU) of OpenCV 4.x for one right-hand side: Cramer's rule in float
    (Matx_FastSolveOp<float, 3, 1>), zeros when the determinant is exactly 0."""
    a = lambda i, j: H[:, i, j]
    bb = lambda i: b[:, i]
    det = (a(0, 0) * (a(1, 1) * a(2, 2) - a(2, 1) * a(1, 2)) - a(0, 1) * (a(1, 0) * a(2, 2) - a(2, 0) * a(1, 2))
           + a(0, 2) * (a(1, 0) * a(2, 1) - a(2, 0) * a(1, 1)))
    ok = det != 0
    d = np.where(ok, F32(1) / np.where(ok, det, F32(1)), F32(0)).astype(np.float32)
    x0 = d * (bb(0) * (a(1, 1) * a(2, 2) - a(1, 2) * a(2, 1)) - a(0, 1) * (bb(1) * a(2, 2) - a(1, 2) * bb(2))
              + a(0, 2) * (bb(1) * a(2, 1) - a(1, 1) * bb(2)))
    x1 = d * (a(0, 0) * (bb(1) * a(2, 2) - a(1, 2) * bb(2)) - bb(0) * (a(1, 0) * a(2, 2) - a(1, 2) * a(2, 0))
              + a(0, 2) * (a(1, 0) * bb(2) - bb(1) * a(2, 0)))
    x2 = d * (a(0, 0) * (a(1, 1) * bb(2) - bb(1) * a(2, 1)) - a(0, 1) * (a(1, 0) * bb(2) - bb(1) * a(2, 0))
              + bb(0) * (a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0)))
    x = np.stack([x0, x1, x2], -1).astype(np.float32)
    return np.where(ok[:, None], x, F32(0))


def refine(dog_o, o, layer, r, c, with_margins=False):
    """adjustLocalExtrema for the candidates of octave o. Returns the kept keypoints (internal fields) and, with
    with_margins, the relative margins of the contrast and edge tests (for the candidates that reached them), the
    distance of the closest offset to the 0.5 convergence bound (every candidate), the indices of the candidates that
    reached the tests and which of those were kept."""
    D = np.stack(dog_o)
    rows, cols = D.shape[1:]
    n = len(r)
    layer = layer.astype(np.int64).copy(); r = r.astype(np.int64).copy(); c = c.astype(np.int64).copy()
    alive = np.ones(n, bool); done = np.zeros(n, bool)
    X = np.zeros((n, 3), np.float32)
    conv_margin = np.full(n, np.inf)
    for _ in range(MAX_STEPS):
        idx = np.nonzero(alive & ~done)[0]
        if len(idx) == 0:
            break
        dD, H, *_ = _derivs(D, layer[idx], r[idx], c[idx])
        x = -solve3(H, dD)
        X[idx] = x
        conv_margin[idx] = np.minimum(conv_margin[idx], np.abs(np.abs(x) - F32(0.5)).min(1))
        conv = (np.abs(x) < F32(0.5)).all(1)
        done[idx[conv]] = True
        idx = idx[~conv]; x = x[~conv]
        big = (np.abs(x) > F32((2 ** 31 - 1) // 3)).any(1)
        alive[idx[big]] = False
        idx = idx[~big]; x = x[~big]
        c[idx] += np.rint(x[:, 0]).astype(np.int64)
        r[idx] += np.rint(x[:, 1]).astype(np.int64)
        layer[idx] += np.rint(x[:, 2]).astype(np.int64)
        out = ((layer[idx] < 1) | (layer[idx] > N_LAYERS) | (c[idx] < BORDER) | (c[idx] >= cols - BORDER)
               | (r[idx] < BORDER) | (r[idx] >= rows - BORDER))
        alive[idx[out]] = False
    notconv = alive & ~done
    alive[notconv] = False
    idx = np.nonzero(alive)[0]
    xc, xr, xi = X[idx, 0], X[idx, 1], X[idx, 2]
    dD, _, dxx, dyy, dxy = _derivs(D, layer[idx], r[idx], c[idx])
    t = F32(0) + dD[:, 0] * xc
    t = t + dD[:, 1] * xr
    t = t + dD[:, 2] * xi
    contr = D[layer[idx], r[idx], c[idx]] * IMG_SCALE + t * F32(0.5)
    low = np.abs(contr) * F32(N_LAYERS) < CONTRAST
    tr = dxx + dyy
    det = dxx * dyy - dxy * dxy
    lhs = tr * tr * EDGE
    rhs = F32((EDGE + 1) * (EDGE + 1)) * det
    edge = (det <= 0) | (lhs >= rhs)
    keep = ~low & ~edge
    margins = None
    if with_margins:
        margins = {"contrast": np.abs(np.abs(contr) * F32(N_LAYERS) - CONTRAST) / CONTRAST,
                   "edge": np.where(det > 0, np.abs(lhs - rhs) / np.maximum(np.abs(rhs), 1e-30), np.inf),
                   "converge": conv_margin}
    k = idx[keep]
    xc, xr, xi, contr = xc[keep], xr[keep], xi[keep], contr[keep]
    s = F32(1 << o)
    kp = {"x": c[k].astype(np.float32) + xc, "y": r[k].astype(np.float32) + xr}
    kp["x"] = (kp["x"] * s).astype(np.float32); kp["y"] = (kp["y"] * s).astype(np.float32)
    oct_field = o + (layer[k] << 8) + (np.rint((xi.astype(np.float64) + 0.5) * 255).astype(np.int64) << 16)
    kp["octave"] = oct_field.astype(np.int64)
    kp["size"] = (SIGMA * np.power(F32(2), (layer[k].astype(np.float32) + xi) / F32(N_LAYERS)) * s * F32(2)).astype(np.float32)
    kp["response"] = np.abs(contr).astype(np.float32)
    kp["o"] = np.full(len(k), o); kp["layer"] = layer[k]; kp["r"] = r[k]; kp["c"] = c[k]
    if with_margins:
        return kp, margins, idx, keep
    return kp


# ------------------------------------------------------------------------------ orientation
def fast_atan2(y, x):
    """cv::hal::fastAtan2 (degrees, [0, 360)), the SIMD form: polynomial with fused multiply-adds."""
    p1 = F32(0.9997878412794807 * 180 / np.pi); p3 = F32(-0.3258083974640975 * 180 / np.pi)
    p5 = F32(0.1555786518463281 * 180 / np.pi); p7 = F32(-0.04432655554792128 * 180 / np.pi)
    y = np.asarray(y, np.float32); x = np.asarray(x, np.float32)
    ax, ay = np.abs(x), np.abs(y)
    c = np.minimum(ax, ay) / (np.maximum(ax, ay) + F32(np.finfo(np.float64).eps))
    cc = c * c
    a = _fma(_fma(_fma(cc, p7, p5), cc, p3), cc, p1) * c
    a = np.where(ax >= ay, a, F32(90) - a)
    a = np.where(x < 0, F32(180) - a, a)
    a = np.where(y < 0, F32(360) - a, a)
    return a.astype(np.float32)


def _grad(img, yy, xx):
    dx = img[yy, xx + 1] - img[yy, xx - 1]
    dy = img[yy - 1, xx] - img[yy + 1, xx]
    return dx, dy


def orientation_hist(img, r, c, radius, sigma):
    """calcOrientationHist -> (smoothed hist float32[36], max)."""
    rows, cols = img.shape
    ii, jj = np.meshgrid(np.arange(-radius, radius + 1), np.arange(-radius, radius + 1), indexing="ij")
    yy, xx = r + ii, c + jj
    ok = (yy > 0) & (yy < rows - 1) & (xx > 0) & (xx < cols - 1)
    ii, jj, yy, xx = ii[ok], jj[ok], yy[ok], xx[ok]
    scale = F32(-1) / (F32(2) * sigma * sigma)
    dx, dy = _grad(img, yy, xx)
    w = np.exp((ii * ii + jj * jj).astype(np.float32) * scale).astype(np.float32)
    ori = fast_atan2(dy, dx)
    mag = np.sqrt(_fma(dx, dx, dy * dy)).astype(np.float32)
    b = np.rint(F32(ORI_BINS / 360.0) * ori).astype(np.int64)
    b = np.where(b >= ORI_BINS, b - ORI_BINS, b); b = np.where(b < 0, b + ORI_BINS, b)
    t = np.zeros(ORI_BINS, np.float32)
    np.add.at(t, b, (w * mag).astype(np.float32))
    tn = lambda s: np.roll(t, -s)
    h = _fma(tn(-2) + tn(2), F32(1 / 16), _fma(tn(-1) + tn(1), F32(4 / 16), t * F32(6 / 16)))
    return h, h.max()


def orientations(gauss, kp, with_margins=False):
    """One keypoint per accepted histogram peak (findScaleSpaceExtrema after adjustLocalExtrema)."""
    out = {k: [] for k in kp}
    out["angle"] = []
    margins = []
    for i in range(len(kp["x"])):
        o, layer = int(kp["o"][i]), int(kp["layer"][i])
        scl = kp["size"][i] * F32(0.5) / F32(1 << o)
        h, omax = orientation_hist(gauss[o][layer], int(kp["r"][i]), int(kp["c"][i]),
                                   int(np.rint(F32(4.5) * scl)), F32(1.5) * scl)
        thr = F32(omax * F32(0.8))
        for j in range(ORI_BINS):
            hl, hr, hj = h[j - 1], h[(j + 1) % ORI_BINS], h[j]
            if hj > hl and hj > hr:
                if with_margins and hj < thr:
                    margins.append(float((thr - hj) / thr))
                if hj >= thr:
                    if with_margins:
                        margins.append(float((hj - thr) / thr))
                    b = F32(j) + F32(0.5) * (hl - hr) / (hl - F32(2) * hj + hr)
                    b = b + F32(ORI_BINS) if b < 0 else (b - F32(ORI_BINS) if b >= ORI_BINS else b)
                    ang = F32(360) - F32(10) * F32(b)
                    if abs(ang - F32(360)) < FLT_EPS:
                        ang = F32(0)
                    for k in kp:
                        out[k].append(kp[k][i])
                    out["angle"].append(ang)
    res = {k: np.asarray(v, dtype=kp[k].dtype if k in kp else np.float32) for k, v in out.items()}
    if with_margins:
        return res, margins
    return res


# ------------------------------------------------------------------------------ selection
def sort_order(kp):
    """The engine's output order: response descending, then x, y, size, angle ascending (then octave)."""
    return np.lexsort((kp["octave"], kp["angle"], kp["size"], kp["y"], kp["x"], -kp["response"].astype(np.float64)))


def select(kp, nfeatures):
    """removeDuplicatedSorted + retainBest(nfeatures), then the firstOctave = -1 rescale (detectAndCompute).
    Returns the keypoints in sort_order."""
    kp = {k: v[sort_order(kp)] for k, v in kp.items()}
    n = len(kp["x"])
    if n:
        key = np.stack([kp["x"], kp["y"], kp["size"], kp["angle"]], 1)
        dup = np.zeros(n, bool)
        dup[1:] = (key[1:] == key[:-1]).all(1)
        kp = {k: v[~dup] for k, v in kp.items()}
    if nfeatures > 0 and len(kp["x"]) > nfeatures:
        cut = kp["response"][nfeatures - 1]
        kp = {k: v[kp["response"] >= cut] for k, v in kp.items()}
    kp["x"] = kp["x"] * F32(0.5); kp["y"] = kp["y"] * F32(0.5); kp["size"] = kp["size"] * F32(0.5)
    kp["octave"] = (kp["octave"] & ~255) | ((kp["octave"] - 1) & 255)
    return kp


# ------------------------------------------------------------------------------ descriptors
def descriptor(img, ptx, pty, ori, scl):
    """calcSIFTDescriptor on the Gaussian level of the keypoint (octave coordinates) -> float32[128] (integers)."""
    d, n = DESC_D, DESC_N
    rows, cols = img.shape
    px, py = int(np.rint(ptx)), int(np.rint(pty))
    cos_t = np.cos(np.float32(ori * F32(np.pi / 180))).astype(np.float32)
    sin_t = np.sin(np.float32(ori * F32(np.pi / 180))).astype(np.float32)
    bins_per_rad = F32(n / 360.0)
    exp_scale = F32(-1.0 / (d * d * 0.5))
    hist_width = F32(3) * scl
    radius = int(np.rint(hist_width * F32(1.4142135623730951) * F32(d + 1) * F32(0.5)))
    radius = min(radius, int(np.sqrt(float(cols) * cols + float(rows) * rows)))
    cos_t = cos_t / hist_width; sin_t = sin_t / hist_width
    ii, jj = np.meshgrid(np.arange(-radius, radius + 1), np.arange(-radius, radius + 1), indexing="ij")
    fi, fj = ii.astype(np.float32), jj.astype(np.float32)
    c_rot = fj * cos_t - fi * sin_t
    r_rot = fj * sin_t + fi * cos_t
    rbin = r_rot + F32(d // 2) - F32(0.5)
    cbin = c_rot + F32(d // 2) - F32(0.5)
    rr, cc = py + ii, px + jj
    ok = (rbin > -1) & (rbin < d) & (cbin > -1) & (cbin < d) & (rr > 0) & (rr < rows - 1) & (cc > 0) & (cc < cols - 1)
    rbin, cbin, rr, cc, c_rot, r_rot = rbin[ok], cbin[ok], rr[ok], cc[ok], c_rot[ok], r_rot[ok]
    dx, dy = _grad(img, rr, cc)
    w = np.exp((c_rot * c_rot + r_rot * r_rot) * exp_scale).astype(np.float32)
    o = fast_atan2(dy, dx)
    mag = np.sqrt(_fma(dx, dx, dy * dy)).astype(np.float32) * w
    obin = (o - ori) * bins_per_rad
    r0, c0, o0 = np.floor(rbin).astype(np.int64), np.floor(cbin).astype(np.int64), np.floor(obin).astype(np.int64)
    rbin = rbin - r0.astype(np.float32); cbin = cbin - c0.astype(np.float32); obin = obin - o0.astype(np.float32)
    o0 = np.where(o0 < 0, o0 + n, o0); o0 = np.where(o0 >= n, o0 - n, o0)
    v_r1 = mag * rbin; v_r0 = mag - v_r1
    v_rc11 = v_r1 * cbin; v_rc10 = v_r1 - v_rc11
    v_rc01 = v_r0 * cbin; v_rc00 = v_r0 - v_rc01
    v111 = v_rc11 * obin; v110 = v_rc11 - v111
    v101 = v_rc10 * obin; v100 = v_rc10 - v101
    v011 = v_rc01 * obin; v010 = v_rc01 - v011
    v001 = v_rc00 * obin; v000 = v_rc00 - v001
    idx = ((r0 + 1) * (d + 2) + c0 + 1) * (n + 2) + o0
    R, C = (d + 2) * (n + 2), n + 2
    offs = np.array([0, 1, C, C + 1, R, R + 1, R + C, R + C + 1])
    vals = np.stack([v000, v001, v010, v011, v100, v101, v110, v111], 1)
    hist = np.zeros((d + 2) * (d + 2) * (n + 2), np.float32)
    np.add.at(hist, (idx[:, None] + offs[None]).ravel(), vals.ravel())     # sample-major: OpenCV's order per bin
    dst = np.zeros(d * d * n, np.float32)
    for i in range(d):
        for j in range(d):
            b = ((i + 1) * (d + 2) + (j + 1)) * (n + 2)
            hist[b] += hist[b + n]
            hist[b + 1] += hist[b + n + 1]
            dst[(i * d + j) * n:(i * d + j + 1) * n] = hist[b:b + n]
    nrm2 = F32(np.sum(dst.astype(np.float64) ** 2))
    thr = np.sqrt(nrm2) * F32(0.2)
    dst = np.minimum(dst, thr)
    nrm2 = F32(np.sum(dst.astype(np.float64) ** 2))
    nrm2 = F32(512) / max(np.sqrt(nrm2), FLT_EPS)
    return np.clip(np.rint(dst * nrm2), 0, 255).astype(np.float32)


def descriptors(gauss, kp):
    """calcDescriptors for keypoints in input-pixel coordinates (select()'s output)."""
    out = np.zeros((len(kp["x"]), 128), np.float32)
    for i in range(len(kp["x"])):
        octv = int(kp["octave"][i]) & 255
        layer = (int(kp["octave"][i]) >> 8) & 255
        octv = octv if octv < 128 else octv - 256
        scale = F32(1.0 / (1 << octv)) if octv >= 0 else F32(1 << -octv)
        size = kp["size"][i] * scale
        ang = F32(360) - kp["angle"][i]
        if abs(ang - F32(360)) < FLT_EPS:
            ang = F32(0)
        out[i] = descriptor(gauss[octv + 1][layer], kp["x"][i] * scale, kp["y"][i] * scale, ang, size * F32(0.5))
    return out


# ------------------------------------------------------------------------------ whole detector
def detect_from_pyramid(gauss, dog, with_margins=False):
    """Extrema + refinement + orientation over every octave -> pre-selection keypoints (internal coordinates)."""
    parts, margins = [], {"contrast": [], "edge": [], "peak": []}
    for o in range(len(dog)):
        layer, r, c = find_extrema(dog[o])
        if len(r) == 0:
            continue
        if with_margins:
            kp, m, idx, keep = refine(dog[o], o, layer, r, c, with_margins=True)
            margins["contrast"].append(m["contrast"]); margins["edge"].append(m["edge"])
            kp, pm = orientations(gauss, kp, with_margins=True)
            margins["peak"].extend(pm)
        else:
            kp = orientations(gauss, refine(dog[o], o, layer, r, c))
        parts.append(kp)
    keys = ["x", "y", "size", "angle", "response", "octave", "o", "layer", "r", "c"]
    if parts:
        kp = {k: np.concatenate([p[k] for p in parts]) for k in keys}
    else:
        kp = {k: np.zeros(0, np.float32 if k in ("x", "y", "size", "angle", "response") else np.int64) for k in keys}
    if with_margins:
        return kp, {k: (np.concatenate(v) if k != "peak" and v else np.asarray(v, np.float64)) for k, v in margins.items()}
    return kp


def detect_and_compute(gray_u8, nfeatures=0):
    """cv2.SIFT_create(nfeatures).detectAndCompute(gray_u8, None) -> (keypoints dict in sort_order, descriptors)."""
    gauss, dog = build_pyramid(gray_u8)
    kp = select(detect_from_pyramid(gauss, dog), nfeatures)
    return kp, descriptors(gauss, kp)


# ------------------------------------------------------------------------------ explaining a difference
def decision_margins(gauss, dog, o, layer, r, c, angle=None):
    """Relative margins of every threshold decision taken for a keypoint at internal octave o, DoG layer, pixel
    (r, c) (and orientation `angle`, degrees): the 26-neighbour test, the contrast and edge tests of the refinement
    started there, and the 0.8 orientation-peak test of the histogram bin nearest to `angle`. A keypoint that one
    implementation keeps and the other drops must sit near one of these thresholds."""
    m = {}
    D = np.stack(dog[o])
    rows, cols = D.shape[1:]
    if not (1 <= layer <= N_LAYERS and 1 <= r < rows - 1 and 1 <= c < cols - 1):
        return {"outside": 0.0}
    v = D[layer, r, c]
    nb = np.delete(D[layer - 1:layer + 2, r - 1:r + 2, c - 1:c + 2].ravel(), 13)
    ref = nb.max() if v > 0 else nb.min()
    m["extremum"] = float(abs(v - ref) / max(abs(v), 1e-30))
    m["threshold"] = float(abs(abs(v) - THRESHOLD) / THRESHOLD)
    kp, mm, idx, keep = refine(dog[o], o, np.array([layer]), np.array([r]), np.array([c]), with_margins=True)
    m["converge"] = float(mm["converge"][0])
    if len(idx):
        m["contrast"] = float(mm["contrast"][0]); m["edge"] = float(mm["edge"][0])
    else:
        m["refine"] = 0.0
    if angle is not None and len(kp["x"]):
        scl = kp["size"][0] * F32(0.5) / F32(1 << o)
        h, omax = orientation_hist(gauss[o][int(kp["layer"][0])], int(kp["r"][0]), int(kp["c"][0]),
                                   int(np.rint(F32(4.5) * scl)), F32(1.5) * scl)
        j = int(np.rint((360.0 - angle) / 10.0)) % ORI_BINS
        thr = omax * F32(0.8)
        m["peak"] = float(min(abs(h[jj] - thr) / thr for jj in (j - 1, j, (j + 1) % ORI_BINS)))
        m["local_max"] = float(min(abs(h[jj] - h[jj - 1]) / omax for jj in (j - 1, j, (j + 1) % ORI_BINS)))
    return m
