"""ORACLE (test infrastructure only, never imported by the product path).

float64 restatements of the stages of the pose back end (map-free-reloc_b200/csrc/geometry.cu), one function per
stage, each fed with the stage's input as it was read from the device. The E-mat path is normalise -> hypotheses
(emat_hyp_kernel) -> top-4 selection and pose choice (emat_stage_in, emat_choose_pose) -> local optimisation
(emat_lo_kernel) -> final model and mask (emat_final_kernel); the PnP path is depth minimum -> compaction and lift
(pnp_prepare_kernel) -> hypotheses (pnp_hyp_kernel) -> mask and LM (pnp_final_kernel). The minimal solvers come from
the library's host hooks (mfr_host_five_point, mfr_host_p3p, mfr_host_decompose_essential): they are the kernels' own
__host__ __device__ code, tested against OpenCV in tests/test_solvers_host.py, so what is restated here is everything
around them. Points are numpy arrays; hypotheses and LM iterations are Python loops over them.
"""
import ctypes
import math

import numpy as np

U32 = 2.0 ** -24                      # fp32 unit roundoff
M64 = (1 << 64) - 1
HYP_PER_BLOCK = 128                   # kHypPerBlock
LO_TOPK, LO_ROUNDS, LO_INNER, LO_MAX_PTS, TIGHT_ROUNDS = 4, 6, 5, 1024, 3
LO_SCHEDULE = (3.0, 2.0, 1.5, 1.0, 1.0, 1.0)
PNP_ITERS = 20
HYP_DTYPE = np.dtype({"names": ["cost", "count", "valid", "model"], "formats": ["<f8", "<i4", "<i4", ("<f8", 12)],
                      "offsets": [0, 8, 12, 16], "itemsize": 112})     # HypResult
LO_DTYPE = np.dtype({"names": ["cost", "R", "t"], "formats": ["<f8", ("<f8", 9), ("<f8", 3)],
                     "offsets": [0, 8, 80], "itemsize": 104})          # LoResult


def _lib():
    from mfr_b200 import lib
    return lib.load()


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ------------------------------------------------------------------------------------------------ RNG and launch shape
def splitmix64(s):
    """One step of the kernels' splitmix64: (new state, output)."""
    s = (s + 0x9E3779B97F4A7C15) & M64
    z = s
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return s, z ^ (z >> 31)


def sample_distinct(st, n, k):
    """sample_distinct<K>: K indices in [0, n); a drawn index equal to an earlier one is redrawn, at most 64 draws per
    slot, and the 64th draw is kept even when it repeats one."""
    idx = []
    for _ in range(k):
        v = 0
        for _ in range(64):
            st, z = splitmix64(st)
            v = z % n
            if v not in idx:
                break
        idx.append(v)
    return idx


def emat_state(seed, pair, h):
    return (seed ^ (0xD1B54A32D192ED03 * (pair + 1)) ^ (0x9E3779B97F4A7C15 * (h + 1))) & M64


def pnp_state(seed, pair, h):
    return (seed ^ (0xA24BAED4963EE407 * (pair + 1)) ^ (0x9E3779B97F4A7C15 * (h + 1))) & M64


def emat_hyp_per_block(P, num_hyp, sm_count):
    """emat_ransac's launch rule: 128 hypotheses per block, halved (down to 32) while P * blocks < sm_count / 2."""
    hpb = HYP_PER_BLOCK
    while hpb > 32 and P * -(-num_hyp // hpb) < sm_count // 2:
        hpb //= 2
    return hpb


# ------------------------------------------------------------------------------------------------ small maths
def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def essential_from_rt(R, t):
    return skew(np.asarray(t, np.float64)) @ np.asarray(R, np.float64).reshape(3, 3)


def so3_exp(w):
    """geometry_solvers.cuh so3_exp, same branch at 1e-8."""
    th2 = float(w @ w)
    th = math.sqrt(th2)
    if th < 1e-8:
        a, b = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0
    else:
        a, b = math.sin(th) / th, (1.0 - math.cos(th)) / th2
    x, y, z = w
    return np.array([[1.0 - b * (y * y + z * z), -a * z + b * x * y, a * y + b * x * z],
                     [a * z + b * x * y, 1.0 - b * (x * x + z * z), -a * x + b * y * z],
                     [-a * y + b * x * z, a * x + b * y * z, 1.0 - b * (x * x + y * y)]])


def tangent_basis(t):
    ax, ay, az = np.abs(t)
    a = np.zeros(3)
    if ax <= ay and ax <= az:
        a[0] = 1.0
    elif ay <= az:
        a[1] = 1.0
    else:
        a[2] = 1.0
    b1 = np.cross(t, a)
    b1 = b1 / np.linalg.norm(b1)
    return b1, np.cross(t, b1)


def solve_damped(H, g, lam):
    """solve_damped: (H + lam (diag(H) + 1e-12)) d = -g by Gaussian elimination with partial pivoting; None when a
    pivot is below 1e-300."""
    n = len(g)
    A = np.concatenate([H.copy(), -g.reshape(n, 1)], 1)
    A[np.arange(n), np.arange(n)] += lam * (np.diag(H) + 1e-12)
    for k in range(n):
        pr = k + int(np.argmax(np.abs(A[k:, k])))
        if abs(A[pr, k]) < 1e-300:
            return None
        if pr != k:
            A[[k, pr]] = A[[pr, k]]
        for i in range(k + 1, n):
            A[i, k:] -= A[i, k] / A[k, k] * A[k, k:]
    d = np.zeros(n)
    for i in range(n - 1, -1, -1):
        d[i] = (A[i, n] - A[i, i + 1:n] @ d[i + 1:]) / A[i, i]
    return d


def decompose_essential(E):
    l = _lib()
    E = np.ascontiguousarray(np.asarray(E, np.float64).reshape(9))
    R1, R2, t = np.zeros(9), np.zeros(9), np.zeros(3)
    l.mfr_host_decompose_essential(_p(E), _p(R1), _p(R2), _p(t))
    return R1.reshape(3, 3), R2.reshape(3, 3), t


def five_point(x0, x1):
    """Candidate essential matrices [n, 9] of one 5-point sample (x0, x1 [5, 2] float64)."""
    E = np.zeros((10, 9))
    n = _lib().mfr_host_five_point(_p(np.ascontiguousarray(x0, np.float64)), _p(np.ascontiguousarray(x1, np.float64)),
                                   _p(E))
    return E[:n]


def p3p(X, f):
    R, t = np.zeros((4, 9)), np.zeros((4, 3))
    n = _lib().mfr_host_p3p(_p(np.ascontiguousarray(X, np.float64)), _p(np.ascontiguousarray(f, np.float64)), _p(R),
                            _p(t))
    return R[:n].reshape(-1, 3, 3), t[:n]


# ------------------------------------------------------------------------------------------------ E-mat
def normalise(kpts0, kpts1, K0, K1):
    """emat_normalise_kernel in float32: (k - c) / f, [N, 4] = (x0, y0, x1, y1)."""
    k0, k1 = np.asarray(kpts0, np.float32), np.asarray(kpts1, np.float32)
    K0, K1 = np.asarray(K0, np.float32).reshape(3, 3), np.asarray(K1, np.float32).reshape(3, 3)
    return np.stack([(k0[:, 0] - K0[0, 2]) / K0[0, 0], (k0[:, 1] - K0[1, 2]) / K0[1, 1],
                     (k1[:, 0] - K1[0, 2]) / K1[0, 0], (k1[:, 1] - K1[1, 2]) / K1[1, 1]], 1).astype(np.float32)


def emat_threshold(pix_thr, K0, K1):
    """emat_threshold in float32: pix_thr / ((K0.fx + K1.fy + (K0.fy + K1.fx)) * 0.25). Returns (thr, thr * thr) as
    the float32 values the hypothesis kernel compares with."""
    K0, K1 = np.asarray(K0, np.float32).reshape(3, 3), np.asarray(K1, np.float32).reshape(3, 3)
    m = ((K0[0, 0] + K1[1, 1]) + (K0[1, 1] + K1[0, 0])) * np.float32(0.25)
    thr = np.float32(pix_thr) / np.float32(m)
    return np.float32(thr), np.float32(thr * thr)


def sampson_sq(E, pts):
    """Squared Sampson distance [..., N] in float64 of the float32 points pts [N, 4] under E [..., 9]
    (geometry_solvers.cuh sampson_sq)."""
    E = np.asarray(E, np.float64)[..., None, :]
    x0, y0, x1, y1 = (np.asarray(pts, np.float64)[:, k] for k in range(4))
    a0 = E[..., 0] * x0 + E[..., 1] * y0 + E[..., 2]
    a1 = E[..., 3] * x0 + E[..., 4] * y0 + E[..., 5]
    a2 = E[..., 6] * x0 + E[..., 7] * y0 + E[..., 8]
    b0 = E[..., 0] * x1 + E[..., 3] * y1 + E[..., 6]
    b1 = E[..., 1] * x1 + E[..., 4] * y1 + E[..., 7]
    num = x1 * a0 + y1 * a1 + a2
    return num * num / (a0 * a0 + a1 * a1 + b0 * b0 + b1 * b1)


def sampson_sq_f_bound(E, pts, e_abs=0.0):
    """(d2, lo, hi) [..., N]: float64 Sampson^2 of the float32 model E [..., 9] and an interval [lo, hi] that holds the
    kernel's float32 evaluation sampson_sq_f. Each of a0..a2, b0, b1 is two fmaf (|err| <= 2u sum |terms|); num is two
    more fmaf on those; den is four fmaf / fmul on their squares; num * num is one rounding and __fdividef is within
    2 ulp (4u). The interval is that of num^2 / den over those errors, widened by the last two roundings. ``e_abs`` adds
    an absolute error of every coefficient of E: the kernel may score a model that differs by that much from E."""
    E = np.asarray(E, np.float64)[..., None, :]
    x0, y0, x1, y1 = (np.asarray(pts, np.float64)[:, k] for k in range(4))
    c = 2 * U32

    def lin(e0, e1, e2, s, t):
        v = e0 * s + e1 * t + e2
        return v, c * (np.abs(e0 * s) + np.abs(e1 * t) + np.abs(e2)) + e_abs * (np.abs(s) + np.abs(t) + 1.0)
    a0, da0 = lin(E[..., 0], E[..., 1], E[..., 2], x0, y0)
    a1, da1 = lin(E[..., 3], E[..., 4], E[..., 5], x0, y0)
    a2, da2 = lin(E[..., 6], E[..., 7], E[..., 8], x0, y0)
    b0, db0 = lin(E[..., 0], E[..., 3], E[..., 6], x1, y1)
    b1, db1 = lin(E[..., 1], E[..., 4], E[..., 7], x1, y1)
    num = x1 * a0 + y1 * a1 + a2
    n_abs = np.abs(x1) * (np.abs(a0) + da0) + np.abs(y1) * (np.abs(a1) + da1) + np.abs(a2) + da2
    dnum = np.abs(x1) * da0 + np.abs(y1) * da1 + da2 + 2 * U32 * n_abs
    den = a0 * a0 + a1 * a1 + b0 * b0 + b1 * b1
    sq = lambda v, dv: 2 * np.abs(v) * dv + dv * dv
    d_abs = (np.abs(a0) + da0) ** 2 + (np.abs(a1) + da1) ** 2 + (np.abs(b0) + db0) ** 2 + (np.abs(b1) + db1) ** 2
    dden = sq(a0, da0) + sq(a1, da1) + sq(b0, db0) + sq(b1, db1) + 4 * U32 * d_abs
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        d2 = num * num / den
        hi = (np.abs(num) + dnum) ** 2 / np.maximum(den - dden, 0.0) * (1 + 5.01 * U32)
        lo = np.maximum(np.abs(num) - dnum, 0.0) ** 2 / (den + dden) * (1 - 5.01 * U32)
    return d2, np.minimum(lo, d2), np.where(np.isnan(hi), np.inf, np.maximum(hi, d2))


def msac_f_bound(E32, pts, thr2_f, e_abs=0.0):
    """(cost, bound, d2, lo, hi) for the kernel's float32 MSAC cost sum min(d2, thr2) of the float32 models E32 [C, 9]:
    the float64 cost; a bound on the kernel's cost from the per-point intervals of ``sampson_sq_f_bound`` clamped at thr2
    (a point surely outside adds exactly thr2) plus the float32 summation (N / 32 sequential adds per lane, five shuffle
    levels); and the per-point d2 and its interval."""
    thr2 = float(thr2_f)
    d2, lo, hi = sampson_sq_f_bound(E32, pts, e_abs)
    m = np.minimum(d2, thr2)
    err = np.maximum(np.minimum(hi, thr2) - m, m - np.minimum(lo, thr2))
    cost = m.sum(-1)
    n = len(pts)
    bound = err.sum(-1) + (-(-n // 32) + 6) * U32 * (cost + err.sum(-1))
    return cost, bound, d2, lo, hi


def emat_hypotheses(pts, N, num_hyp, hpb, seed, pair):
    """Every hypothesis of one pair in the kernel's order. Returns a list over blocks of lists of candidate records
    (warp, lane, c, E [9] float64), for hypotheses h = block * hpb + thread < num_hyp."""
    x = np.asarray(pts[:N], np.float64)
    blocks = -(-num_hyp // hpb)
    out = []
    for b in range(blocks):
        cands = []
        for th in range(hpb):
            h = b * hpb + th
            if h >= num_hyp:
                break
            idx = sample_distinct(emat_state(seed, pair, h), N, 5)
            for c, E in enumerate(five_point(x[idx, 0:2], x[idx, 2:4])):
                cands.append((th >> 5, th & 31, c, E))
        out.append(cands)
    return out


def emat_select(res):
    """emat_stage_in: block indices of the (up to) four cheapest valid block winners, cheapest first, ties in block
    order. ``res``: the HYP_DTYPE records of one pair."""
    valid = [k for k in range(len(res)) if res[k]["valid"]]
    return sorted(valid, key=lambda k: (float(res[k]["cost"]), k))[:LO_TOPK]


def cheirality(R, t, pts):
    """cheirality_ok for every point: both triangulated depths positive and below 1e9."""
    x = np.asarray(pts, np.float64)
    d0 = np.stack([x[:, 0], x[:, 1], np.ones(len(x))], 1)
    d1 = np.stack([x[:, 2], x[:, 3], np.ones(len(x))], 1)
    a = d0 @ np.asarray(R).reshape(3, 3).T
    aa, bb, ab = (a * a).sum(1), (d1 * d1).sum(1), (a * d1).sum(1)
    at, bt = a @ t, d1 @ t
    det = aa * bb - ab * ab
    with np.errstate(divide="ignore", invalid="ignore"):
        l0 = (-at * bb + ab * bt) / det
        l1 = (aa * bt - ab * at) / det
    return (np.abs(det) > 1e-300) & (l0 > 0) & (l1 > 0) & (l0 < 1e9) & (l1 < 1e9)


def choose_pose(E, pts, thr2):
    """emat_choose_pose: the decomposition (R1, t), (R2, t), (R1, -t), (R2, -t) with the most points in front of both
    cameras among those with Sampson^2 < thr2, the first on ties. Returns (R, t, votes [4], near) where ``near`` counts
    the points whose Sampson^2 lies within 1e-12 relative of thr2 (where float64 rounding order can decide the vote)."""
    R1, R2, t = decompose_essential(E)
    d2 = sampson_sq(np.asarray(E).reshape(9), pts)
    inl = d2 < thr2
    near = int((np.abs(d2 - thr2) <= 1e-12 * thr2).sum())
    cands = [(R1, t), (R2, t), (R1, -t), (R2, -t)]
    votes = [int((inl & cheirality(R, tt, pts)).sum()) for R, tt in cands]
    b = 0
    for k in range(1, 4):
        if votes[k] > votes[b]:
            b = k
    return cands[b][0], cands[b][1], votes, near


def msac(R, t, pts, thr2):
    """emat_msac: sum min(Sampson^2, thr2) in float64."""
    return float(np.minimum(sampson_sq(essential_from_rt(R, t).reshape(9), pts), thr2).sum())


def sampson_res_jac(R, t, b1, b2, pts):
    """sampson_res_jac for every point: signed Sampson residual r [N] and its Jacobian J [N, 5] with respect to
    (rotation increment, tangent increment of t)."""
    x = np.asarray(pts, np.float64)
    n = len(x)
    x0 = np.stack([x[:, 0], x[:, 1], np.ones(n)], 1)
    x1 = np.stack([x[:, 2], x[:, 3], np.ones(n)], 1)
    y = x0 @ R.T
    a = np.cross(t, y)
    w = np.cross(t, x1)
    b = -(w @ R)
    num = (x1 * a).sum(1)
    s = a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2
    is_ = 1.0 / np.sqrt(s)
    r = num * is_
    c2 = -0.5 * num * is_ ** 3
    J = np.zeros((n, 5))
    for k in range(5):
        if k < 3:
            ek = np.eye(3)[k]
            da = np.cross(t, np.cross(ek, y))
            db = np.cross(ek, w) @ R
        else:
            bj = b1 if k == 3 else b2
            da = np.cross(bj, y)
            db = -(np.cross(bj, x1) @ R)
        dn = (x1 * da).sum(1)
        ds = 2.0 * (a[:, 0] * da[:, 0] + a[:, 1] * da[:, 1] + b[:, 0] * db[:, 0] + b[:, 1] * db[:, 1])
        J[:, k] = dn * is_ + c2 * ds
    return r, J


def lm_round(R, t, pts, T2, step=1, hard=False, max_it=LO_INNER):
    """emat_lm_round: LM on the Tukey biweight (or, hard, the truncated least squares) of the Sampson residual with
    cut-off sqrt(T2), over every ``step``-th point, from (R, t). Returns the last accepted (R, t)."""
    sub = np.asarray(pts)[::step]
    lam, prev_cost, done = 1e-6, 1e300, False
    pR, pt = R.copy(), t.copy()
    H = np.zeros((5, 5)); g = np.zeros(5)
    for it in range(max_it + 1):
        if done:
            break
        b1, b2 = tangent_basis(t)
        r, J = sampson_res_jac(R, t, b1, b2, sub)
        q = r * r / T2
        m = q < 1.0
        u = 1.0 - q[m]
        wgt = np.ones(m.sum()) if hard else u * u
        Jm = J[m]
        Hn = (Jm * wgt[:, None]).T @ Jm
        gn = Jm.T @ (wgt * r[m])
        cost = float((q[m] if hard else 1.0 - u ** 3).sum() + (~m).sum())
        if cost <= prev_cost:
            if prev_cost - cost <= 1e-10 * cost:
                done = True
            prev_cost = cost
            pR, pt = R.copy(), t.copy()
            H, g = Hn, gn
            lam = max(lam * 0.1, 1e-12)
        else:
            lam *= 10.0
        pb1, pb2 = tangent_basis(pt)
        d = solve_damped(H, g, lam) if it < max_it else None
        if d is not None:
            R = so3_exp(d[:3]) @ pR
            tn = pt + d[3] * pb1 + d[4] * pb2
            t = tn / np.linalg.norm(tn)
        else:
            R, t = pR.copy(), pt.copy()
    return pR, pt


def emat_lo(E, pts, thr2, lo):
    """emat_lo_kernel for one candidate: pose choice from E, then (lo != 0) the six LM rounds at cut-offs
    {3, 2, 1.5, 1, 1, 1} x thr over every ceil(N / 1024)-th point; cost = float64 MSAC at thr2 over all points.
    Returns (cost, R, t, votes [4] of the pose choice, near)."""
    N = len(pts)
    R, t, votes, near = choose_pose(E, pts, thr2)
    if lo:
        step = -(-N // LO_MAX_PTS)
        for s in LO_SCHEDULE:
            R, t = lm_round(R, t, pts, s * s * thr2, step)
    return msac(R, t, pts, thr2), R, t, votes, near


def tighten_cutoff(R, t, pts, thr):
    """One tightening round's cut-off of emat_final_kernel: the 256-bin histogram of sqrt(d2 / thr2) over the points
    with d2 < thr2, the median bin, sigma = 1.4826 (med + 1) / 256 thr, cut-off clamp(3 sigma, 0.02 thr, thr). Returns
    (cut-off, edge) with ``edge`` the number of points within 1e-12 of a bin edge or of thr2 (where float64 rounding
    can move a point to the next bin)."""
    thr2 = thr * thr
    d2 = sampson_sq(essential_from_rt(R, t).reshape(9), pts)
    m = d2 < thr2
    v = np.sqrt(d2[m] / thr2) * 256.0
    k = np.round(v)
    edge = int(((np.abs(v - k) <= 1e-12 * np.maximum(v, 1.0)) & (k >= 1) & (k <= 255)).sum()
               + (np.abs(d2 - thr2) <= 1e-12 * thr2).sum())
    hist = np.bincount(np.minimum(255, v.astype(np.int64)), minlength=256)
    tot = int(hist.sum())
    acc = np.cumsum(hist)
    hit = np.nonzero(2 * acc >= tot)[0]
    med = int(hit[0]) if len(hit) else 255
    sigma = 1.4826 * (med + 1) / 256.0 * thr
    return min(thr, max(3.0 * sigma, 0.02 * thr)), edge


def emat_final(lo_res, pts, thr, lo):
    """emat_final_kernel after the stage-in: the cheapest LO candidate (first on ties), with lo & 1 three tightening
    rounds and the 1.02 safeguard, with lo & 2 four hard LM rounds at thr, then the pose choice under the final E and the
    mask Sampson^2 < thr2 and cheirality. Returns dict(R, t, mask, votes [4], near, edge, failed)."""
    thr2 = thr * thr
    costs = [float(r["cost"]) for r in lo_res]
    bc = 0
    for c in range(1, LO_TOPK):
        if costs[c] < costs[bc]:
            bc = c
    out = {"near": 0, "edge": 0, "failed": not costs[bc] < 1e299}
    if out["failed"]:
        return out
    best_cost = costs[bc]
    bR, bt = np.asarray(lo_res[bc]["R"], np.float64).reshape(3, 3), np.asarray(lo_res[bc]["t"], np.float64)
    R, t = bR.copy(), bt.copy()
    if lo:
        for _ in range(TIGHT_ROUNDS):
            T, e = tighten_cutoff(R, t, pts, thr)
            out["edge"] += e
            R, t = lm_round(R, t, pts, T * T)
        cost = msac(R, t, pts, thr2)
        if cost > 1.02 * best_cost:
            R, t = bR.copy(), bt.copy()
        if lo & 2:
            for _ in range(4):
                R, t = lm_round(R, t, pts, thr2, 1, True, 8)
    E = essential_from_rt(R, t)
    Rc, tc, votes, near = choose_pose(E, pts, thr2)
    d2 = sampson_sq(E.reshape(9), pts)
    mask = (d2 < thr2) & cheirality(Rc, tc, pts)
    out.update(R=Rc, t=tc, mask=mask, votes=votes, near=near + int((np.abs(d2 - thr2) <= 1e-12 * thr2).sum()))
    out["failed"] = not mask.any()
    return out


# ------------------------------------------------------------------------------------------------ scale from depth
def inverse_K_f32(K):
    """inverse_K_f32: the adjugate of the float32 K over its determinant in float64, rounded to float32."""
    A = np.asarray(K, np.float32).astype(np.float64).reshape(9)
    d = (A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]))
    inv = np.array([A[4] * A[8] - A[5] * A[7], A[2] * A[7] - A[1] * A[8], A[1] * A[5] - A[2] * A[4],
                    A[5] * A[6] - A[3] * A[8], A[0] * A[8] - A[2] * A[6], A[2] * A[3] - A[0] * A[5],
                    A[3] * A[7] - A[4] * A[6], A[1] * A[6] - A[0] * A[7], A[0] * A[4] - A[1] * A[3]]) / d
    return inv.astype(np.float32).reshape(3, 3)


def backproject(Ki, uv, z):
    """backproject: z * (Ki @ (u, v, 1)) in float64 from the float32 inverse and integer pixels."""
    uv = np.asarray(uv, np.float64)
    h = np.stack([uv[:, 0], uv[:, 1], np.ones(len(uv))], 1)
    return np.asarray(z, np.float64)[:, None] * (h @ np.asarray(Ki, np.float64).T)


def scale_consensus(R, t, mask, kpts0, kpts1, depth0, depth1, K0, K1, scale_thr):
    """scale_consensus_kernel for one pair: per masked point with both truncated pixels inside the images and both
    depths > 0, the scale (X1 - R X0) . t; the first scale with the most others within scale_thr. Returns (R, t_metric,
    count) or None on failure (NaN pose or no valid point)."""
    if not (np.isfinite(R).all() and np.isfinite(t).all()):
        return None
    H, W = depth0.shape
    i0, i1 = np.asarray(kpts0, np.float32).astype(np.int32), np.asarray(kpts1, np.float32).astype(np.int32)
    ok = np.asarray(mask, bool) & (i0[:, 0] >= 0) & (i0[:, 0] < W) & (i0[:, 1] >= 0) & (i0[:, 1] < H)
    ok &= (i1[:, 0] >= 0) & (i1[:, 0] < W) & (i1[:, 1] >= 0) & (i1[:, 1] < H)
    z0 = np.zeros(len(ok), np.float32); z1 = np.zeros(len(ok), np.float32)
    z0[ok] = depth0[i0[ok, 1], i0[ok, 0]]; z1[ok] = depth1[i1[ok, 1], i1[ok, 0]]
    ok &= (z0 > 0) & (z1 > 0)
    if not ok.any():
        return None
    X0 = backproject(inverse_K_f32(K0), i0[ok], z0[ok])
    X1 = backproject(inverse_K_f32(K1), i1[ok], z1[ok])
    s = (X1 - X0 @ np.asarray(R, np.float64).T) @ np.asarray(t, np.float64)
    cnt = (np.abs(s[None, :] - s[:, None]) < scale_thr).sum(1)
    b = int(np.argmax(cnt))
    return np.asarray(R, np.float64), s[b] * np.asarray(t, np.float64), int(cnt[b])


# ------------------------------------------------------------------------------------------------ PnP
def depth_min(depth):
    """depth_min_kernel: the map minimum clamped at 0 (the reference's depth0.min() for the dataset's non-negative
    depths)."""
    return np.float32(max(float(np.min(depth)), 0.0))


def pnp_prepare(kpts0, kpts1, depth0, K0, dmin):
    """pnp_prepare_kernel for one pair: keypoints of image 0 truncated toward zero (np.int32), valid iff inside the image
    and depth > dmin, in order. Returns (vidx, Xw [n, 3] float64 camera-0 points, uv [n, 2] float32 kpts1)."""
    H, W = depth0.shape
    k0 = np.asarray(kpts0, np.float32)
    ik = k0.astype(np.int32)
    inside = (ik[:, 0] >= 0) & (ik[:, 0] < W) & (ik[:, 1] >= 0) & (ik[:, 1] < H)
    z = np.zeros(len(k0), np.float32)
    z[inside] = depth0[ik[inside, 1], ik[inside, 0]]
    vidx = np.nonzero(inside & (z > dmin))[0]
    return vidx, backproject(inverse_K_f32(K0), ik[vidx], z[vidx]), np.asarray(kpts1, np.float32)[vidx]


def pnp_model(Xw, uv, K1, idx):
    """One PnP hypothesis: P3P on the first three sampled points (bearings from the float32 uv and K1 in float64), the
    solution that reprojects the 4th point best among those in front of the camera. Returns (R, t) or None."""
    K1 = np.asarray(K1, np.float32).reshape(3, 3).astype(np.float64)
    fx, fy, cx, cy = K1[0, 0], K1[1, 1], K1[0, 2], K1[1, 2]
    u = np.asarray(uv, np.float64)
    b = np.stack([(u[idx[:3], 0] - cx) / fx, (u[idx[:3], 1] - cy) / fy, np.ones(3)], 1)
    f = b / np.sqrt((b * b).sum(1))[:, None]
    Rs, ts = p3p(Xw[idx[:3]], f)
    best, out = 1e300, None
    for R, t in zip(Rs, ts):
        Xc = R @ Xw[idx[3]] + t
        if not Xc[2] > 1e-9:
            continue
        e = (fx * Xc[0] / Xc[2] + cx - u[idx[3], 0]) ** 2 + (fy * Xc[1] / Xc[2] + cy - u[idx[3], 1]) ** 2
        if e < best:
            best, out = e, (R, t)
    return out


def pnp_count_bound(R, t, Xw, uv, K1, thr):
    """(lo, hi) [N] bool: the points the kernel's float32 reprojection test (R, t and X rounded to float32, fmaf chains,
    1 / zc, fmaf projection, du^2 + dv^2 < thr^2) must count (lo) and may count (hi). The float64 squared error e of the
    float32-rounded inputs is bounded by first-order propagation of u per operation, with a factor 2 for the terms
    dropped; points with zc near 1e-6 count as undecided."""
    K1 = np.asarray(K1, np.float32).reshape(3, 3).astype(np.float64)
    fx, fy, cx, cy = K1[0, 0], K1[1, 1], K1[0, 2], K1[1, 2]
    R32 = np.asarray(R, np.float32).astype(np.float64).reshape(3, 3)
    t32 = np.asarray(t, np.float32).astype(np.float64)
    X = np.asarray(Xw, np.float32).astype(np.float64)
    u = np.asarray(uv, np.float64)
    Xc = X @ R32.T + t32
    S = np.abs(X) @ np.abs(R32).T + np.abs(t32)
    dX = 4 * U32 * S
    xc, yc, zc = Xc[:, 0], Xc[:, 1], Xc[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        px, py = xc / zc, yc / zc
        dpx = dX[:, 0] / np.abs(zc) + np.abs(px) * (dX[:, 2] / np.abs(zc) + 3 * U32)
        dpy = dX[:, 1] / np.abs(zc) + np.abs(py) * (dX[:, 2] / np.abs(zc) + 3 * U32)
        du = fx * px + cx - u[:, 0]
        dv = fy * py + cy - u[:, 1]
        ddu = fx * dpx + 2 * U32 * (np.abs(fx * px) + abs(cx) + np.abs(u[:, 0]))
        ddv = fy * dpy + 2 * U32 * (np.abs(fy * py) + abs(cy) + np.abs(u[:, 1]))
        e = du * du + dv * dv
        de = 2 * (2 * np.abs(du) * ddu + ddu * ddu + 2 * np.abs(dv) * ddv + ddv * ddv + 2 * U32 * e)
    thr2 = float(np.float32(np.float32(thr) * np.float32(thr)))
    front_sure = zc - dX[:, 2] > 1e-6
    front_may = zc + dX[:, 2] > 1e-6
    lo = front_sure & (e + de < thr2)
    hi = front_may & ~(e - de >= thr2)
    return lo, hi


def pnp_hypotheses(Xw, uv, K1, num_hyp, seed, pair):
    """Every PnP hypothesis of one pair in the kernel's order: list over blocks of lists of (warp, lane, R, t)."""
    N = len(Xw)
    out = []
    for b in range(-(-num_hyp // HYP_PER_BLOCK)):
        cands = []
        for th in range(HYP_PER_BLOCK):
            h = b * HYP_PER_BLOCK + th
            if h >= num_hyp:
                break
            m = pnp_model(Xw, uv, K1, sample_distinct(pnp_state(seed, pair, h), N, 4))
            if m is not None:
                cands.append((th >> 5, th & 31) + m)
        out.append(cands)
    return out


def pnp_winner(res):
    """pnp_final_kernel's record: the first valid block with the lowest cost (-count), or None."""
    b = None
    for k in range(len(res)):
        if res[k]["valid"] and (b is None or res[k]["cost"] < res[b]["cost"]):
            b = k
    return b


def pnp_inliers(R, t, Xw, uv, K1, thr):
    """pnp_final_kernel's inlier test in float64 under the winning record: (inlier [N], near [N]) where ``near`` marks
    points within 1e-12 relative of thr^2."""
    K1 = np.asarray(K1, np.float32).reshape(3, 3).astype(np.float64)
    fx, fy, cx, cy = K1[0, 0], K1[1, 1], K1[0, 2], K1[1, 2]
    Xc = np.asarray(Xw, np.float64) @ np.asarray(R, np.float64).reshape(3, 3).T + np.asarray(t, np.float64)
    thr2 = float(np.float32(thr)) ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        du = fx * Xc[:, 0] / Xc[:, 2] + cx - uv[:, 0]
        dv = fy * Xc[:, 1] / Xc[:, 2] + cy - uv[:, 1]
        e = du * du + dv * dv
    front = Xc[:, 2] > 1e-9
    return front & (e < thr2), front & (np.abs(e - thr2) <= 1e-12 * thr2)


def pnp_lm(R, t, Xw, uv, K1, iters=PNP_ITERS):
    """pnp_final_kernel's LM on a fixed inlier set: reprojection residuals, parameters = left rotation increment and
    translation increment, the same accept / reject and damping as emat_lm_round, ``iters`` steps."""
    K1 = np.asarray(K1, np.float32).reshape(3, 3).astype(np.float64)
    fx, fy, cx, cy = K1[0, 0], K1[1, 1], K1[0, 2], K1[1, 2]
    X = np.asarray(Xw, np.float64)
    u = np.asarray(uv, np.float64)
    R, t = np.asarray(R, np.float64).reshape(3, 3).copy(), np.asarray(t, np.float64).copy()
    pR, pt = R.copy(), t.copy()
    lam, prev = 1e-6, 1e300
    H = np.zeros((6, 6)); g = np.zeros(6)
    for it in range(iters + 1):
        RX = X @ R.T
        Xc = RX + t
        iz = 1.0 / Xc[:, 2]
        ru = fx * Xc[:, 0] * iz + cx - u[:, 0]
        rv = fy * Xc[:, 1] * iz + cy - u[:, 1]
        a0, a2 = fx * iz, -fx * Xc[:, 0] * iz * iz
        b1, b2 = fy * iz, -fy * Xc[:, 1] * iz * iz
        z = np.zeros(len(X))
        Ju = np.stack([a2 * RX[:, 1], a0 * RX[:, 2] - a2 * RX[:, 0], -a0 * RX[:, 1], a0, z, a2], 1)
        Jv = np.stack([-b1 * RX[:, 2] + b2 * RX[:, 1], -b2 * RX[:, 0], b1 * RX[:, 0], z, b1, b2], 1)
        cost = float((ru * ru + rv * rv).sum())
        if cost <= prev:
            prev = cost
            pR, pt = R.copy(), t.copy()
            H = Ju.T @ Ju + Jv.T @ Jv
            g = Ju.T @ ru + Jv.T @ rv
            lam = max(lam * 0.1, 1e-12)
        else:
            lam *= 10.0
        d = solve_damped(H, g, lam) if it < iters else None
        if d is not None:
            R = so3_exp(d[:3]) @ pR
            t = pt + d[3:]
        else:
            R, t = pR.copy(), pt.copy()
    return pR, pt


def pnp_final(res, Xw, uv, K1, thr):
    """pnp_final_kernel for one pair from its block records: dict(failed, mask over the compacted points, near, n_in,
    R, t). n_in < 4 fails; n_in >= 6 runs the LM on the fixed inlier set; |t| > 1000 fails."""
    b = pnp_winner(res) if len(Xw) >= 4 else None
    if b is None:
        return {"failed": True, "mask": np.zeros(len(Xw), bool), "near": np.zeros(len(Xw), bool), "n_in": 0}
    R0 = np.asarray(res[b]["model"][:9], np.float64).reshape(3, 3)
    t0 = np.asarray(res[b]["model"][9:], np.float64)
    inl, near = pnp_inliers(R0, t0, Xw, uv, K1, thr)
    n_in = int(inl.sum())
    out = {"mask": inl, "near": near, "n_in": n_in, "R": R0, "t": t0, "record": b}
    if n_in < 4:
        out.update(failed=True, mask=np.zeros(len(Xw), bool))
        return out
    if n_in >= 6:
        out["R"], out["t"] = pnp_lm(R0, t0, Xw[inl], uv[inl], K1)
    out["failed"] = not np.linalg.norm(out["t"]) <= 1000.0
    if out["failed"]:
        out["mask"] = np.zeros(len(Xw), bool)
    return out


# ------------------------------------------------------------------------------------------------ Procrustes
def procrustes_state(seed, pair, h):
    return (seed ^ (0xC2B2AE3D27D4EB4F * (pair + 1)) ^ (0x9E3779B97F4A7C15 * (h + 1))) & M64


def kabsch_sums(p, q):
    """Moment sums (n, sum p [3], sum q [3], sum p q^T [9]) of p, q [n, 3]."""
    return float(len(p)), p.sum(0), q.sum(0), (p[:, :, None] * q[:, None, :]).sum(0).ravel()


def kabsch(n, sp, sq, spq):
    """kabsch_from_sums through its host hook mfr_host_kabsch: (R [3, 3], t [3]) or None."""
    R, t = np.zeros(9), np.zeros(3)
    c = lambda a: np.ascontiguousarray(a, np.float64)
    sp, sq, spq = c(sp), c(sq), c(spq)
    if not _lib().mfr_host_kabsch(float(n), _p(sp), _p(sq), _p(spq), _p(R), _p(t)):
        return None
    return R.reshape(3, 3), t


def procrustes_prepare(kpts0, kpts1, depth0, depth1, K0, K1, dmin0, dmin1):
    """procrustes_prepare_kernel for one pair: both keypoints truncated toward zero and inside both images, valid iff
    depth > dmin on both sides, in order. Returns (vidx, X0 [n, 3], X1 [n, 3]) float64 camera points."""
    H, W = depth0.shape
    i0, i1 = np.asarray(kpts0, np.float32).astype(np.int32), np.asarray(kpts1, np.float32).astype(np.int32)
    inside = ((i0[:, 0] >= 0) & (i0[:, 0] < W) & (i0[:, 1] >= 0) & (i0[:, 1] < H) &
              (i1[:, 0] >= 0) & (i1[:, 0] < W) & (i1[:, 1] >= 0) & (i1[:, 1] < H))
    z0 = np.zeros(len(i0), np.float32); z1 = np.zeros(len(i0), np.float32)
    z0[inside] = depth0[i0[inside, 1], i0[inside, 0]]; z1[inside] = depth1[i1[inside, 1], i1[inside, 0]]
    vidx = np.nonzero(inside & (z0 > dmin0) & (z1 > dmin1))[0]
    return (vidx, backproject(inverse_K_f32(K0), i0[vidx], z0[vidx]), backproject(inverse_K_f32(K1), i1[vidx], z1[vidx]))


def procrustes_count_bound(R, t, X0, X1, max_dist):
    """(lo, hi) [N] bool: the points procrustes_hyp_kernel's float32 test (R, t, X0, X1 rounded to float32, three fmaf
    per component, a subtraction, d2 = fmaf(dx, dx, fmaf(dy, dy, dz * dz)) < float32 max_dist^2) must count (lo) and may
    count (hi). Each component's error is at most 4 u of the sum of the magnitudes it is made of, d2's at most 3 u of
    d2 on top of the propagated component errors."""
    R32 = np.asarray(R, np.float32).astype(np.float64).reshape(3, 3)
    t32 = np.asarray(t, np.float32).astype(np.float64)
    P = np.asarray(X0, np.float32).astype(np.float64)
    Q = np.asarray(X1, np.float32).astype(np.float64)
    d = P @ R32.T + t32 - Q
    dd = 4 * U32 * (np.abs(P) @ np.abs(R32).T + np.abs(t32) + np.abs(Q))
    e = (d * d).sum(1)
    de = (2 * np.abs(d) * dd + dd * dd).sum(1) + 3 * U32 * (e + (2 * np.abs(d) * dd + dd * dd).sum(1))
    thr2 = float(np.float32(np.float32(max_dist) * np.float32(max_dist)))
    return e + de < thr2, ~(e - de >= thr2)


def procrustes_hypotheses(X0, X1, num_hyp, seed, pair):
    """Every Procrustes hypothesis of one pair in the kernel's order: list over blocks of lists of (warp, lane, R, t)
    for the 3-point samples whose Kabsch model exists."""
    N = len(X0)
    out = []
    for b in range(-(-num_hyp // HYP_PER_BLOCK)):
        cands = []
        for th in range(HYP_PER_BLOCK):
            h = b * HYP_PER_BLOCK + th
            if h >= num_hyp:
                break
            idx = sample_distinct(procrustes_state(seed, pair, h), N, 3)
            m = kabsch(*kabsch_sums(X0[idx], X1[idx]))
            if m is not None:
                cands.append((th >> 5, th & 31) + m)
        out.append(cands)
    return out


def procrustes_final(res, X0, X1, max_dist):
    """procrustes_final_kernel for one pair from its block records: the first valid block with the lowest cost, then
    two refits on the inliers (d^2 < max_dist^2 in float64) and a final count. Returns dict(failed, R, t, n, near) where
    ``near`` counts points within 1e-12 (relative) of the threshold in any round."""
    thr2 = float(np.float32(max_dist)) ** 2
    b = pnp_winner(res) if len(X0) >= 3 else None
    if b is None:
        return {"failed": True, "n": 0, "near": 0}
    R = np.asarray(res[b]["model"][:9], np.float64).reshape(3, 3)
    t = np.asarray(res[b]["model"][9:], np.float64)
    near = 0
    for rnd in range(3):
        d2 = ((X0 @ R.T + t - X1) ** 2).sum(1)
        inl = d2 < thr2
        near += int((np.abs(d2 - thr2) <= 1e-12 * thr2).sum())
        if rnd < 2:
            m = kabsch(*kabsch_sums(X0[inl], X1[inl]))
            if m is not None:
                R, t = m
    n = int(inl.sum())
    return {"failed": n < 3, "R": R, "t": t, "n": n, "near": near, "record": b}


# ------------------------------------------------------------------------------------------------ ICP
def icp_clouds(depth0, depth1, K0, K1):
    """The clouds icp_assoc_kernel lifts: every pixel with depth > 0, through the float32 inverse of K, row-major.
    Returns (X0 [n0, 3], X1 [n1, 3]) float64."""
    H, W = depth0.shape
    vv, uu = np.mgrid[0:H, 0:W]
    uv = np.stack([uu.ravel(), vv.ravel()], 1)
    m0, m1 = depth0.ravel() > 0, depth1.ravel() > 0
    return (backproject(inverse_K_f32(K0), uv[m0], depth0.ravel()[m0]),
            backproject(inverse_K_f32(K1), uv[m1], depth1.ravel()[m1]))


def icp_assoc(X0, X1, R, t, max_dist, tree=None):
    """One association pass of icp_assoc_kernel, exact: the nearest target point within D (float64 of the float32
    max_dist) of every transformed source point by cKDTree. Source points at z <= D + 1 mm in camera 1 are not
    associated, as in the kernel. Returns dict(n, sums [16] = (sum p, sum q, sum p q^T), sse, rmse, near, P, Q, ok)
    with ``near`` the count of points whose distance lies within 1e-9 (relative) of D."""
    from scipy.spatial import cKDTree
    D = float(np.float32(max_dist))
    tree = cKDTree(X1) if tree is None else tree
    P = X0 @ np.asarray(R, np.float64).reshape(3, 3).T + np.asarray(t, np.float64)
    front = P[:, 2] > D + 1e-3
    d, j = tree.query(P, k=1, distance_upper_bound=D * (1 + 1e-9))
    fin = np.isfinite(d)
    near = int((fin & front & (np.abs(d - D) <= 1e-9 * D)).sum())
    ok = fin & front & (d < D)
    Pm, Qm = P[ok], X1[j[ok]]
    n = int(ok.sum())
    sse = float((((Pm - Qm) ** 2).sum(1)).sum())
    _, sp, sq, spq = kabsch_sums(Pm, Qm)
    return {"n": n, "sums": np.concatenate([sp, sq, spq]), "sse": sse, "rmse": np.sqrt(sse / n) if n else 0.0,
            "near": near, "ok": ok}


def icp_update(state_prev, a, n_src, it, rel_fit, rel_rmse):
    """icp_update_kernel for one pair: state_prev = (R [3, 3], t [3], fitness, rmse) of the previous pass, a = icp_assoc
    at R, t. Returns (R, t, fitness, rmse, stop): stop when it > 0 and both changes are below the criteria, when n < 3,
    or when Kabsch fails; otherwise the Kabsch update composed onto the pose."""
    R, t, fit0, rmse0 = state_prev
    n = a["n"]
    fit = n / n_src if n_src > 0 else 0.0
    rmse = a["rmse"]
    if (it > 0 and abs(fit0 - fit) < rel_fit and abs(rmse0 - rmse) < rel_rmse) or n < 3:
        return R, t, fit, rmse, True
    m = kabsch(n, a["sums"][:3], a["sums"][3:6], a["sums"][6:])
    if m is None:
        return R, t, fit, rmse, True
    Ru, tu = m
    return Ru @ R, Ru @ t + tu, fit, rmse, False


def icp_loop(X0, X1, R, t, max_dist, max_iter=30, rel_fit=1e-4, rel_rmse=1e-4):
    """mfr_icp_refine restated: passes it = 0 .. max_iter of association + update (the last pass only evaluates).
    Returns (R, t, fitness, rmse, stop pass, converged flag)."""
    from scipy.spatial import cKDTree
    tree = cKDTree(X1)
    R, t = np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64)
    fit, rmse = 0.0, 0.0
    for it in range(max_iter + 1):
        last = it == max_iter
        a = icp_assoc(X0, X1, R, t, max_dist, tree)
        R, t, fit, rmse, stop = icp_update((R, t, fit, rmse), a, len(X0), it, 1e300 if last else rel_fit,
                                           1e300 if last else rel_rmse)
        if stop:
            return R, t, fit, rmse, it, True
    return R, t, fit, rmse, max_iter, False
