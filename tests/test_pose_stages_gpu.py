"""Each stage of the pose back end (csrc/geometry.cu) against a float64 restatement, fed with the device's own input.

Every check reads the stage's input from the solver handle (``PoseBackend.debug_tensor``: the normalised points, the
block winners, the LO candidates, the final fp64 pose, PnP's compacted points) and recomputes the stage with
``oracle/pose_stages_oracle.py``, so the error of one stage does not add up with the error of the stages before it. The
RNG (splitmix64 seeded from seed, pair and hypothesis index) and the minimal solvers (the library's host hooks) are
restated too, so the hypothesis kernels are checked block by block.

Bars. The normalisation, the PnP compaction, the candidate order, the vote counts and the masks are exact (a mask bit
may differ only at a point within 1e-12 relative of the threshold). The float32 hypothesis scoring is held to a bound
derived from its arithmetic (``sampson_sq_f_bound``, ``pnp_count_bound``): the stored cost within the bound of the
float64 cost of the stored model, no candidate of the block cheaper by more than the two bounds, the inlier count
between the counts of the points surely and possibly inside. The other candidates of a block are the host solver's,
which stand for the kernel's only up to the solver bar below; their bound includes that difference as an absolute error
of every coefficient of the unit-norm E. The float64 stages (pose choice, LO, the final refit,
PnP's LM) must agree with the restatement to summation-order noise; where no bar follows from the arithmetic, the bar
is at most 4x the maximum measured on one NVIDIA H100 80GB HBM3 (700 W power limit) over all cases:

  stage                                          bar                 measured
  emat winner model vs host 5-point candidate    1e-4 (unit E)       6.3e-5
  emat block cost                                |d| / bound <= 1    0.15
  pose choice (lo = 0)                           1e-12               1.6e-15
  LO pose (lo = 1, 3)                            2.4e-9              5.9e-10
  LO cost, relative                              3.7e-12             2.8e-12
  final pose Rd / td (lo = 0, 1)                 1e-12 / 7e-9        2.6e-15
  final pose Rd / td (lo = 3)                    7e-9                1.8e-9
  PnP winner model vs host P3P candidate         7e-9                1.9e-9
  PnP Xw                                         4 ulp               0
  PnP pose vs the LM restatement (float32 R, t)  1.1e-7              2.8e-8
  PnP LM vs cv2.solvePnPGeneric (ITERATIVE)      1.2e-7              3.0e-8

The 5-point solver runs in the kernel with multiply-adds contracted into FMAs and on the host without: on the
ill-conditioned samples (the largest in the benchmark-shaped case) the two builds' candidates differ by up to 6e-5,
far below the distance between two candidates of one sample. The LM stages stop at the first accepted step that improves the
cost by less than 1e-10 of it; near the minimum a step of relative size ~1e-8 changes the cost by float64 rounding only,
so float64 summation order decides whether it is taken, which is what the 1e-9-level pose differences of the LO and
truncated least-squares rounds are. The "outliers" case holds pairs of 5 to 8 unrelated correspondences: a model fits
its own five sample points, and their front-of-camera votes split over the four decompositions, so the vote ties at the
top (the case asserts that it does) and the first-on-ties rule of the pose choice is checked.
"""
import numpy as np
import pytest
import torch

from helpers import rot_angle, synth
from oracle import pose_stages_oracle as so

pytestmark = pytest.mark.gpu

H, W = 240, 320
K_BASE = np.array([[300.0, 0, 159.5], [0, 300.0, 119.5], [0, 0, 1]])
SEED = 0x5EED
PIX_THR, REPROJ_THR = 2.0, 3.0
MAX_PTS = 8192
MODEL_BAR = 1e-4       # kernel vs host 5-point candidate, max abs difference of the unit-norm E
STATS = {}


def _stat(key, v):
    STATS[key] = max(STATS.get(key, 0.0), float(v))


# ------------------------------------------------------------------------------------------------ inputs
def _pair(seed, n, ratio=0.6, noise=0.3, edit=()):
    """One pair at 240x320 from synth.make_correspondences; ``edit`` names edge cases applied on top:
    k1  another K1 (kpts1 re-expressed in it, so that the geometry stays consistent)   k0  another K0 for both images
    oob keypoints at negative coordinates, beyond W - 1 and on x.5 values   dup duplicated correspondences
    zero depth 0 at a third of the keypoint pixels   min depth at a third of the keypoint pixels = the map minimum"""
    K = K_BASE.copy()
    if "k0" in edit:
        K = np.array([[280.0, 0, 150.25], [0, 290.0, 121.5], [0, 0, 1]])
    c = synth.make_correspondences(seed, n=max(n, 1), inlier_ratio=ratio, noise_px=noise, h=H, w=W, K=K)
    k0, k1 = c["kpts0"][:n].copy(), c["kpts1"][:n].copy()
    K0 = K.astype(np.float32); K1 = K.astype(np.float32)
    d0, d1 = c["depth0"].copy(), c["depth1"].copy()
    rng = np.random.default_rng(seed + 7)
    if "k1" in edit:
        K1 = np.array([[330.0, 0, 161.0], [0, 310.0, 118.0], [0, 0, 1]], np.float32)
        x = (k1.astype(np.float64) - K[:2, 2]) / np.diag(K)[:2]
        k1 = (x * np.diag(K1)[:2].astype(np.float64) + K1[:2, 2]).astype(np.float32)
    if "oob" in edit and n >= 12:
        k0[0] = (-0.5, 10.0); k0[1] = (W - 0.5, 20.0); k0[2] = (-3.25, -2.0); k0[3] = (W + 2.0, H + 1.0)
        k1[4] = (30.0, -0.75); k1[5] = (W - 1.0 + 0.5, H - 0.5)
        k0[6:12] = np.floor(k0[6:12]) + 0.5
        k1[6:12] = np.floor(k1[6:12]) + 0.5
    if "dup" in edit and n >= 20:
        j = rng.choice(n, n // 5, replace=False)
        k0[j[: len(j) // 2]] = k0[j[len(j) // 2: 2 * (len(j) // 2)]]
        k1[j[: len(j) // 2]] = k1[j[len(j) // 2: 2 * (len(j) // 2)]]
    ik0 = np.clip(k0.astype(np.int32), 0, [W - 1, H - 1]); ik1 = np.clip(k1.astype(np.int32), 0, [W - 1, H - 1])
    if "zero" in edit:
        j = rng.choice(n, n // 3, replace=False)
        d0[ik0[j, 1], ik0[j, 0]] = 0.0
        d1[ik1[j[::2], 1], ik1[j[::2], 0]] = 0.0
    if "min" in edit:
        j = rng.choice(n, n // 3, replace=False)
        d0[ik0[j, 1], ik0[j, 0]] = d0.min()
    return {"kpts0": k0, "kpts1": k1, "K0": K0, "K1": K1, "depth0": d0.astype(np.float32), "depth1": d1.astype(np.float32)}


def _batch(specs):
    return [_pair(*s) if isinstance(s, tuple) else _pair(**s) for s in specs]


# name -> (pairs, num_hyp, hypotheses per block on 132 SMs)
CASES = {
    "hpb32": ([(101, 1000)], 2048, 32),
    "hpb64": ([(102, 700), (103, 1025, 0.5, 0.5, ("k1",)), (104, 33, 0.8, 0.2)], 2048, 64),
    # the benchmark's shape: 16 pairs x 1024 hypotheses, with an empty pair and a pair of 4 in the middle
    "bench": ([(110 + i, n, 0.5 + 0.03 * (i % 5), 0.2 + 0.1 * (i % 3), e) for i, (n, e) in enumerate([
        (1024, ()), (1025, ("k1",)), (4100, ("k0",)), (33, ()), (0, ()), (800, ("oob",)), (4, ()), (1500, ("dup",)),
        (600, ("zero",)), (900, ("min",)), (2000, ("k0", "k1")), (6, ()), (5, ()), (1200, ("oob", "dup")), (700, ()),
        (3000, ())])], 1024, 128),
    "partial1": ([(120, 300), (121, 50)], 1, 32),
    "partial100": ([(122, 500), (123, 64, 0.9, 0.1)], 100, 32),
    "partial1000": ([(124, 900, 0.4, 0.5), (125, 260)], 1000, 32),
    "noise_free": ([(130, 600, 0.7, 0.0), (131, 5, 1.0, 0.0), (132, 6, 1.0, 0.0), (133, 40, 1.0, 0.0, ("dup",))], 512, 32),
    "max_pts": ([(140, 8192, 0.5, 0.3), (141, 8300, 0.5, 0.3)], 256, 32),
    # outliers only: a model fits its own five sample points, whose front-of-camera votes split over the four
    # decompositions, so the pose choice meets ties at the top
    "outliers": ([(170 + i, n, 0.0, 0.0) for i, n in enumerate([5, 6, 7, 8, 5, 6, 7, 8])], 256, 32),
}
LO_CASES = [("hpb32", 1), ("hpb64", 1), ("bench", 0), ("bench", 1), ("bench", 3), ("partial100", 1), ("noise_free", 0),
            ("noise_free", 1), ("noise_free", 3), ("max_pts", 1), ("outliers", 0), ("outliers", 1)]


def _upload(pairs, dev):
    off = np.cumsum([0] + [len(p["kpts0"]) for p in pairs]).astype(np.int32)
    cat = lambda k: torch.tensor(np.concatenate([p[k] for p in pairs]).reshape(-1, 2), device=dev).contiguous()
    st = lambda k: torch.tensor(np.stack([p[k] for p in pairs]), device=dev).contiguous()
    return (cat("kpts0"), cat("kpts1"), torch.tensor(off, device=dev), st("K0"), st("K1"), st("depth0"), st("depth1"),
            off)


@pytest.fixture(scope="module")
def backend():
    from mfr_b200 import pose_solver as ps
    be = ps.PoseBackend(max_pairs=16, max_pts=MAX_PTS, max_hyp=2048)
    yield be
    be.close()


def _records(be, name, dtype, rows, cols):
    words = rows * cols * dtype.itemsize // 4
    raw = be.debug_tensor(name, (words,), torch.int32).cpu().numpy()
    return raw.view(dtype).reshape(rows, cols)


# ------------------------------------------------------------------------------------------------ E-mat hypotheses
def _check_emat_block(r, cands, pts, thr2_f, key):
    """The four per-block checks of emat_hyp_kernel against the block's restated candidates."""
    if not cands:
        assert r["valid"] == 0 and r["cost"] == 1e300
        return
    assert r["valid"] == 1
    Es = np.stack([c[3] for c in cands])
    Ew = np.asarray(r["model"][:9], np.float64)
    unit = lambda E: E / np.linalg.norm(E, axis=-1, keepdims=True)
    d = np.minimum(np.abs(unit(Es) - unit(Ew)).max(1), np.abs(unit(Es) + unit(Ew)).max(1))
    _stat(f"{key} winner model vs host candidate", d.min())
    assert d.min() < MODEL_BAR, "block winner is none of the block's hypotheses"
    cost, bound, d2, lo, hi = so.msac_f_bound(Ew.astype(np.float32)[None], pts, thr2_f)
    cost, bound, lo, hi = cost[0], bound[0], lo[0], hi[0]
    _stat(f"{key} cost |d| / bound", abs(r["cost"] - cost) / bound)
    assert abs(r["cost"] - cost) <= bound, (r["cost"], cost, bound)
    # the host candidates stand for the kernel's only up to the solver bar, which enters their bound as an absolute
    # error of every (unit-norm) coefficient
    lo_cost = np.inf
    for i in range(0, len(Es), 128):
        E32 = unit(Es[i:i + 128]).astype(np.float32)
        c, bd, _, _, _ = so.msac_f_bound(E32, pts, thr2_f, e_abs=MODEL_BAR + so.U32)
        lo_cost = min(lo_cost, float((c + bd).min()))
    assert lo_cost >= cost - bound, ("a candidate of the block is cheaper than its winner", lo_cost, cost, bound)
    thr2 = float(thr2_f)
    n_lo, n_hi = int((hi < thr2).sum()), int((lo < thr2).sum())
    assert n_lo <= r["count"] <= n_hi, (r["count"], n_lo, n_hi)


@pytest.mark.parametrize("case", list(CASES))
def test_emat_normalise_and_hypotheses(backend, case):
    """emat_normalise_kernel bit-exact; emat_hyp_kernel block by block at the hypotheses-per-block value the launch rule
    picks (32, 64 and 128 on 132 SMs)."""
    specs, num_hyp, hpb_132 = CASES[case]
    pairs = _batch(specs)
    be, P = backend, len(pairs)
    k0, k1, off, K0, K1, d0, d1, off_np = _upload(pairs, be.device)
    be.emat(k0, k1, off, K0, K1, PIX_THR, num_hyp, SEED, 1)
    torch.cuda.synchronize()
    sm = be._l.mfr_device_sm_count()
    hpb = so.emat_hyp_per_block(P, num_hyp, sm)
    if sm == 132:
        assert hpb == hpb_132
    blocks = -(-num_hyp // hpb)
    pts_all = be.debug_tensor("pts_norm", (16, MAX_PTS, 4), torch.float32).cpu().numpy()
    res = _records(be, "hyp_results", so.HYP_DTYPE, 16, blocks)
    for p, pr in enumerate(pairs):
        N = min(len(pr["kpts0"]), MAX_PTS)
        pts = pts_all[p, :N]
        ref = so.normalise(pr["kpts0"][:N], pr["kpts1"][:N], pr["K0"], pr["K1"])
        assert np.array_equal(pts.view(np.uint32), ref.view(np.uint32)), "normalised points differ"
        if N < 5:
            assert (res[p]["valid"] == 0).all() and (res[p]["cost"] == 1e300).all()
            continue
        _, thr2_f = so.emat_threshold(PIX_THR, pr["K0"], pr["K1"])
        for b, cands in enumerate(so.emat_hypotheses(pts, N, num_hyp, hpb, SEED, p)):
            _check_emat_block(res[p, b], cands, pts, thr2_f, "emat")
    print(f"\n[{case}] hpb {hpb} on {sm} SMs; " + "; ".join(f"{k} {v:.3g}" for k, v in sorted(STATS.items())))


# ------------------------------------------------------------------------------------------------ E-mat LO and final
def _thr(pr):
    thr_f, _ = so.emat_threshold(PIX_THR, pr["K0"], pr["K1"])
    thr = float(thr_f)
    return thr, thr * thr


@pytest.mark.parametrize("case,lo", LO_CASES)
def test_emat_lo_and_final(backend, case, lo):
    """Selection, pose choice, LO (emat_lo_kernel) and the final model and mask (emat_final_kernel), each restated from
    the kernel's own input (the block records for LO, the LO records for the final stage)."""
    specs, num_hyp, _ = CASES[case]
    pairs = _batch(specs)
    be, P = backend, len(pairs)
    k0, k1, off, K0, K1, d0, d1, off_np = _upload(pairs, be.device)
    R, t, n, mask = be.emat(k0, k1, off, K0, K1, PIX_THR, num_hyp, SEED, lo)
    torch.cuda.synchronize()
    hpb = so.emat_hyp_per_block(P, num_hyp, be._l.mfr_device_sm_count())
    blocks = -(-num_hyp // hpb)
    pts_all = be.debug_tensor("pts_norm", (16, MAX_PTS, 4), torch.float32).cpu().numpy()
    res = _records(be, "hyp_results", so.HYP_DTYPE, 16, blocks)
    lor = _records(be, "lo_results", so.LO_DTYPE, 16, so.LO_TOPK)
    Rd = be.debug_tensor("Rd", (16, 9), torch.float64).cpu().numpy()
    td = be.debug_tensor("td", (16, 3), torch.float64).cpu().numpy()
    R, t, n, mask = R.cpu().numpy(), t.cpu().numpy(), n.cpu().numpy(), mask.cpu().numpy()
    lo_bar, final_bar = (1e-12, 1e-12) if lo == 0 else (2.4e-9, 7e-9)
    ties = 0
    for p, pr in enumerate(pairs):
        Nall = len(pr["kpts0"])
        N = min(Nall, MAX_PTS)
        m_k = mask[off_np[p]:off_np[p + 1]]
        if N < 5:
            assert (lor[p]["cost"] == 1e300).all()
            assert n[p] == 0 and np.isnan(R[p]).all() and np.isnan(t[p]).all() and not m_k.any()
            continue
        pts = pts_all[p, :N]
        thr, thr2 = _thr(pr)
        cand = so.emat_select(res[p])
        for c in range(so.LO_TOPK):
            if c >= len(cand) or (lo == 0 and c > 0):
                assert lor[p, c]["cost"] == 1e300
                continue
            cost, Rr, tr, votes, near = so.emat_lo(res[p, cand[c]]["model"][:9], pts, thr2, lo)
            assert near == 0, ("a pose vote within rounding of the threshold", near)
            ties += votes.count(max(votes)) > 1
            dR = np.abs(lor[p, c]["R"] - Rr.ravel()).max()
            dt = np.abs(lor[p, c]["t"] - tr).max()
            # relative to the cost, or to N thr^2 where every point fits (N = 5: the cost is rounding noise)
            dc = abs(lor[p, c]["cost"] - cost) / max(cost, N * thr2)
            _stat(f"lo{lo} pose", max(dR, dt)); _stat(f"lo{lo} cost rel", dc)
            assert max(dR, dt) < lo_bar and dc < 3.7e-12, (p, c, dR, dt, dc)
        fin = so.emat_final(lor[p], pts, thr, lo)
        if fin["failed"]:
            assert n[p] == 0 and np.isnan(Rd[p]).all() and np.isnan(R[p]).all() and not m_k.any()
            continue
        assert fin["edge"] == 0, ("a point within rounding of a histogram bin edge", fin["edge"])
        dp = max(np.abs(Rd[p] - fin["R"].ravel()).max(), np.abs(td[p] - fin["t"]).max())
        _stat(f"final lo{lo} pose", dp)
        assert dp < final_bar, (p, dp)
        # the mask under the kernel's own final pose: exact but at points within 1e-12 of thr^2
        E = so.essential_from_rt(Rd[p].reshape(3, 3), td[p]).ravel()
        d2 = so.sampson_sq(E, pts)
        exp = (d2 < thr2) & so.cheirality(Rd[p].reshape(3, 3), td[p], pts)
        free = np.abs(d2 - thr2) <= 1e-12 * thr2
        assert np.array_equal(m_k[:N].astype(bool) | free, exp | free), (p, int((m_k[:N].astype(bool) != exp).sum()))
        assert not m_k[N:].any(), "points beyond max_pts are in the mask"
        assert n[p] == int(m_k.sum())
        assert n[p] == max(fin["votes"]) or fin["near"], (p, n[p], fin["votes"], fin["near"])
        ties += fin["votes"].count(max(fin["votes"])) > 1
        assert np.array_equal(R[p].ravel(), Rd[p].astype(np.float32)) and np.array_equal(t[p], td[p].astype(np.float32))
    if case == "outliers":
        assert ties > 0, "no pose vote tied at the top: the first-on-ties rule was not exercised"
    print(f"\n[{case} lo={lo}] vote ties {ties}; " + "; ".join(f"{k} {v:.3g}" for k, v in sorted(STATS.items())))


# ------------------------------------------------------------------------------------------------ PnP
PNP_CASES = {
    "bench": (CASES["bench"][0] + [], 1024),
    "lm_rules": ([(150, 6, 1.0, 0.5), (151, 4, 1.0, 0.3), (152, 5, 1.0, 0.5), (153, 7, 1.0, 0.5), (154, 300, 0.7, 0.3, ("zero",)),
                  (155, 300, 0.7, 0.3, ("min",))], 256),
    "chunks": ([(160, 4100, 0.5, 0.5, ("zero",)), (161, 8192, 0.6, 0.3, ("oob",)), (162, 2048, 0.6, 0.3, ("k0", "k1"))], 300),
}


@pytest.mark.parametrize("case", list(PNP_CASES))
def test_pnp_stages(backend, case):
    """depth_min_kernel, pnp_prepare_kernel (ordered compaction across 1024-thread chunks, lift), pnp_hyp_kernel block by
    block, pnp_final_kernel (mask under the winning record, n_in rules, LM), each from the device's own input.
    depth_min_kernel clamps the map minimum at 0 where the reference takes depth0.min() as it is; the two differ only for
    negative depths, which the dataset's depth images cannot hold."""
    import cv2
    specs, num_hyp = PNP_CASES[case]
    pairs = _batch(specs)
    be, P = backend, len(pairs)
    k0, k1, off, K0, K1, d0, d1, off_np = _upload(pairs, be.device)
    R, t, n, mask = be.pnp(k0, k1, off, K0, K1, d0, REPROJ_THR, num_hyp, SEED)
    torch.cuda.synchronize()
    blocks = -(-num_hyp // so.HYP_PER_BLOCK)
    dmin = be.debug_tensor("dmin", (16,), torch.float32).cpu().numpy()
    nvalid = be.debug_tensor("nvalid", (16,), torch.int32).cpu().numpy()
    vidx = be.debug_tensor("vidx", (16, MAX_PTS), torch.int32).cpu().numpy()
    uv = be.debug_tensor("uv", (16, MAX_PTS, 2), torch.float32).cpu().numpy()
    Xw = be.debug_tensor("Xw", (16, MAX_PTS, 3), torch.float64).cpu().numpy()
    res = _records(be, "hyp_results", so.HYP_DTYPE, 16, blocks)
    R, t, n, mask = R.cpu().numpy(), t.cpu().numpy(), n.cpu().numpy(), mask.cpu().numpy()
    seen = set()
    for p, pr in enumerate(pairs):
        N = min(len(pr["kpts0"]), MAX_PTS)
        dm = so.depth_min(pr["depth0"])
        assert dmin[p].view(np.uint32) == dm.view(np.uint32)
        vr, Xr, ur = so.pnp_prepare(pr["kpts0"][:N], pr["kpts1"][:N], pr["depth0"], pr["K0"], dm)
        nv = int(nvalid[p])
        assert nv == len(vr) and np.array_equal(vidx[p, :nv], vr) and np.array_equal(uv[p, :nv], ur)
        Xk, uk = Xw[p, :nv], uv[p, :nv]
        ulp = np.abs(Xk - Xr) / np.maximum(np.spacing(np.abs(Xr)), 1e-300)
        _stat("pnp Xw ulp", ulp.max(initial=0))
        assert ulp.max(initial=0) <= 4
        if nv >= 4:
            for b, cands in enumerate(so.pnp_hypotheses(Xk, uk, pr["K1"], num_hyp, SEED, p)):
                r = res[p, b]
                if not cands:
                    assert r["valid"] == 0
                    continue
                assert r["valid"] == 1
                Rw, tw = np.asarray(r["model"][:9]), np.asarray(r["model"][9:])
                d = min(max(np.abs(c[2].ravel() - Rw).max(), np.abs(c[3] - tw).max() / max(1.0, np.abs(tw).max()))
                        for c in cands)
                _stat("pnp winner model vs host candidate", d)
                assert d < 7e-9
                lo_w, hi_w = so.pnp_count_bound(Rw, tw, Xk, uk, pr["K1"], REPROJ_THR)
                assert lo_w.sum() <= r["count"] <= hi_w.sum() and r["cost"] == -r["count"]
                best_lo = max(int(so.pnp_count_bound(c[2], c[3], Xk, uk, pr["K1"], REPROJ_THR)[0].sum()) for c in cands)
                assert best_lo <= hi_w.sum(), ("a hypothesis of the block has more inliers than its winner", best_lo)
        fin = so.pnp_final(res[p], Xk, uk, pr["K1"], REPROJ_THR)
        m_k = mask[off_np[p]:off_np[p + 1]].astype(bool)
        if fin["failed"]:
            assert n[p] == 0 and np.isnan(R[p]).all() and np.isnan(t[p]).all() and not m_k.any()
            continue
        seen.add(fin["n_in"])
        exp = np.zeros(len(m_k), bool)
        exp[vr[fin["mask"]]] = True
        free = np.zeros(len(m_k), bool)
        free[vr[fin["near"]]] = True
        assert np.array_equal(m_k | free, exp | free)
        assert n[p] == fin["n_in"]
        dp = max(np.abs(R[p].astype(np.float64) - fin["R"]).max(), np.abs(t[p] - fin["t"]).max() / max(1.0, np.abs(fin["t"]).max()))
        _stat("pnp pose vs LM restatement", dp)
        assert dp < 1.1e-7, (p, dp)
        if fin["n_in"] >= 6:
            rv, _ = cv2.Rodrigues(np.asarray(res[p, fin["record"]]["model"][:9]).reshape(3, 3))
            inl = fin["mask"]
            ok, rvs, tvs, _ = cv2.solvePnPGeneric(Xk[inl], uk[inl].astype(np.float64), pr["K1"].astype(np.float64), None,
                                                  useExtrinsicGuess=True, rvec=rv,
                                                  tvec=np.asarray(res[p, fin["record"]]["model"][9:]).reshape(3, 1),
                                                  flags=cv2.SOLVEPNP_ITERATIVE)
            Rc, _ = cv2.Rodrigues(rvs[0])
            dcv = max(rot_angle(Rc, fin["R"]), np.abs(tvs[0].ravel() - fin["t"]).max())
            _stat("pnp LM vs cv2.solvePnPGeneric", dcv)
            assert dcv < 1.2e-7
    if case == "lm_rules":
        assert 6 in seen and seen & {4, 5}, seen         # both sides of the n_in >= 6 refinement rule were reached
    print(f"\n[pnp {case}] " + "; ".join(f"{k} {v:.3g}" for k, v in sorted(STATS.items())))
