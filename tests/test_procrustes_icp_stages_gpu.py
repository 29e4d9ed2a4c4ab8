"""Each stage of the Procrustes RANSAC and of its ICP refinement (csrc/geometry.cu) against a float64 restatement
(oracle/pose_stages_oracle.py), fed with the device's own input, as tests/test_pose_stages_gpu.py does for E-mat and PnP.

Procrustes: depth minima, compaction and lift exact (Xw / X1w within 4 ulp); every block winner one of its block's
3-point Kabsch candidates (the host hook mfr_host_kabsch runs the kernel's own code; the two builds differ by FMA
contraction only); the winner's count between the counts of the points surely and possibly inside under the float32
scoring (``procrustes_count_bound``), and no candidate of the block surely above the winner; the final R, t the float32
rounding of the float64 refit (up to ties within 1e-12 of a rounding midpoint), its count exact (no point lies within
1e-12 of the threshold in any case: asserted).

ICP: every association pass against a k-d tree on the same clouds (lifted through the float32 inverse of K, as the
kernel lifts them): the correspondence count exact (a point within 1e-9 of D may go either way: counted and allowed),
rmse within 1e-12, fitness = n / valid source points and n_inliers = int(fitness * valid target points) bit for bit, the
stop pass and flag the restatement's. ``max_iter = k`` leaves the pose after k updates in "icp_state", so the pose of
update k is checked against the restated Kabsch update from the device's pose k - 1. The kernel's sums and the oracle's
differ in summation order only; the bars below that come from measurement are at most 4x the maximum measured on one
NVIDIA H100 80GB HBM3 (700 W power limit) over all cases:

  stage                                              bar       measured
  Procrustes winner model vs host Kabsch candidate   8.4e-13   2.1e-13
  ICP pose of update k vs restated update            2.7e-12   6.8e-13
  ICP whole loop vs the restatement and vs
    icp_point_to_point (float32 R, t)                1.2e-7    3.0e-8

Reproducibility: a pair gives the same bits alone and inside a batch of 16, in two calls, and in a CUDA graph replay.
"""
import numpy as np
import pytest
import torch

from helpers import synth
from oracle import pose_solver_oracle as po
from oracle import pose_stages_oracle as so

pytestmark = pytest.mark.gpu

SEED = 0x5EED
DIST = 0.05
MAX_PTS = 8192
MODEL_BAR = 8.4e-13
ICP_STEP_BAR = 2.7e-12
ICP_LOOP_BAR = 1.2e-7
STATS = {}


def _stat(key, v):
    STATS[key] = max(STATS.get(key, 0.0), float(v))


def _report(tag):
    print(f"\n[{tag}] " + "; ".join(f"{k} {v:.3g}" for k, v in sorted(STATS.items())))


@pytest.fixture(scope="module")
def backend():
    from mfr_b200 import pose_solver as ps
    be = ps.PoseBackend(max_pairs=16, max_pts=MAX_PTS, max_hyp=2048)
    yield be
    be.close()


def _f32_rounding(got, ref):
    """got (float32) is the rounding of ref (float64), up to ties within 1e-12 (relative) of a rounding midpoint."""
    ref = np.asarray(ref, np.float64).ravel()
    d = np.abs(np.asarray(got, np.float64).ravel() - ref)
    return bool((d <= 0.5 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + 1e-12 * np.abs(ref)).all())


# ------------------------------------------------------------------------------------------------ Procrustes inputs
H, W = 540, 720
K_BENCH = np.array([[590.0, 0, 359.5], [0, 590.0, 269.5], [0, 0, 1]])


def _pair(seed, n, ratio=0.6, noise=0.3, edit=(), scale=1.0):
    """One 540x720 pair from synth.make_correspondences. ``edit``: k0 / k1 another K0 for both images / K1 (kpts1
    re-expressed in it), oob keypoints outside the images and on x.5 values, dup duplicated correspondences, zero depth 0
    at a third of the keypoint pixels, min depth = the map minimum there, same every correspondence a copy of the first.
    ``scale`` multiplies both depth maps (and so the translation): x10 puts the scene at 10-80 m."""
    K = K_BENCH.copy()
    if "k0" in edit:
        K = np.array([[575.0, 0, 351.25], [0, 585.0, 272.5], [0, 0, 1]])
    c = synth.make_correspondences(seed, n=max(n, 1), inlier_ratio=ratio, noise_px=noise, h=H, w=W, K=K)
    k0, k1 = c["kpts0"][:n].copy(), c["kpts1"][:n].copy()
    K0 = K.astype(np.float32); K1 = K.astype(np.float32)
    d0, d1 = c["depth0"] * np.float32(scale), c["depth1"] * np.float32(scale)
    rng = np.random.default_rng(seed + 7)
    if "k1" in edit:
        K1 = np.array([[610.0, 0, 362.0], [0, 600.0, 266.0], [0, 0, 1]], np.float32)
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
    if "same" in edit:
        k0[:] = k0[0]; k1[:] = k1[0]
    ik0 = np.clip(k0.astype(np.int32), 0, [W - 1, H - 1]); ik1 = np.clip(k1.astype(np.int32), 0, [W - 1, H - 1])
    if "zero" in edit:
        j = rng.choice(n, n // 3, replace=False)
        d0[ik0[j, 1], ik0[j, 0]] = 0.0
        d1[ik1[j[::2], 1], ik1[j[::2], 0]] = 0.0
    if "min" in edit:
        j = rng.choice(n, n // 3, replace=False)
        d0[ik0[j, 1], ik0[j, 0]] = d0.min()
    return {"kpts0": k0, "kpts1": k1, "K0": K0, "K1": K1, "depth0": d0.astype(np.float32), "depth1": d1.astype(np.float32)}


BENCH = [(300 + i, n, 0.5 + 0.03 * (i % 5), 0.2 + 0.1 * (i % 3), e) for i, (n, e) in enumerate([
    (1024, ()), (4100, ("k1",)), (0, ()), (2, ()), (3, ()), (4, ()), (800, ("oob",)), (1500, ("dup",)),
    (600, ("zero",)), (900, ("min",)), (2000, ("k0", "k1")), (3000, ("k0",)), (1200, ("oob", "dup")), (700, ()),
    (2500, ()), (1800, ("zero", "min"))])]
# name -> (pair specs, num_hyp)
CASES = {
    "bench": (BENCH, 2048),
    "far": ([dict(seed=320 + i, n=n, edit=e, scale=10.0) for i, (n, e) in enumerate([(1500, ()), (800, ("k1",)),
                                                                                      (3000, ("zero",))])], 1024),
    "budget1": ([(330, 400), (331, 60)], 1),
    "budget100": ([(332, 500), (333, 64, 0.9, 0.1)], 100),
    "budget1000": ([(334, 900, 0.4, 0.5), (335, 260)], 1000),
    "max_pts": ([(340, 8192, 0.5, 0.3), (341, 8300, 0.5, 0.3)], 256),
    "degenerate": ([(350, 50, 1.0, 0.0, ("same",)), (351, 3, 1.0, 0.0, ("same",))], 256),
    "noise_free": ([(360, 600, 0.7, 0.0), (361, 3, 1.0, 0.0), (362, 40, 1.0, 0.0, ("dup",))], 512),
}


def _batch(specs):
    return [_pair(*s) if isinstance(s, tuple) else _pair(**s) for s in specs]


def _upload(pairs, dev):
    off = np.cumsum([0] + [len(p["kpts0"]) for p in pairs]).astype(np.int32)
    cat = lambda k: torch.tensor(np.concatenate([p[k] for p in pairs]).reshape(-1, 2), device=dev).contiguous()
    st = lambda k: torch.tensor(np.stack([p[k] for p in pairs]), device=dev).contiguous()
    return cat("kpts0"), cat("kpts1"), torch.tensor(off, device=dev), st("K0"), st("K1"), st("depth0"), st("depth1")


def _records(be, rows, cols):
    raw = be.debug_tensor("hyp_results", (rows * cols * so.HYP_DTYPE.itemsize // 4,), torch.int32).cpu().numpy()
    return raw.view(so.HYP_DTYPE).reshape(rows, cols)


def _run_procrustes(be, pairs, num_hyp):
    args = _upload(pairs, be.device)
    R, t, n = be.procrustes(*args, DIST, num_hyp, SEED)
    torch.cuda.synchronize()
    return R.cpu().numpy(), t.cpu().numpy(), n.cpu().numpy(), _records(be, 16, -(-num_hyp // so.HYP_PER_BLOCK))


@pytest.mark.parametrize("case", list(CASES))
def test_procrustes_stages(backend, case):
    """depth_min_kernel on both maps, procrustes_prepare_kernel (ordered compaction, lift), procrustes_hyp_kernel block
    by block, procrustes_final_kernel (winner, two refits, count), each from the device's own input."""
    specs, num_hyp = CASES[case]
    pairs = _batch(specs)
    be = backend
    R, t, n, res = _run_procrustes(be, pairs, num_hyp)
    dmin = be.debug_tensor("dmin", (16,), torch.float32).cpu().numpy()
    dmin1 = be.debug_tensor("dmin1", (16,), torch.float32).cpu().numpy()
    nvalid = be.debug_tensor("nvalid", (16,), torch.int32).cpu().numpy()
    Xw = be.debug_tensor("Xw", (16, MAX_PTS, 3), torch.float64).cpu().numpy()
    X1w = be.debug_tensor("X1w", (16, MAX_PTS, 3), torch.float64).cpu().numpy()
    for p, pr in enumerate(pairs):
        N = min(len(pr["kpts0"]), MAX_PTS)
        dm0, dm1 = so.depth_min(pr["depth0"]), so.depth_min(pr["depth1"])
        assert dmin[p].view(np.uint32) == dm0.view(np.uint32) and dmin1[p].view(np.uint32) == dm1.view(np.uint32)
        vidx, X0r, X1r = so.procrustes_prepare(pr["kpts0"][:N], pr["kpts1"][:N], pr["depth0"], pr["depth1"], pr["K0"],
                                               pr["K1"], dm0, dm1)
        nv = int(nvalid[p])
        assert nv == len(vidx), (p, nv, len(vidx))
        X0k, X1k = Xw[p, :nv], X1w[p, :nv]
        for Xk, Xr in ((X0k, X0r), (X1k, X1r)):
            ulp = np.abs(Xk - Xr) / np.maximum(np.spacing(np.abs(Xr)), 1e-300)
            _stat("procrustes X ulp", ulp.max(initial=0))
            assert ulp.max(initial=0) <= 4, "compaction order or lift differs"
        if nv >= 3:
            for b, cands in enumerate(so.procrustes_hypotheses(X0k, X1k, num_hyp, SEED, p)):
                r = res[p, b]
                if not cands:
                    assert r["valid"] == 0
                    continue
                assert r["valid"] == 1
                Rw, tw = np.asarray(r["model"][:9]), np.asarray(r["model"][9:])
                d = min(max(np.abs(c[2].ravel() - Rw).max(), np.abs(c[3] - tw).max() / max(1.0, np.abs(tw).max()))
                        for c in cands)
                _stat("procrustes winner vs host candidate", d)
                assert d < MODEL_BAR, "block winner is none of the block's hypotheses"
                lo_w, hi_w = so.procrustes_count_bound(Rw, tw, X0k, X1k, DIST)
                assert lo_w.sum() <= r["count"] <= hi_w.sum(), (p, b, r["count"], lo_w.sum(), hi_w.sum())
                best_lo = max(int(so.procrustes_count_bound(c[2], c[3], X0k, X1k, DIST)[0].sum()) for c in cands)
                assert best_lo <= hi_w.sum(), ("a hypothesis of the block has more inliers than its winner", best_lo)
        fin = so.procrustes_final(res[p], X0k, X1k, DIST)
        if fin["failed"]:
            assert n[p] == 0 and np.isnan(R[p]).all() and np.isnan(t[p]).all(), (p, n[p])
            continue
        assert fin["near"] == 0, ("a point within rounding of the threshold", fin["near"])
        assert n[p] == fin["n"], (p, n[p], fin["n"])
        assert _f32_rounding(R[p], fin["R"]) and _f32_rounding(t[p], fin["t"]), (p, R[p], fin["R"], t[p], fin["t"])
    if case == "degenerate":
        assert (n[:len(pairs)] == 0).all() and np.isnan(R[:len(pairs)]).all()
    _report(f"procrustes {case}")


def test_procrustes_alone_equals_batched(backend):
    """Pair 0 of the benchmark-shaped batch gives the same bits (pose, count, block records) when it runs alone."""
    pairs = _batch(CASES["bench"][0])
    R, t, n, res = _run_procrustes(backend, pairs, 2048)
    res0 = res[0].copy()
    R1, t1, n1, res1 = _run_procrustes(backend, pairs[:1], 2048)
    assert np.array_equal(R1[0].view(np.uint32), R[0].view(np.uint32)) and np.array_equal(t1[0].view(np.uint32), t[0].view(np.uint32))
    assert n1[0] == n[0] and res1[0].tobytes() == res0.tobytes()


# ------------------------------------------------------------------------------------------------ ICP
K_SCANNET = np.array([[577.0, 0, 319.5], [0, 577.0, 239.5], [0, 0, 1]])


def _scene(seed, h=480, w=640, K=K_SCANNET, rot=0.01, trans=0.02, shift=(0.0, 0.0, 0.0)):
    """synth.make_pair at the ScanNet shape with a start pose perturbed from the ground truth."""
    p = synth.make_pair(seed, h=h, w=w, K=K)
    rng = np.random.default_rng(seed)
    R0 = synth.rodrigues(rng.normal(0, rot, 3)) @ p["R_gt"]
    t0 = p["t_gt"] + rng.normal(0, trans, 3) + np.asarray(shift)
    return {"depth0": p["depth0"], "depth1": p["depth1"], "K0": p["K_color0"], "K1": p["K_color1"],
            "R0": R0.astype(np.float32), "t0": t0.astype(np.float32)}


def _hole_scene():
    """A plane 0.2 m in front of both cameras, identity pose, columns 221-419 of depth1 empty: at 0.2 m the radius bound
    reaches ~195 pixels, so the nearest neighbours of the source points in the middle of the hole lie beyond the
    96-pixel window clamp."""
    d0 = np.full((480, 640), 0.2, np.float32)
    d1 = d0.copy()
    d1[:, 221:420] = 0.0
    K = K_SCANNET.astype(np.float32)
    return {"depth0": d0, "depth1": d1, "K0": K, "K1": K, "R0": np.eye(3, dtype=np.float32), "t0": np.zeros(3, np.float32)}


def _icp(be, scenes, max_iter, rel=1e-4):
    dev = be.device
    st = lambda k: torch.tensor(np.stack([s[k] for s in scenes]), device=dev).contiguous()
    R, t, n = be.icp(st("R0"), st("t0"), st("K0"), st("K1"), st("depth0"), st("depth1"), DIST, max_iter, rel, rel)
    torch.cuda.synchronize()
    state = be.debug_tensor("icp_state", (16, 18), torch.float64).cpu().numpy()[:len(scenes)].copy()
    return R.cpu().numpy(), t.cpu().numpy(), n.cpu().numpy(), state


def _check_assoc(st, s, X0, X1, tree, key):
    """The association at the state's pose: n (state[15]) exact but for points within 1e-9 of D, rmse within 1e-12,
    fitness = n / valid source points. Returns the oracle's association."""
    a = so.icp_assoc(X0, X1, st[:9], st[9:12], DIST, tree)
    assert abs(st[15] - a["n"]) <= a["near"], (key, st[15], a["n"], a["near"])
    if a["near"] == 0:
        assert st[15] == a["n"]
        if a["n"]:
            _stat("icp rmse rel", abs(st[13] - a["rmse"]) / a["rmse"])
            assert abs(st[13] - a["rmse"]) <= 1e-12 * a["rmse"], (key, st[13], a["rmse"])
    assert st[12] == (st[15] / st[16] if st[16] > 0 else 0.0)
    return a


def _check_icp_scene(be, s, key, max_iter=30, rel=1e-4, trace=True):
    """Pass by pass (trace) and the whole loop of one scene against the restatement."""
    from scipy.spatial import cKDTree
    X0, X1 = so.icp_clouds(s["depth0"], s["depth1"], s["K0"], s["K1"])
    tree = cKDTree(X1) if len(X1) else None
    R0, t0 = s["R0"].astype(np.float64), s["t0"].astype(np.float64)
    Rf, tf, nf, stf = _icp(be, [s], max_iter, rel)
    assert stf[0, 16] == len(X0) and stf[0, 17] == len(X1)
    if len(X1) == 0 or len(X0) == 0:         # nothing to associate: the start pose stands, fitness 0
        assert stf[0, 14] == 1 and stf[0, 15] == 0 and nf[0] == 0
        assert np.array_equal(Rf[0].ravel(), s["R0"].ravel()) and np.array_equal(tf[0], s["t0"])
        return
    Rl, tl, fitl, rmsel, stop, conv = so.icp_loop(X0, X1, R0, t0, DIST, max_iter, rel, rel)
    assert stf[0, 14] == 1
    assert nf[0] == int(stf[0, 12] * stf[0, 17]), "n_inliers is not int(fitness * valid target points)"
    dl = max(np.abs(Rf[0].astype(np.float64) - Rl.ravel().reshape(3, 3)).max(), np.abs(tf[0] - tl).max())
    _stat("icp loop vs restatement", dl)
    assert dl < ICP_LOOP_BAR, (key, dl)
    _check_assoc(stf[0], s, X0, X1, tree, key)
    if trace:
        prev = None
        for k in range(0, stop + 1):
            _, _, _, st = _icp(be, [s], max(k, 1)) if k > 0 else (None, None, None, None)
            if k == 0:   # pass 0 at the start pose: its association is the one max_iter = 1 evaluates first
                st0 = np.concatenate([R0.ravel(), t0, [0.0, 0.0, 0.0, 0.0, len(X0), len(X1)]])
                a = so.icp_assoc(X0, X1, R0, t0, DIST, tree)
                prev = (st0, a)
                continue
            st = st[0]
            sp, ap = prev
            Ru, tu, _, _, stopped = so.icp_update((sp[:9].reshape(3, 3), sp[9:12], 0.0, 0.0), ap, len(X0), 0, 0.0, 0.0)
            if not stopped:
                d = max(np.abs(st[:9] - Ru.ravel()).max(), np.abs(st[9:12] - tu).max())
                _stat("icp update vs restated", d)
                assert d < ICP_STEP_BAR, (key, k, d)
            a = _check_assoc(st, s, X0, X1, tree, f"{key} pass {k}")
            prev = (st, a)
        # the stop pass: max_iter = stop leaves the state of the full run, max_iter = stop - 1 does not
        if stop >= 2 and conv and stop < max_iter:
            _, _, _, s_at = _icp(be, [s], stop, rel)
            _, _, _, s_before = _icp(be, [s], stop - 1, rel)
            assert np.array_equal(s_at[0], stf[0]) and not np.array_equal(s_before[0, :12], stf[0, :12]), key
    # the reference-side oracle (Open3D's algorithm on a k-d tree) on the same clouds
    T0 = np.eye(4); T0[:3, :3] = R0; T0[:3, 3] = t0
    T, fo, _ = po.icp_point_to_point(X0, X1, T0, float(np.float32(DIST)), max_iter, rel, rel)
    do = max(np.abs(Rf[0] - T[:3, :3]).max(), np.abs(tf[0] - T[:3, 3]).max())
    _stat("icp loop vs icp_point_to_point", do)
    assert do < ICP_LOOP_BAR and abs(nf[0] - int(fo * len(X1))) <= 1, (key, do, nf[0], int(fo * len(X1)))


ICP_CASES = {
    "scene3": lambda: _scene(3),
    "scene8": lambda: _scene(8),
    "scene540x720": lambda: _scene(5, 540, 720, synth.K_DEFAULT),
    "near_range_hole": _hole_scene,
    "projects_outside": lambda: _scene(9, shift=(0.35, -0.2, 0.0)),
    "zero_depth0": lambda: dict(_scene(3), depth0=np.zeros((480, 640), np.float32)),
    "zero_depth1": lambda: dict(_scene(3), depth1=np.zeros((480, 640), np.float32)),
}


@pytest.mark.parametrize("case", list(ICP_CASES))
def test_icp_passes(backend, case):
    _check_icp_scene(backend, ICP_CASES[case](), case)
    _report(f"icp {case}")


def test_icp_max_iter_without_convergence(backend):
    """Criteria that cannot be met (0): the loop runs max_iter updates and evaluates the last pose."""
    _check_icp_scene(backend, _scene(4, rot=0.03, trans=0.05), "max_iter", max_iter=4, rel=0.0, trace=False)
    _report("icp max_iter")


def test_icp_nan_start(backend):
    """A NaN start pose (failed RANSAC) passes through as NaN, 0 inliers, next to a pair that runs."""
    s = _scene(3)
    bad = dict(s, R0=np.full((3, 3), np.nan, np.float32))
    R, t, n, st = _icp(backend, [s, bad], 30)
    assert np.isnan(R[1]).all() and np.isnan(t[1]).all() and n[1] == 0 and np.isfinite(R[0]).all() and n[0] > 0


def _batch16():
    Ks = [np.array([[560.0 + 5 * i, 0, 316.0 + i], [0, 565.0 + 4 * i, 238.0 - i], [0, 0, 1]]) for i in range(16)]
    return [_scene(20 + i, 240, 320, Ks[i] * [[0.5], [0.5], [1.0]]) for i in range(16)]


def test_icp_batch_of_16_with_different_K(backend):
    """16 pairs with 16 intrinsics in one call: each pair's whole loop against the restatement."""
    scenes = _batch16()
    R, t, n, st = _icp(backend, scenes, 30)
    for p, s in enumerate(scenes):
        X0, X1 = so.icp_clouds(s["depth0"], s["depth1"], s["K0"], s["K1"])
        Rl, tl, fit, rmse, stop, conv = so.icp_loop(X0, X1, s["R0"].astype(np.float64), s["t0"].astype(np.float64), DIST)
        d = max(np.abs(R[p] - Rl).max(), np.abs(t[p] - tl).max())
        _stat("icp loop vs restatement", d)
        assert d < ICP_LOOP_BAR, (p, d)
        assert n[p] == int(st[p, 12] * st[p, 17]) and abs(st[p, 12] - fit) * len(X0) <= 1, (p, st[p, 12], fit)
    _report("icp batch16")


def test_icp_reproducible(backend):
    """Bitwise: two calls; pair 0 alone vs inside a batch of 16 at 480x640 (the association grid depends on the frame
    only); a CUDA graph replay (after a warm-up call, which allocates the ICP scratch)."""
    base = [_scene(3), _scene(8), _hole_scene()]
    scenes = [dict(base[i % 3], R0=(synth.rodrigues([0.002 * i, 0, 0]) @ base[i % 3]["R0"]).astype(np.float32))
              for i in range(16)]
    a = _icp(backend, scenes, 30)
    b = _icp(backend, scenes, 30)
    assert a[3].tobytes() == b[3].tobytes() and a[0].tobytes() == b[0].tobytes() and np.array_equal(a[2], b[2])
    alone = _icp(backend, scenes[:1], 30)
    assert alone[3][0].tobytes() == a[3][0].tobytes(), ("pair alone differs from the same pair in a batch of 16",
                                                        alone[3][0] - a[3][0])
    assert alone[0][0].tobytes() == a[0][0].tobytes() and alone[2][0] == a[2][0]
    dev = backend.device
    stk = lambda k: torch.tensor(np.stack([s[k] for s in scenes]), device=dev).contiguous()
    ins = [stk(k) for k in ("R0", "t0", "K0", "K1", "depth0", "depth1")]
    backend.icp(*ins, DIST)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = backend.icp(*ins, DIST)
    g.replay()
    torch.cuda.synchronize()
    state = backend.debug_tensor("icp_state", (16, 18), torch.float64).cpu().numpy()
    assert state.tobytes() == a[3].tobytes() and out[0].cpu().numpy().tobytes() == a[0].tobytes()
