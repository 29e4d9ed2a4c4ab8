"""CONFIDENCE escalation on the device (mfr_emat_ransac_escalate / mfr_pnp_ransac_escalate):

1. batch contract: each pair's outputs equal, bit for bit, those of the fixed-budget call on the same batch at the budget
   the pair stopped at, and that budget is the plugins' host rule replayed over the fixed calls at every budget;
2. single pair: the device escalation gives what the single-pair plugins' host loop gives, budget included;
3. the escalating calls make no host round trip: captured in a CUDA graph they replay to the eager result;
4. RelocPipeline with escalating stages gives what the synchronous stage calls give.
"""
import numpy as np
import pytest
import torch

from helpers import synth
from test_pipeline_cfg_host import _cfg

pytestmark = pytest.mark.gpu

RATIOS = (0.8, 0.5, 0.3, 0.2, 0.1)
CONF, CAP = 0.9999, 32768
PIX_THR, SCALE_THR, REPROJ_THR = 2.0, 0.1, 3.0
EMAT_SEQ, PNP_SEQ = (2048, 8192, 32768), (1024, 4096, 16384, 32768)
CFG = {"EMAT_RANSAC": {"PIX_THRESHOLD": PIX_THR, "SCALE_THRESHOLD": SCALE_THR, "CONFIDENCE": CONF},
       "PNP": {"RANSAC_ITER": 1000, "REPROJECTION_INLIER_THRESHOLD": REPROJ_THR, "CONFIDENCE": CONF},
       "GPU_RANSAC": {"MAX_HYPOTHESES": CAP}}
FOUR, OUTLIERS, EMPTY = 5, 6, 7          # indices of the extra sets


def _sets():
    """Inlier ratios 0.8 .. 0.1 at N = 2000, then 4 correspondences, pure outliers without valid depth in frame 0 (no
    PnP lift, no metric scale) and an empty set."""
    sets = [synth.make_correspondences(300 + i, n=2000, inlier_ratio=r) for i, r in enumerate(RATIOS)]
    sets.append(synth.make_correspondences(310, n=4, inlier_ratio=1.0))
    out = synth.make_correspondences(311, n=2000, inlier_ratio=0.0)
    out["depth0"] = np.zeros_like(out["depth0"])
    sets.append(out)
    empty = dict(sets[0])
    empty["kpts0"], empty["kpts1"] = np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32)
    sets.append(empty)
    return sets


def _batch(sets):
    cat = lambda k: torch.from_numpy(np.concatenate([s[k] for s in sets]).astype(np.float32)).reshape(-1, 2).cuda().contiguous()
    stack = lambda k: torch.from_numpy(np.stack([np.asarray(s[k], np.float32) for s in sets])).cuda().contiguous()
    off = torch.tensor(np.concatenate([[0], np.cumsum([len(s["kpts0"]) for s in sets])]), dtype=torch.int32).cuda()
    return cat("kpts0"), cat("kpts1"), off, stack("K_color0"), stack("K_color1"), stack("depth0"), stack("depth1")


def _bits(x):
    return x.contiguous().view(torch.int32) if x.dtype == torch.float32 else x


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _host_rule(sample_size, counts, N, seq):
    """The plugins' loop (pose_solver._SolverBase) replayed over the inlier counts of fixed calls at every budget."""
    from mfr_b200 import pose_solver
    rule = object.__new__(pose_solver._SolverBase)
    rule.max_hyp, rule.SAMPLE_SIZE = seq[-1], sample_size
    if N < sample_size:
        return 0
    for h in seq:
        if rule._satisfied(CONF, counts[h], N, h):
            return h
    return seq[-1]


def _check_pairs(name, esc, fixed, budgets, off, mask_idx=None):
    """Pair p of the escalating outputs `esc` equals pair p of the fixed call at budgets[p] (round 0's call when 0)."""
    for p in range(len(budgets)):
        h = budgets[p] or min(fixed)
        ref = fixed[h]
        for k, (a, b) in enumerate(zip(esc, ref)):
            if k == mask_idx:
                a, b = a[off[p]:off[p + 1]], b[off[p]:off[p + 1]]
            else:
                a, b = a[p], b[p]
            assert _same(a, b), (name, p, h, k)


def test_batch_contract():
    from mfr_b200 import pose_solver
    sets = _sets()
    k0, k1, off, K0, K1, d0, d1 = _batch(sets)
    P, off_h = len(sets), off.tolist()
    Ns = [min(off_h[p + 1] - off_h[p], 8192) for p in range(P)]
    be = pose_solver.PoseBackend(max_pairs=P, max_pts=8192, max_hyp=CAP)
    b_emat, b_metric, b_pnp = (torch.full((P,), -1, dtype=torch.int32, device="cuda") for _ in range(3))

    emat = be.emat(k0, k1, off, K0, K1, PIX_THR, EMAT_SEQ[0], lo=3, confidence=CONF, max_hyp=CAP, budgets=b_emat)
    metric = be.emat_metric(k0, k1, off, K0, K1, d0, d1, PIX_THR, SCALE_THR, EMAT_SEQ[0], lo=3, confidence=CONF,
                            max_hyp=CAP, budgets=b_metric)
    pnp = be.pnp(k0, k1, off, K0, K1, d0, REPROJ_THR, PNP_SEQ[0], confidence=CONF, max_hyp=CAP, budgets=b_pnp)
    emat_fixed = {h: be.emat(k0, k1, off, K0, K1, PIX_THR, h, lo=3) for h in EMAT_SEQ}
    metric_fixed = {h: be.emat_metric(k0, k1, off, K0, K1, d0, d1, PIX_THR, SCALE_THR, h, lo=3) for h in EMAT_SEQ}
    pnp_fixed = {h: be.pnp(k0, k1, off, K0, K1, d0, REPROJ_THR, h) for h in PNP_SEQ}
    torch.cuda.synchronize()

    b_emat, b_metric, b_pnp = b_emat.tolist(), b_metric.tolist(), b_pnp.tolist()
    # the budgets: the host rule over the E-mat (also for the metric solver) and PnP inlier counts of the fixed calls
    want_emat = [_host_rule(5, {h: int(emat_fixed[h][2][p]) for h in EMAT_SEQ}, Ns[p], EMAT_SEQ) for p in range(P)]
    want_pnp = [_host_rule(4, {h: int(pnp_fixed[h][2][p]) for h in PNP_SEQ}, Ns[p], PNP_SEQ) for p in range(P)]
    print("budgets emat", b_emat, "pnp", b_pnp)
    assert b_emat == want_emat and b_metric == want_emat and b_pnp == want_pnp

    _check_pairs("emat", emat, emat_fixed, b_emat, off_h, mask_idx=3)
    _check_pairs("emat_metric", metric, metric_fixed, b_metric, off_h)
    _check_pairs("pnp", pnp, pnp_fixed, b_pnp, off_h, mask_idx=3)

    for b, seq in ((b_emat, EMAT_SEQ), (b_pnp, PNP_SEQ)):
        assert any(x > seq[0] for x in b) and any(x == seq[0] for x in b)
        assert b[OUTLIERS] == CAP and b[EMPTY] == 0
    assert b_emat[FOUR] == 0 and torch.isnan(emat[0][FOUR]).all() and int(emat[2][FOUR]) == 0
    for R, t, n in (metric, pnp[:3]):        # no depth in frame 0: no scale, no lift
        assert torch.isnan(R[OUTLIERS]).all() and torch.isnan(t[OUTLIERS]).all() and int(n[OUTLIERS]) == 0
    for R, t, n in (emat[:3], metric, pnp[:3]):
        assert torch.isnan(R[EMPTY]).all() and int(n[EMPTY]) == 0
    # a cap above the handle's is refused, not clipped
    from mfr_b200 import lib
    with pytest.raises(lib.MfrError):
        be.pnp(k0, k1, off, K0, K1, d0, REPROJ_THR, PNP_SEQ[0], confidence=CONF, max_hyp=2 * CAP)
    be.close()


def test_single_pair_matches_plugins():
    from mfr_b200 import pose_solver
    be = pose_solver.PoseBackend(max_pairs=1, max_pts=pose_solver.MAX_PTS_LIMIT, max_hyp=CAP)
    budget = torch.zeros(1, dtype=torch.int32, device="cuda")
    as_np = lambda R, t: (R[0].double().cpu().numpy(), t[0].double().cpu().numpy().ravel())
    for i, s in enumerate(_sets()):
        data = {k: s[k] for k in ("K_color0", "K_color1", "depth0", "depth1")}
        k0, k1, off, K0, K1, d0, d1 = _batch([s])
        for kind in ("emat", "emat_metric", "pnp"):
            plugin = {"emat": pose_solver.EssentialMatrixSolver, "emat_metric": pose_solver.EssentialMatrixMetricSolver,
                      "pnp": pose_solver.PnPSolver}[kind](CFG)
            Rp, tp, n_p = plugin.estimate_pose(s["kpts0"], s["kpts1"], data)
            budget.fill_(-1)
            if kind == "emat":
                R, t, n, _ = be.emat(k0, k1, off, K0, K1, PIX_THR, plugin.num_hyp, plugin.seed, plugin.lo,
                                     confidence=CONF, max_hyp=CAP, budgets=budget)
            elif kind == "emat_metric":
                R, t, n = be.emat_metric(k0, k1, off, K0, K1, d0, d1, PIX_THR, SCALE_THR, plugin.num_hyp, plugin.seed,
                                         plugin.lo, confidence=CONF, max_hyp=CAP, budgets=budget)
            else:
                R, t, n, _ = be.pnp(k0, k1, off, K0, K1, d0, REPROJ_THR, plugin.num_hyp, plugin.seed, confidence=CONF,
                                    max_hyp=CAP, budgets=budget)
            Rd, td = as_np(R, t)
            assert np.array_equal(Rd, np.asarray(Rp), equal_nan=True), (i, kind)
            assert np.array_equal(td, np.asarray(tp).ravel(), equal_nan=True), (i, kind)
            assert int(n[0]) == n_p and int(budget[0]) == plugin.last_num_hyp, (i, kind, int(budget[0]), plugin.last_num_hyp)
            plugin.backend.close()
    be.close()


def test_cuda_graph_replay():
    from mfr_b200 import pose_solver
    sets = _sets()
    k0, k1, off, K0, K1, d0, d1 = _batch(sets)
    P = len(sets)
    be = pose_solver.PoseBackend(max_pairs=P, max_pts=8192, max_hyp=CAP)
    bm, bp = (torch.zeros(P, dtype=torch.int32, device="cuda") for _ in range(2))

    def calls():
        m = be.emat_metric(k0, k1, off, K0, K1, d0, d1, PIX_THR, SCALE_THR, EMAT_SEQ[0], lo=3, confidence=CONF,
                           max_hyp=CAP, budgets=bm)
        p = be.pnp(k0, k1, off, K0, K1, d0, REPROJ_THR, PNP_SEQ[0], confidence=CONF, max_hyp=CAP, budgets=bp)
        return list(m) + list(p[:3]) + [bm, bp]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = [x.clone() for x in calls()]
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = calls()
    for _ in range(2):
        for x in outs:
            x.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        for k, (a, b) in enumerate(zip(outs, eager)):
            assert _same(a, b), k
    assert max(eager[-2].tolist()) > EMAT_SEQ[0] and max(eager[-1].tolist()) > PNP_SEQ[0]
    del g
    be.close()


H, W, B, NQ = 240, 320, 2, 6
K_SMALL = np.array([[300.0, 0, 159.5], [0, 300.0, 119.5], [0, 0, 1]])


def test_stream_with_escalation():
    from mfr_b200 import parallel, pipeline, pose_solver, sift
    from mfr_b200.pipeline import EMatMetricStage, PnPStage, RelocPipeline
    eng = sift.SIFTPairs(B, H, W)
    be = pose_solver.PoseBackend(max_pairs=B, max_pts=min(eng.max_pts_per_pair, pose_solver.MAX_PTS_LIMIT), max_hyp=8192)
    s = synth.make_scene(61, NQ, h=H, w=W, K=K_SMALL)
    gray = lambda x: torch.from_numpy(synth.rgb_to_gray_u8(x))
    g0 = gray(s["image0"])[None].expand(NQ, H, W).contiguous()
    g1 = torch.stack([gray(q["image1"]) for q in s["queries"]])
    d0 = torch.from_numpy(s["depth0"])[None].expand(NQ, H, W).contiguous()
    d1 = torch.stack([torch.from_numpy(q["depth1"]) for q in s["queries"]])
    K0 = torch.from_numpy(s["K_color0"])[None].expand(NQ, 3, 3).contiguous()
    K1 = torch.stack([torch.from_numpy(q["K_color1"]) for q in s["queries"]])
    fr = (g0, g1, d0, d1, K0, K1)
    pinned = [x.pin_memory() for x in fr]
    # first budget 128: pairs below ~0.6 (E-mat) / ~0.5 (PnP) inlier ratio escalate
    stages = {"emat_metric": EMatMetricStage(PIX_THR, 0.3, 128, confidence=CONF, max_hyp=8192),
              "pnp": PnPStage(REPROJ_THR, 128, confidence=CONF, max_hyp=8192)}
    for name, stage in stages.items():
        seq = []
        for k in range(0, NQ, B):
            gb0, gb1, db0, db1, Kb0, Kb1 = (x[k:k + B].cuda() for x in fr)
            eng.forward_async(gb0, gb1)
            with torch.cuda.stream(eng.stream):
                R, t, n = stage(be, *eng.pose_inputs(), Kb0, Kb1, db0, db1)
            torch.cuda.synchronize()
            seq.append((R.cpu(), t.cpu(), n.cpu()))
        R, t, n = (torch.cat([o[j] for o in seq]) for j in range(3))
        assert int(n.max()) > 8, name
        pipe = RelocPipeline(eng, be, depth_hw=(H, W), solver=stage)
        pg0, pg1, pd0, pd1, pK0, pK1 = pinned
        paired = parallel.run_stream(NQ, B, lambda ids: pipe.submit_host(pg0[ids], pg1[ids], pd0[ids], pd1[ids], pK0[ids],
                                                                         pK1[ids]), pipe.drain)
        assert torch.equal(paired[:, 1], n.to(torch.float64)), name
        assert torch.allclose(paired[:, 2:11], R.reshape(NQ, 9).double(), atol=1e-6, equal_nan=True), name
        assert torch.allclose(paired[:, 11:14], t.double(), atol=1e-6, equal_nan=True), name
        pipe.reset()
        pipe.set_map(g0[0], torch.from_numpy(s["depth0"]), torch.from_numpy(s["K_color0"]))
        shared = parallel.run_stream(NQ, B, lambda ids: pipe.submit_host_queries(pg1[ids], pd1[ids], pK1[ids]), pipe.drain)
        assert torch.equal(shared.isnan(), paired.isnan()) and torch.equal(shared.nan_to_num(), paired.nan_to_num()), name
        pipe.reset()
        print(f"{name}: inliers {n.tolist()}")
    eng.close(); be.close()

    pipe = pipeline.from_cfg(_cfg("sift_pnp_dptkitti"), B, escalate=True)
    assert (pipe.solver.confidence, pipe.solver.max_hyp, pipe.solver.num_hyp) == (CONF, CAP, 1024)
    assert pipe.be.max_hyp >= CAP
    pipe.eng.close(); pipe.be.close()
    pipe = pipeline.from_cfg(_cfg("sift_pnp_dptkitti"), B)
    assert pipe.solver.confidence is None and pipe.be.max_hyp == 1024
    pipe.eng.close(); pipe.be.close()
