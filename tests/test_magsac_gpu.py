"""MAGSAC++ E-mat RANSAC on the device (mfr_emat_magsac, PoseBackend.emat(..., scoring="magsac")):

1. the scores: block winners' costs against the oracle's sum of rho of the stored models (float32 scoring), the LO
   candidates' costs against it in fp64;
2. noise-free data: the rotation to 1e-6 rad;
3. against cv.findEssentialMat(USAC_MAGSAC), the estimator of the reference: the GPU result is at least as good under
   the reference's own objective, and the masks agree where cv2 finds the true inliers;
4. the escalation contract and CUDA-graph replay, as for mfr_emat_ransac_escalate; a pair gives the same bits alone
   and as pair 0 of a batch of 16;
5. the surface: the single-pair plugin with GPU_RANSAC.SCORING 'magsac' and a from_cfg stream.

Bars set from measurements state them beside the bar, measured on one NVIDIA H100 80GB HBM3 (700 W power limit)."""
import numpy as np
import pytest
import torch

import magsac_oracle as mo
from helpers import rot_angle, synth
from oracle import pose_solver_oracle as po
from oracle import pose_stages_oracle as so
from test_pipeline_cfg_host import _cfg
from test_ransac_escalation_gpu import _batch, _host_rule, _same

pytestmark = pytest.mark.gpu

PIX_THR, SCALE_THR, CONF, CAP = 2.0, 0.1, 0.9999, 32768
EMAT_SEQ = (2048, 8192, 32768)
MAGSAC = {"GPU_RANSAC": {"SCORING": "magsac"}}
HYP_COST_RTOL, LO_COST_RTOL = 1e-4, 1e-9
OBJECTIVE_SLACK = 1e-3           # GPU sum rho <= (1 + slack) x cv2's, per pair (measured: at most 0.9971 x)
MASK_IOU_BAR = 0.94              # mask IoU against cv2 where cv2 recovers >= 95 % of the true inliers (measured: 0.9425)


def _sigma(pix_thr, K0, K1):
    """sigma_max as the kernels compute it: the float32 normalised threshold."""
    return float(so.emat_threshold(pix_thr, K0, K1)[0])


def _E(R, t):
    t = np.asarray(t, np.float64).ravel()
    return po._skew(t) @ np.asarray(R, np.float64).reshape(3, 3)


def _records(be, name, dtype, rows, cols):
    words = rows * cols * dtype.itemsize // 4
    return be.debug_tensor(name, (words,), torch.int32).cpu().numpy().view(dtype).reshape(rows, cols)


def test_scores_against_oracle():
    from mfr_b200 import pose_solver
    sets = [synth.make_correspondences(900 + i, n=n, inlier_ratio=r) for i, (n, r) in
            enumerate([(1000, 0.8), (2000, 0.5), (1500, 0.3), (600, 0.2), (2000, 0.6), (1200, 0.4)])]
    P, num_hyp = len(sets), 2048
    k0, k1, off, K0, K1, _, _ = _batch(sets)
    be = pose_solver.PoseBackend(max_pairs=P, max_pts=8192, max_hyp=num_hyp)
    be.emat(k0, k1, off, K0, K1, PIX_THR, num_hyp, scoring="magsac")
    torch.cuda.synchronize()
    blocks = -(-num_hyp // so.emat_hyp_per_block(P, num_hyp, be._l.mfr_device_sm_count()))
    pts_all = be.debug_tensor("pts_norm", (P, 8192, 4), torch.float32).cpu().numpy()
    hyp = _records(be, "hyp_results", so.HYP_DTYPE, P, blocks)
    lo = _records(be, "lo_results", so.LO_DTYPE, P, so.LO_TOPK)
    worst_hyp = worst_lo = 0.0
    for p, s in enumerate(sets):
        N = len(s["kpts0"])
        pts = pts_all[p, :N].astype(np.float64)
        sigma = _sigma(PIX_THR, s["K_color0"], s["K_color1"])
        for r in hyp[p]:
            if not r["valid"]:
                continue
            want = mo.sum_rho_E(r["model"][:9], pts[:, :2], pts[:, 2:], sigma)
            worst_hyp = max(worst_hyp, abs(r["cost"] - want) / want)
        for r in lo[p]:
            assert r["cost"] < 1e299                     # MAGSAC++ optimises every one of the 4 candidates
            want = mo.sum_rho_E(_E(r["R"], r["t"]), pts[:, :2], pts[:, 2:], sigma)
            worst_lo = max(worst_lo, abs(r["cost"] - want) / want)
        # the candidates are the 4 cheapest block winners, and each is at least as good as its start after LO
        starts = sorted(float(r["cost"]) for r in hyp[p] if r["valid"])[:so.LO_TOPK]
        assert sorted(float(c) for c in lo[p]["cost"])[0] <= starts[0] * (1 + HYP_COST_RTOL)
    print(f"max relative error: block winners {worst_hyp:.2e}, LO candidates {worst_lo:.2e}")
    assert worst_hyp <= HYP_COST_RTOL and worst_lo <= LO_COST_RTOL
    be.close()


def test_noise_free():
    """Exact correspondences without outliers. (With outliers, those within k sigma_max of the epipolar line keep a
    weight, so the optimum of sum rho moves off the true pose: DESIGN §3.4.)"""
    from mfr_b200 import pose_solver
    c = synth.make_correspondences(77, n=1000, inlier_ratio=1.0, noise_px=0.0)
    k0, k1, off, K0, K1, _, _ = _batch([c])
    be = pose_solver.PoseBackend(max_pairs=1, max_pts=8192, max_hyp=CAP)
    R, t, n, _ = be.emat(k0, k1, off, K0, K1, PIX_THR, 2048, scoring="magsac", confidence=CONF, max_hyp=CAP)
    err = rot_angle(R[0].double().cpu().numpy(), c["R_gt"])
    print(f"rotation error {err:.2e} rad, inliers {int(n[0])}")
    assert err < 1e-6 and int(n[0]) == 1000
    be.close()


CELLS = [(n, r) for n in (500, 2000) for r in (0.2, 0.3, 0.5, 0.8)]


@pytest.mark.parametrize("n,ratio", CELLS)
def test_against_cv2(n, ratio):
    """8 seeds per cell, one batch: sum rho (the oracle's, fp64, over all correspondences) of the GPU pose against that
    of cv2's pose, and the mask IoU where cv2 recovers >= 95 % of the true inliers."""
    from mfr_b200 import pose_solver
    sets = [synth.make_correspondences(5000 + 100 * int(10 * ratio) + n + s, n=n, inlier_ratio=ratio, noise_px=0.5)
            for s in range(8)]
    k0, k1, off, K0, K1, _, _ = _batch(sets)
    be = pose_solver.PoseBackend(max_pairs=len(sets), max_pts=8192, max_hyp=CAP)
    R, t, cnt, mask = be.emat(k0, k1, off, K0, K1, PIX_THR, 2048, scoring="magsac", confidence=CONF, max_hyp=CAP)
    R, t, mask, off_h = R.double().cpu().numpy(), t.double().cpu().numpy(), mask.cpu().numpy(), off.tolist()
    ratios, ious = [], []
    for p, s in enumerate(sets):
        Rc, tc, nc, mc = po.essential_matrix_solver(s["kpts0"], s["kpts1"], s["K_color0"], s["K_color1"], PIX_THR, CONF)
        args = (s["kpts0"], s["kpts1"], s["K_color0"], s["K_color1"], PIX_THR)
        ours = mo.sum_rho(R[p], t[p], *args)
        ref = mo.sum_rho(Rc, tc, *args) if nc > 0 else np.inf
        ratios.append(ours / ref)
        m_gpu = mask[off_h[p]:off_h[p + 1]].astype(bool)
        if nc > 0:
            m_cv = np.asarray(mc).ravel().astype(bool)
            if (m_cv & s["inlier_gt"]).sum() >= 0.95 * s["inlier_gt"].sum():
                ious.append((m_gpu & m_cv).sum() / max(1, (m_gpu | m_cv).sum()))
    print(f"N={n} ratio={ratio}: sum-rho ratio GPU/cv2 max {max(ratios):.6f} median {np.median(ratios):.6f}; "
          f"mask IoU vs cv2 min {min(ious) if ious else float('nan'):.4f} over {len(ious)} pairs")
    assert max(ratios) <= 1.0 + OBJECTIVE_SLACK
    assert all(i >= MASK_IOU_BAR for i in ious)
    be.close()


def _esc_sets():
    sets = [synth.make_correspondences(400 + i, n=2000, inlier_ratio=r) for i, r in enumerate((0.8, 0.5, 0.3, 0.2))]
    sets.append(synth.make_correspondences(410, n=4, inlier_ratio=1.0))
    empty = dict(sets[0])
    empty["kpts0"], empty["kpts1"] = np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32)
    sets.append(empty)
    return sets


def test_escalation_contract_and_graph():
    from mfr_b200 import pose_solver
    sets = _esc_sets()
    k0, k1, off, K0, K1, d0, d1 = _batch(sets)
    P, off_h = len(sets), off.tolist()
    be = pose_solver.PoseBackend(max_pairs=P, max_pts=8192, max_hyp=CAP)
    budgets = torch.full((P,), -1, dtype=torch.int32, device="cuda")
    esc = be.emat(k0, k1, off, K0, K1, PIX_THR, EMAT_SEQ[0], scoring="magsac", confidence=CONF, max_hyp=CAP,
                  budgets=budgets)
    esc = [x.clone() for x in esc]
    fixed = {h: [x.clone() for x in be.emat(k0, k1, off, K0, K1, PIX_THR, h, scoring="magsac")] for h in EMAT_SEQ}
    torch.cuda.synchronize()
    b = budgets.tolist()
    Ns = [off_h[p + 1] - off_h[p] for p in range(P)]
    want = [_host_rule(5, {h: int(fixed[h][2][p]) for h in EMAT_SEQ}, Ns[p], EMAT_SEQ) for p in range(P)]
    print("budgets", b)
    assert b == want and any(x > EMAT_SEQ[0] for x in b) and b[-2:] == [0, 0]
    for p in range(P):
        ref = fixed[b[p] or EMAT_SEQ[0]]
        for k in range(3):
            assert _same(esc[k][p], ref[k][p]), (p, k)
        assert _same(esc[3][off_h[p]:off_h[p + 1]], ref[3][off_h[p]:off_h[p + 1]]), p
    assert torch.isnan(esc[0][4]).all() and int(esc[2][5]) == 0

    # the metric solver through the same entry, captured in a CUDA graph
    bm = torch.zeros(P, dtype=torch.int32, device="cuda")

    def calls():
        m = be.emat_metric(k0, k1, off, K0, K1, d0, d1, PIX_THR, SCALE_THR, EMAT_SEQ[0], confidence=CONF, max_hyp=CAP,
                           budgets=bm, scoring="magsac")
        e = be.emat(k0, k1, off, K0, K1, PIX_THR, EMAT_SEQ[0], scoring="magsac", confidence=CONF, max_hyp=CAP,
                    budgets=budgets)
        return list(m) + list(e) + [bm, budgets]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = [x.clone() for x in calls()]
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for k in range(3, 7):
        assert _same(eager[k], esc[k - 3]), k
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = calls()
    for _ in range(2):
        for x in outs:
            x.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        for k, (a, c) in enumerate(zip(outs, eager)):
            assert _same(a, c), k
    del g
    be.close()


def test_batch_independence():
    """Pair 0 alone and as pair 0 of a batch of 16 (seeds depend on the pair index; the hypothesis budget is one at
    which both launches put 128 hypotheses in a block)."""
    from mfr_b200 import pose_solver
    num_hyp = 16384
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    assert so.emat_hyp_per_block(1, num_hyp, sm) == so.emat_hyp_per_block(16, num_hyp, sm)
    sets = [synth.make_correspondences(600 + i, n=300 + 97 * i, inlier_ratio=0.25 + 0.04 * i) for i in range(16)]
    be = pose_solver.PoseBackend(max_pairs=16, max_pts=8192, max_hyp=num_hyp)
    k0, k1, off, K0, K1, _, _ = _batch(sets)
    batch = [x.clone() for x in be.emat(k0, k1, off, K0, K1, PIX_THR, num_hyp, scoring="magsac")]
    a0, a1, aoff, aK0, aK1, _, _ = _batch(sets[:1])
    alone = be.emat(a0, a1, aoff, aK0, aK1, PIX_THR, num_hyp, scoring="magsac")
    torch.cuda.synchronize()
    n0 = len(sets[0]["kpts0"])
    for k in range(3):
        assert _same(alone[k][0], batch[k][0]), k
    assert _same(alone[3][:n0], batch[3][:n0])
    assert int(alone[2][0]) > 0
    be.close()


def test_plugin_matches_backend():
    from mfr_b200 import config, pose_solver
    cfg = config.get_default_cfg()
    cfg.merge_from_dict({"EMAT_RANSAC": {"PIX_THRESHOLD": PIX_THR, "SCALE_THRESHOLD": SCALE_THR, "CONFIDENCE": CONF},
                         **MAGSAC})
    be = pose_solver.PoseBackend(max_pairs=1, max_pts=pose_solver.MAX_PTS_LIMIT, max_hyp=CAP)
    budget = torch.zeros(1, dtype=torch.int32, device="cuda")
    for i, s in enumerate(_esc_sets()[:5]):
        data = {k: s[k] for k in ("K_color0", "K_color1", "depth0", "depth1")}
        plugin = pose_solver.EssentialMatrixMetricSolver(cfg)
        assert plugin.scoring == "magsac"
        Rp, tp, n_p = plugin.estimate_pose(s["kpts0"], s["kpts1"], data)
        k0, k1, off, K0, K1, d0, d1 = _batch([s])
        R, t, n = be.emat_metric(k0, k1, off, K0, K1, d0, d1, PIX_THR, SCALE_THR, plugin.num_hyp, plugin.seed,
                                 confidence=CONF, max_hyp=CAP, budgets=budget, scoring="magsac")
        assert np.array_equal(R[0].double().cpu().numpy(), np.asarray(Rp), equal_nan=True), i
        assert np.array_equal(t[0].double().cpu().numpy().ravel(), np.asarray(tp).ravel(), equal_nan=True), i
        assert int(n[0]) == n_p, i
        if len(s["kpts0"]) >= 5:
            assert int(budget[0]) == plugin.last_num_hyp, i
        plugin.backend.close()
    be.close()


def test_from_cfg_stream():
    """sift_emat_dptkitti with SCORING 'magsac' streams what the batched back end gives on the engine's own matches."""
    from mfr_b200 import parallel, pipeline
    H, W, B, NQ = 240, 320, 2, 6
    pipe = pipeline.from_cfg(_cfg("sift_emat_dptkitti", {"DATASET": {"HEIGHT": H, "WIDTH": W}, **MAGSAC}), B,
                             depth_hw=(H, W))
    assert pipe.method.scoring == "magsac" and pipe.solver.scoring == "magsac"
    s = synth.make_scene(61, NQ, h=H, w=W, K=np.array([[300.0, 0, 159.5], [0, 300.0, 119.5], [0, 0, 1]]))
    gray = lambda x: torch.from_numpy(synth.rgb_to_gray_u8(x))
    fr = (gray(s["image0"])[None].expand(NQ, H, W).contiguous(), torch.stack([gray(q["image1"]) for q in s["queries"]]),
          torch.from_numpy(s["depth0"])[None].expand(NQ, H, W).contiguous(),
          torch.stack([torch.from_numpy(q["depth1"]) for q in s["queries"]]),
          torch.from_numpy(s["K_color0"])[None].expand(NQ, 3, 3).contiguous(),
          torch.stack([torch.from_numpy(q["K_color1"]) for q in s["queries"]]))
    eng, be, spec = pipe.eng, pipe.be, pipe.method
    seq = []
    for k in range(0, NQ, B):
        g0, g1, d0, d1, K0, K1 = (x[k:k + B].cuda() for x in fr)
        eng.forward_async(g0, g1)
        with torch.cuda.stream(eng.stream):
            R, t, n = be.emat_metric(*eng.pose_inputs(), K0, K1, d0, d1, spec.pix_thr, spec.scale_thr, spec.num_hyp,
                                     spec.seed, scoring="magsac")
        torch.cuda.synchronize()
        seq.append((R.cpu(), t.cpu(), n.cpu()))
    R, t, n = (torch.cat([o[j] for o in seq]) for j in range(3))
    assert int(n.max()) > 8
    pinned = [x.pin_memory() for x in fr]
    pg0, pg1, pd0, pd1, pK0, pK1 = pinned
    got = parallel.run_stream(NQ, B, lambda ids: pipe.submit_host(pg0[ids], pg1[ids], pd0[ids], pd1[ids], pK0[ids],
                                                                  pK1[ids]), pipe.drain)
    assert torch.equal(got[:, 1], n.to(torch.float64))
    assert torch.equal(got[:, 2:11].isnan(), R.reshape(NQ, 9).double().isnan())
    assert torch.equal(got[:, 2:11].nan_to_num(), R.reshape(NQ, 9).double().nan_to_num())
    assert torch.equal(got[:, 11:14].nan_to_num(), t.double().nan_to_num())
    print(f"stream inliers {n.tolist()}")
    pipe.eng.close(); pipe.be.close()
