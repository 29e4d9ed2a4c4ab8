"""RelocPipeline with every pair engine (LoFTR, SuperPoint + SuperGlue, SIFT) and every pose stage (EMatMetric, EMat,
PnP, Procrustes, Procrustes + ICP): through parallel.run_stream, the pipeline must give, one call late, what the
synchronous sequence gives (engine forward, then the same PoseBackend call on the same batch), and the shared-map path
(set_map + submit_*_queries) what the paired path gives with the map frame repeated."""
import numpy as np
import pytest
import torch

from helpers import synth

pytestmark = pytest.mark.gpu
H, W, B, N = 240, 320, 2, 6          # 6 queries: 3 batches
K_SMALL = np.array([[300.0, 0, 159.5], [0, 300.0, 119.5], [0, 0, 1]])


def _stages():
    from mfr_b200.pipeline import EMatMetricStage, EMatStage, PnPStage, ProcrustesStage
    return {"emat_metric": EMatMetricStage(2.0, 0.3, 512), "emat": EMatStage(2.0, 512, seed=11, lo=3),
            "pnp": PnPStage(3.0, 512), "procrustes": ProcrustesStage(0.05, 512),
            "procrustes_icp": ProcrustesStage(0.05, 512, seed=5, refine=True)}


def _engine(matcher):
    from mfr_b200 import loftr, sift, spsg
    if matcher == "loftr":
        return loftr.LoFTR(loftr.functional_state_dict(), batch=B, height=H, width=W, cfg={"thr": 0.2}, graph=True)
    if matcher == "spsg":
        sp, sg = spsg.synthetic_state_dicts(0)
        # match_threshold 0: the synthetic SuperGlue weights give no match above the default 0.2
        return spsg.SuperPointSuperGlue(sp, sg, batch=B, height=H, width=W, cfg={"max_keypoints": 512, "match_threshold": 0.0},
                                        graph=True)
    return sift.SIFTPairs(B, H, W)


def _frames(s, dtype):
    """Map frame and queries of scene s as [n,H,W] images of the engine's dtype, depths and intrinsics (host)."""
    gray = lambda x: torch.from_numpy(synth.rgb_to_gray_u8(x))
    img = gray if dtype == torch.uint8 else (lambda x: gray(x).float() / 255.0)
    g0 = img(s["image0"])[None].expand(N, H, W).contiguous()
    g1 = torch.stack([img(q["image1"]) for q in s["queries"]])
    d0 = torch.from_numpy(s["depth0"])[None].expand(N, H, W).contiguous()
    d1 = torch.stack([torch.from_numpy(q["depth1"]) for q in s["queries"]])
    K0 = torch.from_numpy(s["K_color0"])[None].expand(N, 3, 3).contiguous()
    K1 = torch.stack([torch.from_numpy(q["K_color1"]) for q in s["queries"]])
    return g0, g1, d0, d1, K0, K1


def _sequential(eng, be, stage, fr):
    """Synchronous reference: per batch, the engine forward, then the stage's PoseBackend calls on the engine stream."""
    out = []
    for k in range(0, N, B):
        g0, g1, d0, d1, K0, K1 = (x[k:k + B].cuda() for x in fr)
        eng.forward_async(g0, g1)
        with torch.cuda.stream(eng.stream):
            R, t, n = stage(be, *eng.pose_inputs(), K0, K1, d0, d1)
        torch.cuda.synchronize()
        out.append((R.cpu(), t.cpu(), n.cpu()))
    return (torch.cat([o[0] for o in out]), torch.cat([o[1] for o in out]), torch.cat([o[2] for o in out]))


@pytest.mark.parametrize("matcher", ["loftr", "spsg", "sift"])
def test_pipeline_methods(matcher):
    from mfr_b200 import parallel, pose_solver
    from mfr_b200.pipeline import RelocPipeline
    eng = _engine(matcher)
    be = pose_solver.PoseBackend(max_pairs=B, max_pts=min(eng.max_pts_per_pair, pose_solver.MAX_PTS_LIMIT), max_hyp=512)
    s = synth.make_scene(61, N, h=H, w=W, K=K_SMALL)
    fr = _frames(s, eng.input_dtype)
    pinned = [x.pin_memory() for x in fr]
    g0, g1, d0, d1, K0, K1 = pinned
    for name, stage in _stages().items():
        R, t, n = _sequential(eng, be, stage, fr)
        assert int(n.max()) > 8, f"{matcher}/{name}: the synthetic scene should give solvable poses"
        pipe = RelocPipeline(eng, be, depth_hw=(H, W), solver=stage)
        paired = parallel.run_stream(N, B, lambda ids: pipe.submit_host(g0[ids], g1[ids], d0[ids], d1[ids], K0[ids], K1[ids]),
                                     pipe.drain)
        assert torch.equal(paired[:, 1], n.to(torch.float64)), name
        assert torch.allclose(paired[:, 2:11], R.reshape(N, 9).double(), atol=1e-6, equal_nan=True), name
        assert torch.allclose(paired[:, 11:14], t.double(), atol=1e-6, equal_nan=True), name
        pipe.reset()
        pipe.set_map(fr[0][0], torch.from_numpy(s["depth0"]), torch.from_numpy(s["K_color0"]))
        shared = parallel.run_stream(N, B, lambda ids: pipe.submit_host_queries(g1[ids], d1[ids], K1[ids]), pipe.drain)
        assert torch.equal(shared.isnan(), paired.isnan()) and torch.equal(shared.nan_to_num(), paired.nan_to_num()), name
        pipe.reset()                                  # and the device-resident query path
        got = [pipe.submit_device_queries(*(x[k:k + B].cuda() for x in (g1, d1, K1))) for k in range(0, N, B)] + [pipe.drain()]
        assert got[0] is None
        n_dev = torch.cat([r[2] for r in got[1:]])
        assert torch.equal(n_dev.to(torch.float64), shared[:, 1]), name
        print(f"{matcher}/{name}: inliers {n.tolist()}")
    eng.close(); be.close()
