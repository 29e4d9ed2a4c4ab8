"""Cross-check of the oracle restatements against outputs of the UNMODIFIED reference modules, stored in
tests/golden/oracle_vs_reference.npz and tests/golden/spsg_real_reference.npz (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest
import torch

from helpers import pose_case
from oracle import build_ref, loftr_oracle, pose_solver_oracle as po

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden():
    return np.load(os.path.join(GOLDEN, "oracle_vs_reference.npz"))


def _checksum(*arrays):
    return float(sum(np.float64(np.asarray(a, dtype=np.float64)).sum() for a in arrays))


def test_pose_solver_module_matches_oracle():
    G = _golden()
    c = pose_case(1)
    assert _checksum(c["kpts0"], c["kpts1"], c["depth0"], c["depth1"]) == pytest.approx(float(G["pose_checksum"]), rel=1e-12)
    for solver in ("EssentialMatrixMetric", "PNP"):
        if solver == "PNP":
            Ro, to, no = po.pnp_solver(c["kpts0"], c["kpts1"], c["depth0"], c["K_color0"], c["K_color1"], 1000, 3, 0.9999)
        else:
            Ro, to, no = po.essential_matrix_metric_solver(c["kpts0"], c["kpts1"], c["depth0"], c["depth1"],
                                                           c["K_color0"], c["K_color1"], 2.0, 0.9999, 0.1)
        np.testing.assert_allclose(G[solver + "_R"], np.float32(Ro), atol=1e-6)
        np.testing.assert_allclose(G[solver + "_t"], np.float32(to).ravel(), atol=1e-6)
        assert int(G[solver + "_inliers"]) == no


def test_loftr_module_matches_oracle():
    G = _golden()
    sd = loftr_oracle.make_state_dict(3)
    # the oracle's state dict carries exactly the reference model's parameters and buffers
    assert set(sd) - {k for k in sd if "num_batches_tracked" in k} == set(G["loftr_param_names"].tolist())
    g = torch.Generator().manual_seed(5)
    i0 = torch.rand(1, 1, 96, 64, generator=g)
    i1 = torch.roll(i0, (8, 8), (2, 3))
    assert _checksum(i0.numpy()) == pytest.approx(float(G["loftr_checksum"]), rel=1e-12)
    with torch.no_grad():
        o = loftr_oracle.loftr_forward(i0, i1, sd, {"thr": 0.0}, True)
    assert torch.equal(torch.from_numpy(G["loftr_i_ids"]), o["i_ids"]) and torch.equal(torch.from_numpy(G["loftr_j_ids"]), o["j_ids"])
    torch.testing.assert_close(torch.from_numpy(G["loftr_conf_matrix"]), o["conf"], rtol=1e-5, atol=1e-12)
    torch.testing.assert_close(torch.from_numpy(G["loftr_mkpts1_f"]), o["mkpts1_f"], atol=2e-4, rtol=0)


@pytest.mark.skipif(not build_ref.available(), reason="oracle/_ref assets not staged")
def test_spsg_modules_match_oracle_with_real_weights():
    """The in-tree SuperPoint/SuperGlue weights on the ScanNet sample pair: identical keypoints, descriptors and matches
    to the reference (the reference README's known-answer pair, SuperGlue/README.md:121-127)."""
    from helpers import spsg_real_cases
    from oracle import spsg_oracle as so
    G = np.load(os.path.join(GOLDEN, "spsg_real_reference.npz"))
    sp_sd = torch.load(os.path.join(build_ref.weights_dir(), "superpoint_v1.pth"), map_location="cpu")
    sg_sd = torch.load(os.path.join(build_ref.weights_dir(), "superglue_indoor.pth"), map_location="cpu")
    name, i0, i1 = next(c for c in spsg_real_cases() if c[0] == "readme")
    with torch.no_grad():
        k0, s0, d0 = so.superpoint(i0, sp_sd)
        k1, s1, d1 = so.superpoint(i1, sp_sd)
        m0, ms0 = so.superglue(k0, s0, d0, k1, s1, d1, 480, 640, sg_sd)
    assert torch.equal(k0, torch.from_numpy(G[name + "_keypoints0"])) and torch.equal(k1, torch.from_numpy(G[name + "_keypoints1"]))
    torch.testing.assert_close(d0[::8, ::4], torch.from_numpy(G[name + "_descriptors0_sample"]), atol=1e-6, rtol=0)
    assert torch.equal(m0, torch.from_numpy(G[name + "_matches0"])) and int((m0 > -1).sum()) > 100
    torch.testing.assert_close(ms0, torch.from_numpy(G[name + "_matching_scores0"]), atol=1e-5, rtol=0)
