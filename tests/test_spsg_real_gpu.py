"""SuperPoint + SuperGlue CUDA engine with the reference's REAL in-tree weights against vectors of the UNMODIFIED
reference (tests/golden/spsg_real_reference.npz): the SuperGlue README's known-answer ScanNet pair (382 / 391 keypoints
with match_pairs.py's uint8 resize, README.md:121-127; 371 / 376 with the float resize of the FMB matcher plugin) and
a synthetic 540x720 pair at BASELINE config C3 (1024 keypoints). The weights and the two sample images are staged by
oracle/build_ref.py into oracle/_ref/ (git-ignored, travels with the gpurun snapshot); without them the tests skip.

Bars: fp32x3 (3xTF32 split GEMMs): keypoint coordinates and match indices IDENTICAL to the reference's fp32 result
(they are integer outputs); tf32: keypoint-set IoU >= 0.9, match-set IoU >= 0.8 (TF32 moves detections whose score is
near the 0.005 threshold or near a neighbour's inside the 9x9 NMS window by one pixel)."""
import numpy as np
import pytest
import torch

from helpers import GOLDEN, checksum, spsg_real_cases
from oracle import build_ref

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not build_ref.available(), reason="oracle/_ref assets not staged (python oracle/build_ref.py)")]


@pytest.fixture(scope="module")
def real_weights():
    w = build_ref.weights_dir()
    return (torch.load(w + "/superpoint_v1.pth", map_location="cpu"), torch.load(w + "/superglue_indoor.pth", map_location="cpu"))


@pytest.fixture(scope="module")
def cases():
    return {n: (a, b) for n, a, b in spsg_real_cases()}


def _run(real_weights, i0, i1, precision):
    from mfr_b200 import spsg
    sp, sg = real_weights
    H, W = i0.shape[-2:]
    eng = spsg.SuperPointSuperGlue(sp, sg, batch=1, height=H, width=W, graph=False, precision=precision)
    o = eng.forward(i0.cuda(), i1.cuda())
    n0, n1 = int(o["counts"][0]), int(o["counts"][1])
    res = {"k0": o["keypoints"][0, :n0].cpu().numpy(), "k1": o["keypoints"][1, :n1].cpu().numpy(),
           "s0": o["scores"][0, :n0].cpu().numpy(), "m0": o["matches0"][0, :n0].cpu().numpy(),
           "ms0": o["matching_scores0"][0, :n0].cpu().numpy()}
    eng.close()
    return res


def _match_pairs(k0, k1, m0):
    return {(tuple(k0[i].astype(int)), tuple(k1[j].astype(int))) for i, j in enumerate(m0) if j > -1}


@pytest.mark.parametrize("name", ["readme_u8", "readme", "synth1000"])
def test_fp32x3_identical_keypoints_and_matches(real_weights, cases, name):
    G = np.load(GOLDEN + "/spsg_real_reference.npz")
    i0, i1 = cases[name]
    assert abs(checksum(i0.numpy(), i1.numpy()) - float(G[name + "_checksum"])) < 1e-6 * abs(float(G[name + "_checksum"]))
    r = _run(real_weights, i0, i1, "fp32x3")
    if name == "readme_u8":
        assert (len(r["k0"]), len(r["k1"])) == (382, 391)          # SuperGlue/README.md:121-127
    for side in ("0", "1"):
        got = {tuple(x) for x in r["k" + side].astype(int).tolist()}
        exp = {tuple(x) for x in G[f"{name}_keypoints{side}"].astype(int).tolist()}
        assert got == exp, f"keypoint set of image {side} differs: {len(got ^ exp)} of {len(exp)}"
    # scores of the same keypoints
    gi = {tuple(x): n for n, x in enumerate(r["k0"].astype(int).tolist())}
    order = [gi[tuple(x)] for x in G[name + "_keypoints0"].astype(int).tolist()]
    np.testing.assert_allclose(r["s0"][order], G[name + "_scores0"], rtol=0, atol=3e-4)   # measured <= 9e-5 (3xTF32 through 11 conv layers + softmax)
    got_m = _match_pairs(r["k0"], r["k1"], r["m0"])
    exp_m = _match_pairs(G[name + "_keypoints0"], G[name + "_keypoints1"], G[name + "_matches0"])
    assert got_m == exp_m, f"matches differ: {len(got_m ^ exp_m)} of {len(exp_m)}"
    ms = r["ms0"][order]
    sel = G[name + "_matches0"] > -1
    np.testing.assert_allclose(ms[sel], G[name + "_matching_scores0"][sel], rtol=0, atol=1e-3)


@pytest.mark.parametrize("name", ["readme_u8", "synth1000"])
def test_tf32_close_to_reference(real_weights, cases, name):
    G = np.load(GOLDEN + "/spsg_real_reference.npz")
    i0, i1 = cases[name]
    r = _run(real_weights, i0, i1, "tf32")
    for side in ("0", "1"):
        got = {tuple(x) for x in r["k" + side].astype(int).tolist()}
        exp = {tuple(x) for x in G[f"{name}_keypoints{side}"].astype(int).tolist()}
        assert len(got & exp) >= 0.9 * len(got | exp)          # keypoint-set IoU
    got_m = _match_pairs(r["k0"], r["k1"], r["m0"])
    exp_m = _match_pairs(G[name + "_keypoints0"], G[name + "_keypoints1"], G[name + "_matches0"])
    assert len(got_m & exp_m) >= 0.8 * len(got_m | exp_m)      # match-set IoU
