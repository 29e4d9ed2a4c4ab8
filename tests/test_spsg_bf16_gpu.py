"""The SuperPoint + SuperGlue engine's bf16 mode (precision="bf16": bf16 conv / GEMM operands and the fused softmax
attention of sg_attention.cu) against the torch fp32 CPU oracle (oracle/spsg_oracle.py) on synthetic seeded weights,
its structure (no materialised attention scores, fewer launches than tf32), its determinism, and, when oracle/_ref is
staged, the reference's results with the real in-tree weights.

Bars (synthetic weights, the frame of test_spsg_gpu.py): score map and dense descriptors within 5e-2 of max magnitude,
keypoint-set IoU >= 0.8; SuperGlue alone on the oracle's keypoints: score matrix within 5e-2, matches agree on >= 0.8 of
the union. Real weights: keypoint-set IoU >= 0.85, match-set IoU >= 0.75 (measured on an H100: keypoint IoU 0.887 /
0.938 and match IoU 0.775 on readme_u8, 0.886 / 0.914 and 0.791 on synth1000, rounded down to 0.05)."""
import numpy as np
import pytest
import torch

from helpers import GOLDEN, spsg_real_cases, synth
from oracle import build_ref
from oracle import spsg_oracle as so

pytestmark = pytest.mark.gpu
H, W, K = 240, 320, 256


@pytest.fixture(scope="module")
def weights():
    from mfr_b200 import spsg
    return spsg.synthetic_state_dicts(0)


def _crop(p, dy, dx):
    g0 = synth.rgb_to_gray_u8(synth.make_pair(p)["image0"]).astype(np.float32) / 255.0
    return torch.from_numpy(g0[40 + dy:40 + dy + H, 30 + dx:30 + dx + W].copy())[None, None]


def _pair(p=5):
    return _crop(p, 0, 0), _crop(p, 8, 16)


def _rel(a, b):
    a = a.float().cpu(); b = b.float().cpu()
    return ((a - b).abs().max() / b.abs().max()).item()


def _iou(a, b):
    return len(a & b) / max(1, len(a | b))


def test_superpoint_bf16_matches_oracle(weights):
    from mfr_b200 import spsg
    sp, sg = weights
    i0, i1 = _pair()
    cfg = {"max_keypoints": K}
    eng = spsg.SuperPointSuperGlue(sp, sg, batch=1, height=H, width=W, cfg=cfg, graph=False, precision="bf16")
    out = eng.forward(i0.cuda(), i1.cuda())
    h8, w8 = H // 8, W // 8
    for n, img in enumerate((i0, i1)):
        with torch.no_grad():
            sc, desc = so.superpoint_dense(img, sp)
            k, s, d = so.superpoint(img, sp, cfg)
        e_sc = _rel(eng.debug_tensor("scores", (2, h8 * 8, w8 * 8))[n], sc[0])
        e_d = _rel(eng.debug_tensor("dense_desc", (2, h8, w8, 256))[n], desc[0].permute(1, 2, 0))
        cnt = int(out["counts"][n])
        got = {tuple(x) for x in out["keypoints"][n, :cnt].cpu().numpy().astype(int).tolist()}
        exp = {tuple(x) for x in k.numpy().astype(int).tolist()}
        print(f"image {n}: score map {e_sc:.3e}, dense descriptors {e_d:.3e}, keypoint IoU {_iou(got, exp):.3f}")
        assert e_sc < 5e-2 and e_d < 5e-2
        assert _iou(got, exp) >= 0.8
    eng.close()


def test_superglue_bf16_stage_matches_oracle(weights):
    """SuperGlue alone on the oracle's keypoints / descriptors (ragged: n0 != n1), match threshold 0."""
    from mfr_b200 import spsg
    sp, sg = weights
    i0, i1 = _pair()
    cfg = {"max_keypoints": K, "match_threshold": 0.0}
    with torch.no_grad():
        k0, s0, d0 = so.superpoint(i0, sp, cfg)
        k1, s1, d1 = so.superpoint(i1, sp, cfg)
        k1, s1, d1 = k1[:K - 37], s1[:K - 37], d1[:, :K - 37]
        m0, ms0, scores, Z = so.superglue(k0, s0, d0, k1, s1, d1, H, W, sg, cfg, return_scores=True)
    eng = spsg.SuperPointSuperGlue(sp, sg, batch=1, height=H, width=W, cfg=cfg, graph=False, precision="bf16")
    counts = np.array([len(k0), len(k1)], np.int32)
    kp = np.zeros((2, K, 2), np.float32); sc = np.zeros((2, K), np.float32); de = np.zeros((2, K, 256), np.float32)
    kp[0, :len(k0)] = k0.numpy(); kp[1, :len(k1)] = k1.numpy()
    sc[0, :len(k0)] = s0.numpy(); sc[1, :len(k1)] = s1.numpy()
    de[0, :len(k0)] = d0.t().numpy(); de[1, :len(k1)] = d1.t().numpy()
    out = eng.forward_superglue(counts, kp, sc, de)
    S = eng.debug_tensor("sg_scores", (1, K, K))[0, :len(k0), :len(k1)]
    e_s = _rel(S, scores)
    got = out["matches0"][0, :len(k0)].cpu().long()
    assert (got >= -1).all() and (got < len(k1)).all()
    both = (got > -1) & (m0 > -1)
    union = ((got > -1) | (m0 > -1)).sum().item()
    agree = (both & (got == m0)).sum().item()
    print(f"score matrix {e_s:.3e}, matches agree on {agree} of {union}")
    assert e_s < 5e-2
    assert union > 30 and agree >= 0.8 * union
    eng.close()


def test_bf16_structure(weights):
    from mfr_b200 import lib as _lib, spsg
    sp, sg = weights
    cfg = {"max_keypoints": K}
    e32 = spsg.SuperPointSuperGlue(sp, sg, batch=1, height=H, width=W, cfg=cfg, graph=False)
    e16 = spsg.SuperPointSuperGlue(sp, sg, batch=1, height=H, width=W, cfg=cfg, graph=False, precision="bf16")
    # 18 layers x (4 attention launches -> 1), one shadow refresh after the keypoint encoder and after 17 of the layers
    print(f"launches: tf32 {e32.num_launches()}, bf16 {e16.num_launches()}")
    assert e32.num_launches() - e16.num_launches() >= 35
    for name in ("attn_scores", "attn_vt"):
        e32.debug_tensor(name, (1,))
        with pytest.raises(_lib.MfrError):
            e16.debug_tensor(name, (1,))
    i0, i1 = _pair()
    e16.forward(i0.cuda(), i1.cuda())
    assert e16.debug_tensor("qkv", (2, K, 768)).dtype == torch.bfloat16
    assert e16.debug_tensor("msg", (2, K, 256)).dtype == torch.bfloat16
    assert e32.debug_tensor("qkv", (2, K, 768)).dtype == torch.float32
    e32.close(); e16.close()


def _outputs(o, p):
    n0, n1 = int(o["counts"][2 * p]), int(o["counts"][2 * p + 1])
    return {"counts": (n0, n1),
            "kpts0": o["keypoints"][2 * p, :n0].cpu(), "kpts1": o["keypoints"][2 * p + 1, :n1].cpu(),
            "desc0": o["descriptors"][2 * p, :n0].cpu(), "desc1": o["descriptors"][2 * p + 1, :n1].cpu(),
            "m0": o["matches0"][p, :n0].cpu(), "ms0": o["matching_scores0"][p, :n0].cpu()}


def _same(a, b):
    assert a["counts"] == b["counts"]
    for k in ("kpts0", "kpts1", "desc0", "desc1", "m0", "ms0"):
        assert torch.equal(a[k], b[k]), k


def test_bf16_deterministic_graph_and_batch(weights):
    from mfr_b200 import spsg
    sp, sg = weights
    cfg = {"max_keypoints": K, "match_threshold": 0.0}
    pairs = [_pair(5), _pair(6), _pair(7)]
    e1 = spsg.SuperPointSuperGlue(sp, sg, batch=1, height=H, width=W, cfg=cfg, graph=True, precision="bf16")
    a = _outputs(e1.forward(pairs[1][0].cuda(), pairs[1][1].cuda()), 0)    # captures the graph
    b = _outputs(e1.forward(pairs[1][0].cuda(), pairs[1][1].cuda()), 0)    # replay
    c = _outputs(e1.forward(pairs[1][0].cuda(), pairs[1][1].cuda()), 0)    # replay
    assert len(a["m0"]) > 10 and (a["m0"] > -1).sum() > 10
    _same(a, b); _same(b, c)
    e3 = spsg.SuperPointSuperGlue(sp, sg, batch=3, height=H, width=W, cfg=cfg, graph=True, precision="bf16")
    i0 = torch.cat([p[0] for p in pairs]).cuda(); i1 = torch.cat([p[1] for p in pairs]).cuda()
    _same(_outputs(e3.forward(i0, i1), 1), a)
    e1.close(); e3.close()


@pytest.fixture(scope="module")
def real_weights():
    w = build_ref.weights_dir()
    return (torch.load(w + "/superpoint_v1.pth", map_location="cpu"), torch.load(w + "/superglue_indoor.pth", map_location="cpu"))


def _match_pairs(k0, k1, m0):
    return {(tuple(k0[i].astype(int)), tuple(k1[j].astype(int))) for i, j in enumerate(m0) if j > -1}


@pytest.mark.skipif(not build_ref.available(), reason="oracle/_ref assets not staged (python oracle/build_ref.py)")
@pytest.mark.parametrize("name", ["readme_u8", "synth1000"])
def test_bf16_real_weights_close_to_reference(real_weights, name):
    from mfr_b200 import spsg
    G = np.load(GOLDEN + "/spsg_real_reference.npz")
    i0, i1 = {n: (a, b) for n, a, b in spsg_real_cases()}[name]
    sp, sg = real_weights
    h, w = i0.shape[-2:]
    eng = spsg.SuperPointSuperGlue(sp, sg, batch=1, height=h, width=w, graph=False, precision="bf16")
    o = eng.forward(i0.cuda(), i1.cuda())
    n0, n1 = int(o["counts"][0]), int(o["counts"][1])
    k = [o["keypoints"][0, :n0].cpu().numpy(), o["keypoints"][1, :n1].cpu().numpy()]
    m0 = o["matches0"][0, :n0].cpu().numpy()
    eng.close()
    ious = []
    for side in (0, 1):
        got = {tuple(x) for x in k[side].astype(int).tolist()}
        exp = {tuple(x) for x in G[f"{name}_keypoints{side}"].astype(int).tolist()}
        ious.append(_iou(got, exp))
    got_m = _match_pairs(k[0], k[1], m0)
    exp_m = _match_pairs(G[name + "_keypoints0"], G[name + "_keypoints1"], G[name + "_matches0"])
    print(f"{name}: keypoint IoU {ious[0]:.3f} / {ious[1]:.3f}, match IoU {_iou(got_m, exp_m):.3f} "
          f"({len(got_m)} matches, reference {len(exp_m)})")
    assert min(ious) >= 0.85
    assert _iou(got_m, exp_m) >= 0.75
