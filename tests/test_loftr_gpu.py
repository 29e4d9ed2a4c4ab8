"""GPU parity of the CUDA LoFTR engine: stage-wise against the torch fp32 CPU oracle, end to end
against the committed reference vectors, and bit-exact match selection at the conf-matrix boundary.

Tolerances (TF32 tensor-core inputs, fp32 accumulate; the reference's own GPU path runs cuDNN convs in
TF32 too): feature maps within 2e-2 of the tensor's max magnitude; fine-level keypoints within 0.25 px;
integer outputs (i_ids / j_ids) bit-exact given the same confidence matrix."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import GOLDEN, loftr_case
from oracle import loftr_oracle as lo

pytestmark = pytest.mark.gpu

FEAT_TOL = 2e-2
PIX_TOL = 0.25


def _rel(a, b):
    a = a.float().cpu(); b = b.float().cpu()
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.fixture(scope="module")
def sd():
    return lo.make_state_dict(0)


def _pairs(B, H, W):
    from mfr_b200 import synth
    i0, i1 = [], []
    for b in range(B):
        p = synth.make_pair(20 + b)
        g0 = synth.rgb_to_gray_u8(p["image0"]).astype(np.float32) / 255.0
        g1 = synth.rgb_to_gray_u8(p["image1"]).astype(np.float32) / 255.0
        i0.append(g0[40:40 + H, 30:30 + W])
        i1.append(g0[48:48 + H, 46:46 + W] if b % 2 == 0 else g1[40:40 + H, 30:30 + W])
    return torch.from_numpy(np.stack(i0))[:, None], torch.from_numpy(np.stack(i1))[:, None]


@pytest.mark.parametrize("B,H,W,graph", [(1, 96, 128, False), (2, 160, 120, True)])
def test_stages_match_oracle(sd, B, H, W, graph):
    from mfr_b200 import loftr
    i0, i1 = _pairs(B, H, W)
    with torch.no_grad():
        o = lo.loftr_forward(i0, i1, sd, {"thr": 0.0}, True)
        fcb, ffb = lo.backbone(torch.cat([i0, i1], 0), sd)
    eng = loftr.LoFTR(sd, batch=B, height=H, width=W, cfg={"thr": 0.0}, graph=graph)
    assert eng.num_kernels() > 100      # the launch list is our own kernels, not a library call
    out = eng.forward(i0.cuda(), i1.cuda())
    out2 = eng.forward(i0.cuda(), i1.cuda())       # second call: CUDA-graph replay must reproduce it
    h8, w8 = H // 8, W // 8
    L = h8 * w8
    assert _rel(eng.debug_tensor("feat_c_backbone", (2 * B, h8, w8, 256)), fcb.permute(0, 2, 3, 1)) < FEAT_TOL
    assert _rel(eng.debug_tensor("feat_f", (2 * B, H // 2, W // 2, 128)), ffb.permute(0, 2, 3, 1)) < FEAT_TOL
    tok = eng.debug_tensor("tok", (2 * B, L, 512))[:, :, :256]
    assert _rel(tok[:B], o["feat_c0"]) < FEAT_TOL and _rel(tok[B:], o["feat_c1"]) < FEAT_TOL
    assert _rel(eng.debug_tensor("sim", (B, L, L)), o["sim"]) < FEAT_TOL
    # matches: ordered by (pair, i) like torch.where; compare as sets (TF32 may flip near-ties)
    keys = list(zip(out["b_ids"].tolist(), out["i_ids"].tolist()))
    assert keys == sorted(keys)
    assert out["M"] == out2["M"] and torch.equal(out["i_ids"], out2["i_ids"]) and torch.equal(out["j_ids"], out2["j_ids"])
    e = {k: n for n, k in enumerate(zip(out["b_ids"].tolist(), out["i_ids"].tolist(), out["j_ids"].tolist()))}
    r = {k: n for n, k in enumerate(zip(o["b_ids"].tolist(), o["i_ids"].tolist(), o["j_ids"].tolist()))}
    common = sorted(set(e) & set(r))
    assert len(common) >= 0.8 * max(1, len(set(e) | set(r)))
    ie = torch.tensor([e[k] for k in common]); io = torch.tensor([r[k] for k in common])
    assert torch.equal(out["mkpts0_f"].cpu()[ie], o["mkpts0_f"][io])          # grid points: exact
    assert (out["mkpts1_f"].cpu()[ie] - o["mkpts1_f"][io]).abs().max().item() < PIX_TOL
    eng.close()


def test_bf16_backbone_mode(sd):
    """precision="bf16": bf16 storage + bf16 wgmma inputs in the ResNet-FPN (fp32 accumulate). Features
    stay within bf16 round-off of the fp32 oracle and the match set stays close to the TF32 engine's."""
    from mfr_b200 import loftr
    B, H, W = 2, 160, 120
    i0, i1 = _pairs(B, H, W)
    with torch.no_grad():
        fcb, ffb = lo.backbone(torch.cat([i0, i1], 0), sd)
    ref = loftr.LoFTR(sd, batch=B, height=H, width=W, cfg={"thr": 0.0}, graph=False)
    o_ref = ref.forward(i0.cuda(), i1.cuda())
    eng = loftr.LoFTR(sd, batch=B, height=H, width=W, cfg={"thr": 0.0}, graph=True, precision="bf16")
    out = eng.forward(i0.cuda(), i1.cuda())
    out = eng.forward(i0.cuda(), i1.cuda())
    h8, w8 = H // 8, W // 8
    assert _rel(eng.debug_tensor("feat_c_backbone", (2 * B, h8, w8, 256)), fcb.permute(0, 2, 3, 1)) < 4e-2
    assert _rel(eng.debug_tensor("feat_f", (2 * B, H // 2, W // 2, 128)), ffb.permute(0, 2, 3, 1)) < 4e-2
    e = set(zip(out["b_ids"].tolist(), out["i_ids"].tolist(), out["j_ids"].tolist()))
    r = set(zip(o_ref["b_ids"].tolist(), o_ref["i_ids"].tolist(), o_ref["j_ids"].tolist()))
    # synthetic weights give a nearly flat confidence surface, so near-ties flip between precisions;
    # the correlation input itself stays within bf16 round-off of the fp32 oracle
    with torch.no_grad():
        o = lo.loftr_forward(i0, i1, sd, {"thr": 0.0}, True)
    L = h8 * w8
    assert _rel(eng.debug_tensor("sim", (B, L, L)), o["sim"]) < 4e-2
    assert len(e & r) >= 0.4 * max(1, len(e | r))
    ref.close(); eng.close()


@pytest.mark.parametrize("ci", range(2))
def test_end_to_end_vs_reference_golden(sd, ci):
    """CUDA engine vs vectors produced by the UNMODIFIED reference LoFTR (tests/golden)."""
    from mfr_b200 import loftr
    G = np.load(GOLDEN + "/loftr_reference.npz")
    i0, i1, thr = loftr_case(ci)
    eng = loftr.LoFTR(sd, batch=1, height=i0.shape[2], width=i0.shape[3], cfg={"thr": thr}, graph=False)
    out = eng.forward(i0.cuda(), i1.cuda())
    ref = set(zip(G[f"c{ci}_i_ids"].tolist(), G[f"c{ci}_j_ids"].tolist()))
    got = set(zip(out["i_ids"].tolist(), out["j_ids"].tolist()))
    assert len(ref & got) >= 0.8 * len(ref | got)
    ridx = {k: n for n, k in enumerate(zip(G[f"c{ci}_i_ids"].tolist(), G[f"c{ci}_j_ids"].tolist()))}
    gidx = {k: n for n, k in enumerate(zip(out["i_ids"].tolist(), out["j_ids"].tolist()))}
    for k in ref & got:
        assert np.abs(out["mkpts1_f"][gidx[k]].cpu().numpy() - G[f"c{ci}_mkpts1_f"][ridx[k]]).max() < PIX_TOL
        assert np.array_equal(out["mkpts0_f"][gidx[k]].cpu().numpy(), G[f"c{ci}_mkpts0_f"][ridx[k]])
    eng.close()


def _coarse_match(mfr, mat, h_c, w_c, thr, border, is_conf):
    lib = mfr.load()
    B, L, _ = mat.shape
    dev = mat.device
    cnt = torch.zeros(1, dtype=torch.int32, device=dev); off = torch.zeros(B + 1, dtype=torch.int32, device=dev)
    ids = [torch.zeros(B * L, dtype=torch.int32, device=dev) for _ in range(3)]
    mconf = torch.zeros(B * L, device=dev); mk0 = torch.zeros(B * L, 2, device=dev); mk1 = torch.zeros(B * L, 2, device=dev)
    mfr.check(lib.mfr_coarse_match(mfr.ptr(mat), B, h_c, w_c, thr, border, 8.0, int(is_conf), mfr.ptr(cnt), mfr.ptr(off),
                                   mfr.ptr(ids[0]), mfr.ptr(ids[1]), mfr.ptr(ids[2]), mfr.ptr(mconf), mfr.ptr(mk0),
                                   mfr.ptr(mk1), mfr.cur_stream()))
    m = int(cnt.item())
    return [t[:m].cpu() for t in ids] + [mconf[:m].cpu(), mk0[:m].cpu(), mk1[:m].cpu(), off.cpu()]


@pytest.mark.parametrize("h_c,w_c", [(12, 9), (11, 9)])      # L = 108: fused passes; L = 99 (not a multiple of 4): the row / column kernels
def test_selection_bit_exact_given_conf(mfr, h_c, w_c):
    """Stage boundary: identical fp32 confidence matrix in -> identical int indices out, including exact
    ties (lowest column wins, coarse_matching.py:187-193) and the 2-cell border removal (:8-25)."""
    g = torch.Generator().manual_seed(3)
    B = 2
    L = h_c * w_c
    conf = torch.rand(B, L, L, generator=g) * 0.15
    perm = torch.randperm(L, generator=g)
    for b in range(B):
        for i in range(0, L, 2):
            conf[b, i, perm[i]] = 0.3 + 0.6 * torch.rand(1, generator=g).item()
    conf[0, 30, 40] = conf[0, 30, 41] = 0.99   # exact tie inside one row
    conf[1, 50, 20] = conf[1, 51, 20] = 0.98   # exact tie inside one column
    bo, io, jo, mo = lo.coarse_select(conf, h_c, w_c, h_c, w_c, 0.2, 2)
    b_, i_, j_, mc, mk0, mk1, off = _coarse_match(mfr, conf.cuda().contiguous(), h_c, w_c, 0.2, 2, True)
    assert torch.equal(b_.long(), bo) and torch.equal(i_.long(), io) and torch.equal(j_.long(), jo)
    assert torch.equal(mc, mo)
    assert torch.equal(mk0, torch.stack([io % w_c, io // w_c], 1).float() * 8)
    assert torch.equal(mk1, torch.stack([jo % w_c, jo // w_c], 1).float() * 8)
    assert off.tolist() == [0, int((bo == 0).sum()), len(bo)]


@pytest.mark.parametrize("h_c,w_c,thr", [(16, 11, 0.2), (15, 11, 0.2), (16, 11, 0.0), (16, 11, 0.05)])
def test_dual_softmax_selection_matches_oracle(mfr, h_c, w_c, thr):
    """Dual softmax + mutual NN from the similarity matrix. thr > 0: the confidence pass screens entries (only candidates of
    conf > thr are evaluated); thr = 0: exhaustive pass; L = 165 (not a multiple of 4): the unfused row / column kernels."""
    g = torch.Generator().manual_seed(4)
    B = 1
    L = h_c * w_c
    f0 = torch.randn(B, L, 64, generator=g)
    f1 = f0[:, torch.randperm(L, generator=g)] + 0.05 * torch.randn(B, L, 64, generator=g)
    sim = torch.einsum("nlc,nsc->nls", f0, f1) / 0.8
    conf = torch.softmax(sim, 1) * torch.softmax(sim, 2)
    bo, io, jo, mo = lo.coarse_select(conf, h_c, w_c, h_c, w_c, thr, 2)
    b_, i_, j_, mc, _, _, _ = _coarse_match(mfr, sim.cuda().contiguous(), h_c, w_c, thr, 2, False)
    assert len(io) > 20
    assert torch.equal(i_.long(), io) and torch.equal(j_.long(), jo)
    torch.testing.assert_close(mc, mo, rtol=1e-4, atol=1e-6)


def test_empty_match_set(sd):
    from mfr_b200 import loftr
    i0, i1 = _pairs(1, 96, 96)
    eng = loftr.LoFTR(sd, batch=1, height=96, width=96, cfg={"thr": 0.999}, graph=False)
    out = eng.forward(i0.cuda(), i1.cuda())
    assert out["M"] == 0 and out["mkpts0_f"].shape == (0, 2)
    m = loftr.LoFTR_matcher.__new__(loftr.LoFTR_matcher)
    m.engine, m.resize = eng, (96, 96)
    pts = m.match_arrays(i0[0, 0].numpy(), i1[0, 0].numpy())
    assert pts.shape == (1, 4) and np.isnan(pts).all()      # matchers.py:58-59 NaN row
    eng.close()


def _lin_att_ref(q, k, v, heads, eps=1e-6):
    """linear_attention.py:31-45 on already feature-mapped q', k' (fp64 restatement; the v / S ... * S pair cancels)."""
    n, L, C = q.shape
    d = C // heads
    Q = q.double().view(n, L, heads, d); K = k.double().view(n, -1, heads, d); V = v.double().view(n, -1, heads, d)
    KV = torch.einsum("nshd,nshv->nhdv", K, V)
    Z = 1 / (torch.einsum("nlhd,nhd->nlh", Q, K.sum(dim=1)) + eps)
    return torch.einsum("nlhd,nhdv,nlh->nlhv", Q, KV, Z).reshape(n, L, C)


@pytest.mark.parametrize("windows,n,L,S", [(0, 3, 301, 417), (0, 2, 64, 4800), (1, 37, 25, 25)])
@pytest.mark.parametrize("bf16", [0, 1])
def test_linear_attention_stage(mfr, windows, n, L, S, bf16):
    """Coarse (8 x 32) and fine-window (8 x 16) linear attention on feature-mapped q, k: the fp32 SIMT kernels against an
    fp64 restatement, tolerance 1e-4 of the output range. Ragged L / S exercise the zero-filled slab tails. bf16 = 1
    (bf16 tensors with pre-mapped q, k) is rejected, so that such a caller gets an error instead of q and k mapped twice
    (bf16 takes raw q, k: test_linear_attention_raw_qk)."""
    lib = mfr.load()
    g = torch.Generator().manual_seed(11 + windows)
    C = 128 if windows else 256
    q = torch.nn.functional.elu(torch.randn(n, L, C, generator=g)) + 1
    k = torch.nn.functional.elu(torch.randn(n, S, C, generator=g)) + 1
    v = torch.randn(n, S, C, generator=g)
    dt = torch.bfloat16 if bf16 else torch.float32
    qd, kd, vd = (x.to(dt).cuda().contiguous() for x in (q, k, v))
    out = torch.full((n, L, C), float("nan"), dtype=dt, device="cuda")
    rc = lib.mfr_linear_attention(mfr.ptr(qd), mfr.ptr(kd), mfr.ptr(vd), mfr.ptr(out), n, L, S, windows, bf16,
                                  mfr.cur_stream())
    torch.cuda.synchronize()
    if bf16:
        assert rc == 3                                  # MFR_ERR_UNSUPPORTED
        assert torch.isnan(out).all()                   # nothing was written
        return
    mfr.check(rc)
    ref = _lin_att_ref(qd.cpu().float(), kd.cpu().float(), vd.cpu().float(), 8)
    got = out.cpu().double()
    assert torch.isfinite(got).all()
    assert ((got - ref).abs().max() / ref.abs().max()).item() < 1e-4


@pytest.mark.parametrize("NI,H,W", [(2, 720, 544), (3, 96, 128), (1, 75, 61)])
def test_stem_tcgen05_matches_reference(mfr, NI, H, W):
    """(The name predates the port: the stem under test is the mma.sync one.) The tensor-core stem with bf16 output (hi/lo-split operands) against an fp64 convolution of the same image
    and weights. Ragged sizes exercise the clipped edge rows."""
    lib = mfr.load()
    g = torch.Generator().manual_seed(17 + H)
    img = torch.rand(NI, H, W, generator=g).cuda()
    w = (torch.randn(128, 49, generator=g) / 7.0).cuda()
    bias = torch.randn(128, generator=g).cuda()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = torch.full((NI, Ho, Wo, 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    mfr.check(lib.mfr_stem_conv7x7(mfr.ptr(img), mfr.ptr(w), mfr.ptr(bias), mfr.ptr(out), NI, H, W, 1, 0, mfr.cur_stream()))
    torch.cuda.synchronize()
    o = out.float().cpu()
    ref = torch.relu(F.conv2d(img.cpu().double()[:, None], w.cpu().double().view(128, 1, 7, 7), bias.cpu().double(), stride=2, padding=3))
    ref = ref.permute(0, 2, 3, 1)
    scale = ref.abs().max().item()
    assert torch.isfinite(o).all()
    assert ((o.double() - ref).abs().max().item()) <= 2.0 ** -8 * scale     # bf16 rounding of the output


@pytest.mark.parametrize("windows,n,L,S", [(0, 3, 301, 417), (0, 2, 64, 4800), (1, 37, 25, 25)])
def test_linear_attention_raw_qk(mfr, windows, n, L, S):
    """bf16 = 2: the tensor-core attention kernels take raw q, k (the projection GEMM's output) and apply elu + 1 to their
    fragments; the result must equal the fp64 restatement on the bf16-rounded feature-mapped inputs within the bf16
    tolerance 2e-2 of the output range (bf16 operands and bf16-rounded KV: 8-bit mantissas, sums of <= 4800 positive
    terms in fp32). Ragged L / S: the zero-filled token padding must stay zero (elu(0) + 1 = 1 would count as tokens)."""
    lib = mfr.load()
    g = torch.Generator().manual_seed(23 + windows)
    C = 128 if windows else 256
    q = torch.randn(n, L, C, generator=g).to(torch.bfloat16)
    k = torch.randn(n, S, C, generator=g).to(torch.bfloat16)
    v = torch.randn(n, S, C, generator=g).to(torch.bfloat16)
    qd, kd, vd = (x.cuda().contiguous() for x in (q, k, v))
    out = torch.full((n, L, C), float("nan"), dtype=torch.bfloat16, device="cuda")
    mfr.check(lib.mfr_linear_attention(mfr.ptr(qd), mfr.ptr(kd), mfr.ptr(vd), mfr.ptr(out), n, L, S, windows, 2, mfr.cur_stream()))
    torch.cuda.synchronize()
    qf = (torch.nn.functional.elu(q.float()) + 1).to(torch.bfloat16).float()
    kf = (torch.nn.functional.elu(k.float()) + 1).to(torch.bfloat16).float()
    ref = _lin_att_ref(qf, kf, v.float(), 8)
    got = out.cpu().double()
    assert torch.isfinite(got).all()
    assert ((got - ref).abs().max() / ref.abs().max()).item() < 2e-2
