"""Each LoFTR engine stage after the backbone against a float64 restatement, fed with the engine's own input.

Every check reads the stage input from the engine (``LoFTR.debug_tensor``) and recomputes the stage in torch float64 on
the GPU with ``oracle/loftr_oracle.py``'s functions, so the error of one stage does not add up with the error of the
stages before it and the bars can follow each precision's rounding model. All checks run for the three engine
precisions, with two pairs per batch (B = 2) whose match sets differ, so that a mix-up of ``b_ids`` shows.

One encoder layer at a time: a layer whose norm2 gain and bias are zero returns ``x + 0 = x`` exactly (the LayerNorm
kernel of tf32 / fp32x3 and bf16's fused encoder tail, which also rewrites the bf16 shadow, both compute
``(x - mean) * rstd * 0 + 0``), so with norm2 zeroed in every layer but k the transformer's output is layer k applied
to its input (``tests/test_loftr_stages_host.py`` checks that on the oracle). Every bf16 check runs the one bf16 path
the engine has: raw q, k into the tensor-core attention kernels, then the fused tail.

Bars. Single-kernel stages have bounds derived from the kernel's arithmetic (a K-term fp32 dot product is within
``(c_op + K * 2^-24) * sum |a| |b|`` of the exact one, with c_op the operand rounding of the precision). The encoder
layers are multi-kernel stages: their bar is a multiple of the precision's unit roundoff u (bf16 2^-8, tf32 2^-11,
fp32x3 2^-22 for the split operands) on the layer's residual branch, ``|(out - in) - branch_ref| / max |branch_ref|``.
The maxima measured on one H100 80GB HBM3 (700 W power limit) are quoted next to each bar."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import U32, branch_err, dot_bound, fullres_inputs
from oracle import loftr_oracle as lo

pytestmark = pytest.mark.gpu

PRECISIONS = ["tf32", "bf16", "fp32x3"]
C_OP = {"tf32": 2 * 2.0 ** -10, "bf16": 2 * 2.0 ** -10, "fp32x3": 2.0 ** -20}   # operand term of the fp32-input GEMMs
# residual-branch bars of one encoder layer, as multiples of the unit roundoff (measured maxima in the test docstrings)
COARSE_BAR = {"tf32": 4 * 2.0 ** -11, "bf16": 4 * 2.0 ** -8, "fp32x3": 32 * 2.0 ** -22}
FINE_BAR = {"tf32": 4 * 2.0 ** -11, "bf16": 4 * 2.0 ** -8, "fp32x3": 32 * 2.0 ** -22}


# ------------------------------------------------------------------------------------------------ harness
def isolate_layer(sd, prefix, n_layers, keep):
    """Copy of a reference-format state dict in which every ``{prefix}.layers.{i}`` but ``keep`` has norm2 = 0 (weight and
    bias), so that it returns its input unchanged. ``keep=None`` zeroes all of them."""
    out = dict(sd)
    for i in range(n_layers):
        if i != keep:
            for t in ("weight", "bias"):
                k = f"{prefix}.layers.{i}.norm2.{t}"
                out[k] = torch.zeros_like(sd[k])
    return out


def hybrid_state_dict():
    """The functional matcher's backbone and coarse transformer (many, well separated matches) with the seeded random
    fine level (down_proj, merge_feat and both fine encoder layers do real arithmetic)."""
    from mfr_b200 import loftr
    sd = loftr.functional_state_dict()
    rnd = loftr.synthetic_state_dict(0)
    sd.update({k: v for k, v in rnd.items() if k.startswith(("fine_preprocess.", "loftr_fine."))})
    return sd


_GRAY = {}


def _gray(seed):
    if seed not in _GRAY:
        from mfr_b200 import synth
        p = synth.make_pair(seed)
        _GRAY[seed] = tuple(synth.rgb_to_gray_u8(p[k]).astype(np.float32) / 255.0 for k in ("image0", "image1"))
    return _GRAY[seed]


def images(kind, H, W):
    """B = 2 batches of two scenes. "shifted": a crop and the same view shifted by (8, 16) px in pair 0, (16, 8) px in
    pair 1 (about 160 matches each at 160x120, border_rm 0, functional weights). "identical": each crop with itself (M
    close to the capacity B * L). "views": the two views of each scene cropped at the same place (6 and 10 matches at
    96x128 in the CPU oracle)."""
    i0, i1 = [], []
    for b, (dy, dx) in enumerate(((8, 16), (16, 8))):
        g0, g1 = _gray(20 + b)
        a = g0[40:40 + H, 30:30 + W]
        if kind == "shifted":
            c = g0[40 + dy:40 + dy + H, 30 + dx:30 + dx + W]
        elif kind == "identical":
            c = a
        else:
            c = g1[40:40 + H, 30:30 + W]
        i0.append(a); i1.append(c)
    return torch.from_numpy(np.stack(i0))[:, None].cuda(), torch.from_numpy(np.stack(i1))[:, None].cuda()


def engine(sd, precision, H, W, cfg=None, graph=False):
    from mfr_b200 import loftr
    return loftr.LoFTR(sd, batch=2, height=H, width=W, cfg=cfg, graph=graph, precision=precision)


def d64(sd):
    return {k: v.double().cuda() for k, v in sd.items()}


def bf16_view(eng, name, shape):
    """A bf16 debug buffer: ``shape`` in bf16 elements (the last axis even), read through the float32 view."""
    return eng.debug_tensor(name, (*shape[:-1], shape[-1] // 2)).view(torch.bfloat16)


def posenc(sd, h8, w8):
    from mfr_b200 import loftr
    return torch.from_numpy(loftr.prepare_weights(sd, h8, w8)["pos_enc"]).cuda().view(h8 * w8, 256)


def live(eng, M):
    """Fine-level tensors of the last forward, cloned, on their live rows."""
    Mc = eng.capacity
    R = Mc * 25
    return {"cin": eng.debug_tensor("fine_cin", (2, Mc, 256))[:, :M].clone(),
            "cproj": eng.debug_tensor("fine_cproj", (2, Mc, 128))[:, :M].clone(),
            "win": eng.debug_tensor("fine_win", (2, R, 256))[:, :25 * M].clone(),
            "ftok": eng.debug_tensor("fine_tok", (2, R, 256))[:, :25 * M, :128].clone()}


# ------------------------------------------------------------------------------------------------ coarse transformer
def _coarse_layer(eng, sd, k, H, W, ims=None):
    """Runs the engine with only coarse layer k active; returns (engine input, engine output, fp64 reference)."""
    h8, w8 = H // 8, W // 8
    L = h8 * w8
    sdk = isolate_layer(sd, "loftr_coarse", 8, k)
    eng.load_state_dict(sdk)
    eng.forward(*(ims or images("shifted", H, W)))
    fcb = eng.debug_tensor("feat_c_backbone", (4, L, 256)).clone()
    x_in = fcb + posenc(sdk, h8, w8)[None]                 # one fp32 add, as posenc_kernel
    x_out = eng.debug_tensor("tok", (4, L, 512))[:, :, :256].clone()
    s64 = d64(sdk)
    p = f"loftr_coarse.layers.{k}"
    x = x_in.double()
    if k % 2 == 0:
        r = torch.cat([lo.encoder_layer(x[:2], x[:2], s64, p, 8), lo.encoder_layer(x[2:], x[2:], s64, p, 8)])
    else:      # cross: feat1 attends to the engine's updated feat0
        r = torch.cat([lo.encoder_layer(x[:2], x[2:], s64, p, 8), lo.encoder_layer(x[2:], x_out[:2].double(), s64, p, 8)])
    return x_in, x_out, r


@pytest.mark.parametrize("precision", PRECISIONS)
def test_posenc_and_identity_layers(precision):
    """All eight coarse layers zeroed: the tokens after the transformer are exactly feat_c_backbone + pos_enc (one fp32
    add per element, row l of every image gets row l of the table) and, in bf16 mode, the shadow is their bf16
    rounding."""
    from mfr_b200 import loftr
    H, W = 160, 120
    sd = isolate_layer(loftr.synthetic_state_dict(0), "loftr_coarse", 8, None)
    eng = engine(sd, precision, H, W, {"thr": 0.0, "border_rm": 0})
    eng.forward(*images("shifted", H, W))
    L = 300
    fcb = eng.debug_tensor("feat_c_backbone", (4, L, 256))
    tok = eng.debug_tensor("tok", (4, L, 512))[:, :, :256]
    assert torch.equal(tok, fcb + posenc(sd, H // 8, W // 8)[None])
    if precision == "bf16":
        assert torch.equal(bf16_view(eng, "tok_bf16", (4, L, 512))[:, :, :256].view(torch.int16),
                           tok.to(torch.bfloat16).view(torch.int16))
    eng.close()


@pytest.mark.parametrize("layer", range(8))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_coarse_layer(precision, layer):
    """One coarse encoder layer (even = self, odd = cross) at 160x120 (L = 300) on the engine's own input, residual branch
    against fp64. Bars 4 u (tf32, 1.95e-3), 4 u (bf16, 1.56e-2), 32 u (fp32x3, 7.6e-6); measured maxima over the
    eight layers: tf32 7.3e-4, bf16 5.6e-3, fp32x3 2.8e-6."""
    from mfr_b200 import loftr
    H, W = 160, 120
    sd = loftr.synthetic_state_dict(0)
    eng = engine(sd, precision, H, W, {"thr": 0.0})
    x_in, x_out, ref = _coarse_layer(eng, sd, layer, H, W)
    err = branch_err(x_in, x_out, ref)
    print(f"coarse {precision} layer {layer}: branch err {err:.3e} (bar {COARSE_BAR[precision]:.3e})")
    assert err < COARSE_BAR[precision], err
    eng.close()


@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_coarse_layer_bench_frame(precision, layer):
    """Layers 0 (self) and 1 (cross) at the benchmark frame 720x544 (L = 6120): long attention sums, many GEMM tiles.
    Same bars as at L = 300;
    measured maxima: tf32 7.9e-4, bf16 5.5e-3."""
    from mfr_b200 import loftr
    H, W = 720, 544
    sd = loftr.synthetic_state_dict(0)
    eng = engine(sd, precision, H, W, {"thr": 0.0})
    i0, i1 = fullres_inputs()                   # two 720x540 pairs, zero-padded to the frame by the engine
    x_in, x_out, ref = _coarse_layer(eng, sd, layer, H, W, (i0.cuda(), i1.cuda()))
    err = branch_err(x_in, x_out, ref)
    print(f"coarse@bench {precision} layer {layer}: branch err {err:.3e}")
    assert err < COARSE_BAR[precision], err
    eng.close()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_coarse_layer_small_message(precision, layer):
    """Layer 0 (self) or 1 (cross) with merge.weight scaled by 2^-10: the LayerNorm1 input of layer 1 then has a variance
    of about 8e-6 per row (8.3 at scale 1 in the oracle), the size of LayerNorm's eps = 1e-5, so a LayerNorm path with
    another eps or a mis-rounded variance fails here (layernorm_kernel in tf32 / fp32x3, the fused tail in bf16). Bars as
    for the other coarse layers; measured maxima for layer 1: tf32 5.8e-4, bf16 4.8e-3, fp32x3 2.8e-6."""
    from mfr_b200 import loftr
    H, W = 160, 120
    sd = loftr.synthetic_state_dict(0)
    k = f"loftr_coarse.layers.{layer}.merge.weight"
    sd[k] = sd[k] * 2.0 ** -10
    eng = engine(sd, precision, H, W, {"thr": 0.0})
    x_in, x_out, ref = _coarse_layer(eng, sd, layer, H, W)
    err = branch_err(x_in, x_out, ref)
    print(f"coarse small message {precision} layer {layer}: branch err {err:.3e}")
    assert err < COARSE_BAR[precision], err
    eng.close()


# ------------------------------------------------------------------------------------------------ bf16 shadows
FINE_CASES = [("shifted", 160, 120), ("identical", 96, 128)]


@pytest.mark.parametrize("kind,H,W", FINE_CASES)
def test_bf16_shadows_coherent(kind, H, W):
    """After a bf16 forward, the bf16 copies the token GEMMs read are the round-to-nearest-even bf16 of the fp32 tokens,
    bit for bit: the coarse tokens on all 2B * L rows, the fine tokens on the 25 * M live rows of both sides (last
    written by the fused tail). "identical" fills M close to the capacity B * L."""
    from mfr_b200 import loftr
    L = (H // 8) * (W // 8)
    eng = engine(loftr.synthetic_state_dict(0), "bf16", H, W, {"thr": 0.0, "border_rm": 0})
    out = eng.forward(*images(kind, H, W))
    M = out["M"]
    assert M > 0
    tok = eng.debug_tensor("tok", (4, L, 512))[:, :, :256]
    sh = bf16_view(eng, "tok_bf16", (4, L, 512))[:, :, :256]
    assert torch.equal(sh.view(torch.int16), tok.to(torch.bfloat16).view(torch.int16))
    R = eng.capacity * 25
    ft = eng.debug_tensor("fine_tok", (2, R, 256))[:, :25 * M, :128]
    fsh = bf16_view(eng, "fine_tok_bf16", (2, R, 256))[:, :25 * M, :128]
    assert torch.equal(fsh.view(torch.int16), ft.to(torch.bfloat16).view(torch.int16))
    eng.close()


# ------------------------------------------------------------------------------------------------ correlation
@pytest.mark.parametrize("precision", PRECISIONS)
def test_correlation(precision):
    """sim = <t0_i, t1_j> / (256 T) element by element within the dot-product bound
    |d_ij| <= (c_op + (256 + 2) 2^-24) alpha sum_k |a_ik| |b_jk|, alpha = 1 / (256 T); bf16 mode reads the tokens' bf16
    shadow (products exact: c_op = 0), tf32 truncates both operands to 10 bits (c_op = 2^-9), fp32x3 drops lo * lo and
    rounds lo (c_op = 2^-20). The + 2 covers the fp32 alpha and the epilogue multiply."""
    from mfr_b200 import loftr
    H, W = 160, 120
    L = 300
    eng = engine(loftr.synthetic_state_dict(0), precision, H, W, {"thr": 0.0})
    eng.forward(*images("shifted", H, W))
    if precision == "bf16":
        t = bf16_view(eng, "tok_bf16", (4, L, 512))[:, :, :256].double()
        c_op = 0.0
    else:
        t = eng.debug_tensor("tok", (4, L, 512))[:, :, :256].double()
        c_op = C_OP[precision]
    sim = eng.debug_tensor("sim", (2, L, L)).double()
    alpha = 1.0 / (256 * 0.1)
    ref = torch.einsum("blc,bsc->bls", t[:2], t[2:]) * alpha
    bound = (c_op + 258 * U32) * alpha * torch.einsum("blc,bsc->bls", t[:2].abs(), t[2:].abs())
    ratio = ((sim - ref).abs() / bound).max().item()
    print(f"correlation {precision}: max |d| / bound {ratio:.3e}")
    assert ratio <= 1.0, ratio
    eng.close()


# ------------------------------------------------------------------------------------------------ match selection
@pytest.mark.parametrize("thr,border", [(0.2, 2), (0.0, 0)])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_selection_on_engine_sim(precision, thr, border):
    """The oracle's coarse_select on the dual-softmax of the engine's own sim (computed in fp64, stored in fp32 like the
    reference's confidence matrix) gives exactly the engine's b_ids / i_ids / j_ids and m_offsets, and mconf within
    rtol 1e-4 of the fp64 confidence (functional weights). A flipped near-tie is reported with the relative gap between
    the two largest confidences of its row and column, to be compared with the fp32 ulp."""
    from mfr_b200 import loftr
    H, W = 160, 120
    h8, w8 = H // 8, W // 8
    L = h8 * w8
    eng = engine(loftr.functional_state_dict(), precision, H, W, {"thr": thr, "border_rm": border})
    out = eng.forward(*images("shifted", H, W))
    sim = eng.debug_tensor("sim", (2, L, L)).double()
    conf64 = torch.softmax(sim, 1) * torch.softmax(sim, 2)
    conf = conf64.float()        # the fp32 confidence of the reference: values below 1.4e-45 are 0, so not above thr 0
    b, i, j, mconf = lo.coarse_select(conf, h8, w8, h8, w8, thr, border)
    mconf = conf64[b, i, j]
    got = (out["b_ids"].long(), out["i_ids"].long(), out["j_ids"].long())
    assert (b == 0).any() and (b == 1).any()
    if not all(torch.equal(g, r) for g, r in zip(got, (b, i, j))):
        e = set(zip(*(t.tolist() for t in got)))
        r = set(zip(b.tolist(), i.tolist(), j.tolist()))
        lines = []
        for (bb, ii, jj) in sorted(e ^ r)[:8]:
            gaps = []
            for name, v in (("row", conf[bb, ii]), ("column", conf[bb, :, jj])):
                top = torch.topk(v.double(), 2).values
                gaps.append(f"{name} top-2 {top.tolist()} rel gap {((top[0] - top[1]) / top[0]).item():.3e}")
            lines.append(f"{'engine' if (bb, ii, jj) in e else 'oracle'} only: ({bb},{ii},{jj}) conf "
                         f"{conf[bb, ii, jj].item():.9g}; " + "; ".join(gaps) + " (fp32 ulp 6e-8)")
        pytest.fail("selection differs from the oracle on the engine's sim:\n" + "\n".join(lines))
    assert out["m_offsets"].tolist() == [0, int((b == 0).sum()), len(b)]
    # atol only matters below 1e-37: there the fp32 conf is subnormal and keeps its leading bits only
    torch.testing.assert_close(out["mconf"].double(), mconf, rtol=1e-4, atol=1e-41)
    eng.close()


# ------------------------------------------------------------------------------------------------ fine level
def _edge_matches(out, w8):
    """Matches whose window reaches outside the 1/2-resolution map (cell row or column 0 on either side)."""
    i, j = out["i_ids"].long(), out["j_ids"].long()
    return int(((i % w8 == 0) | (i // w8 == 0) | (j % w8 == 0) | (j // w8 == 0)).sum())


@pytest.mark.parametrize("kind,H,W", FINE_CASES)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_fine_gather_and_projections(precision, kind, H, W):
    """border_rm = 0: fine_cin is the exact copy of the matched coarse tokens, fine_win the exact 5x5 windows of feat_f
    at stride 4 with zero padding outside the map (the case has edge matches) next to the projected coarse token,
    fine_cproj (down_proj, fp32 operands even in bf16 mode) and the merge_feat output (both fine layers zeroed) within
    the per-element dot-product bound. "identical" fills M close to the capacity B * L."""
    from mfr_b200 import loftr
    h8, w8 = H // 8, W // 8
    L = h8 * w8
    sd = isolate_layer(hybrid_state_dict(), "loftr_fine", 2, None)
    eng = engine(sd, precision, H, W, {"thr": 0.2, "border_rm": 0})
    out = eng.forward(*images(kind, H, W))
    M = out["M"]
    assert _edge_matches(out, w8) > 0
    if kind == "identical":
        assert M >= 0.8 * eng.capacity, (M, eng.capacity)
    f = live(eng, M)
    b, i, j = out["b_ids"].long(), out["i_ids"].long(), out["j_ids"].long()
    tok = eng.debug_tensor("tok", (4, L, 512))[:, :, :256]
    assert torch.equal(f["cin"][0], tok[b, i]) and torch.equal(f["cin"][1], tok[2 + b, j])
    featf = eng.debug_tensor("feat_f", (4, H // 2, W // 2, 128)).permute(0, 3, 1, 2)
    u = F.unfold(featf, kernel_size=5, stride=4, padding=2).view(4, 128, 25, L).permute(0, 3, 2, 1)   # img, cell, tap, c
    for s, (img, cell) in enumerate(((b, i), (2 + b, j))):
        w = f["win"][s].view(M, 25, 256)
        assert torch.equal(w[:, :, :128], u[img, cell])
        assert torch.equal(w[:, :, 128:], f["cproj"][s][:, None, :].expand(M, 25, 128))
    c_op = C_OP[precision]
    Wd, bd = sd["fine_preprocess.down_proj.weight"].cuda(), sd["fine_preprocess.down_proj.bias"].cuda()
    ref = f["cin"].double() @ Wd.double().t() + bd.double()
    assert ((f["cproj"].double() - ref).abs() <= dot_bound(f["cin"], Wd, c_op, bd)).all()
    Wm, bm = sd["fine_preprocess.merge_feat.weight"].cuda(), sd["fine_preprocess.merge_feat.bias"].cuda()
    ref = f["win"].double() @ Wm.double().t() + bm.double()
    d = (f["ftok"].double() - ref).abs() / dot_bound(f["win"], Wm, c_op, bm)
    print(f"fine merge {precision} {kind}: M {M} max |d| / bound {d.max().item():.3e}")
    assert d.max().item() <= 1.0
    eng.close()


@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("kind,H,W", FINE_CASES)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_fine_layer(precision, kind, H, W, layer):
    """One fine encoder layer (0 = self, 1 = cross over the 5x5 windows) on the merge_feat output of the same engine
    (both fine layers zeroed), residual branch against fp64. "identical" fills M close to the capacity B * L. Bars as
    for the coarse layers; measured maxima on "shifted": tf32 6.4e-4, bf16 4.5e-3, fp32x3 2.8e-6."""
    base = hybrid_state_dict()
    eng = engine(base, precision, H, W, {"thr": 0.2, "border_rm": 0})
    ims = images(kind, H, W)
    eng.load_state_dict(isolate_layer(base, "loftr_fine", 2, None))
    M = eng.forward(*ims)["M"]
    a = live(eng, M)
    sdk = isolate_layer(base, "loftr_fine", 2, layer)
    eng.load_state_dict(sdk)
    assert eng.forward(*ims)["M"] == M
    o = live(eng, M)
    assert torch.equal(o["win"], a["win"])            # same upstream bits
    x = a["ftok"].view(2, M, 25, 128).double()
    y = o["ftok"].view(2, M, 25, 128)
    s64 = d64(sdk)
    p = f"loftr_fine.layers.{layer}"
    if layer == 0:
        r = torch.stack([lo.encoder_layer(x[0], x[0], s64, p, 8), lo.encoder_layer(x[1], x[1], s64, p, 8)])
    else:
        r = torch.stack([lo.encoder_layer(x[0], x[1], s64, p, 8), lo.encoder_layer(x[1], y[0].double(), s64, p, 8)])
    err = branch_err(x, y, r)
    print(f"fine {precision} {kind} layer {layer}: M {M} branch err {err:.3e}")
    assert err < FINE_BAR[precision], err
    eng.close()


@pytest.mark.parametrize("weights", ["functional", "hybrid"])
@pytest.mark.parametrize("kind,H,W", FINE_CASES)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_fine_match(precision, kind, H, W, weights):
    """fine_match_kernel from the engine's final fine tokens against the fp64 expectation (fine_matching of the oracle).
    sim_r = <f0_12, f1_r> / sqrt(128) is within d = 130 * 2^-24 * sum |f0| |f1| / sqrt(128) (fp32 fmaf chain, scale);
    the softmax turns that into a relative heatmap error e = expm1(2 d + exp error + 8 u), with the __expf error
    (2 + 1.2 |x|) 2^-23 + u |x| at x = sim - max; |d ex|, |d ey| <= e + 8 u; mkpts1_f = mkpts1_c + 4 ex adds one rounding.
    std = sqrt(max(var_x, 1e-10)) + sqrt(max(var_y, 1e-10)) with var = sum h g^2 - ex^2 loses its digits to cancellation
    when the heatmap is peaked (the functional weights take the clamp branch), so |d std| <= 2 sqrt(d_var) with
    d_var = sum h g^2 (e + 16 u) + 2 |ex| (e + 8 u) + (e + 8 u)^2."""
    from mfr_b200 import loftr
    sd = loftr.functional_state_dict() if weights == "functional" else hybrid_state_dict()
    eng = engine(sd, precision, H, W, {"thr": 0.2, "border_rm": 0})
    out = eng.forward(*images(kind, H, W))
    M = out["M"]
    assert M > 0
    f = live(eng, M)["ftok"].view(2, M, 25, 128)
    mk1c = eng.device_outputs()["mkpts1_c"][:M].double()
    u = U32
    f0, f1 = f[0].double(), f[1].double()
    c = f0[:, 12]
    sim = torch.einsum("mc,mrc->mr", c, f1) / math.sqrt(128)
    dsim = 130 * u * torch.einsum("mc,mrc->mr", c.abs(), f1.abs()) / math.sqrt(128)
    x = (sim - sim.max(1, keepdim=True).values).abs().max(1).values
    e = torch.expm1(2 * dsim.max(1).values + (2 + 1.2 * x) * 2.0 ** -23 + u * x + 8 * u)
    ex_err = e + 8 * u
    _, mk1_ref, expec_ref = lo.fine_matching(f0, f1, mk1c * 0, mk1c * 0, 2.0)
    heat = torch.softmax(sim, 1)
    lin = torch.linspace(-1, 1, 5, device=sim.device, dtype=torch.float64)
    g2 = torch.stack([(heat * lin.repeat(5) ** 2).sum(1), (heat * lin.repeat_interleave(5) ** 2).sum(1)], 1)
    d_var = g2 * (e + 16 * u)[:, None] + 2 * expec_ref[:, :2].abs() * ex_err[:, None] + ex_err[:, None] ** 2
    ex = out["expec_f"].double()
    assert torch.isfinite(ex).all()
    assert ((ex[:, :2] - expec_ref[:, :2]).abs() <= ex_err[:, None]).all(), (ex[:, :2] - expec_ref[:, :2]).abs().max()
    mk_ref = mk1c + mk1_ref
    mk_bar = 4 * ex_err[:, None] + 2 * u * mk_ref.abs()
    assert ((out["mkpts1_f"].double() - mk_ref).abs() <= mk_bar).all()
    std_bar = 2 * d_var.max(1).values.sqrt() + 4 * u * expec_ref[:, 2]
    dstd = (ex[:, 2] - expec_ref[:, 2]).abs()
    clamped = int((expec_ref[:, 2] < 1e-4).sum())
    print(f"fine_match {precision} {kind} {weights}: M {M} clamped {clamped} max d std / bar {(dstd / std_bar).max().item():.3e}")
    assert (dstd <= std_bar).all(), (dstd / std_bar).max()
    if weights == "functional" and kind == "identical":
        assert clamped > 0            # the peaked heatmaps reach the variance clamp
    eng.close()


# ------------------------------------------------------------------------------------------------ graph replays
def _snapshot(eng, out):
    M = out["M"]
    s = {k: out[k].clone() for k in ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_f", "mkpts1_f", "expec_f")}
    s["m_offsets"] = out["m_offsets"].clone()
    s["M"] = M
    s["ftok"] = live(eng, M)["ftok"]
    return s


@pytest.mark.parametrize("precision", PRECISIONS)
def test_graph_replays_follow_dynamic_m(precision):
    """One CUDA-graph engine runs large M (image pairs with themselves), small M (the two views of each scene), large M again; every
    call's live outputs equal, bit for bit, those of a fresh eager engine on that batch alone (the LoFTR path has no float
    atomics, so the engine is deterministic)."""
    from mfr_b200 import loftr
    H, W = 96, 128
    sd = loftr.functional_state_dict()
    cfg = {"thr": 0.2, "border_rm": 0}
    batches = [images("identical", H, W), images("views", H, W)]
    ref = []
    for ims in batches:
        e = engine(sd, precision, H, W, cfg, graph=False)
        ref.append(_snapshot(e, e.forward(*ims)))
        e.close()
    assert ref[0]["M"] >= 0.8 * 2 * 192 and ref[1]["M"] < 0.25 * ref[0]["M"], (ref[0]["M"], ref[1]["M"])
    g = engine(sd, precision, H, W, cfg, graph=True)
    for call, bi in enumerate([0, 1, 0]):
        got = _snapshot(g, g.forward(*batches[bi]))
        for k, v in ref[bi].items():
            same = v == got[k] if k == "M" else torch.equal(v, got[k])
            assert same, f"call {call} (batch {bi}): {k} differs from the eager engine"
    g.close()
