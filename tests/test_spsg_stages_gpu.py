"""Each SuperPoint + SuperGlue engine stage against a float64 restatement, fed with the engine's own input.

Every check reads the stage input from the engine (``SuperPointSuperGlue.debug_tensor`` and its outputs) and recomputes
the stage in torch float64 on the GPU with ``oracle/spsg_oracle.py``'s functions, so the error of one stage does not add
up with the error of the stages before it. All checks run for the three engine precisions, on B = 2 pairs of different
content (a mix-up between pairs shows), at 240x320 with K = 256 and at the product frame 720x540 (w8 = 67: the score map
is 536 wide and the 2x2 pools drop a column) with K = 1024.

One GNN layer at a time: a layer whose ``mlp.3`` weight and bias are zero returns ``x + 0 = x`` exactly (tf32 and fp32x3
add an exact 0 in the residual epilogue; bf16 adds mlp.3's fp32 output to the fp32 tokens and rebuilds the x half of the
bf16 shadow from them), so with mlp.3 zeroed in every layer but k the GNN output is layer k applied to the keypoint
encoder's output, both images updated from the old tokens (``tests/test_spsg_stages_host.py`` checks that on the oracle).

Bars. The exact stages (NMS, keypoint selection, compaction) are compared with ``==``. Single-kernel float stages have
bounds derived from the kernel's arithmetic; a K-term fp32 GEMM is within ``(c_op + (K + 2) 2^-24) sum |a| |b|`` of the
exact one (``helpers.dot_bound``), c_op being the operand rounding: tf32 2^-9, fp32x3 2^-20, 2^-9 for the rounded weights
of a bf16 conv. The keypoint encoder and the GNN layers are multi-kernel stages: their bar is a multiple of the
precision's unit roundoff u (bf16 2^-8, tf32 2^-11, fp32x3 2^-22; the keypoint encoder is a tf32 GEMM chain in bf16 mode)
on the stage's residual branch, ``|(out - in) - branch_ref| / max |branch_ref|``, less the rounding of the fp32 sum
``in + branch`` itself. In fp32x3 the operand split is not what limits them: the fp32 accumulation of sums that cancel
and, in the GNN, the softmax's __expf (2 + 1.2 |x| ulp at logits x of up to ~20) do, hence the larger multiples. Sinkhorn
has an absolute bar on the log couplings Z. Maxima measured on one H100 80GB HBM3 (700 W power limit), over both frames
and, where it runs them, the ragged and K = 2048 cases:

  stage                        bar                           tf32      bf16      fp32x3
  detector head                |d| / __expf bound <= 1       0.196     0.197     0.192
  descriptor head              |d| / dot bound <= 1          0.142     0.393     0.067
  descriptor sampling          |d| / position bound <= 1     4.4e-3    4.5e-3    4.5e-3
  keypoint encoder             16 u_tf32, 16 u_tf32, 64 u    4.2e-3    4.0e-3    5.9e-6
                               (7.8e-3, 7.8e-3, 1.5e-5)
  GNN layers 0, 1, 17          8 u, 2 u, 128 u               1.9e-3    3.6e-3    1.5e-5
                               (3.9e-3, 7.8e-3, 3.1e-5)
  final_proj, score GEMM       |d| / dot bound <= 1          0.661     0.625     0.376
  Sinkhorn                     |dZ| < 4e-5                   1.2e-5    9.7e-6    8.4e-6
  softmax rows (K = 2048)      |d| / bound <= 1              0.158     -         0.082
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import U32, branch_err, dot_bound, fullres_inputs, synth
from oracle import spsg_oracle as so

pytestmark = pytest.mark.gpu

PRECISIONS = ["tf32", "bf16", "fp32x3"]
FRAMES = {"small": (240, 320, 256), "product": (720, 540, 1024)}
# operand rounding of the fp32-input GEMMs (tf32 keeps 10 mantissa bits of both operands, fp32x3 drops lo * lo): the
# keypoint encoder, final_proj and the score matrix, which are tf32 GEMMs in bf16 mode too
C_OP = {"tf32": 2 * 2.0 ** -10, "bf16": 2 * 2.0 ** -10, "fp32x3": 2.0 ** -20}
# the SuperPoint heads: in bf16 mode the stored bf16 input is exact and only the weights are rounded (to nearest)
C_OP_HEAD = {"tf32": 2 * 2.0 ** -10, "bf16": 2.0 ** -9, "fp32x3": 2.0 ** -20}
U = {"tf32": 2.0 ** -11, "bf16": 2.0 ** -8, "fp32x3": 2.0 ** -22}
KENC_BAR = {"tf32": 16 * U["tf32"], "bf16": 16 * U["tf32"], "fp32x3": 64 * U["fp32x3"]}
GNN_BAR = {"tf32": 8 * U["tf32"], "bf16": 2 * U["bf16"], "fp32x3": 128 * U["fp32x3"]}
SK_BAR = 4e-5
# about half of the mutual nearest neighbours of the synthetic weights score above it, so that the threshold decides
# rows both ways (the reference's 0.2 keeps one or two per pair)
MATCH_THR = 0.008
GNN_LAYERS = [0, 1, 17]


# ------------------------------------------------------------------------------------------------ harness
def isolate_gnn_layer(sg, keep):
    """Copy of a SuperGlue state dict in which every ``gnn.layers.{i}`` but ``keep`` has mlp.3 = 0 (weight and bias), so
    that it returns its input unchanged. ``keep=None`` zeroes all of them."""
    out = dict(sg)
    for i in range(18):
        if i != keep:
            for t in ("weight", "bias"):
                k = f"gnn.layers.{i}.mlp.3.{t}"
                out[k] = torch.zeros_like(sg[k])
    return out


def decisions(Z, thr, bar):
    """The match decision of superglue.py:266-276 on log couplings Z [(n0 + 1) x (n1 + 1)] (float64, bins last) ->
    (matches0 [n0], mscores0 [n0], stable [n0]). A row is stable when no perturbation of Z within ``bar`` can change its
    decision: its arg-max leads the runner-up of the row by more than 2 bar, that column's arg-max (the mutual check)
    leads its runner-up by more than 2 bar, and log(thr) is more than 2 bar away from the row's maximum."""
    core = Z[:-1, :-1]
    n0, n1 = core.shape
    if n0 == 0 or n1 == 0:
        return (torch.full((n0,), -1, dtype=torch.long, device=Z.device), Z.new_zeros(n0),
                torch.ones(n0, dtype=torch.bool, device=Z.device))
    rt = core.topk(min(2, n1), dim=1)
    ct = core.topk(min(2, n0), dim=0)
    i0, max0 = rt.indices[:, 0], rt.values[:, 0]
    mutual = ct.indices[0][i0] == torch.arange(n0, device=Z.device)
    ms = torch.where(mutual, max0.exp(), Z.new_zeros(()))
    m0 = torch.where(mutual & (ms > thr), i0, torch.full_like(i0, -1))
    inf = torch.full_like(max0, math.inf)
    row_gap = rt.values[:, 0] - rt.values[:, 1] if n1 > 1 else inf
    col_gap = (ct.values[0] - ct.values[1])[i0] if n0 > 1 else inf
    thr_gap = (max0 - math.log(thr)).abs() if thr > 0 else inf
    stable = (row_gap > 2 * bar) & (col_gap > 2 * bar) & (thr_gap > 2 * bar)
    return m0, ms, stable


@pytest.fixture(scope="module")
def weights():
    from mfr_b200 import spsg
    return spsg.synthetic_state_dicts(0)


def d64(sd):
    return {k: v.double().cuda() for k, v in sd.items()}


def _crop(p, dy, dx, H, W):
    g0 = synth.rgb_to_gray_u8(synth.make_pair(p)["image0"]).astype(np.float32) / 255.0
    return torch.from_numpy(g0[40 + dy:40 + dy + H, 30 + dx:30 + dx + W].copy())[None]


def images(frame):
    """B = 2 pairs. small: a crop and the same view shifted by (8, 16) px in pair 0, another scene shifted by (16, 8) px in
    pair 1. product: the two views of two synthetic scenes at 720x540."""
    if frame == "product":
        i0, i1 = fullres_inputs()
        return i0.cuda(), i1.cuda()
    H, W, _ = FRAMES[frame]
    i0 = torch.cat([_crop(5, 0, 0, H, W), _crop(6, 0, 0, H, W)])
    i1 = torch.cat([_crop(5, 8, 16, H, W), _crop(6, 16, 8, H, W)])
    return i0.cuda(), i1.cuda()


def engine(weights, precision, frame, B=2, K=None, cfg=None):
    from mfr_b200 import spsg
    H, W, K0 = FRAMES[frame]
    sp, sg = weights
    c = {"max_keypoints": K or K0, "match_threshold": MATCH_THR, **(cfg or {})}
    return spsg.SuperPointSuperGlue(sp, sg, batch=B, height=H, width=W, cfg=c, graph=False, precision=precision)


def snapshot(eng, out):
    """The engine's outputs (the keypoint scores as "kp_scores") and stage buffers after a forward, cloned."""
    B, K, H, W = eng.B, eng.K, eng.H, eng.W
    NI = 2 * B
    h8, w8 = H // 8, W // 8
    s = {("kp_scores" if k == "scores" else k): v.clone() for k, v in out.items()}   # "scores": the score map
    for name, shape in (("logits", (NI, h8 * w8, 65)), ("scores", (NI, h8 * 8, w8 * 8)),
                        ("nms_mask", (NI, h8 * 8, w8 * 8)), ("cDa", (NI, h8 * w8, 256)),
                        ("dense_desc", (NI, h8, w8, 256)), ("tokens", (NI, K, 512)), ("mdesc", (NI, K, 256)),
                        ("sg_scores", (B, K, K)), ("sk_u", (B, K + 1)), ("sk_v", (B, K + 1))):
        s[name] = eng.debug_tensor(name, shape).clone()
    return s


_SNAP = {}


def forward_snapshot(weights, precision, frame, K=None, cfg=None):
    """Snapshot of one forward of a B = 2 engine on images(frame), cached per configuration."""
    key = (precision, frame, K, tuple(sorted((cfg or {}).items())))
    if key not in _SNAP:
        eng = engine(weights, precision, frame, K=K, cfg=cfg)
        _SNAP[key] = snapshot(eng, eng.forward(*images(frame)))
        eng.close()
    return _SNAP[key]


def live_rows(t, counts):
    """[NI, K, ...] -> the live rows of every image, concatenated."""
    return torch.cat([t[n, :int(c)] for n, c in enumerate(counts.tolist())])


# ------------------------------------------------------------------------------------------------ SuperPoint
@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_detector_head(weights, precision, frame):
    """scores = softmax over the 65 logits of each 8x8 cell, dustbin dropped, depth-to-space. score_map_kernel is fp32
    with __expf in every precision: each exponential is within (2 + 1.2 |x|) 2^-23 + |x| 2^-24 relative of exp(x) (CUDA's
    __expf bound and the rounded argument x = l - max), the 65-term sum, its reciprocal and the product add 68 u; values
    below 2^-125 may flush to zero."""
    s = forward_snapshot(weights, precision, frame)
    H, W, _ = FRAMES[frame]
    h8, w8 = H // 8, W // 8
    lg = s["logits"].double().view(-1, h8, w8, 65)
    NI = lg.shape[0]
    ref = torch.softmax(lg, -1)[..., :64].reshape(NI, h8, w8, 8, 8).permute(0, 1, 3, 2, 4).reshape(NI, h8 * 8, w8 * 8)
    x = (lg - lg.max(-1, keepdim=True).values).abs().max(-1).values
    rel = 2 * ((2 + 1.2 * x) * 2.0 ** -23 + x * U32) + 68 * U32
    rel = rel.repeat_interleave(8, 1).repeat_interleave(8, 2)
    ratio = ((s["scores"].double() - ref).abs() / (rel * ref + 2.0 ** -125)).max().item()
    print(f"detector head {precision} {frame}: max |d| / bound {ratio:.3e}")
    assert ratio <= 1.0


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_nms(weights, precision, frame):
    """The separable NMS on the engine's own scores equals simple_nms exactly (max and == are exact)."""
    s = forward_snapshot(weights, precision, frame)
    sc, mask = s["scores"], s["nms_mask"]
    assert ((mask == 0) | (mask == 1)).all()
    assert torch.equal(torch.where(mask > 0, sc, torch.zeros_like(sc)), so.simple_nms(sc, 4))


@pytest.mark.parametrize("arg", ["nms_radius", "remove_borders"])
def test_negative_radius_or_border_rejected(weights, arg):
    from mfr_b200 import lib as _lib
    with pytest.raises(_lib.MfrError):
        engine(weights, "tf32", "small", cfg={arg: -1})


def select_ref(sc, mask, thr, border, K):
    """Keypoint selection of superpoint.py:170-187 on one image's scores and NMS mask: (x, y) [n, 2], scores [n] and the
    number of candidates. All candidates in row-major order when there are at most K, else the K highest scores, lower
    pixel index first on ties (the engine's stated order)."""
    Hs, Ws = sc.shape
    yy = torch.arange(Hs, device=sc.device)[:, None].expand(Hs, Ws)
    xx = torch.arange(Ws, device=sc.device)[None].expand(Hs, Ws)
    cand = (mask > 0) & (sc > torch.tensor(thr, dtype=torch.float32, device=sc.device))
    cand &= (yy >= border) & (yy < Hs - border) & (xx >= border) & (xx < Ws - border)
    idx = torch.nonzero(cand.flatten())[:, 0]
    v = sc.flatten()[idx]
    n = len(idx)
    if n > K:
        order = torch.from_numpy(np.lexsort((idx.cpu().numpy(), -v.double().cpu().numpy()))[:K]).to(sc.device)
        idx, v = idx[order], v[order]
    return torch.stack([idx % Ws, idx // Ws], 1).float(), v, n


# (frame, K, nms_radius, remove_borders): bitonic top-k (4, 4) and (4, 0); all candidates in row-major order at K = 2048
# and 240x320, with border 0 (keypoints on the first and last rows and columns) and border 3 (about 28 candidates on
# column W - 3 and 10 on row H - 3, just outside it); nms_radius 1 at 720x540: about 30k candidates, more than the 16384
# the kernel keeps in shared memory
SELECT_CASES = [("small", None, 4, 4), ("small", 2048, 4, 0), ("small", 2048, 4, 3), ("product", None, 4, 4),
                ("product", None, 4, 0), ("product", None, 1, 4), ("product", None, 1, 0)]


@pytest.mark.parametrize("frame,K,radius,border", SELECT_CASES)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_keypoint_selection(weights, precision, frame, K, radius, border):
    """Counts, coordinates and scores equal the reference selection on the engine's own scores and mask, exactly; unused
    slots are zero."""
    cfg = {"nms_radius": radius, "remove_borders": border}
    s = forward_snapshot(weights, precision, frame, K, cfg)
    K = K or FRAMES[frame][2]
    if radius != 4:   # the mask of this configuration (the NMS test covers radius 4)
        assert torch.equal(torch.where(s["nms_mask"] > 0, s["scores"], 0 * s["scores"]), so.simple_nms(s["scores"], radius))
    ncand = []
    for n in range(s["scores"].shape[0]):
        kp, v, nc = select_ref(s["scores"][n], s["nms_mask"][n], 0.005, border, K)
        ncand.append(nc)
        c = int(s["counts"][n])
        assert c == min(nc, K), (n, c, nc)
        assert torch.equal(s["keypoints"][n, :c], kp), n
        assert torch.equal(s["kp_scores"][n, :c], v), n
        assert not s["keypoints"][n, c:].any() and not s["kp_scores"][n, c:].any()
    print(f"selection {precision} {frame} K {K} r {radius} b {border}: candidates {ncand}")
    if K == 2048:
        assert max(ncand) <= K
        if border == 0:
            assert all((s["keypoints"][n, :, 0] == 0).any() and (s["keypoints"][n, :, 1] == 0).any() for n in range(4))
    elif radius == 1 and frame == "product":
        assert min(ncand) > 16384
    else:
        assert min(ncand) > K


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_descriptor_head(weights, precision, frame):
    """dense_desc = L2-normalised convDb(cDa) (1x1 conv) within the per-element bound e_i + |n_i| ||e|| + 260 u |n_i|,
    e = dot bound / ||raw|| (the normalisation's first-order error plus its own sum of squares and scaling)."""
    s = forward_snapshot(weights, precision, frame)
    sp, _ = weights
    x = s["cDa"].double().view(-1, 256)
    Wt, b = sp["convDb.weight"][:, :, 0, 0].cuda(), sp["convDb.bias"].cuda()
    raw = x @ Wt.double().t() + b.double()
    nrm = raw.norm(dim=1, keepdim=True)
    ref = raw / nrm
    e = dot_bound(x, Wt, C_OP_HEAD[precision], b) / nrm
    bar = e + ref.abs() * (e.norm(dim=1, keepdim=True) + 260 * U32)
    ratio = ((s["dense_desc"].double().view(-1, 256) - ref).abs() / bar).max().item()
    print(f"descriptor head {precision} {frame}: max |d| / bound {ratio:.3e}")
    assert ratio <= 1.0


def sampling_bound(kp, dmap, raw):
    """Bound of sample_desc_kernel's normalised descriptor: the fp32 keypoint -> grid -> pixel mapping is within
    dp = 4 (max(h, w) + 1) u of the exact position, which moves a bilinear sample of unit vectors by at most 4 dp in norm;
    the four fmaf taps add 8 u; normalising doubles the relative error and adds 260 u."""
    h, w = dmap.shape[:2]
    dp = 4 * (max(h, w) + 1) * U32
    return 2 * (4 * dp + 8 * U32) / raw.norm(dim=1, keepdim=True) + 260 * U32


@pytest.mark.parametrize("frame,K,border", [("small", None, 4), ("product", None, 4), ("small", 2048, 0)])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_descriptor_sampling(weights, precision, frame, K, border):
    """descriptors = normalize(grid_sample(dense_desc, keypoints, align_corners=False, zero padding)) within
    sampling_bound; border 0 puts keypoints on the first and last rows and columns, where the taps reach the zero
    padding. Unused slots are exactly 0."""
    s = forward_snapshot(weights, precision, frame, K, {"remove_borders": border})
    ratio = 0.0
    for n in range(s["scores"].shape[0]):
        c = int(s["counts"][n])
        kp = s["keypoints"][n, :c].double()
        dmap = s["dense_desc"][n].double()
        ref = so.sample_descriptors(kp[None], dmap.permute(2, 0, 1)[None], 8)[0].t()
        h, w = dmap.shape[:2]
        g = (kp - 3.5) / kp.new_tensor([w * 8 - 4.5, h * 8 - 4.5]) * 2 - 1
        raw = F.grid_sample(dmap.permute(2, 0, 1)[None], g.view(1, 1, -1, 2), align_corners=False)[0, :, 0].t()
        d = (s["descriptors"][n, :c].double() - ref).abs()
        ratio = max(ratio, (d / sampling_bound(kp, dmap, raw)).max().item())
        assert not s["descriptors"][n, c:].any()
    print(f"descriptor sampling {precision} {frame} border {border}: max |d| / bound {ratio:.3e}")
    assert ratio <= 1.0


# ------------------------------------------------------------------------------------------------ SuperGlue
_ISO = {}


def isolated_runs(weights, precision, frame):
    """Tokens of a B = 2 engine with every mlp.3 zeroed (the keypoint encoder's output) and with only layer k live, for k
    in GNN_LAYERS, plus the SuperPoint outputs they were computed from."""
    key = (precision, frame)
    if key not in _ISO:
        sp, sg = weights
        eng = engine((sp, isolate_gnn_layer(sg, None)), precision, frame)
        ims = images(frame)
        out = eng.forward(*ims)
        r = {k: out[k].clone() for k in ("counts", "keypoints", "scores", "descriptors")}
        r["tokens"] = {None: eng.debug_tensor("tokens", (4, eng.K, 512))[:, :, :256].clone()}
        for k in GNN_LAYERS:
            eng.load_state_dicts(sp, isolate_gnn_layer(sg, k))
            o = eng.forward(*ims)
            assert torch.equal(o["counts"], r["counts"]) and torch.equal(o["descriptors"], r["descriptors"])
            r["tokens"][k] = eng.debug_tensor("tokens", (4, eng.K, 512))[:, :, :256].clone()
        eng.close()
        _ISO[key] = r
    return _ISO[key]


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_keypoint_encoder(weights, precision, frame):
    """All GNN layers zeroed: tokens = descriptors + kenc([normalised x, y, score]) on every live row, the encoder branch
    against fp64 (bar KENC_BAR)."""
    r = isolated_runs(weights, precision, frame)
    H, W, _ = FRAMES[frame]
    sg64 = d64(isolate_gnn_layer(weights[1], None))
    cnt = r["counts"]
    kp, sc = live_rows(r["keypoints"], cnt).double(), live_rows(r["scores"], cnt).double()
    desc = live_rows(r["descriptors"], cnt)
    kin = torch.cat([so.normalize_keypoints(kp[None], H, W)[0], sc[:, None]], 1).t()[None]
    ref = desc.double() + so._mlp(kin, sg64, "kenc.encoder", 5)[0].t()
    err = branch_err(desc, live_rows(r["tokens"][None], cnt), ref, U32)
    print(f"keypoint encoder {precision} {frame}: branch err {err:.3e} (bar {KENC_BAR[precision]:.3e})")
    assert err < KENC_BAR[precision]


@pytest.mark.parametrize("layer", GNN_LAYERS)
@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_gnn_layer(weights, precision, frame, layer):
    """Only layer k live: its output on the engine's encoder output against fp64 _attention_layer (self for even k, cross
    for odd k, both images from the old tokens), residual branch over the live rows of all four images (bar GNN_BAR)."""
    r = isolated_runs(weights, precision, frame)
    sg64 = d64(isolate_gnn_layer(weights[1], layer))
    cnt = r["counts"].tolist()
    x = [r["tokens"][None][n, :cnt[n]].double().t()[None] for n in range(4)]
    pre = f"gnn.layers.{layer}"
    ref = []
    for n in range(4):
        src = x[n ^ 1] if layer % 2 else x[n]
        ref.append((x[n] + so._attention_layer(x[n], src, sg64, pre))[0].t())
    err = branch_err(live_rows(r["tokens"][None], r["counts"]), live_rows(r["tokens"][layer], r["counts"]), torch.cat(ref),
                     U32)
    print(f"gnn {precision} {frame} layer {layer}: branch err {err:.3e} (bar {GNN_BAR[precision]:.3e})")
    assert err < GNN_BAR[precision]


def check_scores(s, fp_w, fp_b, c_op, pairs):
    """final_proj and the score GEMM of the given pairs within the per-element dot bound; returns the larger ratio."""
    x = s["tokens"][:, :, :256].reshape(-1, 256)
    m = s["mdesc"].reshape(-1, 256)
    r1 = ((m.double() - (x.double() @ fp_w.double().t() + fp_b.double())).abs() / dot_bound(x, fp_w, c_op, fp_b)).max()
    r2 = 0.0
    for p in pairs:
        a, b = s["mdesc"][2 * p].double(), s["mdesc"][2 * p + 1].double()
        ref = a @ b.t() / 16
        bound = (c_op + 258 * U32) * (a.abs() @ b.abs().t()) / 16
        r2 = max(r2, ((s["sg_scores"][p].double() - ref).abs() / bound).max().item())
    return max(r1.item(), r2)


def check_sinkhorn_and_matches(s, p, alpha, iters=20):
    """Z = S + u + v - norm of pair p from the engine against fp64 log_optimal_transport on the engine's own S (bar
    SK_BAR); matches0 against the fp64 decision on every stable row, mscores0 within the bar there, rows past n0 empty.
    Returns (max |dZ|, number of unstable rows, number of matches)."""
    n0, n1 = int(s["counts"][2 * p]), int(s["counts"][2 * p + 1])
    K = s["sg_scores"].shape[1]
    m0 = s["matches0"][p].long()
    ms0 = s["matching_scores0"][p].double()
    assert (m0[n0:] == -1).all() and not ms0[n0:].any()
    if n0 == 0 or n1 == 0:
        assert (m0 == -1).all() and not ms0.any()
        return 0.0, 0, 0
    S = s["sg_scores"][p, :n0, :n1].double()
    a = torch.tensor(float(alpha), dtype=torch.float64, device=S.device)
    Zref = so.log_optimal_transport(S[None], a, iters)[0]
    Zs = torch.full((n0 + 1, n1 + 1), float(alpha), dtype=torch.float64, device=S.device)
    Zs[:n0, :n1] = S
    norm = -math.log(n0 + n1)
    Z = Zs + s["sk_u"][p, :n0 + 1].double()[:, None] + s["sk_v"][p, :n1 + 1].double()[None] - norm
    dz = (Z - Zref).abs().max().item()
    assert dz < SK_BAR, dz
    ref_m0, ref_ms, stable = decisions(Zref, MATCH_THR, SK_BAR)
    assert torch.equal(m0[:n0][stable], ref_m0[stable])
    d = (ms0[:n0] - ref_ms)[stable].abs()
    assert (d <= ref_ms[stable] * math.expm1(SK_BAR) + 2.0 ** -20).all(), d.max()
    return dz, int((~stable).sum()), int((m0 > -1).sum())


def check_compaction(s):
    """m_offsets and the compacted keypoints follow matches0 exactly, pair by pair."""
    off = s["m_offsets"].tolist()
    assert off[0] == 0
    for p in range(len(off) - 1):
        m0 = s["matches0"][p].long()
        rows = torch.nonzero(m0 > -1)[:, 0]
        assert off[p + 1] - off[p] == len(rows), (p, off)
        assert torch.equal(s["mkpts0"][off[p]:off[p + 1]], s["keypoints"][2 * p][rows])
        assert torch.equal(s["mkpts1"][off[p]:off[p + 1]], s["keypoints"][2 * p + 1][m0[rows]])


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_scores_sinkhorn_matches(weights, precision, frame):
    """final_proj, the score GEMM (alpha = 1/16), Sinkhorn, the match decision and the compaction on the full forward."""
    s = forward_snapshot(weights, precision, frame)
    sg = weights[1]
    ratio = check_scores(s, sg["final_proj.weight"][:, :, 0].cuda(), sg["final_proj.bias"].cuda(), C_OP[precision], (0, 1))
    res = [check_sinkhorn_and_matches(s, p, sg["bin_score"]) for p in (0, 1)]
    check_compaction(s)
    print(f"scores {precision} {frame}: max |d| / bound {ratio:.3e}; sinkhorn max |dZ| {max(r[0] for r in res):.3e}, "
          f"unstable rows {[r[1] for r in res]}, matches {[r[2] for r in res]}")
    assert ratio <= 1.0
    if frame == "small":
        assert all(r[2] > 10 for r in res)


def superglue_inputs(src, K, plan):
    """Host arrays for forward_superglue: pair p of ``plan`` = ((image a, n0), (image b, n1)) takes the first n rows of
    the snapshot's images a and b; the rest is zero."""
    NI = 2 * len(plan)
    cnt = np.zeros(NI, np.int32)
    kp = np.zeros((NI, K, 2), np.float32); sc = np.zeros((NI, K), np.float32); de = np.zeros((NI, K, 256), np.float32)
    for p, sides in enumerate(plan):
        for side, (img, n) in enumerate(sides):
            i = 2 * p + side
            cnt[i] = n
            kp[i, :n] = src["keypoints"][img, :n].cpu().numpy()
            sc[i, :n] = src["kp_scores"][img, :n].cpu().numpy()
            de[i, :n] = src["descriptors"][img, :n].cpu().numpy()
    return cnt, kp, sc, de


@pytest.mark.parametrize("precision", PRECISIONS)
def test_ragged_pairs(weights, precision):
    """B = 5 through forward_superglue with counts (K, K), (K - 37, 5), (1, 1), (0, 40), (40, 0): every live pair passes the
    score, Sinkhorn and match checks, empty pairs have no matches and leave m_offsets where it was, and the tokens are
    finite on every row, padding included."""
    src = forward_snapshot(weights, precision, "small")
    K = FRAMES["small"][2]
    assert (src["counts"] == K).all()
    plan = [((0, K), (1, K)), ((2, K - 37), (3, 5)), ((1, 1), (0, 1)), ((3, 0), (2, 40)), ((0, 40), (3, 0))]
    eng = engine(weights, precision, "small", B=5)
    s = snapshot(eng, eng.forward_superglue(*superglue_inputs(src, K, plan)))
    eng.close()
    assert torch.isfinite(s["tokens"]).all()
    sg = weights[1]
    ratio = check_scores(s, sg["final_proj.weight"][:, :, 0].cuda(), sg["final_proj.bias"].cuda(), C_OP[precision],
                         range(5))
    res = [check_sinkhorn_and_matches(s, p, sg["bin_score"]) for p in range(5)]
    check_compaction(s)
    off = s["m_offsets"].tolist()
    assert off[3] == off[4] == off[5]
    print(f"ragged {precision}: max |d| / bound {ratio:.3e}; sinkhorn max |dZ| {max(r[0] for r in res):.3e}, "
          f"unstable rows {[r[1] for r in res]}, matches {[r[2] for r in res]}, m_offsets {off}")
    assert ratio <= 1.0
    assert res[0][2] > 0 and res[1][2] + res[2][2] > 0


@pytest.mark.parametrize("precision", ["tf32", "fp32x3"])
def test_softmax_k2048(weights, precision):
    """K = 2048 (the softmax rows' second code path, past 1024 keys) with counts 1500 and 1100: the last layer's attention
    probabilities (a cross layer; attn_scores holds P after the forward) against an fp64 masked softmax of Q K^T / 8 from
    the engine's qkv. Per row, |P - P_ref| <= P_ref expm1(2 D + (2 + 1.2 X) 2^-23 + X u + 40 u) + 2^-125, with D the dot
    bound of the scores and X the row's largest |S - max S|; rows and columns past the counts are exactly 0. The score,
    Sinkhorn and match checks run on the same forward."""
    K, n = 2048, (1500, 1100)
    g = torch.Generator().manual_seed(7)
    H, W, _ = FRAMES["small"]
    kp = torch.stack([torch.randint(0, W, (2, K), generator=g), torch.randint(0, H, (2, K), generator=g)], -1).float()
    sc = torch.rand(2, K, generator=g)
    de = F.normalize(torch.randn(2, K, 256, generator=g), dim=-1)
    cnt = np.array(n, np.int32)
    for i in range(2):
        kp[i, n[i]:] = 0; sc[i, n[i]:] = 0; de[i, n[i]:] = 0
    eng = engine(weights, precision, "small", B=1, K=K)
    out = eng.forward_superglue(cnt, kp.numpy(), sc.numpy(), de.numpy())
    qkv = eng.debug_tensor("qkv", (2, K, 768)).double()
    P = eng.debug_tensor("attn_scores", (2, 4, K, K))
    ratio = 0.0
    for img in range(2):
        nq, nk = n[img], n[img ^ 1]
        assert not P[img, :, nq:].any() and not P[img, :, :, nk:].any()
        for h in range(4):
            q = qkv[img, :nq, 64 * h:64 * h + 64]
            k = qkv[img ^ 1, :nk, 256 + 64 * h:256 + 64 * h + 64]
            S = q @ k.t() / 8
            D = ((C_OP[precision] + 66 * U32) * (q.abs() @ k.abs().t()) / 8).max(1, keepdim=True).values
            X = (S - S.max(1, keepdim=True).values).abs().max(1, keepdim=True).values
            ref = torch.softmax(S, 1)
            bound = ref * torch.expm1(2 * D + (2 + 1.2 * X) * 2.0 ** -23 + X * U32 + 40 * U32) + 2.0 ** -125
            ratio = max(ratio, ((P[img, h, :nq, :nk].double() - ref).abs() / bound).max().item())
    s = snapshot(eng, out)
    eng.close()
    sg = weights[1]
    r2 = check_scores(s, sg["final_proj.weight"][:, :, 0].cuda(), sg["final_proj.bias"].cuda(), C_OP[precision], (0,))
    dz, unstable, nm = check_sinkhorn_and_matches(s, 0, sg["bin_score"])
    check_compaction(s)
    print(f"softmax K 2048 {precision}: max |d| / bound {ratio:.3e}; scores {r2:.3e}; sinkhorn {dz:.3e}, "
          f"unstable {unstable}, matches {nm}")
    assert ratio <= 1.0 and r2 <= 1.0
