"""ORACLE (test infrastructure only — never imported by the product path).

Plain PyTorch fp32 CPU restatement of the SuperPoint + SuperGlue inference path that the reference's
``SuperGlue_matcher`` runs (etc/feature_matching_baselines/matchers.py:62-120 ->
SuperGlue/models/matching.py:56-84, superpoint.py:145-202, superglue.py:228-283), written
functionally over reference-format state dicts (``superpoint_v1.pth`` / ``superglue_*.pth`` layout)
so the same weights feed the reference modules, this oracle and the CUDA engine.

Pinned against the reference modules (real in-tree weights, imported from /root/reference in the
build container) by tests/test_oracle_vs_reference.py and the vectors in tests/golden/.
"""
import torch
import torch.nn.functional as F

SP_CFG = {"nms_radius": 4, "keypoint_threshold": 0.005, "max_keypoints": 1024, "remove_borders": 4}  # matchers.py:65-68
SG_CFG = {"sinkhorn_iterations": 20, "match_threshold": 0.2}                                          # matchers.py:70-71


# ------------------------------------------------------------------------------ SuperPoint
def simple_nms(scores, r):
    """superpoint.py:47-62."""
    def mp(x):
        return F.max_pool2d(x, kernel_size=r * 2 + 1, stride=1, padding=r)
    zeros = torch.zeros_like(scores)
    max_mask = scores == mp(scores)
    for _ in range(2):
        supp_mask = mp(max_mask.float()) > 0
        supp_scores = torch.where(supp_mask, zeros, scores)
        new_max_mask = supp_scores == mp(supp_scores)
        max_mask = max_mask | (new_max_mask & (~supp_mask))
    return torch.where(max_mask, scores, zeros)


def sample_descriptors(kpts, desc, s=8):
    """superpoint.py:80-92; torch 2.x => grid_sample align_corners default (False), see :87."""
    b, c, h, w = desc.shape
    kpts = kpts - s / 2 + 0.5
    kpts = kpts / torch.tensor([(w * s - s / 2 - 0.5), (h * s - s / 2 - 0.5)]).to(kpts)[None]
    kpts = kpts * 2 - 1
    d = F.grid_sample(desc, kpts.view(b, 1, -1, 2), mode="bilinear", align_corners=False)
    return F.normalize(d.reshape(b, c, -1), p=2, dim=1)


def superpoint_dense(img, sd):
    """Encoder + heads (superpoint.py:147-166,190-192): img [1,1,H,W] -> (scores [1,H8*8,W8*8] before
    NMS, dense L2-normalised descriptors [1,256,H8,W8])."""
    x = img
    for name in ("1a", "1b", "P", "2a", "2b", "P", "3a", "3b", "P", "4a", "4b"):
        if name == "P":
            x = F.max_pool2d(x, 2, 2)
        else:
            x = F.relu(F.conv2d(x, sd[f"conv{name}.weight"], sd[f"conv{name}.bias"], 1, 1))
    cPa = F.relu(F.conv2d(x, sd["convPa.weight"], sd["convPa.bias"], 1, 1))
    scores = F.conv2d(cPa, sd["convPb.weight"], sd["convPb.bias"])
    scores = F.softmax(scores, 1)[:, :-1]
    b, _, h, w = scores.shape
    scores = scores.permute(0, 2, 3, 1).reshape(b, h, w, 8, 8).permute(0, 1, 3, 2, 4).reshape(b, h * 8, w * 8)
    cDa = F.relu(F.conv2d(x, sd["convDa.weight"], sd["convDa.bias"], 1, 1))
    desc = F.normalize(F.conv2d(cDa, sd["convDb.weight"], sd["convDb.bias"]), p=2, dim=1)
    return scores, desc


def superpoint(img, sd, cfg=None):
    """SuperPoint.forward for one image [1,1,H,W] -> keypoints [n,2] (x,y) float, scores [n],
    descriptors [256,n]."""
    cfg = {**SP_CFG, **(cfg or {})}
    scores, desc = superpoint_dense(img, sd)
    h8, w8 = desc.shape[2:]
    scores = simple_nms(scores, cfg["nms_radius"])[0]
    kp = torch.nonzero(scores > cfg["keypoint_threshold"])
    sc = scores[tuple(kp.t())]
    bd, hh, ww = cfg["remove_borders"], h8 * 8, w8 * 8
    m = (kp[:, 0] >= bd) & (kp[:, 0] < hh - bd) & (kp[:, 1] >= bd) & (kp[:, 1] < ww - bd)
    kp, sc = kp[m], sc[m]
    k = cfg["max_keypoints"]
    if k >= 0 and k < len(kp):
        sc, idx = torch.topk(sc, k, dim=0)
        kp = kp[idx]
    kp = torch.flip(kp, [1]).float()
    d = sample_descriptors(kp[None], desc, 8)[0]
    return kp, sc, d


# ------------------------------------------------------------------------------ SuperGlue
def _mlp(x, sd, pre, n_layers):
    """MLP of Conv1d(k=1) [+ BatchNorm1d + ReLU between] (superglue.py:49-60); x [1,C,n]."""
    idx = 0
    for i in range(n_layers):
        x = F.conv1d(x, sd[f"{pre}.{idx}.weight"], sd[f"{pre}.{idx}.bias"])
        idx += 1
        if i < n_layers - 1:
            x = F.batch_norm(x, sd[f"{pre}.{idx}.running_mean"], sd[f"{pre}.{idx}.running_var"],
                             sd[f"{pre}.{idx}.weight"], sd[f"{pre}.{idx}.bias"], False, 0.0, 1e-5)
            x = F.relu(x)
            idx += 2
    return x


def normalize_keypoints(kpts, h, w):
    """superglue.py:63-70 (on kpts' device, in its dtype)."""
    size = kpts.new_tensor([[float(w), float(h)]])
    center = size / 2
    scaling = size.max(1, keepdim=True).values * 0.7
    return (kpts - center[:, None, :]) / scaling[:, None, :]


def _attention_layer(x, src, sd, pre):
    """AttentionalPropagation.forward (superglue.py:110-118) incl. the (dim, heads) channel split of
    MultiHeadedAttention (:101-107)."""
    b = x.size(0)
    q, k, v = [F.conv1d(t, sd[f"{pre}.attn.proj.{i}.weight"], sd[f"{pre}.attn.proj.{i}.bias"]).view(b, 64, 4, -1)
               for i, t in enumerate((x, src, src))]
    scores = torch.einsum("bdhn,bdhm->bhnm", q, k) / 64 ** 0.5
    prob = F.softmax(scores, dim=-1)
    msg = torch.einsum("bhnm,bdhm->bdhn", prob, v).contiguous().view(b, 256, -1)
    msg = F.conv1d(msg, sd[f"{pre}.attn.merge.weight"], sd[f"{pre}.attn.merge.bias"])
    return _mlp(torch.cat([x, msg], dim=1), sd, f"{pre}.mlp", 2)


def gnn(d0, d1, sd):
    """AttentionalGNN.forward (superglue.py:130-138): 18 layers, ['self', 'cross'] * 9; both images are updated from the
    previous layer's tokens."""
    for i in range(18):
        pre = f"gnn.layers.{i}"
        s0, s1 = (d1, d0) if i % 2 == 1 else (d0, d1)       # ['self', 'cross'] * 9 (superglue.py:192)
        delta0, delta1 = _attention_layer(d0, s0, sd, pre), _attention_layer(d1, s1, sd, pre)
        d0, d1 = d0 + delta0, d1 + delta1
    return d0, d1


def log_optimal_transport(scores, alpha, iters):
    """superglue.py:141-170."""
    b, m, n = scores.shape
    one = scores.new_tensor(1)
    ms, ns = (m * one).to(scores), (n * one).to(scores)
    bins0 = alpha.expand(b, m, 1)
    bins1 = alpha.expand(b, 1, n)
    al = alpha.expand(b, 1, 1)
    Z = torch.cat([torch.cat([scores, bins0], -1), torch.cat([bins1, al], -1)], 1)
    norm = -(ms + ns).log()
    log_mu = torch.cat([norm.expand(m), ns.log()[None] + norm])[None].expand(b, -1)
    log_nu = torch.cat([norm.expand(n), ms.log()[None] + norm])[None].expand(b, -1)
    u, v = torch.zeros_like(log_mu), torch.zeros_like(log_nu)
    for _ in range(iters):
        u = log_mu - torch.logsumexp(Z + v.unsqueeze(1), dim=2)
        v = log_nu - torch.logsumexp(Z + u.unsqueeze(2), dim=1)
    return Z + u.unsqueeze(2) + v.unsqueeze(1) - norm


def superglue(kpts0, sc0, desc0, kpts1, sc1, desc1, h, w, sd, cfg=None, return_scores=False):
    """SuperGlue.forward (superglue.py:228-283): kpts [n,2], scores [n], desc [256,n] per image ->
    matches0 [n0] int64 (-1 = none), matching_scores0 [n0]."""
    cfg = {**SG_CFG, **(cfg or {})}
    if kpts0.shape[0] == 0 or kpts1.shape[0] == 0:
        return torch.full((kpts0.shape[0],), -1, dtype=torch.int64), torch.zeros(kpts0.shape[0])
    k0 = normalize_keypoints(kpts0[None], h, w)
    k1 = normalize_keypoints(kpts1[None], h, w)
    d0 = desc0[None] + _mlp(torch.cat([k0.transpose(1, 2), sc0[None, None]], 1), sd, "kenc.encoder", 5)
    d1 = desc1[None] + _mlp(torch.cat([k1.transpose(1, 2), sc1[None, None]], 1), sd, "kenc.encoder", 5)
    d0, d1 = gnn(d0, d1, sd)
    m0 = F.conv1d(d0, sd["final_proj.weight"], sd["final_proj.bias"])
    m1 = F.conv1d(d1, sd["final_proj.weight"], sd["final_proj.bias"])
    scores = torch.einsum("bdn,bdm->bnm", m0, m1) / 256 ** 0.5
    Z = log_optimal_transport(scores, sd["bin_score"], cfg["sinkhorn_iterations"])
    max0, max1 = Z[:, :-1, :-1].max(2), Z[:, :-1, :-1].max(1)
    i0, i1 = max0.indices, max1.indices
    ar0 = torch.arange(i0.shape[1])[None]
    mutual0 = ar0 == i1.gather(1, i0)
    ms0 = torch.where(mutual0, max0.values.exp(), Z.new_tensor(0))
    valid0 = mutual0 & (ms0 > cfg["match_threshold"])
    matches0 = torch.where(valid0, i0, i0.new_tensor(-1))[0]
    if return_scores:
        return matches0, ms0[0], scores[0], Z[0]
    return matches0, ms0[0]


def match_pair(img0, img1, sp_sd, sg_sd):
    """Matching.forward + SuperGlue_matcher.match glue (matching.py:56-84, matchers.py:106-120):
    -> [N,4] (x0,y0,x1,y1) float32 tensor (possibly empty)."""
    h, w = img0.shape[2:]
    k0, s0, d0 = superpoint(img0, sp_sd)
    k1, s1, d1 = superpoint(img1, sp_sd)
    m0, _ = superglue(k0, s0, d0, k1, s1, d1, h, w, sg_sd)
    valid = m0 > -1
    return torch.cat([k0[valid], k1[m0[valid]]], 1)
