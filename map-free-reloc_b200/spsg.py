"""Host side of the SuperPoint + SuperGlue matcher: weight preparation for the CUDA engine and the
matcher plugin with the reference's interface (``SuperGlue_matcher(resize, outdoor).match(pair) ->
[N,4]``, etc/feature_matching_baselines/matchers.py:62-120). All network arithmetic runs in
libmfr_b200.so; torch is used for device memory and streams only. No CPU fallback."""
import ctypes
import os

import numpy as np
import torch

from . import lib as _lib
from .image_io import PairMatcher

DEFAULTS = {"nms_radius": 4, "keypoint_threshold": 0.005, "max_keypoints": 1024, "remove_borders": 4,
            "sinkhorn_iterations": 20, "match_threshold": 0.2}          # matchers.py:65-71


def _conv_layout(w):
    co, ci, r, s = w.shape
    return w.permute(0, 2, 3, 1).reshape(co, r * s, ci).contiguous()


def _fold_bn1d(w, b, sd, bn, eps=1e-5):
    """Conv1d(k=1) [Cout, Cin, 1] + BatchNorm1d (eval) -> ([Cout, Cin], [Cout])."""
    g, beta = sd[bn + ".weight"].double(), sd[bn + ".bias"].double()
    mean, var = sd[bn + ".running_mean"].double(), sd[bn + ".running_var"].double()
    s = g / torch.sqrt(var + eps)
    return (w[:, :, 0].double() * s[:, None]).float(), ((b.double() - mean) * s + beta).float()


# SuperGlue splits channels as (dim=64, heads=4): channel c = d*4 + h (superglue.py:104-105). The
# engine wants heads contiguous (c' = h*64 + d); PERM[c'] = c.
_PERM = torch.tensor([d * 4 + h for h in range(4) for d in range(64)])


def prepare_weights(sp_sd, sg_sd):
    """(superpoint_v1.pth-format dict, superglue_*.pth-format dict) -> {engine name: float32 ndarray}."""
    sp = {k: v.detach().float().cpu() for k, v in sp_sd.items()}
    sg = {k: v.detach().float().cpu() for k, v in sg_sd.items()}
    out = {"conv1a.w": sp["conv1a.weight"].reshape(64, 9), "conv1a.b": sp["conv1a.bias"]}
    for n in ("1b", "2a", "2b", "3a", "3b", "4a", "4b", "Pa", "Pb", "Da", "Db"):
        out[f"conv{n}.w"] = _conv_layout(sp[f"conv{n}.weight"])
        out[f"conv{n}.b"] = sp[f"conv{n}.bias"]
    # keypoint encoder: Conv1d/BN/ReLU x4 + Conv1d (superglue.py:73-82); input padded 3 -> 4 channels
    idx = 0
    for i in range(5):
        w, b = sg[f"kenc.encoder.{idx}.weight"], sg[f"kenc.encoder.{idx}.bias"]
        if i < 4:
            w2, b2 = _fold_bn1d(w, b, sg, f"kenc.encoder.{idx + 1}")
            idx += 3
        else:
            w2, b2 = w[:, :, 0], b
        if i == 0:
            w2 = torch.cat([w2, torch.zeros(w2.shape[0], 1)], 1)
        out[f"kenc.{i}.w"], out[f"kenc.{i}.b"] = w2, b2
    for i in range(18):
        p = f"gnn.layers.{i}"
        q = f"gnn.{i}"
        ws = [sg[f"{p}.attn.proj.{j}.weight"][:, :, 0][_PERM] for j in range(3)]
        bs = [sg[f"{p}.attn.proj.{j}.bias"][_PERM] for j in range(3)]
        out[q + ".qkv.w"], out[q + ".qkv.b"] = torch.cat(ws, 0), torch.cat(bs, 0)
        out[q + ".merge.w"] = sg[f"{p}.attn.merge.weight"][:, :, 0][:, _PERM]
        out[q + ".merge.b"] = sg[f"{p}.attn.merge.bias"]
        out[q + ".mlp0.w"], out[q + ".mlp0.b"] = _fold_bn1d(sg[f"{p}.mlp.0.weight"], sg[f"{p}.mlp.0.bias"], sg, f"{p}.mlp.1")
        out[q + ".mlp3.w"], out[q + ".mlp3.b"] = sg[f"{p}.mlp.3.weight"][:, :, 0], sg[f"{p}.mlp.3.bias"]
    out["final_proj.w"], out["final_proj.b"] = sg["final_proj.weight"][:, :, 0], sg["final_proj.bias"]
    out["bin_score"] = sg["bin_score"].reshape(1)
    return {k: np.ascontiguousarray(v.numpy().astype(np.float32)) for k, v in out.items()}


def synthetic_state_dicts(seed=0):
    """Deterministic synthetic SuperPoint / SuperGlue weights in the reference's state_dict formats
    (the real ones live in the reference tree, which does not travel to the GPU box)."""
    g = torch.Generator().manual_seed(seed)

    def conv(co, ci, k):
        return torch.randn(co, ci, k, k, generator=g) * (2.0 / (ci * k * k)) ** 0.5, 0.05 * torch.randn(co, generator=g)

    sp = {}
    for n, ci, co, k in (("1a", 1, 64, 3), ("1b", 64, 64, 3), ("2a", 64, 64, 3), ("2b", 64, 64, 3), ("3a", 64, 128, 3),
                         ("3b", 128, 128, 3), ("4a", 128, 128, 3), ("4b", 128, 128, 3), ("Pa", 128, 256, 3),
                         ("Pb", 256, 65, 1), ("Da", 128, 256, 3), ("Db", 256, 256, 1)):
        sp[f"conv{n}.weight"], sp[f"conv{n}.bias"] = conv(co, ci, k)
    sp["convPb.weight"] *= 6.0     # peaky cell softmax -> a realistic number of detections
    # zero-mean descriptor head: a random ReLU net collapses to nearly parallel descriptors; centring
    # the last (linear) layer on a fixed probe image makes them discriminative enough to match
    import torch.nn.functional as F
    x = torch.rand(1, 1, 96, 96, generator=g)
    with torch.no_grad():
        for n in ("1a", "1b", "P", "2a", "2b", "P", "3a", "3b", "P", "4a", "4b"):
            x = F.max_pool2d(x, 2, 2) if n == "P" else F.relu(F.conv2d(x, sp[f"conv{n}.weight"], sp[f"conv{n}.bias"], 1, 1))
        y = F.conv2d(F.relu(F.conv2d(x, sp["convDa.weight"], sp["convDa.bias"], 1, 1)), sp["convDb.weight"], None)
    sp["convDb.bias"] = -y.mean(dim=(0, 2, 3))
    sg = {}

    def c1(name, ci, co, scale=1.0):
        sg[name + ".weight"] = torch.randn(co, ci, 1, generator=g) * scale / ci ** 0.5
        sg[name + ".bias"] = 0.05 * torch.randn(co, generator=g)

    def bn(name, c):
        sg[name + ".weight"] = 0.75 + 0.5 * torch.rand(c, generator=g)
        sg[name + ".bias"] = 0.1 * torch.randn(c, generator=g)
        sg[name + ".running_mean"] = 0.1 * torch.randn(c, generator=g)
        sg[name + ".running_var"] = 0.5 + torch.rand(c, generator=g)

    chans = [3, 32, 64, 128, 256, 256]
    idx = 0
    for i in range(5):
        c1(f"kenc.encoder.{idx}", chans[i], chans[i + 1])
        idx += 1
        if i < 4:
            bn(f"kenc.encoder.{idx}", chans[i + 1])
            idx += 2
    for i in range(18):
        p = f"gnn.layers.{i}"
        for j in range(3):
            c1(f"{p}.attn.proj.{j}", 256, 256, 2.0)
        c1(f"{p}.attn.merge", 256, 256)
        c1(f"{p}.mlp.0", 512, 512)
        bn(f"{p}.mlp.1", 512)
        c1(f"{p}.mlp.3", 512, 256, 0.05)
        sg[f"{p}.mlp.3.bias"] *= 0.1
    sg["kenc.encoder.12.weight"] *= 0.05
    sg["kenc.encoder.12.bias"] *= 0.05
    # near-identity projection with gain: matching score ~ 12 * cos(desc0, desc1)
    c1("final_proj", 256, 256, 1.0)
    sg["final_proj.weight"] = 14.0 * torch.eye(256)[:, :, None] + 0.5 * sg["final_proj.weight"]
    sg["bin_score"] = torch.tensor(1.0)
    return sp, sg


def load_weights(w, outdoor):
    """(superpoint, superglue) state dicts from ``w``: such a pair, or the directory holding superpoint_v1.pth and
    superglue_{indoor,outdoor}.pth (SuperGlue/models/weights in the reference tree)."""
    if not isinstance(w, str):
        sp, sg = w
        return sp, sg
    return (torch.load(os.path.join(w, "superpoint_v1.pth"), map_location="cpu"),
            torch.load(os.path.join(w, f"superglue_{'outdoor' if outdoor else 'indoor'}.pth"), map_location="cpu"))


class SuperPointSuperGlue(_lib.Engine):
    """CUDA SuperPoint+SuperGlue engine for ``batch`` pairs of [H, W] gray images."""

    input_dtype = torch.float32

    def __init__(self, sp_sd, sg_sd, batch=1, height=720, width=540, cfg=None, device=0, graph=True, precision="tf32"):
        self.cfg = c = {**DEFAULTS, **(cfg or {})}
        self.B, self.H, self.W, self.K = int(batch), int(height), int(width), int(self.cfg["max_keypoints"])
        self.capacity, self.max_pts_per_pair = self.B * self.K, self.K
        self.precision = {"tf32": 0, "bf16": 1, "fp32x3": 2, "fp32": 2}[precision]
        super().__init__("spsg", "mfr_spsg_create_ex", (self.B, self.H, self.W, self.K, int(c["nms_radius"]),
                                                        float(c["keypoint_threshold"]), int(c["remove_borders"]),
                                                        int(c["sinkhorn_iterations"]), float(c["match_threshold"]),
                                                        self.precision), device)
        self._l.mfr_spsg_set_graph(self._h, int(bool(graph)))
        self.load_state_dicts(sp_sd, sg_sd)
        self._o = self._get_outputs(self._l.mfr_spsg_get_outputs, _lib.SpsgOutputs)

    def load_state_dicts(self, sp_sd, sg_sd):
        """Uploads new SuperPoint / SuperGlue weights (reference state_dict formats); a map of set_map is dropped."""
        self._upload_weights(prepare_weights(sp_sd, sg_sd))

    def num_launches(self):
        return self._l.mfr_spsg_num_launches(self._h)

    # buffers stored in bf16 in bf16 mode: the SuperPoint activations, q|k|v, the attention message, the token shadow
    BF16_TENSORS = ("x1a", "x4b", "cPa", "cDa", "qkv", "msg", "tokens_bf16")

    def debug_tensor(self, name, shape):
        """Named engine buffer as a device tensor view. fp32, except in bf16 mode (precision="bf16"), where the
        buffers named in BF16_TENSORS ("qkv" [2B][K][768], "msg" [2B][K][256], ...) are torch.bfloat16 views, and
        "attn_scores" / "attn_vt" do not exist (the fused attention never stores them)."""
        bf = self.precision == 1 and name in self.BF16_TENSORS
        return super().debug_tensor(name, shape, torch.bfloat16 if bf else torch.float32)

    def device_outputs(self):
        o, B, K = self._o, self.B, self.K
        return {"counts": self.view(o.counts, (2 * B,), torch.int32),
                "keypoints": self.view(o.keypoints, (2 * B, K, 2), torch.float32),
                "scores": self.view(o.scores, (2 * B, K), torch.float32),
                "descriptors": self.view(o.descriptors, (2 * B, K, o.desc_ld), torch.float32),
                "matches0": self.view(o.matches0, (B, K), torch.int32),
                "matching_scores0": self.view(o.matching_scores0, (B, K), torch.float32),
                "m_offsets": self.view(o.m_offsets, (B + 1,), torch.int32),
                "mkpts0": self.view(o.mkpts0, (B * K, 2), torch.float32),
                "mkpts1": self.view(o.mkpts1, (B * K, 2), torch.float32)}

    def pose_inputs(self):
        """(kpts0 [capacity, 2], kpts1 [capacity, 2], offsets [B + 1]): device views of the last forward's matches in the
        pose back end's layout."""
        o = self._o
        return (self.view(o.mkpts0, (self.capacity, 2), torch.float32), self.view(o.mkpts1, (self.capacity, 2), torch.float32),
                self.view(o.m_offsets, (self.B + 1,), torch.int32))

    def forward_async(self, img0, img1):
        """Enqueues one batch of pairs (CUDA float32 [B,(1,)H,W] each) on the engine stream."""
        self._call(self._l.mfr_spsg_forward, self._images(img0, self.B, self.H, self.W),
                   self._images(img1, self.B, self.H, self.W))

    def set_map(self, img0):
        """Runs SuperPoint once, eagerly on the engine stream, on the map image img0 (CUDA float32 [(1,)(1,)H,W]). Until
        the next set_map, ``forward_shared[_async](img1)`` gives the bits ``forward[_async]`` gives with img0 repeated for
        every pair; a paired forward in between does not disturb the map."""
        self._call(self._l.mfr_spsg_set_map, self._images(img0, self.H, self.W))

    def forward_shared_async(self, img1):
        """Enqueues one batch of B query images [B,(1,)H,W] against the map of ``set_map``."""
        self._call(self._l.mfr_spsg_forward_shared, self._images(img1, self.B, self.H, self.W))

    def forward_shared(self, img1):
        self.forward_shared_async(img1)
        self.stream.synchronize()
        return self.device_outputs()

    def forward_superglue(self, counts, kpts, scores, desc):
        """SuperGlue only on host numpy arrays: counts [2B] int32, kpts [2B,K,2], scores [2B,K],
        desc [2B,K,256] float32 (pair-interleaved image order)."""
        c = np.ascontiguousarray(counts, dtype=np.int32); k = np.ascontiguousarray(kpts, dtype=np.float32)
        s_ = np.ascontiguousarray(scores, dtype=np.float32); d = np.ascontiguousarray(desc, dtype=np.float32)
        assert k.shape == (2 * self.B, self.K, 2) and d.shape == (2 * self.B, self.K, 256)
        P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        self._call(self._l.mfr_spsg_forward_superglue, P(c), P(k), P(s_), P(d))
        self.stream.synchronize()
        return self.device_outputs()

    def forward(self, img0, img1):
        self.forward_async(img0, img1)
        self.stream.synchronize()
        return self.device_outputs()


class SuperGlue_matcher(PairMatcher):
    """Drop-in for the reference's offline matcher plugin (matchers.py:62-120). ``weights_dir`` holds superpoint_v1.pth
    and superglue_{indoor,outdoor}.pth (SuperGlue/models/weights in the reference tree); ``state_dicts``, a (superpoint,
    superglue) pair, replaces it."""

    def __init__(self, resize, outdoor=False, weights_dir="SuperGlue/models/weights", state_dicts=None, precision="tf32"):
        sp, sg = load_weights(weights_dir if state_dicts is None else state_dicts, outdoor)
        # precision: "tf32" (default), "bf16" (throughput mode, see include/mfr_b200.h) or "fp32x3"
        super().__init__(resize, SuperPointSuperGlue(sp, sg, batch=1, height=int(resize[1]), width=int(resize[0]),
                                                     precision=precision))

    @staticmethod
    def _matches(o):
        m = int(o["m_offsets"][1].item())
        return o["mkpts0"][:m], o["mkpts1"][:m]
