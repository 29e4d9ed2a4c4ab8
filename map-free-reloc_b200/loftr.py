"""Host side of the LoFTR matcher: weight preparation for the CUDA engine and the matcher plugin
with the reference's interface (``LoFTR_matcher(resize, outdoor).match((path0, path1)) -> [N,4]``,
etc/feature_matching_baselines/matchers.py:12-59 of the reference).

All network arithmetic runs in libmfr_b200.so (hand-written sm_90a kernels); torch is used for
device memory and streams only. There is no CPU fallback.
"""
import ctypes
import math

import numpy as np
import torch

from . import lib as _lib
from .image_io import PairMatcher
from .pose_solver import _cfg_get

DEFAULT_CFG = {"thr": 0.2, "border_rm": 2, "temperature": 0.1}  # cvpr_ds_config.py:31-35


def position_encoding(d_model, h, w):
    """Sinusoidal table added to the 1/8 feature map, ``temp_bug_fix=False`` variant
    (LoFTR/src/loftr/utils/position_encoding.py:22-38): the divisor evaluates to -1.0, i.e.
    div_term = exp(-2k). Returned channel-last [h, w, d_model] float32."""
    pe = torch.zeros((d_model, h, w), dtype=torch.float32)
    ypos = torch.arange(1, h + 1, dtype=torch.float32)[:, None].expand(h, w)[None]
    xpos = torch.arange(1, w + 1, dtype=torch.float32)[None, :].expand(h, w)[None]
    k = torch.arange(0, d_model // 2, 2, dtype=torch.float32)
    div = torch.exp(k * float(-math.log(10000.0) / d_model // 2))[:, None, None]
    pe[0::4] = torch.sin(xpos * div)
    pe[1::4] = torch.cos(xpos * div)
    pe[2::4] = torch.sin(ypos * div)
    pe[3::4] = torch.cos(ypos * div)
    return pe.permute(1, 2, 0).contiguous()


def _fold_bn(conv_w, sd, bn, eps=1e-5):
    """Folds an eval-mode BatchNorm2d into the preceding bias-free conv:
    w' = w * g/sqrt(var+eps), b' = beta - mean * g/sqrt(var+eps)."""
    g = sd[bn + ".weight"].double()
    b = sd[bn + ".bias"].double()
    mean = sd[bn + ".running_mean"].double()
    var = sd[bn + ".running_var"].double()
    s = g / torch.sqrt(var + eps)
    w = conv_w.double() * s[:, None, None, None]
    return w.float(), (b - mean * s).float()


def _conv_layout(w):
    """[Cout, Cin, R, S] -> [Cout, R*S, Cin] (channel-last taps, what the implicit GEMM reads)."""
    co, ci, r, s = w.shape
    return w.permute(0, 2, 3, 1).reshape(co, r * s, ci).contiguous()


def prepare_weights(sd, h_c, w_c):
    """Reference-format LoFTR ``state_dict`` -> {engine tensor name: float32 ndarray}."""
    sd = {k[len("matcher."):] if k.startswith("matcher.") else k: v.detach().float().cpu()
          for k, v in sd.items()}  # loftr.py:77-81 strips the Lightning prefix
    out = {}
    w, b = _fold_bn(sd["backbone.conv1.weight"], sd, "backbone.bn1")
    out["stem.w"] = w.reshape(128, 49)
    out["stem.b"] = b
    for li in (1, 2, 3):
        for bi in (0, 1):
            p = f"backbone.layer{li}.{bi}"
            q = f"layer{li}.{bi}"
            for cv, bn in (("conv1", "bn1"), ("conv2", "bn2")):
                w, b = _fold_bn(sd[f"{p}.{cv}.weight"], sd, f"{p}.{bn}")
                out[f"{q}.{cv}.w"] = _conv_layout(w)
                out[f"{q}.{cv}.b"] = b
            if f"{p}.downsample.0.weight" in sd:
                w, b = _fold_bn(sd[f"{p}.downsample.0.weight"], sd, f"{p}.downsample.1")
                out[f"{q}.down.w"] = _conv_layout(w)
                out[f"{q}.down.b"] = b
    for name in ("layer3_outconv", "layer2_outconv", "layer1_outconv"):
        out[name + ".w"] = _conv_layout(sd[f"backbone.{name}.weight"])
    for name in ("layer2_outconv2", "layer1_outconv2"):
        w, b = _fold_bn(sd[f"backbone.{name}.0.weight"], sd, f"backbone.{name}.1")
        out[name + ".0.w"] = _conv_layout(w)
        out[name + ".0.b"] = b
        out[name + ".3.w"] = _conv_layout(sd[f"backbone.{name}.3.weight"])
    out["pos_enc"] = position_encoding(256, h_c, w_c)
    for pre, ref, nl in (("coarse", "loftr_coarse", 8), ("fine", "loftr_fine", 2)):
        for i in range(nl):
            r = f"{ref}.layers.{i}"
            q = f"{pre}.{i}"
            out[q + ".qkv.w"] = torch.cat([sd[r + ".q_proj.weight"], sd[r + ".k_proj.weight"],
                                           sd[r + ".v_proj.weight"]], 0)
            out[q + ".merge.w"] = sd[r + ".merge.weight"]
            out[q + ".mlp0.w"] = sd[r + ".mlp.0.weight"]
            out[q + ".mlp2.w"] = sd[r + ".mlp.2.weight"]
            out[q + ".norm1.g"] = sd[r + ".norm1.weight"]
            out[q + ".norm1.b"] = sd[r + ".norm1.bias"]
            out[q + ".norm2.g"] = sd[r + ".norm2.weight"]
            out[q + ".norm2.b"] = sd[r + ".norm2.bias"]
    out["fine.down_proj.w"] = sd["fine_preprocess.down_proj.weight"]
    out["fine.down_proj.b"] = sd["fine_preprocess.down_proj.bias"]
    out["fine.merge_feat.w"] = sd["fine_preprocess.merge_feat.weight"]
    out["fine.merge_feat.b"] = sd["fine_preprocess.merge_feat.bias"]
    return {k: np.ascontiguousarray(v.numpy().astype(np.float32)) for k, v in out.items()}


# ---- synthetic weights (the real indoor/outdoor checkpoints are not distributed with the reference)
def _state_dict_shapes():
    s = {}
    def bn(p, c):
        s[p + ".weight"] = (c,); s[p + ".bias"] = (c,)
        s[p + ".running_mean"] = (c,); s[p + ".running_var"] = (c,)
    s["backbone.conv1.weight"] = (128, 1, 7, 7)
    bn("backbone.bn1", 128)
    cin = 128
    for li, c in zip((1, 2, 3), (128, 196, 256)):
        for bi in (0, 1):
            p = f"backbone.layer{li}.{bi}"
            s[p + ".conv1.weight"] = (c, cin if bi == 0 else c, 3, 3)
            s[p + ".conv2.weight"] = (c, c, 3, 3)
            bn(p + ".bn1", c)
            bn(p + ".bn2", c)
            if bi == 0 and li > 1:
                s[p + ".downsample.0.weight"] = (c, cin, 1, 1)
                bn(p + ".downsample.1", c)
        cin = c
    s["backbone.layer3_outconv.weight"] = (256, 256, 1, 1)
    s["backbone.layer2_outconv.weight"] = (256, 196, 1, 1)
    s["backbone.layer2_outconv2.0.weight"] = (256, 256, 3, 3)
    bn("backbone.layer2_outconv2.1", 256)
    s["backbone.layer2_outconv2.3.weight"] = (196, 256, 3, 3)
    s["backbone.layer1_outconv.weight"] = (196, 128, 1, 1)
    s["backbone.layer1_outconv2.0.weight"] = (196, 196, 3, 3)
    bn("backbone.layer1_outconv2.1", 196)
    s["backbone.layer1_outconv2.3.weight"] = (128, 196, 3, 3)
    for pre, c, nl in (("loftr_coarse", 256, 8), ("loftr_fine", 128, 2)):
        for i in range(nl):
            p = f"{pre}.layers.{i}"
            for nme in ("q_proj", "k_proj", "v_proj", "merge"):
                s[f"{p}.{nme}.weight"] = (c, c)
            s[p + ".mlp.0.weight"] = (2 * c, 2 * c)
            s[p + ".mlp.2.weight"] = (c, 2 * c)
            for nme in ("norm1", "norm2"):
                s[f"{p}.{nme}.weight"] = (c,)
                s[f"{p}.{nme}.bias"] = (c,)
    s["fine_preprocess.down_proj.weight"] = (128, 256)
    s["fine_preprocess.down_proj.bias"] = (128,)
    s["fine_preprocess.merge_feat.weight"] = (128, 256)
    s["fine_preprocess.merge_feat.bias"] = (128,)
    return s


def synthetic_state_dict(seed=0):
    """Deterministic synthetic LoFTR weights with the reference's state_dict names and shapes
    (the real indoor/outdoor checkpoints are not in the reference tree, SURVEY.md §3.3).
    He-style conv init, Xavier-style linear init, and NON-trivial BatchNorm statistics / affine
    terms / LayerNorm affine terms so that folding and normalisation are actually exercised."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in _state_dict_shapes().items():
        if k.endswith("running_var"):
            v = 0.5 + torch.rand(shp, generator=g)
        elif k.endswith("running_mean"):
            v = 0.1 * torch.randn(shp, generator=g)
        elif ".bn" in k or "downsample.1" in k or "outconv2.1" in k or ".norm" in k:
            if k.endswith(".weight"):
                v = 0.75 + 0.5 * torch.rand(shp, generator=g)
            else:
                v = 0.1 * torch.randn(shp, generator=g)
        elif len(shp) == 4:
            fan_out = shp[0] * shp[2] * shp[3]
            v = torch.randn(shp, generator=g) * (2.0 / fan_out) ** 0.5
        elif len(shp) == 2:
            bound = (6.0 / (shp[0] + shp[1])) ** 0.5
            v = (torch.rand(shp, generator=g) * 2 - 1) * bound
        else:
            v = 0.05 * torch.randn(shp, generator=g)
        sd[k] = v.float().contiguous()
    return sd


def functional_state_dict(coarse_scale=200.0, fine_scale=30.0, ln_gain=40.0, noise=0.0, noise_seed=0):
    """Hand-constructed LoFTR weights (reference state_dict names / shapes) that make the network a
    working matcher on textured scenes, for benchmarking without the real checkpoints (which the
    reference does not ship): every layer runs with its full shape and FLOPs, but the convolutions
    implement a classical patch descriptor instead of learned features.

    * stem: 7x7 Gaussian -> channel 0 = blurred image at 1/2 resolution (all values >= 0, so the
      ReLUs are transparent; BatchNorms are identities);
    * layer1: shift kernels build the 9x9 neighbourhood of channel 0 in other channels (fine
      descriptor, 2 px sample spacing) while the residual path carries channel 0 on;
    * layer2 / layer3.0.conv1: [1 2 1]^2 / 16 blur + stride 2 on channel 0 (down to 1/8), shortcut
      convs zero; layer3: shift kernels build the 7x7 neighbourhood (8 px spacing);
    * layer3_outconv / layer1_outconv2.3: centring matrices (sample - patch mean) and a scale; the
      FPN top-down branches are zeroed;
    * coarse transformer layer 0: message zeroed (norm1 gain 0), MLP = identity (relu(x) - relu(-x)),
      norm2 gain ``ln_gain`` -> x + g * LayerNorm(x): tokens get (almost) unit norm, so the dual
      softmax matches by normalised cross-correlation; the other layers are identities;
    * fine level: merge_feat passes the window features through, transformer identity.

    ``noise`` > 0 adds seeded Gaussian noise of that standard deviation to EVERY conv / linear weight, so that no
    tensor-core operand is structurally zero: the constructed weights above are 99.8 % zeros, and a chip multiplying
    zeros draws far less power (and clocks higher) than one running a trained checkpoint. The perturbed network is
    still a working matcher (the descriptor is a few hundred times larger than the perturbation), which is what the
    throughput benchmark needs: dense operands AND a few thousand matches per pair for the fine level and RANSAC.
    """
    sd = {k: torch.zeros(shp) for k, shp in _state_dict_shapes().items()}
    for k in sd:                                                       # identity BatchNorms / LayerNorm gains off
        if k.endswith("running_var"):
            sd[k] = torch.ones_like(sd[k])
        elif (".bn" in k or "downsample.1" in k or "outconv2.1" in k) and k.endswith(".weight"):
            sd[k] = torch.ones_like(sd[k])
    ax = torch.arange(7, dtype=torch.float32) - 3
    g1 = torch.exp(-ax ** 2 / (2 * 1.5 ** 2)); g1 = g1 / g1.sum()
    sd["backbone.conv1.weight"][0, 0] = g1[:, None] * g1[None, :]
    b3 = torch.tensor([1.0, 2.0, 1.0]) / 4
    blur3 = b3[:, None] * b3[None, :]

    def shift_kernel(dy, dx):            # out(y, x) = in(y + dy, x + dx)  (cross-correlation convention)
        k = torch.zeros(3, 3); k[1 + dy, 1 + dx] = 1.0
        return k

    def grow(w, src, dst_base):
        """src: {offset: channel}; add a ring: every offset within max|o|+1 gets a channel >= dst_base
        fed from a neighbouring source offset through a one-hot 3x3 kernel. Returns {offset: channel}."""
        r = max(max(abs(a), abs(b)) for a, b in src) + 1
        out = {}
        c = dst_base
        for oy in range(-r, r + 1):
            for ox in range(-r, r + 1):
                sy, sx = max(-r + 1, min(r - 1, oy)), max(-r + 1, min(r - 1, ox))
                w[c, src[(sy, sx)]] = shift_kernel(oy - sy, ox - sx)
                out[(oy, ox)] = c
                c += 1
        return out

    # ---- layer1 (1/2 res, 128 ch): ch 0 = blurred image, fine-descriptor samples in 1.. ; residual keeps ch 0
    o = grow(sd["backbone.layer1.0.conv1.weight"], {(0, 0): 0}, 1)             # 3x3  -> internal ch 1..9
    o = grow(sd["backbone.layer1.0.conv2.weight"], o, 1)                       # 5x5  -> x ch 1..25
    o = grow(sd["backbone.layer1.1.conv1.weight"], o, 1)                       # 7x7  -> internal ch 1..49
    fine = grow(sd["backbone.layer1.1.conv2.weight"], o, 26)                   # 9x9  -> x1 ch 26..106
    # ---- layer2 / layer3: blur + subsample channel 0, then the 7x7 neighbourhood at 1/8
    sd["backbone.layer2.0.conv1.weight"][0, 0] = blur3
    sd["backbone.layer2.0.conv2.weight"][0, 0] = shift_kernel(0, 0)
    sd["backbone.layer3.0.conv1.weight"][0, 0] = blur3
    o = grow(sd["backbone.layer3.0.conv2.weight"], {(0, 0): 0}, 0)             # 3x3 -> x ch 0..8
    o = grow(sd["backbone.layer3.1.conv1.weight"], o, 0)                       # 5x5 -> internal ch 0..24
    coarse = grow(sd["backbone.layer3.1.conv2.weight"], o, 9)                  # 7x7 -> x3 ch 9..57 (0..8 keep the 3x3)
    nc = len(coarse)
    cen = (torch.eye(nc) - torch.full((nc, nc), 1.0 / nc)) * coarse_scale
    chans = [coarse[k] for k in sorted(coarse)]
    for r_ in range(nc):
        for c_ in range(nc):
            sd["backbone.layer3_outconv.weight"][r_, chans[c_], 0, 0] = cen[r_, c_]
    # ---- fine branch: select the 81 samples, identity 3x3 (centre tap), centring + scale
    fch = [fine[k] for k in sorted(fine)]
    nf = len(fch)
    for r_ in range(nf):
        sd["backbone.layer1_outconv.weight"][r_, fch[r_], 0, 0] = 1.0
        sd["backbone.layer1_outconv2.0.weight"][r_, r_, 1, 1] = 1.0
    cenf = (torch.eye(nf) - torch.full((nf, nf), 1.0 / nf)) * fine_scale
    sd["backbone.layer1_outconv2.3.weight"][:nf, :nf, 1, 1] = cenf
    # ---- transformers
    for pre, c, nl in (("loftr_coarse", 256, 8), ("loftr_fine", 128, 2)):
        for i in range(nl):
            p = f"{pre}.layers.{i}"
            w0 = torch.zeros(2 * c, 2 * c); w0[:c, :c] = torch.eye(c); w0[c:, :c] = -torch.eye(c)
            sd[p + ".mlp.0.weight"] = w0
            sd[p + ".mlp.2.weight"] = torch.cat([torch.eye(c), -torch.eye(c)], 1)
            for nme in ("q_proj", "k_proj", "v_proj", "merge"):     # attention runs, its message is gated off by norm1
                sd[f"{p}.{nme}.weight"] = torch.eye(c)
    sd["loftr_coarse.layers.0.norm2.weight"] = torch.full((256,), float(ln_gain))
    sd["fine_preprocess.merge_feat.weight"] = torch.cat([torch.eye(128), torch.zeros(128, 128)], 1)
    if noise > 0:
        g = torch.Generator().manual_seed(int(noise_seed))
        for k in sorted(sd):
            if k.endswith(".weight") and sd[k].dim() in (2, 4):
                sd[k] = sd[k] + float(noise) * torch.randn(sd[k].shape, generator=g)
    return {k: v.float().contiguous() for k, v in sd.items()}


class LoFTR(_lib.Engine):
    """CUDA LoFTR engine for ``batch`` pairs of [H, W] images (H, W multiples of 8)."""

    input_dtype = torch.float32

    def __init__(self, state_dict, batch=1, height=720, width=544, cfg=None, device=0, graph=True,
                 precision="tf32", pipelined=False):
        self.cfg = {**DEFAULT_CFG, **(cfg or {})}
        self.B, self.H, self.W = int(batch), int(height), int(width)
        # tf32: fp32 storage, TF32 tensor-core inputs; bf16: bf16 storage + kind::f16 MMAs (backbone, token GEMMs,
        # correlation, attention); fp32x3: fp32 storage, every GEMM as a 3xTF32 split product (fp32-faithful)
        self.precision = {"tf32": 0, "bf16": 1, "fp32x3": 2, "fp32": 2}[precision]
        self.precision_name = {0: "tf32", 1: "bf16", 2: "fp32x3"}[self.precision]
        # pipelined: the engine will run under RelocPipeline, where the pose back end of the previous batch shares the GPU
        # with the first layers of this batch's matcher: those launches then leave 8 SMs to it (reserved_sms of
        # mfr_loftr_create; measured +0.8 % pairs/s in the pipeline, -0.6 % for a matcher running alone)
        reserved_sms = 8 if pipelined else 0
        super().__init__("loftr", "mfr_loftr_create", (self.B, self.H, self.W, float(self.cfg["thr"]),
                                                       int(self.cfg["border_rm"]), float(self.cfg["temperature"]),
                                                       self.precision, reserved_sms), device)
        self._l.mfr_loftr_set_graph(self._h, int(bool(graph)))
        self.load_state_dict(state_dict)
        self._o = self._get_outputs(self._l.mfr_loftr_get_outputs, _lib.LoftrOutputs)
        self.capacity = self._o.capacity
        self.max_pts_per_pair = (self.H // 8) * (self.W // 8)   # one match per coarse cell of image 0 at most
        self._host_counts = torch.zeros(4 + self.B + 1, dtype=torch.int32).pin_memory()

    def load_state_dict(self, state_dict):
        self._upload_weights(prepare_weights(state_dict, self.H // 8, self.W // 8))

    def num_kernels(self):
        return self._l.mfr_loftr_num_kernels(self._h)

    def num_launches(self):
        """Kernel launches of one forward (a step of the launch list may launch several kernels)."""
        return self._l.mfr_loftr_num_launches(self._h)

    def profile(self, img0, img1):
        """Per-step device times of one eager forward: list of (name, kind, ms, flops). Returns when it is done."""
        h, w = img0.shape[-2:]
        img0, img1 = self._images(img0, self.B, h, w), self._images(img1, self.B, h, w)
        n = self.num_kernels()
        ms = np.zeros(n, np.float32); fl = np.zeros(n, np.float64); kinds = np.zeros(n, np.int32)
        names = ctypes.create_string_buffer(32 * n)
        torch.cuda.current_stream(self.device).synchronize()     # the images are written; the engine stream orders the rest
        rc = self._l.mfr_loftr_profile(self._h, _lib.ptr(img0), _lib.ptr(img1), h, w,
                                       ctypes.c_void_p(self.stream.cuda_stream), n, ms.ctypes.data_as(ctypes.c_void_p),
                                       fl.ctypes.data_as(ctypes.c_void_p), kinds.ctypes.data_as(ctypes.c_void_p), names)
        if rc < 0:
            raise _lib.MfrError(f"mfr_loftr_profile failed rc={rc}")
        raw = names.raw
        return [(raw[32 * i:32 * i + 32].split(b"\0")[0].decode(), int(kinds[i]), float(ms[i]), float(fl[i]))
                for i in range(rc)]

    def step_names(self):
        """Names of the steps of the paired forward list, in launch order ("stem", "layer1.0.conv1", "upsample", ...)."""
        names = []
        while (n := self._l.mfr_loftr_step_name(self._h, len(names))) is not None:
            names.append(n.decode())
        return names

    def run_steps(self, begin, end):
        """Runs steps [begin, end) of the forward list eagerly on the engine's buffers as the last call left them (stage
        tests: a forward stages the images first). Ordered after the current stream's work; returns when it is done."""
        self._call(self._l.mfr_loftr_run_steps, int(begin), int(end))
        self.stream.synchronize()

    def forward_async(self, img0, img1):
        """Enqueues one batch on the engine stream. img0/img1: CUDA float32 [B,(1,)h,w] with h <= H,
        w <= W; the engine zero-pads to its [H, W] frame (the reference's pad-to-8)."""
        h, w = img0.shape[-2:]
        self._call(self._l.mfr_loftr_forward, self._images(img0, self.B, h, w), self._images(img1, self.B, h, w), h, w)

    def device_outputs(self):
        """Views of the engine's output buffers (valid until the next forward)."""
        cap = self.capacity
        o = self._o
        return {
            "m_total": self.view(o.m_total, (4,), torch.int32),
            "m_offsets": self.view(o.m_offsets, (self.B + 1,), torch.int32),
            "b_ids": self.view(o.b_ids, (cap,), torch.int32),
            "i_ids": self.view(o.i_ids, (cap,), torch.int32),
            "j_ids": self.view(o.j_ids, (cap,), torch.int32),
            "mconf": self.view(o.mconf, (cap,), torch.float32),
            "mkpts0_f": self.view(o.mkpts0_f, (cap, 2), torch.float32),
            "mkpts1_f": self.view(o.mkpts1_f, (cap, 2), torch.float32),
            "mkpts1_c": self.view(o.mkpts1_c, (cap, 2), torch.float32),
            "expec_f": self.view(o.expec_f, (cap, 3), torch.float32),
        }

    def pose_inputs(self):
        """(kpts0 [capacity, 2], kpts1 [capacity, 2], offsets [B + 1]): device views of the last forward's fine matches in
        the pose back end's layout."""
        d = self.device_outputs()
        return d["mkpts0_f"], d["mkpts1_f"], d["m_offsets"]

    def set_map(self, img0):
        """Encodes the map image img0 (CUDA float32 [(1,)(1,)h,w], h <= H, w <= W) once, eagerly, on the engine stream.
        Until the next set_map or weight upload, ``forward_shared[_async](img1)`` gives the bits ``forward[_async]`` gives
        with img0 repeated for every pair; a paired forward in between does not disturb the map."""
        h, w = img0.shape[-2:]
        self._call(self._l.mfr_loftr_set_map, self._images(img0, h, w), h, w)

    def forward_shared_async(self, img1):
        """Enqueues one batch of B query images [B,(1,)h,w] against the map of ``set_map`` (same h, w; else MfrError)."""
        h, w = img1.shape[-2:]
        self._call(self._l.mfr_loftr_forward_shared, self._images(img1, self.B, h, w), h, w)

    def forward_shared(self, img1):
        """forward_shared_async + the live matches, as ``forward`` returns them."""
        self.forward_shared_async(img1)
        return self._live_outputs()

    def forward(self, img0, img1):
        """Runs the batch and returns the live matches (device tensors, sliced to M)."""
        self.forward_async(img0, img1)
        return self._live_outputs()

    def _live_outputs(self):
        d = self.device_outputs()
        with torch.cuda.stream(self.stream):
            self._host_counts[:4].copy_(d["m_total"], non_blocking=True)
            self._host_counts[4:].copy_(d["m_offsets"], non_blocking=True)
        self.stream.synchronize()
        m = int(self._host_counts[0])
        out = {k: v[:m] for k, v in d.items() if k not in ("m_total", "m_offsets")}
        out["m_offsets"] = self._host_counts[4:].clone()
        out["M"] = m
        return out


def read_image_gray(path, resize):
    """Reference image loader (SuperGlue/models/utils.py:263-285 with resize_float=True):
    grayscale imread, float32 cv2.resize to (W, H), /255 -> float32 [H, W] numpy."""
    import cv2
    image = cv2.imread(str(path), cv2.IMREAD_GRAYSCALE)
    if image is None:
        return None
    w_new, h_new = int(resize[0]), int(resize[1])
    image = cv2.resize(image.astype("float32"), (w_new, h_new))
    return (image / 255.0).astype(np.float32)


def pad_to_8(img):
    """matchers.py:41-46 quirk kept: pads right/bottom by ``size % 8`` (not the complement) and the
    test ``inp.size(1) % 8`` looks at the channel axis (=1), so it always fires. img [.., H, W]."""
    pad_bottom = img.shape[-2] % 8
    pad_right = img.shape[-1] % 8
    return torch.nn.functional.pad(img, (0, pad_right, 0, pad_bottom), value=0.0)


def engine_frame(h, w):
    """The engine frame (H, W) for h x w images: what ``pad_to_8`` makes of them, which must be a multiple of 8."""
    hp, wp = h + h % 8, w + w % 8
    if hp % 8 or wp % 8:
        raise ValueError(f"LoFTR needs a resolution that the reference's padding turns into a multiple of 8, got {h}x{w}")
    return hp, wp


def load_weights(w):
    """The reference-format LoFTR state dict in ``w``: a state dict, a Lightning checkpoint ({'state_dict': ...}), or
    the path of a file holding either."""
    if isinstance(w, str):
        w = torch.load(w, map_location="cpu")
    return w.get("state_dict", w)


def engine_cfg(cfg):
    """The engine's ``cfg`` from a method config's LOFTR.{THR, BORDER_RM, TEMPERATURE} keys, DEFAULT_CFG where unset."""
    return {k: type(v)(_cfg_get(cfg, "LOFTR." + k.upper(), v)) for k, v in DEFAULT_CFG.items()}


class LoFTR_matcher(PairMatcher):
    """Drop-in for the reference's offline matcher plugin (matchers.py:12-59). ``weights``: anything ``load_weights``
    takes; the reference reads LoFTR/weights/{indoor,outdoor}_ot.ckpt, which are not distributed with it."""

    def __init__(self, resize, outdoor=False, weights=None, cfg=None):
        if weights is None:
            weights = "LoFTR/weights/outdoor_ot.ckpt" if outdoor else "LoFTR/weights/indoor_ot.ckpt"
        h, w = engine_frame(int(resize[1]), int(resize[0]))
        super().__init__(resize, LoFTR(load_weights(weights), batch=1, height=h, width=w, cfg=cfg))

    @staticmethod
    def _matches(out):
        return out["mkpts0_f"], out["mkpts1_f"]
