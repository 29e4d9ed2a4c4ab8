"""Each LoFTR backbone stage (stem, every ResNet-FPN conv, both FPN upsample-adds) against float64, fed with the engine's
own input, in the three engine precisions.

The forward overwrites most backbone buffers later in the same list (a0 holds the stem output, then layer1's output;
b1, b2, c1, c2 are reused inside every block), so a forward alone shows only its two outputs. Here one forward stages
the images, then ``LoFTR.run_steps`` walks the forward list one stage at a time: the stage's inputs are copied out of
the engine's buffers (``debug_tensor``), the stage runs (in fp32x3 its ``split3`` step and the conv), and its output is
compared element by element with a float64 restatement on the GPU that uses the folded fp32 tables ``prepare_weights``
uploads (``tests/test_loftr_backbone_host.py`` ties those tables and the stage functions below to the BN-form oracle).

Conv bars, with S = sum |w| |x| + |b| the fp64 conv of |x| and |W| (+ |b|) and K = Cin R^2:
    |y - ref| <= (c_op + (K_acc + 2) 2^-24) S + 2^-24 |res| + u_out |y|
  - K_acc is the number of fp32 products the kernel sums: K, or 3 K in fp32x3, whose GEMM runs over the [hi | lo | hi]
    split (K = 3 Cin per tap), so that the worst-case accumulation bound holds as stated.
  - c_op, the operand rounding: tf32 reads both operands with 10 explicit mantissa bits (2^-10 each, c_op = 2^-9);
    fp32x3 keeps hi.hi + lo.hi + hi.lo of tf32 round-to-nearest splits and drops lo.lo plus the rounding of lo (about
    3 2^-22, c_op = 2^-20 as in the other stage tests); bf16 reads its activations exactly from the engine's bf16
    buffers and the reference uses the round-to-nearest-even bf16 copy of the weights the kernel reads, so c_op = 0.
  - ReLU and LeakyReLU are 1-Lipschitz, so the bound carries through them. The fp32 slope 0.01f differs from 0.01 by
    2.2e-8 relative; on the negative side the conv term of the bound is 100 times larger than needed, which covers it.
  - u_out = 2^-24 for fp32 outputs, 2^-8 for bf16 outputs (round to nearest: |fl(v) - v| <= 2^-8 |fl(v)|).
Stem (K = 49, 7x7 stride 2, pad 3): fp32x3 runs ``stem_kernel``, a 49-term fmaf chain and the bias add (c_op = 0,
K_acc = 49). tf32 and bf16 run ``stem_mma_kernel``: image and weights split into bf16 hi + lo with round to nearest
(|a - ha| <= 2^-8 |a|, the rounding r of lo below 2^-16 |a|); it sums ha.hw + ha.lw + la.hw, so it misses
ha.rw + ra.w + la.lw + la.rw <= (2^-16 + 2^-16 + 2^-16 + 2^-24) |a| |w|: c_op = 3 2^-16, and K_acc = 3 * 49 products.
Upsample-add, dst += bilinear_align_corners(src) with exact fp64 sample positions in the reference:
    |y - ref| <= dy Gy + dx Gx + 8 2^-24 (M + |dst_before|) + u_out |y|
  - ry = fl((Hs - 1) / (Hd - 1)) and sy = fl(ry y) are within 2.01 2^-24 sy of the exact position (dy, dx); the
    interpolant is Lipschitz in each coordinate with the largest neighbour difference Gy (Gx) of src within one pixel
    of the sample cell, which also covers a floor() that lands on the neighbouring cell;
  - the weighted sum of the four samples (largest magnitude M) rounds at most four times and its weights 1 - l once
    (2^-25), the add to dst once: 8 2^-24 (M + |dst_before|) is a generous cover;
  - u_out as for the convs: 2^-24 for the fp32 kernel (tf32, fp32x3) is already in the add term, bf16 adds 2^-8 |y|.
Pad channels: in bf16 mode the 196-channel maps have a pixel stride of 200 so that every row is 16-byte aligned;
``upsample2x_add8_kernel<true>`` reads and writes channels 196..199 and is right only while they hold zero. After
every stage that writes such a map, channels 196..199 are exactly zero.
Teeth: the same bars against perturbed references must fail (ratio > 1): a 196-channel conv whose reference drops the
last 4 input channels, a 3x3 stride-2 conv whose reference pads one pixel off, the 1/8 -> 1/4 upsample with
align_corners=False (small frame; measured tf32 / bf16 / fp32x3: 12.7 / 179 / 83, 141 / 2980 / 1381, and above 2e5).

Frames, B = 2 (4 images), ``synthetic_state_dict(0)`` (dense arithmetic in every layer):
  - bench: 720x544 fed with the two 720x540 ``fullres_inputs()`` (4 zero-padded columns): 1/2, 1/4 and 1/8 maps of
    360x272, 180x136 and 90x68, many tiles per CTA and the TMA traversal stride of the stride-2 convs; all three
    precisions, and bf16 with ``pipelined=True`` as bench.py builds it (the first four convs on a reduced grid);
  - small: 104x152 fed with a 100x150 crop (1/8 map 13x19, odd on both axes, ragged tiles everywhere).

Measured max |d| / bound on one H100 80GB HBM3 (700 W power limit), largest over the 21 convs / the stem / the two
upsample-adds:
  bench  tf32 0.28 / 0.22 / 0.62;  bf16 0.996 / 0.985 / 0.9998 (pipelined: the same bits);  fp32x3 0.060 / 0.067 / 0.62
  small  tf32 0.27 / 0.12 / 0.49;  bf16 0.992 / 0.971 / 0.9998;                              fp32x3 0.061 / 0.057 / 0.49
In bf16 the output rounding is most of the bar: a correctly rounded bf16 value is up to 2^-8 |y| from its fp32 value
when |y| lies just above a power of two, so the maxima sit just below 1 and anything the kernel adds to the rounding
beyond the few 1e-5 relative of the accumulation term fails; the two bf16 convs with fp32 outputs (layer3_outconv,
layer1_outconv2.3) measure 1.1e-2 and 6.3e-3. The whole file runs in about 30 s on that GPU."""
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from helpers import U32, fullres_inputs

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -8       # bf16 unit roundoff
C_OP = {"tf32": 2.0 ** -9, "bf16": 0.0, "fp32x3": 2.0 ** -20}
STEM_C_OP = {"tf32": 3 * 2.0 ** -16, "bf16": 3 * 2.0 ** -16, "fp32x3": 0.0}

# engine buffer -> (resolution divisor, channels); in bf16 mode every backbone map but img, feat_c and feat_f is bf16
# and the 196-channel maps have a pixel stride of 200
BUFFERS = {"img": (1, 1), "a0": (2, 128), "a1": (2, 128), "a2": (2, 128), "b0": (4, 196), "b1": (4, 196),
           "b2": (4, 196), "c0": (8, 256), "c1": (8, 256), "c2": (8, 256), "feat_c_backbone": (8, 256),
           "p4a": (4, 256), "p4b": (4, 256), "p4c": (4, 196), "p2a": (2, 196), "p2b": (2, 196), "feat_f": (2, 128)}
FP32_BUFFERS = ("img", "feat_c_backbone", "feat_f")

Stage = namedtuple("Stage", "step x cin cout r stride res act out")
# the backbone in launch order (loftr_engine.cu: backbone); upsample: x = src, out = dst (in place)
STAGES = [
    Stage("stem", "img", 1, 128, 7, 2, None, "relu", "a0"),
    Stage("layer1.0.conv1", "a0", 128, 128, 3, 1, None, "relu", "a1"),
    Stage("layer1.0.conv2", "a1", 128, 128, 3, 1, "a0", "relu", "a2"),
    Stage("layer1.1.conv1", "a2", 128, 128, 3, 1, None, "relu", "a1"),
    Stage("layer1.1.conv2", "a1", 128, 128, 3, 1, "a2", "relu", "a0"),
    Stage("layer2.0.conv1", "a0", 128, 196, 3, 2, None, "relu", "b1"),
    Stage("layer2.0.down", "a0", 128, 196, 1, 2, None, None, "b2"),
    Stage("layer2.0.conv2", "b1", 196, 196, 3, 1, "b2", "relu", "b0"),
    Stage("layer2.1.conv1", "b0", 196, 196, 3, 1, None, "relu", "b1"),
    Stage("layer2.1.conv2", "b1", 196, 196, 3, 1, "b0", "relu", "b2"),
    Stage("layer3.0.conv1", "b2", 196, 256, 3, 2, None, "relu", "c1"),
    Stage("layer3.0.down", "b2", 196, 256, 1, 2, None, None, "c2"),
    Stage("layer3.0.conv2", "c1", 256, 256, 3, 1, "c2", "relu", "c0"),
    Stage("layer3.1.conv1", "c0", 256, 256, 3, 1, None, "relu", "c1"),
    Stage("layer3.1.conv2", "c1", 256, 256, 3, 1, "c0", "relu", "c2"),
    Stage("layer3_outconv", "c2", 256, 256, 1, 1, None, None, "feat_c_backbone"),
    Stage("layer2_outconv", "b2", 196, 256, 1, 1, None, None, "p4a"),
    Stage("upsample", "feat_c_backbone", 256, 256, None, None, None, None, "p4a"),
    Stage("layer2_outconv2.0", "p4a", 256, 256, 3, 1, None, "leaky", "p4b"),
    Stage("layer2_outconv2.3", "p4b", 256, 196, 3, 1, None, None, "p4c"),
    Stage("layer1_outconv", "a0", 128, 196, 1, 1, None, None, "p2a"),
    Stage("upsample", "p4c", 196, 196, None, None, None, None, "p2a"),
    Stage("layer1_outconv2.0", "p2a", 196, 196, 3, 1, None, "leaky", "p2b"),
    Stage("layer1_outconv2.3", "p2b", 196, 128, 3, 1, None, None, "feat_f"),
]


def stage_id(s):
    return f"upsample.{s.out}" if s.step == "upsample" else s.step


STAGE_IDS = [stage_id(s) for s in STAGES]


# ------------------------------------------------------------------------------------------------ fp64 stage functions
def folded_weights(tables, s):
    """(W [Cout, Cin, R, R], b [Cout] or None) of a conv stage from the engine tables ([Cout][R*R][Cin], BN folded),
    in float64 on the tables' device."""
    w = torch.as_tensor(tables[s.step + ".w"]).double().view(s.cout, s.r, s.r, s.cin).permute(0, 3, 1, 2)
    b = tables.get(s.step + ".b")
    return w, (None if b is None else torch.as_tensor(b).double())


def activation(y, act):
    if act == "relu":
        return F.relu(y)
    if act == "leaky":
        return F.leaky_relu(y, 0.01)
    return y


def conv_stage(x, w, b, s, res=None, pad=None):
    """act(conv(x, W) + b (+ res)), NCHW float64, one image at a time (the im2col of fp64 convs at 1/2 resolution)."""
    pad = s.r // 2 if pad is None else pad
    y = torch.cat([F.conv2d(x[n:n + 1], w, b, s.stride, pad) for n in range(x.shape[0])])
    return activation(y if res is None else y + res, s.act)


def upsample_stage(src, dst, align_corners=True):
    return dst + F.interpolate(src, size=dst.shape[-2:], mode="bilinear", align_corners=align_corners)


def backbone64(img, tables):
    """The whole backbone as the chain of the stage functions: img [N,1,H,W] float64 -> (feat_c, feat_f), NCHW."""
    buf = {"img": img}
    for s in STAGES:
        if s.step == "upsample":
            buf[s.out] = upsample_stage(buf[s.x], buf[s.out])
        else:
            w, b = folded_weights(tables, s)
            buf[s.out] = conv_stage(buf[s.x], w, b, s, buf[s.res] if s.res else None)
    return buf["feat_c_backbone"], buf["feat_f"]


# ------------------------------------------------------------------------------------------------ bounds
def ratio(got, ref, bound):
    """max |got - ref| / bound (elements with got == ref count 0)."""
    d = (got - ref).abs()
    return torch.where(d == 0, torch.zeros_like(d), d / bound).max().item()


def conv_bound(x, w, b, s, precision, got, res, out_bf16):
    if s.step == "stem":
        c_op, k_acc = STEM_C_OP[precision], 49 if precision == "fp32x3" else 3 * 49
    else:
        k = s.cin * s.r * s.r
        c_op, k_acc = C_OP[precision], 3 * k if precision == "fp32x3" else k
    S = conv_stage(x.abs(), w.abs(), None if b is None else b.abs(), s._replace(act=None))
    bound = (c_op + (k_acc + 2) * U32) * S + (U16 if out_bf16 else U32) * got.abs()
    return bound if res is None else bound + U32 * res.abs()


def _gather(t, yi, xi):
    return t[:, :, yi][:, :, :, xi]


def upsample_bound(src, dst, got, out_bf16):
    """Per-element bound of the fp32 upsample-add (derivation in the module docstring). src, dst, got NCHW float64."""
    Hs, Ws = src.shape[-2:]
    Hd, Wd = 2 * Hs, 2 * Ws
    dev = src.device
    yy, xx = torch.arange(Hd, device=dev), torch.arange(Wd, device=dev)
    y0, x0 = yy * (Hs - 1) // (Hd - 1), xx * (Ws - 1) // (Wd - 1)
    y1, x1 = (y0 + 1).clamp(max=Hs - 1), (x0 + 1).clamp(max=Ws - 1)
    pool = lambda t: F.max_pool2d(t, 3, 1, 1)      # max over the cell's one-pixel neighbourhood
    m = pool(src.abs())
    M = torch.maximum(_gather(m, y0, x0), _gather(m, y1, x1))
    gy = pool(F.pad((src[:, :, 1:] - src[:, :, :-1]).abs(), (0, 0, 0, 1)))
    gx = pool(F.pad((src[..., 1:] - src[..., :-1]).abs(), (0, 1)))
    Gy = torch.maximum(_gather(gy, y0, x0), _gather(gy, y0, x1))
    Gx = torch.maximum(_gather(gx, y0, x0), _gather(gx, y1, x0))
    dy = (2.01 * U32 * yy.double() * (Hs - 1) / (Hd - 1))[:, None]
    dx = (2.01 * U32 * xx.double() * (Ws - 1) / (Wd - 1))[None, :]
    bound = dy * Gy + dx * Gx + 8 * U32 * (M + dst.abs())
    return bound + U16 * got.abs() if out_bf16 else bound + U32 * got.abs()


# ------------------------------------------------------------------------------------------------ the step walk
FRAMES = {"bench": (720, 544), "small": (104, 152)}
WALKS = {"bench-tf32": ("bench", "tf32", False), "bench-bf16": ("bench", "bf16", False),
         "bench-fp32x3": ("bench", "fp32x3", False), "bench-bf16-pipelined": ("bench", "bf16", True),
         "small-tf32": ("small", "tf32", False), "small-bf16": ("small", "bf16", False),
         "small-fp32x3": ("small", "fp32x3", False)}
TEETH = {"channel_tail": "layer2.1.conv1", "padding_shift": "layer2.0.conv1", "align_corners": "upsample.p4a"}


def frame_inputs(frame):
    i0, i1 = fullres_inputs()                     # two 720x540 pairs; the engine zero-pads them to its frame
    if frame == "small":
        i0, i1 = i0[..., 300:400, 200:350], i1[..., 300:400, 200:350]
    return i0.contiguous().cuda(), i1.contiguous().cuda()


def read(eng, name, H, W, bf):
    """An engine buffer as a channel-last tensor [4, h, w, pixel stride] (bf16 or fp32, a view)."""
    if name == "img":
        return eng.debug_tensor("img", (4, H, W, 1))
    div, c = BUFFERS[name]
    if bf and name not in FP32_BUFFERS:
        ld = 200 if c == 196 else c
        return eng.debug_tensor(name, (4, H // div, W // div, ld // 2)).view(torch.bfloat16)
    return eng.debug_tensor(name, (4, H // div, W // div, c))


def nchw64(t, c):
    return t[..., :c].permute(0, 3, 1, 2).double()       # a float64 copy


def walk(frame, precision, pipelined):
    """Builds the engine, runs one forward, then re-runs the backbone stage by stage. Returns the step names, the
    stages checked in order, their max |d| / bound, the pad-channel checks (bf16) and the teeth ratios (small frame)."""
    from mfr_b200 import loftr
    H, W = FRAMES[frame]
    sd = loftr.synthetic_state_dict(0)
    tables = {k: torch.from_numpy(v).cuda() for k, v in loftr.prepare_weights(sd, H // 8, W // 8).items()}
    eng = loftr.LoFTR(sd, batch=2, height=H, width=W, graph=False, precision=precision, pipelined=pipelined)
    eng.forward(*frame_inputs(frame))
    bf = precision == "bf16"
    out = {"names": eng.step_names(), "checked": [], "ratio": {}, "rel": {}, "pads": {}, "teeth": {}}
    names, i = out["names"], 0
    for s in STAGES:
        sid = stage_id(s)
        conv = s.step not in ("stem", "upsample")
        n_split = 1 if precision == "fp32x3" and conv else 0
        if names[i:i + n_split + 1] != ["split3"] * n_split + [s.step]:
            break
        x = nchw64(read(eng, s.x, H, W, bf), s.cin)
        res = nchw64(read(eng, s.res, H, W, bf), s.cout) if s.res else None
        dst = nchw64(read(eng, s.out, H, W, bf), s.cout) if s.step == "upsample" else None
        eng.run_steps(i, i + n_split + 1)
        i += n_split + 1
        raw = read(eng, s.out, H, W, bf)
        got = nchw64(raw, s.cout)
        out_bf16 = raw.dtype == torch.bfloat16
        if raw.shape[-1] > s.cout:
            out["pads"][sid] = bool((raw[..., s.cout:] == 0).all())
        if s.step == "upsample":
            ref = upsample_stage(x, dst)
            bound = upsample_bound(x, dst, got, out_bf16)
            bad = {"align_corners": lambda: upsample_stage(x, dst, align_corners=False)}
        else:
            w, b = folded_weights(tables, s)
            if bf and conv:
                w = w.float().bfloat16().double()
            ref = conv_stage(x, w, b, s, res)
            bound = conv_bound(x, w, b, s, precision, got, res, out_bf16)
            bad = {"channel_tail": lambda: conv_stage(x[:, :192], w[:, :192], b, s, res),
                   "padding_shift": lambda: conv_stage(F.pad(x, (0, 2, 0, 2)), w, b, s, res, pad=0)}
        out["ratio"][sid] = ratio(got, ref, bound)
        out["rel"][sid] = ((got - ref).abs().max() / ref.abs().max()).item()
        if frame == "small":
            for kind, f in bad.items():
                if TEETH[kind] == sid:
                    out["teeth"][kind] = ratio(got, f(), bound)
        out["checked"].append(s.step)
        print(f"backbone {frame} {precision}{' pipelined' if pipelined else ''} {sid}: max |d| / bound "
              f"{out['ratio'][sid]:.3e}, max |d| / max |ref| {out['rel'][sid]:.2e}")
        del x, res, dst, got, ref, bound
    eng.close()
    torch.cuda.empty_cache()
    return out


_RESULTS = {}


def result(key):
    """The walk of one (frame, precision) engine, run once per module: the tests assert on it stage by stage."""
    if key not in _RESULTS:
        try:
            _RESULTS[key] = walk(*WALKS[key])
        except Exception as e:          # reported by every test of this engine, not re-run
            _RESULTS[key] = e
        torch.cuda.empty_cache()
    r = _RESULTS[key]
    if isinstance(r, Exception):
        raise r
    return r


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("key", list(WALKS))
def test_walk_reaches_every_backbone_step(key):
    """The stages checked, in order, are exactly the backbone part of the forward list (everything before the position
    encoding), with each fp32x3 ``split3`` step folded into the conv that follows it."""
    r = result(key)
    names = r["names"]
    prefix = names[:names.index("posenc")]
    assert [n for n in prefix if n != "split3"] == r["checked"] == [s.step for s in STAGES]
    if WALKS[key][1] == "fp32x3":
        assert all(prefix[k + 1] not in ("split3", "stem", "upsample") for k, n in enumerate(prefix) if n == "split3")
    else:
        assert "split3" not in prefix


@pytest.mark.parametrize("stage", STAGE_IDS)
@pytest.mark.parametrize("key", list(WALKS))
def test_backbone_stage(key, stage):
    """One backbone stage against float64 within its per-element bound (module docstring)."""
    r = result(key)
    assert stage in r["ratio"], f"the step walk did not reach {stage}"
    assert r["ratio"][stage] <= 1.0, f"{key} {stage}: max |d| / bound {r['ratio'][stage]:.3e}"


@pytest.mark.parametrize("key", [k for k, v in WALKS.items() if v[1] == "bf16"])
def test_pad_channels_stay_zero(key):
    """bf16: after every stage that writes a 196-channel map at pixel stride 200 (b0, b1, b2, p4c, p2a, p2b), channels
    196..199 of that map are exactly zero."""
    r = result(key)
    written = {s.out for s in STAGES if BUFFERS[s.out][1] == 196}
    assert {s.out for s in STAGES if stage_id(s) in r["pads"]} == written
    assert all(r["pads"].values()), [k for k, ok in r["pads"].items() if not ok]


@pytest.mark.parametrize("kind", list(TEETH))
@pytest.mark.parametrize("precision", ["tf32", "bf16", "fp32x3"])
def test_bars_bite(precision, kind):
    """The bars reject a subtly wrong stage: the same bound against a perturbed reference (the last 4 of 196 input
    channels dropped, the padding of a stride-2 conv shifted by one pixel, align_corners=False) is exceeded."""
    r = result(f"small-{precision}")
    print(f"teeth {precision} {kind}: max |d| / bound against the perturbed reference {r['teeth'][kind]:.3e}")
    assert r["teeth"][kind] > 1.0,f"{precision} {kind}: perturbed reference within the bar ({r['teeth'][kind]:.3e})"
