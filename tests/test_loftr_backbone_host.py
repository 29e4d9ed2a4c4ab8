"""The references of tests/test_loftr_backbone_stages_gpu.py, tied to the BN-form oracle without a GPU.

1. Every backbone table of ``prepare_weights`` is, bit for bit, the fp32 rounding of the float64 BatchNorm fold
   w g / sqrt(var + 1e-5), beta - mean g / sqrt(var + 1e-5) (stem, every conv1 / conv2 / down, both outconv2.0) or the
   plain copy of the conv weight (the 1x1 outconvs and both outconv2.3), in the engine's [Cout][R*R][Cin] layout.
2. The chain of the stage functions over those tables is ``oracle.loftr_oracle.backbone`` in float64: the only
   difference is the fp32 rounding of the folded tables (2^-24 relative per weight), so both outputs agree within a
   few fp32 units of their largest element."""
import numpy as np
import pytest
import torch

from oracle import loftr_oracle as lo
from test_loftr_backbone_stages_gpu import STAGES, backbone64

EPS = 1e-5


def _fold(sd, conv, bn):
    s = sd[bn + ".weight"].double().numpy() / np.sqrt(sd[bn + ".running_var"].double().numpy() + EPS)
    w = sd[conv].double().numpy() * s[:, None, None, None]
    b = sd[bn + ".bias"].double().numpy() - sd[bn + ".running_mean"].double().numpy() * s
    return w, b


def _layout(w):
    co, ci, r, _ = w.shape
    return w.transpose(0, 2, 3, 1).reshape(co, r * r, ci)


def _expected_tables(sd):
    """{engine name: float64 array} restated from the reference-format state dict."""
    out = {}
    w, b = _fold(sd, "backbone.conv1.weight", "backbone.bn1")
    out["stem.w"], out["stem.b"] = w.reshape(128, 49), b
    for li in (1, 2, 3):
        for bi in (0, 1):
            p, q = f"backbone.layer{li}.{bi}", f"layer{li}.{bi}"
            for cv, bn in (("conv1", "bn1"), ("conv2", "bn2")):
                w, b = _fold(sd, f"{p}.{cv}.weight", f"{p}.{bn}")
                out[f"{q}.{cv}.w"], out[f"{q}.{cv}.b"] = _layout(w), b
            if bi == 0 and li > 1:
                w, b = _fold(sd, f"{p}.downsample.0.weight", f"{p}.downsample.1")
                out[f"{q}.down.w"], out[f"{q}.down.b"] = _layout(w), b
    for n in ("layer2_outconv2", "layer1_outconv2"):
        w, b = _fold(sd, f"backbone.{n}.0.weight", f"backbone.{n}.1")
        out[f"{n}.0.w"], out[f"{n}.0.b"] = _layout(w), b
        out[f"{n}.3.w"] = _layout(sd[f"backbone.{n}.3.weight"].double().numpy())
    for n in ("layer3_outconv", "layer2_outconv", "layer1_outconv"):
        out[n + ".w"] = _layout(sd[f"backbone.{n}.weight"].double().numpy())
    return out


@pytest.mark.parametrize("seed", [0, 1])
def test_folded_tables_are_the_rounded_fp64_fold(seed):
    from mfr_b200 import loftr
    sd = loftr.synthetic_state_dict(seed)
    got = loftr.prepare_weights(sd, 4, 4)
    exp = _expected_tables(sd)
    backbone = {k for k in got if k.startswith(("stem.", "layer"))}
    assert backbone == set(exp)
    assert {s.step for s in STAGES if s.step != "upsample"} == {k.rsplit(".", 1)[0] for k in exp}
    for k, v in exp.items():
        g = got[k]
        assert g.dtype == np.float32 and g.shape == v.shape, (k, g.shape, v.shape)
        assert np.array_equal(g.view(np.int32), v.astype(np.float32).view(np.int32)), k


def test_stage_chain_is_the_oracle_backbone():
    """1 image 48x80 (1/8 map 6x10); max |d| / max |ref| of both outputs below 16 fp32 units."""
    from mfr_b200 import loftr
    sd = loftr.synthetic_state_dict(0)
    g = torch.Generator().manual_seed(5)
    img = torch.rand((1, 1, 48, 80), generator=g, dtype=torch.float64)
    tables = loftr.prepare_weights(sd, 6, 10)
    fc, ff = backbone64(img, tables)
    rc, rf = lo.backbone(img, {k: v.double() for k, v in sd.items()})
    for name, got, ref in (("feat_c", fc, rc), ("feat_f", ff, rf)):
        assert got.shape == ref.shape
        err = ((got - ref).abs().max() / ref.abs().max()).item()
        print(f"{name}: max |d| / max |ref| {err:.3e} ({err / 2.0 ** -24:.2f} fp32 units)")
        assert err < 16 * 2.0 ** -24, (name, err)
