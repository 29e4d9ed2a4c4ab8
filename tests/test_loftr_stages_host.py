"""The layer-isolation trick of tests/test_loftr_stages_gpu.py, checked in float64 on the oracle (no GPU): with norm2
zeroed in every encoder layer but k, the whole transformer returns exactly what a single ``encoder_layer`` call of
layer k returns, including in cross layers, where feat1 attends to the updated feat0."""
import pytest
import torch

from oracle import loftr_oracle as lo
from test_loftr_stages_gpu import isolate_layer


@pytest.fixture(scope="module")
def sd64():
    from mfr_b200 import loftr
    return {k: v.double() for k, v in loftr.synthetic_state_dict(0).items()}


@pytest.mark.parametrize("pre,n_layers,names,shape", [("loftr_coarse", 8, lo.CONFIG["coarse_layers"], (2, 40, 256)),
                                                      ("loftr_fine", 2, lo.CONFIG["fine_layers"], (7, 25, 128))])
def test_isolated_layer_is_one_encoder_layer(sd64, pre, n_layers, names, shape):
    g = torch.Generator().manual_seed(n_layers)
    f0 = torch.randn(shape, generator=g, dtype=torch.float64)
    f1 = torch.randn(shape, generator=g, dtype=torch.float64)
    nh = lo.CONFIG["coarse_heads"]
    none = isolate_layer(sd64, pre, n_layers, None)
    y0, y1 = lo.transformer(f0, f1, none, pre, names, nh)
    assert torch.equal(y0, f0) and torch.equal(y1, f1)
    for k in range(n_layers):
        sdk = isolate_layer(sd64, pre, n_layers, k)
        assert all(torch.equal(sdk[n], sd64[n]) for n in sd64 if not n.startswith(f"{pre}.layers.") or
                   n.startswith(f"{pre}.layers.{k}."))
        y0, y1 = lo.transformer(f0, f1, sdk, pre, names, nh)
        p = f"{pre}.layers.{k}"
        if names[k] == "self":
            r0 = lo.encoder_layer(f0, f0, sd64, p, nh)
            r1 = lo.encoder_layer(f1, f1, sd64, p, nh)
        else:
            r0 = lo.encoder_layer(f0, f1, sd64, p, nh)
            r1 = lo.encoder_layer(f1, r0, sd64, p, nh)
        assert torch.equal(y0, r0) and torch.equal(y1, r1)
        assert not torch.equal(r1, f1)          # the layer does change the tokens
