"""The harness of tests/test_spsg_stages_gpu.py checked without a GPU: the layer-isolation trick in float64 on the oracle
(with mlp.3 zeroed in every GNN layer but k, the 18-layer GNN returns exactly one ``_attention_layer`` step of layer k,
both images updated from the old tokens), and the stable-decision rule on hand-made log couplings."""
import math

import pytest
import torch

from oracle import spsg_oracle as so
from test_spsg_stages_gpu import decisions, isolate_gnn_layer


@pytest.fixture(scope="module")
def sg64():
    from mfr_b200 import spsg
    return {k: v.double() for k, v in spsg.synthetic_state_dicts(0)[1].items()}


def test_isolated_layer_is_one_attention_step(sg64):
    g = torch.Generator().manual_seed(3)
    d0 = torch.randn(1, 256, 50, generator=g, dtype=torch.float64)
    d1 = torch.randn(1, 256, 37, generator=g, dtype=torch.float64)
    y0, y1 = so.gnn(d0, d1, isolate_gnn_layer(sg64, None))
    assert torch.equal(y0, d0) and torch.equal(y1, d1)
    for k in range(18):
        sdk = isolate_gnn_layer(sg64, k)
        assert all(torch.equal(sdk[n], sg64[n]) for n in sg64 if ".mlp.3." not in n or n.startswith(f"gnn.layers.{k}."))
        y0, y1 = so.gnn(d0, d1, sdk)
        p = f"gnn.layers.{k}"
        s0, s1 = (d1, d0) if k % 2 else (d0, d1)
        r0 = d0 + so._attention_layer(d0, s0, sg64, p)
        r1 = d1 + so._attention_layer(d1, s1, sg64, p)
        assert torch.equal(y0, r0) and torch.equal(y1, r1)
        assert not torch.equal(r0, d0) and not torch.equal(r1, d1)    # the layer does change the tokens


def _Z(core, bins=-5.0):
    """Log couplings with the bin row and column appended."""
    core = torch.tensor(core, dtype=torch.float64)
    n0, n1 = core.shape
    Z = torch.full((n0 + 1, n1 + 1), bins, dtype=torch.float64)
    Z[:n0, :n1] = core
    return Z


def test_decisions_follow_superglue():
    """Same matches and scores as the oracle's superglue extraction: mutual arg-max above the threshold."""
    lt = math.log(0.2)
    Z = _Z([[-0.1, -3.0, -4.0],      # row 0 -> 0, mutual, exp(-0.1) > 0.2
            [-3.0, -2.0, -5.0],      # row 1 -> 1, mutual, exp(-2) < 0.2: no match
            [-0.5, -4.0, -6.0],      # row 2 -> 0, not mutual (row 0 wins column 0)
            [-4.0, -4.0, lt + 1]])   # row 3 -> 2, mutual, above the threshold
    m0, ms, stable = decisions(Z, 0.2, 1e-3)
    assert m0.tolist() == [0, -1, -1, 2]
    assert torch.allclose(ms, torch.tensor([math.exp(-0.1), math.exp(-2.0), 0.0, math.exp(lt + 1)], dtype=torch.float64))
    assert stable.all()


def test_decisions_flag_unstable_rows():
    """A row is unstable when its two best entries, the best two of its arg-max column, or its maximum and log(thr) are
    within 2 bar."""
    bar = 1e-3
    lt = math.log(0.2)
    Z = _Z([[-0.1, -0.1 - 1.5 * bar, -4.0, -4.0],   # row tie within 2 bar
            [-4.0, -4.0, -0.2, -4.0],                 # column 2: -0.2 against -0.2 - bar in row 2
            [-4.0, -4.0, -0.2 - bar, -3.0],           # loses column 2 by bar: may become mutual
            [-4.0, -4.0, -5.0, lt + 0.5 * bar],       # maximum at the threshold
            [-3.9, -4.0, -5.0, -5.0]])                # clear: column 0 is row 0's by 3.8, no match
    m0, _, stable = decisions(Z, 0.2, bar)
    assert stable.tolist() == [False, False, False, False, True]
    assert m0[4].item() == -1 and m0[2].item() == -1


def test_decisions_empty_sides():
    for n0, n1 in ((0, 3), (3, 0), (0, 0)):
        m0, ms, stable = decisions(torch.zeros(n0 + 1, n1 + 1, dtype=torch.float64), 0.2, 1e-3)
        assert m0.tolist() == [-1] * n0 and not ms.any() and stable.all()
