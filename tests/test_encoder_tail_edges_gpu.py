"""Edge cases of the fused encoder-layer tail's 128-row tiles (csrc/encoder_tail.cu; two warpgroups of 64 rows each),
against the same torch restatement and bars as tests/test_encoder_tail_gpu.py: no live row, one live row, a last tile
whose second half is empty (128k + 1 live rows) or partial (128k + 65), and fewer row tiles than SMs with an odd tile
count."""
import pytest
import torch

from test_encoder_tail_gpu import _bf, _reference

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("C,n_blocks,rows_cap,live", [(256, 2, 300, 0), (128, 2, 300, 0), (256, 1, 200, 1), (128, 3, 200, 1),
                                                     (256, 2, 128 * 5 + 40, 128 * 5 + 1), (128, 2, 128 * 5 + 40, 128 * 5 + 1),
                                                     (256, 2, 128 * 4 + 100, 128 * 4 + 65), (128, 1, 128 * 7 + 70, 128 * 7 + 65),
                                                     (256, 1, 128 * 13 - 5, None), (128, 1, 128 * 37 - 90, None)])
def test_encoder_tail_tile_edges(mfr, C, n_blocks, rows_cap, live):
    lib = mfr.load()
    g = torch.Generator().manual_seed(7 * C + rows_cap)
    rows = n_blocks * rows_cap
    msg = _bf(torch.randn(rows, C, generator=g))
    x = torch.randn(rows, C, generator=g) * 2.0
    Wm = _bf(torch.randn(C, C, generator=g) / C ** 0.5)
    W0 = _bf(torch.randn(2 * C, 2 * C, generator=g) / (2 * C) ** 0.5)
    W2 = _bf(torch.randn(C, 2 * C, generator=g) / (2 * C) ** 0.5)
    g1 = 0.75 + 0.5 * torch.rand(C, generator=g); b1 = 0.1 * torch.randn(C, generator=g)
    g2 = 0.75 + 0.5 * torch.rand(C, generator=g); b2 = 0.1 * torch.randn(C, generator=g)
    xb = _bf(x)
    ref = _reference(msg, xb, x, Wm, W0, W2, g1, b1, g2, b2)
    dev = "cuda"
    x_d = torch.zeros(rows, 2 * C, device=dev); x_d[:, :C] = x.to(dev); x_d[:, C:] = 7.0
    xb_d = torch.zeros(rows, 2 * C, dtype=torch.bfloat16, device=dev); xb_d[:, :C] = xb.to(dev).to(torch.bfloat16); xb_d[:, C:] = 3.0
    msg_d = msg.to(dev).to(torch.bfloat16).contiguous()
    w = [t.to(dev).to(torch.bfloat16).contiguous() for t in (Wm, W0, W2)]
    nrm = [t.to(dev).contiguous() for t in (g1, b1, g2, b2)]
    dyn = torch.tensor([live], dtype=torch.int32, device=dev) if live is not None else None
    mfr.check(lib.mfr_encoder_tail(mfr.ptr(msg_d), mfr.ptr(xb_d), mfr.ptr(x_d), mfr.ptr(w[0]), mfr.ptr(w[1]), mfr.ptr(w[2]),
                                   mfr.ptr(nrm[0]), mfr.ptr(nrm[1]), mfr.ptr(nrm[2]), mfr.ptr(nrm[3]), C, n_blocks, rows_cap,
                                   mfr.ptr(dyn), 1, mfr.cur_stream()))
    torch.cuda.synchronize()
    got = x_d[:, :C].cpu()
    lim = rows_cap if live is None else live
    keep = torch.zeros(rows, dtype=torch.bool)
    for b in range(n_blocks):
        keep[b * rows_cap: b * rows_cap + lim] = True
    if keep.any():
        assert torch.isfinite(got[keep]).all()
        err = (got[keep] - ref[keep]).abs()
        assert err.max().item() < 4e-2 and err.mean().item() < 1.5e-3, (err.max().item(), err.mean().item())
    assert torch.equal(got[~keep], x[~keep])                                    # dead rows: not written
    assert (x_d[:, C:] == 7.0).all() and (xb_d[:, C:].float() == 3.0).all()    # message halves untouched
    sh = xb_d[:, :C].float().cpu()
    assert torch.equal(sh[keep], _bf(got[keep]))                                # the shadow is the bf16 rounding of the new x
    assert torch.equal(sh[~keep], xb[~keep])                                    # and not written on dead rows
