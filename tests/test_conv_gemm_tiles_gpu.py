"""GPU parity of the conv kernel's exact 200-column N tiles, halo mode at BN = 200 / 256 and the epilogue kinds with a
compile-time body (bf16 / fp32 output, with and without a residual), against an fp64 reference; and the same bits from
every tiling of a shape."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ref(x, w, stride, pad, bias, res, act):
    """x [N, H, W, Cin], w [Cout, R*R, Cin] (any dtype) -> fp64 NHWC reference."""
    Cout, RR, Cin = w.shape
    R = int(round(RR ** 0.5))
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().reshape(Cout, R, R, Cin).permute(0, 3, 1, 2), None,
                 stride=stride, padding=pad).permute(0, 2, 3, 1) + bias.double()
    if res is not None:
        y = y + res.double()
    if act == 1:
        y = torch.relu(y)
    elif act == 2:
        y = torch.where(y > 0, y, 0.01 * y)
    return y


def _bf16_case(mfr, N, H, W, Cin, Cout, R, act, out_bf16, use_res, ldo=None):
    """bf16 operands; the output rows have `ldo` >= Cout channels (the padding must stay untouched)."""
    lib = mfr.load()
    g = torch.Generator(device="cpu").manual_seed(2024)
    Cp = (Cin + 7) // 8 * 8
    ldo = ldo or Cout
    x = torch.zeros(N, H, W, Cp); x[..., :Cin] = torch.randn(N, H, W, Cin, generator=g)
    w = torch.zeros(Cout, R * R, Cp); w[..., :Cin] = torch.randn(Cout, R * R, Cin, generator=g) / (R * R * Cin) ** 0.5
    xb, wb = x.bfloat16().cuda(), w.bfloat16().cuda()
    pad = R // 2
    bias = torch.randn(Cout, generator=g).cuda()
    odt = torch.bfloat16 if out_bf16 else torch.float32
    res = torch.randn(N, H, W, ldo, generator=g).to(odt).cuda() if use_res else None
    out = torch.full((N, H, W, ldo), -7.0, device="cuda", dtype=odt)
    mfr.check(lib.mfr_conv2d_nhwc_bf16(mfr.ptr(xb), N, H, W, Cin, Cp, mfr.ptr(wb), Cp, Cout, R, R, 1, pad,
                                       mfr.ptr(bias), mfr.ptr(res), ldo, act, 1.0, mfr.ptr(out), ldo, int(out_bf16),
                                       mfr.cur_stream()))
    torch.cuda.synchronize()
    ref = _ref(xb[..., :Cin], wb[..., :Cin], 1, pad, bias, res[..., :Cout] if use_res else None, act)
    if ldo != Cout:
        assert (out[..., Cout:] == -7.0).all(), "channel padding of the output rows was written"
    err = (out[..., :Cout].double() - ref).abs().max().item()
    assert err <= 1e-2 * ref.abs().max().item(), err


@pytest.mark.parametrize("force", ["-1,-1,-1", "0,1,-1", "1,1,8", "1,1,16", "1,1,32"])
@pytest.mark.parametrize("N,H,W,Cin,Cout,R,act,out_bf16,use_res,ldo", [
    (2, 37, 50, 196, 196, 3, 1, True, True, 200),     # BN 200, residual, ragged tiles, 200-wide rows
    (2, 24, 32, 256, 196, 3, 0, True, False, 200),    # BN 200, no activation
    (2, 30, 41, 196, 196, 3, 2, True, False, 200),    # BN 200, leaky relu
    (2, 26, 19, 256, 256, 3, 1, True, True, None),    # BN 256, residual
    (2, 26, 19, 196, 128, 3, 0, False, False, None),  # fp32 output
    (2, 21, 33, 256, 256, 3, 0, False, True, None),   # fp32 output with a residual (run-time epilogue)
    (2, 33, 27, 128, 196, 1, 0, True, False, 200),    # 1x1, BN 200
])
def test_bf16_exact_n_and_halo(mfr, monkeypatch, force, N, H, W, Cin, Cout, R, act, out_bf16, use_res, ldo):
    """Force string: halo,MT,TW (-1 = free); a tiling the shape cannot take falls back to the free search."""
    monkeypatch.setenv("MFR_CONV_FORCE", force)
    _bf16_case(mfr, N, H, W, Cin, Cout, R, act, out_bf16, use_res, ldo)


@pytest.mark.parametrize("force", ["-1,-1,-1", "1,1,16", "0,1,-1"])
@pytest.mark.parametrize("Cin,Cout", [(196, 196), (256, 200), (256, 256)])
def test_tf32_exact_n_and_halo(mfr, monkeypatch, force, Cin, Cout):
    """tf32 operands at BN 200 / 256 in generic and halo mode."""
    monkeypatch.setenv("MFR_CONV_FORCE", force)
    lib = mfr.load()
    g = torch.Generator(device="cpu").manual_seed(11)
    N, H, W = 2, 29, 22
    x = torch.randn(N, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, 9, Cin, generator=g) / (9 * Cin) ** 0.5).cuda()
    bias = torch.randn(Cout, generator=g).cuda()
    res = torch.randn(N, H, W, Cout, generator=g).cuda()
    out = torch.full((N, H, W, Cout), float("nan"), device="cuda")
    mfr.check(lib.mfr_conv2d_nhwc_tf32(mfr.ptr(x), N, H, W, Cin, Cin, mfr.ptr(w), Cout, 3, 3, 1, 1, 0,
                                       mfr.ptr(bias), mfr.ptr(res), Cout, 1, 1.0, mfr.ptr(out), Cout, mfr.cur_stream()))
    torch.cuda.synchronize()
    ref = _ref(x, w, 1, 1, bias, res, 1)
    assert torch.isfinite(out).all()
    err = (out.double() - ref).abs().max().item()
    assert err <= 3e-3 * ref.abs().max().item(), err


@pytest.mark.parametrize("Cin,Cout", [(128, 128), (196, 128), (196, 196), (256, 256)])
def test_tiling_does_not_change_bits(mfr, monkeypatch, Cin, Cout):
    """The taps are summed in one order per shape, so per-tap and halo mode (any tile shape) give identical bits."""
    lib = mfr.load()
    g = torch.Generator(device="cpu").manual_seed(5)
    N, H, W = 2, 35, 29
    Cp = (Cin + 7) // 8 * 8
    x = torch.zeros(N, H, W, Cp); x[..., :Cin] = torch.randn(N, H, W, Cin, generator=g)
    w = torch.zeros(Cout, 9, Cp); w[..., :Cin] = torch.randn(Cout, 9, Cin, generator=g) / (9 * Cin) ** 0.5
    xb, wb = x.bfloat16().cuda(), w.bfloat16().cuda()
    bias = torch.randn(Cout, generator=g).cuda()
    outs = []
    for force in ("0,1,-1", "0,2,-1", "1,1,8", "1,1,16", "1,2,16"):
        monkeypatch.setenv("MFR_CONV_FORCE", force)
        out = torch.zeros(N, H, W, Cout, device="cuda")
        mfr.check(lib.mfr_conv2d_nhwc_bf16(mfr.ptr(xb), N, H, W, Cin, Cp, mfr.ptr(wb), Cp, Cout, 3, 3, 1, 1,
                                           mfr.ptr(bias), None, Cout, 0, 1.0, mfr.ptr(out), Cout, 0, mfr.cur_stream()))
        torch.cuda.synchronize()
        outs.append(out)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
