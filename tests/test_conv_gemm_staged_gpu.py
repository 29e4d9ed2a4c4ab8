"""GPU checks of the conv kernel's TMA-store epilogue (the compile-time epilogue kinds): the result is written through a
shared-memory staging buffer by TMA stores whose tensor map clips ragged tiles and the channels >= Cout.

Every case runs the same op twice: once into rows whose stride allows the TMA store, once into rows whose stride is 8
bytes modulo 16, which no tensor map can address, so that the run-time generic epilogue writes them. Both apply the same arithmetic, so the bits
must be identical; the staged result is also checked against an fp64 reference, and nothing outside the output columns
may change."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENTINEL = -7.0


def _ref(x, w, pad, bias, res, act):
    Cout, RR, Cin = w.shape
    R = int(round(RR ** 0.5))
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().reshape(Cout, R, R, Cin).permute(0, 3, 1, 2), None,
                 padding=pad).permute(0, 2, 3, 1) + bias.double()
    if res is not None:
        y = y + res.double()
    if act == 1:
        y = torch.relu(y)
    elif act == 2:
        y = torch.where(y > 0, y, 0.01 * y)
    return y


def _run(mfr, xb, wb, Cin, Cout, R, bias, res, act, out_bf16, ldo):
    lib = mfr.load()
    N, H, W, Cp = xb.shape
    odt = torch.bfloat16 if out_bf16 else torch.float32
    out = torch.full((N, H, W, ldo), SENTINEL, device="cuda", dtype=odt)
    r = None
    if res is not None:   # the residual rows have the output's stride
        r = torch.zeros(N, H, W, ldo, device="cuda", dtype=odt)
        r[..., :Cout] = res
    mfr.check(lib.mfr_conv2d_nhwc_bf16(mfr.ptr(xb), N, H, W, Cin, Cp, mfr.ptr(wb), Cp, Cout, R, R, 1, R // 2,
                                       mfr.ptr(bias), mfr.ptr(r), ldo, act, 1.0, mfr.ptr(out), ldo, int(out_bf16),
                                       mfr.cur_stream()))
    torch.cuda.synchronize()
    assert (out[..., Cout:] == SENTINEL).all(), "columns beyond Cout were written"
    return out[..., :Cout]


@pytest.mark.parametrize("N,H,W,Cin,Cout,R,act,out_bf16,use_res,ldo", [
    (8, 64, 72, 64, 512, 1, 1, True, False, 512),     # BN 256 x 2 N tiles, >= 3 tiles per CTA
    (8, 61, 70, 128, 256, 3, 1, True, True, 256),     # residual reloads over >= 3 tiles per CTA, ragged tiles
    (4, 37, 45, 256, 196, 3, 1, True, True, 200),     # BN 200: narrow last box, residual
    (3, 29, 33, 64, 392, 1, 2, True, False, 400),     # BN 200 x 2 N tiles: the narrow box must not touch the next tile
    (2, 53, 1, 128, 256, 1, 0, True, False, 264),     # W = 1, one column per image, ldo > Cout
    (8, 45, 58, 256, 256, 1, 0, False, False, 256),   # fp32 output: two staging passes
    (4, 31, 27, 128, 196, 3, 0, False, False, 200),   # fp32 output, BN 200: two passes, narrow last box
    (2, 35, 29, 128, 128, 3, 0, False, False, 132),   # fp32 output, BN 128, two sub-tiles per CTA tile
])
def test_staged_epilogue_bits_and_bounds(mfr, N, H, W, Cin, Cout, R, act, out_bf16, use_res, ldo):
    g = torch.Generator(device="cpu").manual_seed(77)
    Cp = (Cin + 7) // 8 * 8
    x = torch.zeros(N, H, W, Cp); x[..., :Cin] = torch.randn(N, H, W, Cin, generator=g)
    w = torch.zeros(Cout, R * R, Cp); w[..., :Cin] = torch.randn(Cout, R * R, Cin, generator=g) / (R * R * Cin) ** 0.5
    xb, wb = x.bfloat16().cuda(), w.bfloat16().cuda()
    bias = torch.randn(Cout, generator=g).cuda()
    odt = torch.bfloat16 if out_bf16 else torch.float32
    res = torch.randn(N, H, W, Cout, generator=g).to(odt).cuda() if use_res else None
    staged = _run(mfr, xb, wb, Cin, Cout, R, bias, res, act, out_bf16, ldo)
    # rows of 8 bytes modulo 16: no tensor map, the run-time generic epilogue
    ld_generic = next(ld for ld in range(Cout + (4 if out_bf16 else 2), Cout + 64, 4 if out_bf16 else 2)
                      if ld * (2 if out_bf16 else 4) % 16 == 8)
    generic = _run(mfr, xb, wb, Cin, Cout, R, bias, res, act, out_bf16, ld_generic)
    assert torch.equal(staged.view(torch.int16) if out_bf16 else staged.view(torch.int32),
                       generic.view(torch.int16) if out_bf16 else generic.view(torch.int32))
    ref = _ref(xb[..., :Cin], wb[..., :Cin], R // 2, bias, res, act)
    err = (staged.double() - ref).abs().max().item()
    assert err <= 1e-2 * ref.abs().max().item(), err
