"""GPU parity of the wgmma implicit-GEMM conv kernel against plain PyTorch fp32 (cuDNN/cuBLAS
with TF32 disabled). TF32 inputs => tolerance 3e-3 of the output range (stated here)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 3e-3


def _run(mfr, x_nhwc, w, stride, pad, bias=None, residual=None, act=0, alpha=1.0, batched=False):
    lib = mfr.load()
    N, H, W, Cin = x_nhwc.shape
    if batched:
        Cout, R, S = w.shape[1], 1, 1
    else:
        Cout, R, S = w.shape[0], w.shape[1], w.shape[2]
    Ho = (H + 2 * pad - R) // stride + 1
    Wo = (W + 2 * pad - S) // stride + 1
    out = torch.full((N, Ho, Wo, Cout), float("nan"), device="cuda", dtype=torch.float32)
    rc = lib.mfr_conv2d_nhwc_tf32(
        mfr.ptr(x_nhwc), N, H, W, Cin, Cin, mfr.ptr(w), Cout, R, S, stride, pad, int(batched),
        mfr.ptr(bias), mfr.ptr(residual), Cout, act, alpha, mfr.ptr(out), Cout, mfr.cur_stream())
    mfr.check(rc)
    torch.cuda.synchronize()
    return out


def _ref(x_nhwc, w, stride, pad, bias=None, residual=None, act=0, alpha=1.0):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x = x_nhwc.permute(0, 3, 1, 2).double()
    wt = w.permute(0, 3, 1, 2).double()  # [Cout][R][S][Cin] -> [Cout][Cin][R][S]
    y = F.conv2d(x, wt, None, stride=stride, padding=pad) * alpha
    y = y.permute(0, 2, 3, 1)
    if bias is not None:
        y = y + bias.double()
    if residual is not None:
        y = y + residual.double()
    if act == 1:
        y = torch.relu(y)
    elif act == 2:
        y = F.leaky_relu(y, 0.01)
    elif act == 3:
        y = F.elu(y) + 1
    return y.float()


def _check(out, ref):
    assert torch.isfinite(out).all(), "non-finite / unwritten outputs"
    scale = ref.abs().max().item()
    err = (out - ref).abs().max().item()
    assert err <= TOL * scale, f"max err {err} vs scale {scale}"


@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,act,use_bias,use_res", [
    (1, 1, 300, 256, 256, 1, 1, 0, False, False),     # plain linear layer
    (1, 1, 300, 512, 512, 1, 1, 1, False, False),     # two N tiles
    (2, 40, 36, 128, 128, 3, 1, 1, True, True),       # residual block conv
    (2, 40, 36, 128, 196, 3, 2, 1, True, False),      # stride-2 conv, odd Cout
    (2, 23, 17, 196, 256, 3, 2, 2, True, False),      # channel tail (196 = 6*32+4), ragged tiles
    (2, 40, 36, 128, 196, 1, 2, 0, True, False),      # 1x1 stride-2 shortcut
    (1, 45, 34, 196, 196, 3, 1, 3, False, False),     # elu+1 epilogue
    (2, 90, 68, 256, 256, 3, 1, 0, False, False),     # coarse-level size
])
def test_conv_matches_torch(mfr, N, H, W, Cin, Cout, R, stride, act, use_bias, use_res):
    g = torch.Generator(device="cpu").manual_seed(1234)
    x = torch.randn(N, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, R, R, Cin, generator=g) / (R * R * Cin) ** 0.5).cuda()
    pad = R // 2
    Ho = (H + 2 * pad - R) // stride + 1
    Wo = (W + 2 * pad - R) // stride + 1
    bias = torch.randn(Cout, generator=g).cuda() if use_bias else None
    res = torch.randn(N, Ho, Wo, Cout, generator=g).cuda() if use_res else None
    out = _run(mfr, x, w, stride, pad, bias, res, act, 0.5)
    ref = _ref(x, w, stride, pad, bias, res, act, 0.5)
    _check(out, ref)


@pytest.mark.parametrize("force", ["0,1,-1", "1,1,8", "1,1,16", "1,2,8,0", "1,2,16,0", "1,2,32,0", "0,2,-1", "1,1,128",
                                   "1,2,8,1", "1,2,16,1", "1,2,32,1", "1,1,16,0,1", "1,2,16,0,1", "1,1,8,0,1"])
@pytest.mark.parametrize("N,H,W,Cin,Cout,use_res", [
    (2, 70, 52, 128, 128, True),      # ragged in x and y for every tile shape
    (1, 37, 50, 196, 196, False),     # BN = 208 (MT stays 1), channel tail in K
    (2, 33, 24, 64, 64, True),        # narrow N
])
def test_conv3x3_tilings_agree(mfr, monkeypatch, force, N, H, W, Cin, Cout, use_res):
    """Every tiling of the 3x3 stride-1 path (per-tap A loads vs halo A box shared by the three ky taps,
    one or two 128-pixel sub-tiles per CTA, tile widths) against the fp64 reference. Force string: halo,MT,TW
    (fields after the third are ignored); shapes a mode cannot take fall back to the free search."""
    monkeypatch.setenv("MFR_CONV_FORCE", force)
    g = torch.Generator(device="cpu").manual_seed(4321)
    x = torch.randn(N, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5).cuda()
    bias = torch.randn(Cout, generator=g).cuda()
    res = torch.randn(N, H, W, Cout, generator=g).cuda() if use_res else None
    out = _run(mfr, x, w, 1, 1, bias, res, 1, 1.0)
    _check(out, _ref(x, w, 1, 1, bias, res, 1, 1.0))


@pytest.mark.parametrize("force", ["0,1,-1", "0,2,-1"])
def test_conv1x1_and_stride2_two_subtiles(mfr, monkeypatch, force):
    monkeypatch.setenv("MFR_CONV_FORCE", force)
    g = torch.Generator(device="cpu").manual_seed(5)
    for (N, H, W, Cin, Cout, R, stride) in [(2, 64, 40, 128, 64, 1, 1), (2, 50, 48, 128, 128, 3, 2), (2, 50, 48, 96, 128, 1, 2)]:
        x = torch.randn(N, H, W, Cin, generator=g).cuda()
        w = (torch.randn(Cout, R, R, Cin, generator=g) / (R * R * Cin) ** 0.5).cuda()
        out = _run(mfr, x, w, stride, R // 2, None, None, 0, 1.0)
        _check(out, _ref(x, w, stride, R // 2, None, None, 0, 1.0))


@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,act,use_res", [
    (2, 48, 64, 128, 128, 3, 1, 1, True), (2, 48, 64, 128, 196, 3, 2, 1, False), (2, 48, 64, 128, 196, 1, 2, 0, False),
    (2, 24, 32, 196, 196, 3, 1, 1, True), (2, 24, 32, 196, 256, 3, 2, 1, False), (2, 24, 32, 196, 256, 1, 2, 0, False),
    (2, 12, 16, 256, 256, 3, 1, 1, True), (2, 12, 16, 256, 256, 1, 1, 0, False), (2, 24, 32, 196, 256, 1, 1, 0, False),
    (2, 24, 32, 256, 256, 3, 1, 2, False), (2, 24, 32, 256, 196, 3, 1, 0, False), (2, 48, 64, 128, 196, 1, 1, 0, False),
    (2, 48, 64, 196, 196, 3, 1, 2, False), (2, 48, 64, 196, 128, 3, 1, 0, False),
    (4, 80, 60, 128, 128, 3, 1, 1, True), (4, 80, 60, 196, 128, 3, 1, 0, False), (4, 40, 30, 256, 196, 3, 1, 0, False),
])
def test_backbone_shapes_small_images(mfr, N, H, W, Cin, Cout, R, stride, act, use_res):
    """The ResNet-FPN conv shapes at the image sizes the engine tests use (few tiles, narrow N tiles)."""
    g = torch.Generator(device="cpu").manual_seed(77)
    x = torch.randn(N, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, R, R, Cin, generator=g) / (R * R * Cin) ** 0.5).cuda()
    pad = R // 2
    Ho = (H + 2 * pad - R) // stride + 1
    Wo = (W + 2 * pad - R) // stride + 1
    bias = torch.randn(Cout, generator=g).cuda()
    res = torch.randn(N, Ho, Wo, Cout, generator=g).cuda() if use_res else None
    out = _run(mfr, x, w, stride, pad, bias, res, act, 1.0)
    _check(out, _ref(x, w, stride, pad, bias, res, act, 1.0))


def test_batched_xyt(mfr):
    g = torch.Generator(device="cpu").manual_seed(7)
    a = torch.randn(2, 1, 300, 256, generator=g).cuda()
    b = torch.randn(2, 500, 256, generator=g).cuda()
    out = _run(mfr, a, b, 1, 0, alpha=1.0 / 25.6, batched=True)
    ref = torch.einsum("nlc,nsc->nls", a[:, 0].double(), b.double()).float() / 25.6
    _check(out[:, 0], ref)


@pytest.mark.parametrize("force", ["-1,-1,-1,0", "1,2,16,1", "1,2,16,0,1", "1,1,-1,0,1"])
def test_bf16_conv_swapped_operands(mfr, monkeypatch, force):
    """bf16 residual block conv (layer1 shape class) under several forced tilings (halo,MT,TW; further fields ignored)."""
    monkeypatch.setenv("MFR_CONV_FORCE", force)
    _bf16_conv_case(mfr, 2, 72, 48, 128, 128, 3, 1, True, True)
    _bf16_conv_case(mfr, 2, 40, 36, 196, 128, 3, 1, False, False)


@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,out_bf16,use_res", [
    (2, 40, 36, 128, 128, 3, 1, True, True),
    (2, 40, 36, 128, 196, 3, 2, True, False),
    (2, 23, 17, 196, 256, 3, 1, False, False),     # Cin 196 padded to 200 in memory (16-byte strides)
    (1, 1, 300, 256, 256, 1, 1, False, False),
])
def test_bf16_conv_matches_torch(mfr, N, H, W, Cin, Cout, R, stride, out_bf16, use_res):
    _bf16_conv_case(mfr, N, H, W, Cin, Cout, R, stride, out_bf16, use_res)


def _bf16_conv_case(mfr, N, H, W, Cin, Cout, R, stride, out_bf16, use_res):
    """bf16 operands / fp32 accumulate vs an fp64 reference on the same bf16-rounded inputs
    (tolerance 1e-2 of the output range covers the bf16 rounding of the output itself)."""
    lib = mfr.load()
    g = torch.Generator(device="cpu").manual_seed(99)
    Cp = (Cin + 7) // 8 * 8
    x = torch.zeros(N, H, W, Cp); x[..., :Cin] = torch.randn(N, H, W, Cin, generator=g)
    w = torch.zeros(Cout, R * R, Cp); w[..., :Cin] = torch.randn(Cout, R * R, Cin, generator=g) / (R * R * Cin) ** 0.5
    xb, wb = x.bfloat16().cuda(), w.bfloat16().cuda()
    pad = R // 2
    Ho = (H + 2 * pad - R) // stride + 1; Wo = (W + 2 * pad - R) // stride + 1
    bias = torch.randn(Cout, generator=g).cuda()
    res = torch.randn(N, Ho, Wo, Cout, generator=g).bfloat16().cuda() if use_res else None
    out = torch.zeros(N, Ho, Wo, Cout, device="cuda", dtype=torch.bfloat16 if out_bf16 else torch.float32)
    mfr.check(lib.mfr_conv2d_nhwc_bf16(mfr.ptr(xb), N, H, W, Cin, Cp, mfr.ptr(wb), Cp, Cout, R, R, stride, pad,
                                       mfr.ptr(bias), mfr.ptr(res), Cout, 1, 1.0, mfr.ptr(out), Cout, int(out_bf16),
                                       mfr.cur_stream()))
    torch.cuda.synchronize()
    xr = xb[..., :Cin].double().permute(0, 3, 1, 2)
    wr = wb[..., :Cin].double().reshape(Cout, R, R, Cin).permute(0, 3, 1, 2)
    ref = F.conv2d(xr, wr, None, stride=stride, padding=pad).permute(0, 2, 3, 1) + bias.double()
    if use_res:
        ref = ref + res.double()
    ref = torch.relu(ref)
    err = (out.double() - ref).abs().max().item()
    assert err <= 1e-2 * ref.abs().max().item(), err


@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,act", [
    (2, 40, 36, 196, 196, 3, 1, 2),      # BN = 256 for 196 channels: the columns past Cout are not stored
    (2, 37, 50, 128, 196, 1, 1, 0),      # 1x1, ragged tiles
    (2, 40, 36, 128, 196, 3, 2, 1),      # stride 2
    (1, 1, 777, 256, 768, 1, 1, 3),      # token GEMM (q|k|v shape): three N tiles, elu+1
    (1, 1, 300, 128, 384, 1, 1, 3),
])
def test_bf16_tma_store_epilogue(mfr, N, H, W, Cin, Cout, R, stride, act):
    """bf16 outputs without a residual (the register epilogue's packed bf16x2 stores): two launches of the same op give
    identical bits, the channel padding of the output rows (stride 200 for 196 channels) stays untouched, and the
    result matches an fp64 reference."""
    lib = mfr.load()
    g = torch.Generator(device="cpu").manual_seed(123)
    Cp, Co = (Cin + 7) // 8 * 8, (Cout + 7) // 8 * 8
    x = torch.zeros(N, H, W, Cp); x[..., :Cin] = torch.randn(N, H, W, Cin, generator=g)
    w = torch.zeros(Cout, R * R, Cp); w[..., :Cin] = torch.randn(Cout, R * R, Cin, generator=g) / (R * R * Cin) ** 0.5
    xb, wb = x.bfloat16().cuda(), w.bfloat16().cuda()
    pad = R // 2
    Ho = (H + 2 * pad - R) // stride + 1; Wo = (W + 2 * pad - R) // stride + 1
    bias = torch.randn(Cout, generator=g).cuda()
    outs = []
    for _ in range(2):
        out = torch.full((N, Ho, Wo, Co), -7.0, device="cuda", dtype=torch.bfloat16)
        mfr.check(lib.mfr_conv2d_nhwc_bf16(mfr.ptr(xb), N, H, W, Cin, Cp, mfr.ptr(wb), Cp, Cout, R, R, stride, pad,
                                           mfr.ptr(bias), None, Co, act, 1.0, mfr.ptr(out), Co, 1, mfr.cur_stream()))
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0][..., :Cout], outs[1][..., :Cout])
    if Co != Cout:   # the row's own channel padding
        assert (outs[0][..., Cout:] == -7.0).all() and (outs[1][..., Cout:] == -7.0).all()
    xr = xb[..., :Cin].double().permute(0, 3, 1, 2)
    wr = wb[..., :Cin].double().reshape(Cout, R, R, Cin).permute(0, 3, 1, 2)
    ref = F.conv2d(xr, wr, None, stride=stride, padding=pad).permute(0, 2, 3, 1) + bias.double()
    if act == 1: ref = torch.relu(ref)
    elif act == 2: ref = torch.where(ref > 0, ref, 0.01 * ref)
    elif act == 3: ref = torch.where(ref > 0, ref + 1, torch.exp(ref))
    err = (outs[0][..., :Cout].double() - ref).abs().max().item()
    assert err <= 1e-2 * ref.abs().max().item(), err
