"""GPU checks of the conv kernel's TMA-store epilogue on token GEMMs with a device row count (the LoFTR fine-level
projections: q|k|v, merge_feat, down_proj), through mfr_token_gemm_dyn_rows.

The output tensor map only knows the capacity, so the tile that crosses the count is copied out by the store warp with
plain stores, its live rows only. Each case runs every row count twice: once into rows whose stride allows the TMA
store, once into rows whose stride is 8 bytes modulo 16, which no tensor map can address, so that the run-time generic
epilogue writes them. Both apply the same arithmetic, so the live rows must be bit-identical; they must also lie within
a dot-product bound of an fp64 reference, and every row at or past the count and every column at or past Cout must
keep the sentinel the output was filled with."""
import re

import pytest
import torch

from helpers import dot_bound

pytestmark = pytest.mark.gpu

SENTINEL = -7.0
SMS = 132
CAP = 400 * 128 + 45                      # ragged capacity: the last tile of a full count is partial too
MANY = 3 * SMS * 128 + 50                 # >= 3 tiles per CTA with one image, one partial
COUNTS = [0, 1, 127, 128, 129, CAP - 1, CAP, MANY]
KINDS = {   # name: (bf16 operands, bf16 output, K)
    "bf16_kBf": (True, True, 128),        # fine q|k|v
    "bf16_kF32": (True, False, 128),
    "tf32_kF32": (False, False, 256),     # fine merge_feat / down_proj
}


def _operands(in_bf16, n_img, K, Cout):
    g = torch.Generator(device="cpu").manual_seed(1000 * K + Cout + n_img)
    x = torch.randn(n_img, CAP, K, generator=g)
    w = torch.randn(Cout, K, generator=g) / K ** 0.5
    bias = torch.randn(Cout, generator=g).cuda()
    dt = torch.bfloat16 if in_bf16 else torch.float32
    return x.to(dt).cuda(), w.to(dt).cuda(), bias


def _launch(mfr, x, w, bias, out, count, in_bf16, out_bf16, Cout, act=0):
    n_img, cap, K = x.shape
    mfr.check(mfr.load().mfr_token_gemm_dyn_rows(mfr.ptr(x), n_img, cap, K, K, mfr.ptr(w), 0, int(in_bf16), Cout,
                                                  mfr.ptr(bias), act, mfr.ptr(out), out.shape[-1], int(out_bf16),
                                                  mfr.ptr(count), mfr.cur_stream()))


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _check_untouched(out, live, Cout):
    assert (out[:, live:] == SENTINEL).all(), "a row at or past the device row count was written"
    assert (out[:, :live, Cout:] == SENTINEL).all(), "a column at or past Cout was written"


@pytest.mark.parametrize("n_img", [1, 2])
@pytest.mark.parametrize("Cout,BN", [(128, 128), (200, 200), (256, 256)])
@pytest.mark.parametrize("kind", list(KINDS))
def test_dyn_rows_staged_epilogue(mfr, capfd, monkeypatch, kind, Cout, BN, n_img):
    in_bf16, out_bf16, K = KINDS[kind]
    x, w, bias = _operands(in_bf16, n_img, K, Cout)
    odt = torch.bfloat16 if out_bf16 else torch.float32
    # staged rows: 16-byte strides; generic rows: 8 bytes modulo 16 (no tensor map)
    ld_staged, ld_generic = (Cout + 8, Cout + 4) if out_bf16 else (Cout + 4, Cout + 2)
    ref = x.double() @ w.double().t() + bias.double()
    c_op = 2.0 ** -8 if out_bf16 else 0.0      # the bf16 rounding of the result
    if not in_bf16:
        c_op += 2.0 ** -9                        # tf32 operands (10 explicit mantissa bits each)
    bound = dot_bound(x, w, c_op, bias)
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    out_s = torch.empty(n_img, CAP, ld_staged, dtype=odt, device="cuda")
    out_g = torch.empty(n_img, CAP, ld_generic, dtype=odt, device="cuda")
    monkeypatch.setenv("MFR_CONV_DEBUG", "1")
    for live in COUNTS:
        count.fill_(live)
        out_s.fill_(SENTINEL)
        out_g.fill_(SENTINEL)
        _launch(mfr, x, w, bias, out_s, count, in_bf16, out_bf16, Cout)
        _launch(mfr, x, w, bias, out_g, count, in_bf16, out_bf16, Cout)
        torch.cuda.synchronize()
        _check_untouched(out_s, live, Cout)
        _check_untouched(out_g, live, Cout)
        s, gen = out_s[:, :live, :Cout], out_g[:, :live, :Cout]
        assert torch.equal(_bits(s), _bits(gen)), f"count {live}: staged and generic epilogues differ"
        if live:
            err = (s.double() - ref[:, :live]).abs() - bound[:, :live]
            assert err.max().item() <= 0, f"count {live}: {err.max().item()} over the fp64 bound"
    tiles = set(int(b) for b in re.findall(r"BN(\d+) nt1 ", capfd.readouterr().err))
    assert tiles == {BN}, f"expected one N tile of BN {BN}, tilings seen: {tiles}"


def test_dyn_rows_graph_replay(mfr):
    """One captured launch, the device count changed between replays."""
    x, w, bias = _operands(True, 2, 128, 256)
    count = torch.full((1,), 129, dtype=torch.int32, device="cuda")
    out = torch.full((2, CAP, 264), SENTINEL, dtype=torch.bfloat16, device="cuda")
    ref_out = torch.empty_like(out)
    _launch(mfr, x, w, bias, out, count, True, True, 256)   # module load and attributes outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _launch(mfr, x, w, bias, out, count, True, True, 256)
    for live in (129, CAP - 1, 0, MANY):
        count.fill_(live)
        out.fill_(SENTINEL)
        g.replay()
        ref_out.fill_(SENTINEL)
        _launch(mfr, x, w, bias, ref_out, count, True, True, 256)
        torch.cuda.synchronize()
        _check_untouched(out, live, 256)
        assert torch.equal(_bits(out), _bits(ref_out)), f"count {live}: the replay differs from a direct launch"
