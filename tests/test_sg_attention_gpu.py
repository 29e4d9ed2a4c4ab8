"""mfr_superglue_attention, the fused bf16 softmax attention of the SuperPoint + SuperGlue engine's bf16 mode, against
an fp64 torch softmax attention (superglue.py:85-89) on the same bf16 q, k and v.

Bar: max |error| <= 1e-2 * max|v| per (image, head), from P and the message being rounded to bf16 (2^-9 relative
each). Rows at or past the query count, and every row of an image whose partner has no keypoint, are exactly 0; every
output is finite; nothing is written past the last image."""
import pytest
import torch

pytestmark = pytest.mark.gpu

PAD = 128   # sentinel rows after the message tensor: a tile that runs past max_kp must not write them


def _lib():
    from mfr_b200 import lib
    return lib.load()


def _qkv(n_img, K, seed, q_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n_img, K, 768, generator=g)
    x[..., :256] *= q_scale
    return x.to(torch.bfloat16)


def _run(qkv, counts, cross):
    n_img, K, _ = qkv.shape
    q = qkv.cuda().contiguous()
    c = torch.tensor(counts, dtype=torch.int32, device="cuda")
    buf = torch.full((n_img * K + PAD, 256), float("nan"), dtype=torch.bfloat16, device="cuda")
    rc = _lib().mfr_superglue_attention(q.data_ptr(), 768, c.data_ptr(), n_img, K, cross, buf.data_ptr(), 256,
                                        torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0
    assert torch.isnan(buf[n_img * K:].float()).all(), "rows past the last image were written"
    return buf[:n_img * K].view(n_img, K, 256)


def _reference(qkv, counts, cross):
    q = qkv.cuda().double()
    n_img, K, _ = q.shape
    out = torch.zeros(n_img, K, 256, dtype=torch.float64, device="cuda")
    for i in range(n_img):
        s = i ^ cross
        nq, nk = counts[i], counts[s]
        if nq == 0 or nk == 0:
            continue
        for h in range(4):
            Q = q[i, :nq, 64 * h:64 * h + 64]
            Kh = q[s, :nk, 256 + 64 * h:256 + 64 * h + 64]
            V = q[s, :nk, 512 + 64 * h:512 + 64 * h + 64]
            out[i, :nq, 64 * h:64 * h + 64] = torch.softmax(Q @ Kh.T / 8.0, dim=1) @ V
    return out


def _check(qkv, counts, cross):
    got = _run(qkv, counts, cross)
    ref = _reference(qkv, counts, cross)
    g = got.double()
    assert torch.isfinite(g).all()
    worst = 0.0
    for i, nq in enumerate(counts):
        assert (got[i, nq:] == 0).all(), f"image {i}: rows past the count are not zero"
        s = i ^ cross
        if counts[s] == 0:
            assert (got[i] == 0).all(), f"image {i}: partner without keypoints must give zero messages"
            continue
        for h in range(4):
            vmax = qkv[s, :counts[s], 512 + 64 * h:576 + 64 * h].double().abs().max().item()
            err = (g[i, :nq, 64 * h:64 * h + 64] - ref[i, :nq, 64 * h:64 * h + 64]).abs().max().item() if nq else 0.0
            worst = max(worst, err / vmax)
            assert err <= 1e-2 * vmax, f"image {i} head {h}: |err| {err:.3e} > 1e-2 * {vmax:.3f}"
    print(f"max |err| / max|v| = {worst:.3e}")
    return got


CASES = [
    # K, counts (pair-interleaved), q scale
    (16, [16, 1], 1.0),
    (16, [0, 16, 15, 7], 1.0),
    (256, [0, 17, 255, 256, 1, 15], 1.0),
    (256, [200, 256, 256, 129], 12.0),         # logits up to about +-60: exercises the running-max rescaling
    (1024, [1, 15, 17, 1023, 1024, 0, 500, 129, 128, 127, 1000, 900, 64, 65, 1024, 3], 1.0),
    (1024, [1024, 1000, 777, 1024], 12.0),
    (2048, [2048, 2047, 0, 1, 17, 15, 1500, 2048, 1024, 1025, 300, 2000, 128, 2048, 999, 1], 1.0),
]


@pytest.mark.parametrize("cross", [0, 1])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_attention_matches_fp64(case, cross):
    K, counts, q_scale = CASES[case]
    qkv = _qkv(len(counts), K, seed=100 + case, q_scale=q_scale)
    if q_scale > 1.0:   # the case is meant to reach large logits
        q = qkv.double()
        s = max((q[i, :, :64] @ q[i ^ 1, :, 256:320].T).abs().max().item() for i in range(len(counts))) / 8.0
        assert s > 40.0
    _check(qkv, counts, cross)


def test_pair_independent_of_batch():
    """Pair 1 of a 4-pair batch gives the same bits alone."""
    K = 1024
    counts = [1024, 700, 513, 1000, 64, 1024, 900, 3]
    qkv = _qkv(len(counts), K, seed=7)
    full = _run(qkv, counts, 1)
    alone = _run(qkv[2:4].clone(), counts[2:4], 1)
    assert torch.equal(full[2:4].view(torch.int16), alone.view(torch.int16))


def test_rejects_bad_arguments():
    l = _lib()
    q = torch.zeros(2, 64, 768, dtype=torch.bfloat16, device="cuda")
    c = torch.zeros(2, dtype=torch.int32, device="cuda")
    m = torch.zeros(2, 64, 256, dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert l.mfr_superglue_attention(q.data_ptr(), 768, c.data_ptr(), 2, 72, 0, m.data_ptr(), 256, st) != 0   # K % 16
    assert l.mfr_superglue_attention(q.data_ptr(), 768, c.data_ptr(), 2, 4096, 0, m.data_ptr(), 256, st) != 0  # K > 2048
    assert l.mfr_superglue_attention(q.data_ptr(), 768, c.data_ptr(), 1, 64, 1, m.data_ptr(), 256, st) != 0    # odd pairs
    assert l.mfr_superglue_attention(q.data_ptr(), 512, c.data_ptr(), 2, 64, 0, m.data_ptr(), 256, st) != 0    # ldq < 768
