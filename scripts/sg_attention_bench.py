"""Times the fused SuperGlue softmax attention (mfr_superglue_attention, csrc/sg_attention.cu) with CUDA events at the
bf16 engine's shapes: n_img = 16 images (8 pairs), K = 1024 and K = 2048 keypoints per image, every count full, both
the self (cross 0) and the cross (cross 1) form.

  python scripts/sg_attention_bench.py [--iters N]

Algorithmic work per image: 4 heads x 2 products (Q K^T, P V) x 2 FLOP x nq x nk x 64. The achieved rate is set
against the H100 SXM data sheet's dense BF16 figure, 989 TFLOP/s (a card allowed 700 W; the card and its power limit
are printed first)."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import mfr_b200  # noqa: E402,F401
from mfr_b200 import lib as mfr  # noqa: E402

PEAK = 989e12

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=50)
args = ap.parse_args()
try:
    smi = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                  text=True).strip()
except Exception as e:
    smi = f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"
print("card:", smi, flush=True)
lib = mfr.load()
st = torch.cuda.current_stream()
for K in (1024, 2048):
    n_img = 16
    g = torch.Generator(device="cuda").manual_seed(K)
    qkv = torch.randn(n_img, K, 768, device="cuda", generator=g).bfloat16()
    counts = torch.full((n_img,), K, dtype=torch.int32, device="cuda")
    msg = torch.empty(n_img, K, 256, device="cuda", dtype=torch.bfloat16)
    flop = n_img * 4 * 2 * 2 * K * K * 64
    for cross in (0, 1):
        def launch():
            rc = lib.mfr_superglue_attention(qkv.data_ptr(), 768, counts.data_ptr(), n_img, K, cross, msg.data_ptr(), 256,
                                             st.cuda_stream)
            assert rc == 0
        for _ in range(5):
            launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(args.iters):
            launch()
        e1.record(st)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        tf = flop / (ms * 1e-3) / 1e12
        print(f"n_img {n_img}, K {K}, cross {cross}: {ms:.4f} ms, {flop / 1e9:.1f} GFLOP, {tf:.1f} TFLOP/s "
              f"({100 * tf * 1e12 / PEAK:.1f} % of the 989 TFLOP/s data-sheet BF16 peak)", flush=True)
