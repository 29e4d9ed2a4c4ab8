"""Times the fused encoder-layer tail (mfr_encoder_tail, csrc/encoder_tail.cu) at the shapes of the bench's engine batch
(16 pairs, 720x544 frames, 60x45 = 2700 coarse tokens per image) and sets each against its floor on the H100.

  python scripts/tail_bench.py [--tree DIR] [--iters N] [--json OUT]

Shapes: C = 256 over 1 x 195 840 rows (a self layer: 72 images x 2720 rows of the token buffer) and 1 x 97 920 (one side
of a cross layer); C = 128 over 2 blocks and 1 block of rows_cap = 25 x 97 920 with 25 x 26 000 live rows (the fine
level with 26 k matches). The floor of a launch is the larger of FLOP / 989 TFLOP/s and HBM bytes / 3.35 TB/s (the
H100 SXM data sheet: dense bf16, HBM3). FLOP per row are 14 C^2 (merge C x C, mlp.0 2C x 2C, mlp.2 C x 2C); HBM bytes
per row are the bf16 message and x shadow read (4 C), the fp32 x read and written (8 C) and the shadow written (2 C).
Then the *.tail steps of LoFTR.profile() are summed for one engine batch (B = 16, bf16, the bench's weights).
`--tree` times another checkout's library instead.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--json", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.tree))

import torch  # noqa: E402
import mfr_b200  # noqa: E402,F401
from mfr_b200 import lib as mfr  # noqa: E402

PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
lib = mfr.load()


def tail_case(C, n_blocks, rows_cap, live, iters):
    g = torch.Generator(device="cuda").manual_seed(C)
    rows = n_blocks * rows_cap
    msg = torch.randn(rows, C, device="cuda", generator=g).bfloat16()
    x = torch.randn(rows, 2 * C, device="cuda", generator=g)
    xb = x.bfloat16()
    w = [(torch.randn(o, i, device="cuda", generator=g) / i ** 0.5).bfloat16() for o, i in ((C, C), (2 * C, 2 * C), (C, 2 * C))]
    nrm = [torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")]
    dyn = torch.tensor([live], dtype=torch.int32, device="cuda") if live is not None else None

    def run(n):
        mfr.check(lib.mfr_encoder_tail(mfr.ptr(msg), mfr.ptr(xb), mfr.ptr(x), mfr.ptr(w[0]), mfr.ptr(w[1]), mfr.ptr(w[2]),
                                       mfr.ptr(nrm[0]), mfr.ptr(nrm[1]), mfr.ptr(nrm[2]), mfr.ptr(nrm[3]), C, n_blocks, rows_cap,
                                       mfr.ptr(dyn), n, mfr.cur_stream()))
    run(3)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run(iters)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    n = n_blocks * (rows_cap if live is None else live)
    flops, nbytes = 14.0 * C * C * n, 14.0 * C * n
    t_f, t_b = flops / PEAK_FLOPS * 1e3, nbytes / PEAK_BW * 1e3
    return dict(C=C, n_blocks=n_blocks, rows_cap=rows_cap, live=live, ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1),
                gb_s=round(nbytes / ms / 1e6, 1), floor_ms=round(max(t_f, t_b), 4), floor_bound="tensor" if t_f > t_b else "HBM")


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
res = {"tree": os.path.abspath(args.tree), "device": torch.cuda.get_device_name(0), "nvidia_smi": smi, "shapes": []}
print(f"{res['tree']}\n{smi}", flush=True)
for C, nb, cap, live in ((256, 1, 195840, None), (256, 1, 97920, None), (128, 2, 25 * 97920, 25 * 26000),
                         (128, 1, 25 * 97920, 25 * 26000)):
    r = tail_case(C, nb, cap, live, args.iters)
    res["shapes"].append(r)
    print(f"C {C} {nb} x {cap} rows (live {live}): {r['ms']:.3f} ms  {r['tflops']:6.1f} TFLOP/s  {r['gb_s']:7.1f} GB/s  "
          f"floor {r['floor_ms']:.3f} ms ({r['floor_bound']})", flush=True)
    torch.cuda.empty_cache()

from mfr_b200 import loftr, synth  # noqa: E402

B, HP, WP = 16, 720, 544
eng = loftr.LoFTR(loftr.functional_state_dict(noise=1e-3), batch=B, height=HP, width=WP, cfg={"thr": 0.2}, graph=False,
                  precision="bf16")
imgs = []
for i in range(B):
    p = synth.make_pair(1000 + i)
    g0 = synth.rgb_to_gray_u8(p["image0"]).astype(np.float32) / 255.0
    g1 = synth.rgb_to_gray_u8(p["image1"]).astype(np.float32) / 255.0
    imgs.append((np.pad(g0, ((0, HP - g0.shape[0]), (0, WP - g0.shape[1]))), np.pad(g1, ((0, HP - g1.shape[0]), (0, WP - g1.shape[1])))))
i0 = torch.from_numpy(np.stack([a for a, _ in imgs])).cuda()
i1 = torch.from_numpy(np.stack([b for _, b in imgs])).cuda()
eng.forward(i0, i1)
runs = [eng.profile(i0, i1) for _ in range(3)]
prof = [(n, float(np.median([r[j][2] for r in runs]))) for j, (n, _, _, _) in enumerate(runs[0])]
tails = [(n, ms) for n, ms in prof if n.endswith(".tail")]
res["engine_tail_steps"] = [{"name": n, "ms": round(ms, 4)} for n, ms in tails]
res["engine_tail_ms"] = round(sum(ms for _, ms in tails), 3)
res["engine_step_ms"] = round(sum(ms for _, ms in prof), 3)
for n, ms in tails:
    print(f"  {n:24s} {ms:8.3f} ms")
print(f"{len(tails)} tail steps: {res['engine_tail_ms']:.2f} ms of {res['engine_step_ms']:.2f} ms profiled per engine batch",
      flush=True)
eng.close()
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump(res, open(args.json, "w"), indent=1)
