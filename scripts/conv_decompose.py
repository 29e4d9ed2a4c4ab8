"""Splits the time of the wgmma conv kernel (conv_gemm_kernel) into a fixed cost per CTA tile and a cost per k-block.

  python scripts/conv_decompose.py [--tree DIR] [--json OUT]

1. 1x1 convs, Cout 256, at the layer2 pixel count of the bench (32 images of 180 x 136), Cin 64 .. 1024, tiling pinned
   to TW16 TH8 MT1 (MFR_CONV_FORCE="0,1,16") so that every launch has the same tiles: the time of one wave of tiles
   over the SMs is fitted as fixed + slope * k-blocks (one k-block = 64 bf16 channels of one tap). `fixed` is the
   prologue + epilogue of a tile, `slope` the main loop's cost per k-block.
2. The 3x3 convs of the ResNet-FPN at their bench shapes: the tiling the library picks, then generic and halo
   mode pinned.
3. Per-launch times of the backbone convs from LoFTR.profile() (B = 16 pairs, bf16, the bench's dense weights).

TFLOP/s and the L2 -> shared-memory operand bytes of every launch come from the tiling the library reports
(MFR_CONV_DEBUG), computed below. `--tree` points at another checkout whose library is timed instead.
"""
import argparse
import json
import math
import os
import re
import sys
import tempfile

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--json", default=None)
ap.add_argument("--iters", type=int, default=20)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.tree))

import torch  # noqa: E402
import mfr_b200  # noqa: E402,F401
from mfr_b200 import lib as mfr  # noqa: E402

lib = mfr.load()
SMS = torch.cuda.get_device_properties(0).multi_processor_count
CFG_RE = re.compile(r"TW(\d+) TH(\d+) MT(\d+) BN(\d+) nt(\d+) halo(\d+)")


def tiling_of(fn):
    """Runs fn() once with MFR_CONV_DEBUG set and parses the tiling the library prints on stderr."""
    os.environ["MFR_CONV_DEBUG"] = "1"
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+b") as f:
        os.dup2(f.fileno(), 2)
        try:
            fn()
            torch.cuda.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["MFR_CONV_DEBUG"]
        f.seek(0)
        text = f.read().decode(errors="replace")
    m = CFG_RE.findall(text)
    if not m:
        raise RuntimeError("no tiling reported: " + text[-300:])
    tw, th, mt, bn, nt, halo = map(int, m[-1])
    return dict(TW=tw, TH=th, MT=mt, BN=bn, nt=nt, halo=halo)


def operand_bytes(t, N, Ho, Wo, Cin, R):
    """L2 -> shared-memory bytes of one launch: A boxes + B tiles of every CTA tile (a 64-channel k-block is 128 B
    per row; a channel tail of <= 16 channels moves as 32-byte rows)."""
    kb = math.ceil(Cin / 64)
    tail = Cin - (kb - 1) * 64
    kbf = (kb - 1) + (0.25 if (tail <= 16 and kb > 1) else 1.0)
    tiles = N * math.ceil(Wo / t["TW"]) * math.ceil(Ho / (t["MT"] * t["TH"])) * t["nt"]
    if t["halo"]:
        a = t["TW"] * (t["MT"] * t["TH"] + 2) * 128 * 3 * kbf
    else:
        a = t["TW"] * t["TH"] * t["MT"] * 128 * R * R * kbf
    b = t["BN"] * 128 * R * R * kbf
    return tiles, tiles * (a + b)


def conv_case(N, H, W, Cin, Cout, R, stride, force=None, iters=20):
    Cp, Co = (Cin + 7) // 8 * 8, (Cout + 7) // 8 * 8
    pad = R // 2
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    x = torch.randn(N, H, W, Cp, device="cuda").bfloat16()
    w = (torch.randn(Cout, R * R, Cp, device="cuda") / (R * R * Cin) ** 0.5).bfloat16()
    bias = torch.randn(Cout, device="cuda")
    out = torch.empty(N, Ho, Wo, Co, device="cuda", dtype=torch.bfloat16)
    if force:
        os.environ["MFR_CONV_FORCE"] = force

    def run():
        mfr.check(lib.mfr_conv2d_nhwc_bf16(mfr.ptr(x), N, H, W, Cin, Cp, mfr.ptr(w), Cp, Cout, R, R, stride, pad,
                                           mfr.ptr(bias), None, Co, 1, 1.0, mfr.ptr(out), Co, 1, mfr.cur_stream()))
    try:
        t = tiling_of(run)
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            run()
        e1.record()
        torch.cuda.synchronize()
    finally:
        os.environ.pop("MFR_CONV_FORCE", None)
    ms = e0.elapsed_time(e1) / iters
    flops = 2.0 * N * Ho * Wo * Cout * Cin * R * R
    tiles, nbytes = operand_bytes(t, N, Ho, Wo, Cin, R)
    waves = math.ceil(tiles / SMS)
    return dict(shape=[N, H, W, Cin, Cout, R, stride], tiling=t, ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1),
                tiles=tiles, waves=waves, us_per_wave=round(ms * 1e3 / waves, 3), operand_gb=round(nbytes / 1e9, 3),
                operand_tb_s=round(nbytes / ms / 1e9, 2), kblocks=R * R * math.ceil(Cin / 64))


res = {"device": torch.cuda.get_device_name(0), "sms": SMS}
print(res["device"], SMS, "SMs", flush=True)

# 1. fixed + slope fit, 1x1 convs with a pinned tiling
fit_rows = []
for cin in (64, 128, 256, 512, 1024):
    r = conv_case(32, 180, 136, cin, 256, 1, 1, force="0,1,16", iters=args.iters)
    fit_rows.append(r)
    print(f"1x1 Cin {cin:5d} Cout 256: {r['ms']:.3f} ms  {r['tflops']:6.1f} TF/s  tiling {r['tiling']}  waves {r['waves']}  "
          f"{r['us_per_wave']:.2f} us/wave  {r['operand_tb_s']:.2f} TB/s operands", flush=True)
kb = np.array([r["kblocks"] for r in fit_rows], np.float64)
tw = np.array([r["us_per_wave"] for r in fit_rows], np.float64)
slope, fixed = np.polyfit(kb, tw, 1)
res["fit_1x1"] = {"rows": fit_rows, "fixed_us_per_tile": round(float(fixed), 3), "us_per_kblock": round(float(slope), 4),
                  "note": "time of one wave of TW16 TH8 MT1 BN256 tiles = fixed + slope * k-blocks (64 bf16 channels)"}
print(f"fit: {fixed:.3f} us fixed per tile + {slope:.4f} us per k-block (BN 256, 128 pixels)", flush=True)

# 2. the 3x3 convs at bench shapes (32 images), free tiling
res["conv3x3"] = []
for (H, W, Cin, Cout) in ((360, 272, 128, 128), (360, 272, 196, 196), (360, 272, 196, 128), (180, 136, 196, 196),
                          (180, 136, 256, 256), (180, 136, 256, 196), (90, 68, 256, 256)):
    for force in (None, "0,-1,-1", "1,-1,-1"):   # the library's choice, then generic and halo mode pinned
        r = conv_case(32, H, W, Cin, Cout, 3, 1, force=force, iters=max(5, args.iters // 2))
        r["force"] = force
        res["conv3x3"].append(r)
        print(f"3x3 {H}x{W} {Cin}->{Cout} force {str(force):9s}: {r['ms']:.3f} ms  {r['tflops']:6.1f} TF/s  tiling {r['tiling']}  "
              f"{r['operand_gb']:.2f} GB operands ({r['operand_tb_s']:.2f} TB/s)", flush=True)

# 3. the backbone launches of the bench engine
from mfr_b200 import loftr, synth  # noqa: E402

B, HP, WP = 16, 720, 544
sd = loftr.functional_state_dict(noise=1e-3)
eng = loftr.LoFTR(sd, batch=B, height=HP, width=WP, cfg={"thr": 0.2}, graph=False, precision="bf16")
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
prof = [(n, k, float(np.median([r[j][2] for r in runs])), f) for j, (n, k, _, f) in enumerate(runs[0])]
bb = [p for p in prof if p[1] == 1 and p[0].startswith("layer")]
res["backbone"] = [{"name": n, "ms": round(ms, 4), "tflops": round(f / ms / 1e9, 1)} for n, _, ms, f in bb]
bb_ms, bb_fl = sum(p[2] for p in bb), sum(p[3] for p in bb)
res["backbone_ms"] = round(bb_ms, 3)
res["backbone_tflops"] = round(bb_fl / bb_ms / 1e9, 1)
res["step_ms"] = round(sum(p[2] for p in prof), 3)
for r in res["backbone"]:
    print(f"  {r['name']:22s} {r['ms']:8.3f} ms {r['tflops']:7.1f} TF/s")
print(f"backbone convs {bb_ms:.2f} ms ({bb_fl / 1e12:.2f} TFLOP, {res['backbone_tflops']} TF/s) of {res['step_ms']:.2f} ms "
      f"profiled per engine batch", flush=True)
eng.close()
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump(res, open(args.json, "w"), indent=1)
