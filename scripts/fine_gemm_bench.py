"""Times the fine-level projection GEMMs of one LoFTR engine batch (fine.down_proj, fine.merge_feat, the q|k|v
projections of fine.0 and both directions of fine.1) at the bench's shape: 16 pairs of 720x544 frames, the bench's
dense functional weights, coarse threshold 0.2 (about 26 k matches, 25 rows per match in the fine token GEMMs).

  python scripts/fine_gemm_bench.py [--tree DIR] [--precision bf16|tf32|fp32x3] [--rounds N] [--json OUT]

The times are the per-step CUDA events of LoFTR.profile() (an eager forward with an event pair around every step). With
`--tree DIR` the library of that other checkout is loaded next to this tree's, each under its own package name, and the
two engines are profiled alternately in one process, `--rounds` times each; the medians are reported. The fused
encoder tails of the fine layers (*.tail) are listed apart: they are not projection GEMMs.
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=None, help="another checkout, profiled alternately with this one")
ap.add_argument("--precision", default="bf16", choices=["bf16", "tf32", "fp32x3"])
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--json", default=None)
args = ap.parse_args()

import torch  # noqa: E402


def load_package(tree, name):
    """The tree's package (its own libmfr_b200.so) under the module name `name`."""
    pkg = os.path.join(os.path.abspath(tree), "map-free-reloc_b200")
    spec = importlib.util.spec_from_file_location(name, os.path.join(pkg, "__init__.py"), submodule_search_locations=[pkg])
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    mod.lib.load()
    return mod


trees = [("this", HERE)] + ([("other", args.tree)] if args.tree else [])
B, HP, WP = 16, 720, 544
engines, inputs = {}, None
for i, (label, tree) in enumerate(trees):
    pkg = load_package(tree, f"mfr_tree{i}")
    loftr = importlib.import_module(f"mfr_tree{i}.loftr")
    synth = importlib.import_module(f"mfr_tree{i}.synth")
    if inputs is None:
        imgs = []
        for b in range(B):
            p = synth.make_pair(1000 + b)
            g0 = synth.rgb_to_gray_u8(p["image0"]).astype(np.float32) / 255.0
            g1 = synth.rgb_to_gray_u8(p["image1"]).astype(np.float32) / 255.0
            imgs.append((np.pad(g0, ((0, HP - g0.shape[0]), (0, WP - g0.shape[1]))),
                         np.pad(g1, ((0, HP - g1.shape[0]), (0, WP - g1.shape[1])))))
        inputs = (torch.from_numpy(np.stack([a for a, _ in imgs])).cuda(), torch.from_numpy(np.stack([b for _, b in imgs])).cuda())
    eng = loftr.LoFTR(loftr.functional_state_dict(noise=1e-3), batch=B, height=HP, width=WP, cfg={"thr": 0.2}, graph=False,
                      precision=args.precision)
    eng.forward(*inputs)
    engines[label] = (os.path.abspath(tree), eng)

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,power.draw", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print(f"{torch.cuda.get_device_name(0)} | {smi} | precision {args.precision}", flush=True)
runs = {label: [] for label in engines}
for _ in range(args.rounds):
    for label, (_, eng) in engines.items():
        runs[label].append(eng.profile(*inputs))

res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi, "precision": args.precision, "rounds": args.rounds, "trees": {}}
for label, (tree, eng) in engines.items():
    r = runs[label]
    steps = [(n, k, float(np.median([x[j][2] for x in r]))) for j, (n, k, _, _) in enumerate(r[0])]
    gemms = [(j, n, ms) for j, (n, k, ms) in enumerate(steps) if k == 1 and n.startswith("fine") and not n.endswith(".tail")]
    tails = [(j, n, ms) for j, (n, k, ms) in enumerate(steps) if k == 1 and n.startswith("fine") and n.endswith(".tail")]
    total = sum(ms for _, _, ms in steps)
    m = int(eng.device_outputs()["m_total"][0].item())
    out = {"tree": tree, "matches": m, "fine_gemm_ms": round(sum(ms for *_, ms in gemms), 3),
           "fine_tail_ms": round(sum(ms for *_, ms in tails), 3), "engine_batch_ms": round(total, 3),
           "fine_gemm_steps": [{"step": j, "name": n, "ms": round(ms, 4)} for j, n, ms in gemms]}
    res["trees"][label] = out
    print(f"[{label}] {tree}: {m} matches", flush=True)
    for j, n, ms in gemms:
        print(f"  {j:4d} {n:24s} {ms:8.3f} ms")
    print(f"  fine GEMMs {out['fine_gemm_ms']:.3f} ms, fine tails {out['fine_tail_ms']:.3f} ms, "
          f"all steps {out['engine_batch_ms']:.3f} ms per engine batch (median of {args.rounds})", flush=True)
    eng.close()
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump(res, open(args.json, "w"), indent=1)
