"""Cost of the CONFIDENCE escalation on the device (PoseBackend(..., confidence=...), from_cfg(..., escalate=True))
against the fixed first budget. One process, one GPU.

  python scripts/ransac_escalation_bench.py        # B=16 ITERS=50 ROUNDS=3 SECONDS=1

backend: E-mat metric (first budget 2048) and PnP (1024), confidence 0.9999, cap 32768, B pairs of N = 2000
  synth.make_correspondences per batch: every pair at inlier ratio r in {0.8, 0.5, 0.3, 0.2, 0.1}, and one mixed batch
  (the five ratios in turn). Fixed and escalating calls alternate ROUNDS times; each timed window is ITERS calls after
  warm-up between CUDA events (closed after a device synchronise); the median ms per call is reported with the
  histogram of the budgets the pairs stopped at. In the r = 0.8 batch no pair escalates: the difference there is the
  cost of the later rounds' launches whose blocks all exit at once.
stream: pairs/s of pipeline.from_cfg(cfg, B, escalate=False / True) for sift_emat_dptkitti and sift_pnp_dptkitti on a
  synthetic 540x720 scene (method_stream_bench's paired arm). The solver stream overlaps the next matcher batch, so
  escalation shows in pairs/s only once a batch's solve outgrows the matcher.
The card, its power limit and its clocks are printed first."""
import collections
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import method_stream_bench as msb  # noqa: E402
import mfr_b200  # noqa: E402,F401
from mfr_b200 import pose_solver, synth  # noqa: E402
from mfr_b200.pipeline import from_cfg  # noqa: E402

B = msb.B
ITERS = int(os.environ.get("ITERS", 50))
ROUNDS = int(os.environ.get("ROUNDS", 3))
N, CONF, CAP = 2000, 0.9999, 32768
RATIOS = (0.8, 0.5, 0.3, 0.2, 0.1)


def batch(ratios, seed):
    sets = [synth.make_correspondences(seed + i, n=N, inlier_ratio=r) for i, r in enumerate(ratios)]
    cat = lambda k: torch.from_numpy(np.concatenate([s[k] for s in sets])).cuda().contiguous()
    stack = lambda k: torch.from_numpy(np.stack([np.asarray(s[k], np.float32) for s in sets])).cuda().contiguous()
    off = torch.arange(0, N * (len(sets) + 1), N, dtype=torch.int32, device="cuda")
    return cat("kpts0"), cat("kpts1"), off, stack("K_color0"), stack("K_color1"), stack("depth0"), stack("depth1")


def ms_per_call(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(ITERS):
        fn()
    torch.cuda.synchronize()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / ITERS


def backend_level():
    be = pose_solver.PoseBackend(max_pairs=B, max_pts=N, max_hyp=CAP)
    budgets = torch.zeros(B, dtype=torch.int32, device="cuda")
    batches = {f"r={r}": batch([r] * B, 1000 + 100 * i) for i, r in enumerate(RATIOS)}
    batches["mixed"] = batch([RATIOS[i % len(RATIOS)] for i in range(B)], 2000)
    out = {}
    for name, (k0, k1, off, K0, K1, d0, d1) in batches.items():
        solvers = {
            "emat_metric": lambda **kw: be.emat_metric(k0, k1, off, K0, K1, d0, d1, 2.0, 0.1, 2048, lo=pose_solver.LO_LSQ, **kw),
            "pnp": lambda **kw: be.pnp(k0, k1, off, K0, K1, d0, 3.0, 1024, **kw)}
        for solver, call in solvers.items():
            variants = {"fixed": lambda: call(), "escalate": lambda: call(confidence=CONF, max_hyp=CAP, budgets=budgets)}
            for fn in variants.values():     # warm-up
                fn()
            times = {v: [] for v in variants}
            for _ in range(ROUNDS):
                for v, fn in variants.items():
                    times[v].append(ms_per_call(fn))
            hist = dict(sorted(collections.Counter(budgets.tolist()).items()))
            r = {v: float(np.median(t)) for v, t in times.items()}
            r.update(rounds=times, budgets=hist, ratio=r["escalate"] / r["fixed"])
            out[f"{solver} {name}"] = r
            print(f"{solver:12s} {name:8s} fixed {r['fixed']:8.3f} ms  escalate {r['escalate']:8.3f} ms  "
                  f"x{r['ratio']:.2f}  budgets {hist}", flush=True)
    be.close()
    return out


def stream_level():
    H, W = msb.H, msb.W
    scene = synth.make_scene(7, B, h=H, w=W)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    g0 = dev(synth.rgb_to_gray_u8(scene["image0"]))
    g1 = dev(np.stack([synth.rgb_to_gray_u8(q["image1"]) for q in scene["queries"]]))
    d0, K0 = dev(scene["depth0"]), dev(scene["K_color0"])
    d1 = dev(np.stack([q["depth1"] for q in scene["queries"]]))
    K1 = dev(np.stack([q["K_color1"] for q in scene["queries"]]))
    G0, D0, KK0 = (x[None].expand(B, *x.shape).contiguous() for x in (g0, d0, K0))
    out = {}
    for name in ("sift_emat_dptkitti", "sift_pnp_dptkitti"):
        pipes = {e: from_cfg(msb.method_cfg(name), B, escalate=e) for e in (False, True)}
        rates = {e: [] for e in pipes}
        for _ in range(ROUNDS):
            for e, pipe in pipes.items():
                pipe.reset()
                rates[e].append(msb.timed(lambda: pipe.submit_device(G0, g1, D0, d1, KK0, K1)))
        for pipe in pipes.values():
            pipe.reset()
            pipe.eng.close(); pipe.be.close()
        r = {"fixed_pairs_s": float(np.median(rates[False])), "escalate_pairs_s": float(np.median(rates[True])),
             "rounds": {str(e): v for e, v in rates.items()}}
        out[name] = r
        print(f"{name:20s} fixed {r['fixed_pairs_s']:8.1f} pairs/s  escalate {r['escalate_pairs_s']:8.1f} pairs/s", flush=True)
        torch.cuda.empty_cache()
    return out


def main():
    print("card (name, power limit, SM clock, max SM clock):", msb.card(), flush=True)
    res = {"card": msb.card(), "batch": B, "backend": backend_level(), "stream": stream_level()}
    out = os.environ.get("OUT")
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
