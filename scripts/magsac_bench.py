"""MAGSAC++ against MSAC scoring of the E-mat stage (PoseBackend.emat(..., scoring="magsac") / the default lo = LO_LSQ
MSAC path), and both against cv2.findEssentialMat(USAC_MAGSAC). One process, one GPU.

  OUT=magsac_bench.json python scripts/magsac_bench.py        # ITERS=20 ROUNDS=3

B = 16 pairs of synth.make_correspondences (0.5 px noise) per cell, N in {1000, 2000, 6000} x inlier ratio in
{20, 50, 80} %, threshold 2 px, one fixed budget of 2048 hypotheses (the stream's default). Time: the two modes alternate
ROUNDS times in one process; each timed window is ITERS calls after a warm-up, between CUDA events closed after a
device synchronise; the median ms per batch is reported. Accuracy: median rotation error and t-direction error against
the synthetic ground truth of the 16 pairs, for MSAC, MAGSAC++ and cv2 (the reference's call, confidence 0.9999). The
card's name and power limit are read in the same run. Prints one JSON document (and writes it to OUT if set)."""
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
from oracle import pose_solver_oracle as po  # noqa: E402

B, NUM_HYP, PIX_THR, CONF = 16, 2048, 2.0, 0.9999
ITERS = int(os.environ.get("ITERS", 20))
ROUNDS = int(os.environ.get("ROUNDS", 3))
NS, RATIOS = (1000, 2000, 6000), (0.2, 0.5, 0.8)


def batch(sets):
    cat = lambda k: torch.from_numpy(np.concatenate([s[k] for s in sets])).cuda().contiguous()
    stack = lambda k: torch.from_numpy(np.stack([np.asarray(s[k], np.float32) for s in sets])).cuda().contiguous()
    off = torch.tensor(np.cumsum([0] + [len(s["kpts0"]) for s in sets]), dtype=torch.int32, device="cuda")
    return cat("kpts0"), cat("kpts1"), off, stack("K_color0"), stack("K_color1")


def ms_per_call(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(ITERS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / ITERS


def errors(Rs, ts, sets):
    rot = [po.rotation_angle(np.asarray(R, np.float64), s["R_gt"]) if np.isfinite(R).all() else np.pi
           for R, s in zip(Rs, sets)]
    tra = [po.vector_angle(t, s["t_gt"]) if np.isfinite(t).all() else np.pi for t, s in zip(ts, sets)]
    return float(np.median(rot)), float(np.median(tra))


def main():
    card = msb.card()
    be = pose_solver.PoseBackend(max_pairs=B, max_pts=8192, max_hyp=NUM_HYP)
    cells = []
    for n in NS:
        for ratio in RATIOS:
            sets = [synth.make_correspondences(7000 + 37 * n + int(100 * ratio) + i, n=n, inlier_ratio=ratio, noise_px=0.5)
                    for i in range(B)]
            k0, k1, off, K0, K1 = batch(sets)
            modes = {"msac": lambda: be.emat(k0, k1, off, K0, K1, PIX_THR, NUM_HYP, lo=pose_solver.LO_LSQ),
                     "magsac": lambda: be.emat(k0, k1, off, K0, K1, PIX_THR, NUM_HYP, scoring="magsac")}
            acc = {}
            for m, fn in modes.items():          # warm-up, and the poses for the accuracy columns
                R, t, _, _ = fn()
                torch.cuda.synchronize()
                acc[m] = errors(R.double().cpu().numpy(), t.double().cpu().numpy(), sets)
            times = {m: [] for m in modes}
            for _ in range(ROUNDS):
                for m, fn in modes.items():
                    times[m].append(ms_per_call(fn))
            cv = [po.essential_matrix_solver(s["kpts0"], s["kpts1"], s["K_color0"], s["K_color1"], PIX_THR, CONF)
                  for s in sets]
            acc["cv2"] = errors([c[0] for c in cv], [c[1] for c in cv], sets)
            ms = {m: float(np.median(v)) for m, v in times.items()}
            cell = {"N": n, "inlier_ratio": ratio, "ms_per_batch": ms, "rounds_ms": times,
                    "magsac_over_msac": ms["magsac"] / ms["msac"],
                    "median_rot_err_rad": {m: a[0] for m, a in acc.items()},
                    "median_t_dir_err_rad": {m: a[1] for m, a in acc.items()}}
            cells.append(cell)
            print(f"N={n:5d} r={ratio:.1f}  msac {ms['msac']:7.3f} ms  magsac {ms['magsac']:7.3f} ms  "
                  f"x{cell['magsac_over_msac']:.2f}  rot " +
                  " ".join(f"{m} {a[0]:.2e}" for m, a in acc.items()) + "  t " +
                  " ".join(f"{m} {a[1]:.2e}" for m, a in acc.items()), file=sys.stderr, flush=True)
    be.close()
    res = {"card": card, "batch": B, "num_hyp": NUM_HYP, "pix_thr": PIX_THR, "iters": ITERS, "rounds": ROUNDS,
           "cells": cells}
    print(json.dumps(res))
    out = os.environ.get("OUT")
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
