"""Times PoseBackend.icp (mfr_icp_refine, PROCRUSTES.REFINE) on 16 pairs at 480x640 (ScanNet) and 540x720 (Map-free),
from perturbed ground-truth start poses over synth.make_pair scenes, 30 iterations at most, radius 0.05 m.

    python scripts/icp_bench.py [--before-lib PATH] [--reps 20]

--before-lib: another build of libmfr_b200.so (e.g. of an earlier commit), timed in the same process, alternating with
this tree's library; its poses are compared with this tree's. Prints the card's name and power limit with the numbers.
CUDA events around each call; the median over --reps calls after two warm-up calls.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__  # noqa: E402,F401
from mfr_b200 import lib as _lib, synth  # noqa: E402

c_vp, c_int, c_f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float


def _load(path):
    l = ctypes.CDLL(path)
    l.mfr_pose_solver_create.argtypes = [c_int, c_int, c_int, ctypes.POINTER(c_vp)]
    l.mfr_pose_solver_destroy.argtypes = [c_vp]
    l.mfr_icp_refine.argtypes = [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_f, c_int, c_f, c_f,
                                 c_vp, c_vp, c_vp, c_vp]
    h = c_vp()
    assert l.mfr_pose_solver_create(16, 64, 128, ctypes.byref(h)) == 0
    return l, h


def _inputs(h, w, K):
    scenes = []
    for i in range(16):
        p = synth.make_pair(40 + i % 4, h=h, w=w, K=K)
        rng = np.random.default_rng(i)
        R0 = synth.rodrigues(rng.normal(0, 0.01, 3)) @ p["R_gt"]
        t0 = p["t_gt"] + rng.normal(0, 0.02, 3)
        scenes.append((p, R0, t0))
    dev = torch.device("cuda")
    st = lambda f: torch.tensor(np.stack([f(s) for s in scenes]), dtype=torch.float32, device=dev).contiguous()
    return (st(lambda s: s[1]), st(lambda s: s[2]), st(lambda s: s[0]["K_color0"]), st(lambda s: s[0]["K_color1"]),
            st(lambda s: s[0]["depth0"]), st(lambda s: s[0]["depth1"]))


def _call(l, h, ins, H, W):
    R0, t0, K0, K1, d0, d1 = ins
    R = torch.empty(16, 3, 3, device="cuda"); t = torch.empty(16, 3, device="cuda")
    n = torch.empty(16, dtype=torch.int32, device="cuda")
    p = lambda x: c_vp(x.data_ptr())
    rc = l.mfr_icp_refine(h, p(d0), p(d1), H, W, 16, p(K0), p(K1), p(R0), p(t0), 0.05, 30, 1e-4, 1e-4, p(R), p(t), p(n),
                          c_vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    return R, t, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--before-lib", default=None)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    arms = {"this tree": _load(_lib.LIB_PATH)}
    if a.before_lib:
        arms["before"] = _load(a.before_lib)
    out = {"gpu": gpu, "pairs": 16, "max_iter": 30, "radius_m": 0.05}
    for name, (H, W, K) in {"480x640": (480, 640, np.array([[577.0, 0, 319.5], [0, 577.0, 239.5], [0, 0, 1]])),
                            "540x720": (540, 720, synth.K_DEFAULT)}.items():
        ins = _inputs(H, W, K)
        res, times = {}, {k: [] for k in arms}
        for k, (l, h) in arms.items():
            for _ in range(2):
                res[k] = _call(l, h, ins, H, W)
        torch.cuda.synchronize()
        for _ in range(a.reps):
            for k, (l, h) in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); _call(l, h, ins, H, W); e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1))
        row = {k: round(float(np.median(v)), 3) for k, v in times.items()}
        if "before" in res:
            Rb, tb, nb = (x.cpu().numpy() for x in res["before"])
            Ra, ta, na = (x.cpu().numpy() for x in res["this tree"])
            row["max |dR|, |dt| vs before"] = float(max(np.abs(Ra - Rb).max(), np.abs(ta - tb).max()))
            row["max |d n_inliers| vs before"] = int(np.abs(na.astype(np.int64) - nb).max())
        out[f"{name} ms per call (median)"] = row
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
