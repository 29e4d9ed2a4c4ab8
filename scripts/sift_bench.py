"""GPU SIFT engine on 16 synthetic 540x720 pairs (synth.make_pair): detect time for the 32 images with a per-stage
split, end-to-end pairs/s (GPU detect -> match_pairs -> emat RANSAC + scale from depth at C1's settings: 3 px, 0.1,
2048 hypotheses) next to the host cv2 path on the same pairs, median pose errors of both detectors against the
synthetic ground truth, and the fraction of cv2's keypoints the engine reproduces. Prints the card and its power limit.

Usage: python scripts/sift_bench.py [--pairs 16] [--iters 20] [--out results/sift_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception as e:   # the card name still comes from torch below
        return f"nvidia-smi unavailable ({e})"


def pose_err(R, t, Rg, tg):
    ang = float(np.degrees(np.arccos(np.clip((np.trace(np.asarray(R, np.float64) @ np.asarray(Rg).T) - 1) / 2, -1, 1))))
    return ang, float(np.linalg.norm(np.asarray(t, np.float64).ravel() - np.asarray(tg, np.float64).ravel()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import cv2
    import torch
    import mfr_b200  # noqa: F401
    from mfr_b200 import model, pose_solver, sift, synth
    from sift_compare import cv_rows, pair
    if not torch.cuda.is_available():
        raise SystemExit("sift_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    P = a.pairs
    pairs = [synth.make_pair(i) for i in range(P)]
    g = np.stack([synth.rgb_to_gray_u8(p[k]) for p in pairs for k in ("image0", "image1")])
    H, W = g.shape[1:]
    imgs = torch.from_numpy(g).to(dev)
    eng = sift.SIFT(2 * P, H, W, nfeatures=2048, root_sift=True)
    for _ in range(3):
        eng.detect(imgs)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        eng.l.mfr_sift_detect(eng.h, mfr_b200.lib.ptr(imgs), mfr_b200.lib.cur_stream())
    e1.record(); torch.cuda.synchronize()
    detect_ms = e0.elapsed_time(e1) / a.iters
    stages = [eng.profile(imgs) for _ in range(5)]
    stage_ms = {k: float(np.median([s[k] for s in stages])) for k in stages[0]}
    be = pose_solver.PoseBackend(max_pairs=P, max_pts=8192, max_hyp=2048)
    K = torch.from_numpy(np.stack([p["K_color0"] for p in pairs]).reshape(P, 9).astype(np.float32)).to(dev)
    d0 = torch.from_numpy(np.stack([p["depth0"] for p in pairs]).astype(np.float32)).to(dev)
    d1 = torch.from_numpy(np.stack([p["depth1"] for p in pairs]).astype(np.float32)).to(dev)

    def gpu_run():
        eng.detect(imgs)
        k0, k1, off = eng.match_pairs(0.8)
        R, t, n = be.emat_metric(k0, k1, off, K, K, d0, d1, 3.0, 0.1, 2048)
        return R.cpu().numpy(), t.cpu().numpy(), off.cpu().numpy()

    gpu_run(); torch.cuda.synchronize()
    t0 = time.perf_counter()
    reps = 5
    for _ in range(reps):
        R, t, off = gpu_run()
    torch.cuda.synchronize()
    gpu_pps = reps * P / (time.perf_counter() - t0)
    gpu_err = [pose_err(R[i], t[i], pairs[i]["R_gt"], pairs[i]["t_gt"]) for i in range(P)]
    # host cv2 path on the same pairs (detect on the host, the rest on the GPU as bench C1 does)
    cs = cv2.SIFT_create(2048)
    be1 = pose_solver.PoseBackend(max_pairs=1, max_pts=8192, max_hyp=2048)
    t0 = time.perf_counter()
    host_err, recall = [], []
    for i in range(P):
        kp0, de0 = cs.detectAndCompute(g[2 * i], None); kp1, de1 = cs.detectAndCompute(g[2 * i + 1], None)
        i1, dd1, _, dd2 = model.knn2_gpu(model.root_sift(de0), model.root_sift(de1))
        good = dd1 < 0.8 * dd2
        p0 = np.float32([kp0[j].pt for j in np.where(good)[0]]).reshape(-1, 2)
        p1 = np.float32([kp1[j].pt for j in i1[good]]).reshape(-1, 2)
        Rh, th, _ = be1.emat_metric(torch.from_numpy(p0).to(dev), torch.from_numpy(p1).to(dev),
                                    torch.tensor([0, len(p0)], dtype=torch.int32, device=dev), K[i:i + 1], K[i:i + 1],
                                    d0[i:i + 1], d1[i:i + 1], 3.0, 0.1, 2048)
        host_err.append(pose_err(Rh[0].cpu().numpy(), th[0].cpu().numpy(), pairs[i]["R_gt"], pairs[i]["t_gt"]))
    host_pps = P / (time.perf_counter() - t0)
    out = eng.detect(imgs)
    for b in range(4):
        kps, _ = cs.detectAndCompute(g[b], None)
        a_, _ = cv_rows(kps)
        n = int(out["counts"][b])
        kp = out["keypoints"][b, :n].cpu().numpy().astype(np.float64)
        recall.append(float((pair(a_, kp) >= 0).mean()))
    res = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "images": 2 * P, "size": [H, W],
           "detect_ms_32_images": detect_ms, "stage_ms": stage_ms, "gpu_pairs_per_s": gpu_pps, "host_cv2_pairs_per_s": host_pps,
           "median_rot_err_deg": {"gpu": float(np.median([e[0] for e in gpu_err])), "cv2": float(np.median([e[0] for e in host_err]))},
           "median_trans_err_m": {"gpu": float(np.median([e[1] for e in gpu_err])), "cv2": float(np.median([e[1] for e in host_err]))},
           "cv2_keypoints_reproduced": float(np.mean(recall)), "matches_per_pair": float(off[-1] / P)}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    eng.close(); be.close(); be1.close()


if __name__ == "__main__":
    main()
