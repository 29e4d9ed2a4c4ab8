"""Pairs/s of every Map-free method config (the reference's config/matching/mapfree/*.yaml over config/mapfree.yaml)
through pipeline.from_cfg, paired and with a shared map frame, and the median pose error against the synthetic ground
truth. One process, one GPU.

  python scripts/method_stream_bench.py            # B=16 SECONDS=1 ROUNDS=2 PRECISION=bf16

Inputs are device-resident synthetic Map-free-style scenes (synth.make_scene: one map frame, B query frames rendered from
it; 540x720 source frames, synthetic depth for both frames). Weights: LoFTR loftr.functional_state_dict(); SP+SG the
real indoor weights when oracle/build_ref.py has staged them, else synthetic ones (printed); SIFT none.
  paired: submit_device(map repeated B times, queries, ...)     shared: set_map once, then submit_device_queries(...)
The _dptkitti / _dptnyu variants of a method differ only in which depth files a scene reader loads: their streams do the
same work, so each distinct method is timed once and its numbers are printed for every config that names it.

The two arms alternate ROUNDS times; each timed window runs at least SECONDS of back-to-back batches between CUDA events
(closed after a device synchronise) and the median of the rounds is reported. Before timing, the shared arm's poses are
checked to be identical to the paired arm's. The card, its power limit and its clocks are printed first."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import mfr_b200  # noqa: E402,F401
from mfr_b200 import config, loftr, spsg, synth  # noqa: E402
from mfr_b200.pipeline import from_cfg, resolve_method  # noqa: E402
from oracle import build_ref  # noqa: E402

B = int(os.environ.get("B", 16))
SECONDS = float(os.environ.get("SECONDS", 1.0))
ROUNDS = int(os.environ.get("ROUNDS", 2))
PRECISION = os.environ.get("PRECISION", "bf16")
H, W = 720, 540

EMAT = lambda pix: {"POSE_SOLVER": "EssentialMatrixMetric",
                    "EMAT_RANSAC": {"PIX_THRESHOLD": pix, "SCALE_THRESHOLD": 0.1, "CONFIDENCE": 0.9999}}
PNP = {"POSE_SOLVER": "PNP", "PNP": {"RANSAC_ITER": 1000, "REPROJECTION_INLIER_THRESHOLD": 3, "CONFIDENCE": 0.9999}}
PROC = {"POSE_SOLVER": "Procrustes", "PROCRUSTES": {"MAX_CORR_DIST": 0.05}}
# the keys of config/matching/mapfree/<name>.yaml
METHODS = {f"{m.lower()}_{s}_{d}": (m, d, EMAT(3.0 if m == "SIFT" else 2.0) if s == "emat" else PNP)
           for m in ("LoFTR", "SG", "SIFT") for s in ("emat", "pnp") for d in ("dptkitti", "dptnyu")}
METHODS["sg_procrustes_dptkitti"] = ("SG", "dptkitti", PROC)


def method_cfg(name):
    matcher, depth, solver = METHODS[name]
    cfg = config.get_default_cfg()
    cfg.merge_from_dict({"DATASET": {"DATA_SOURCE": "MapFree", "HEIGHT": H, "WIDTH": W}})
    cfg.merge_from_dict({"MODEL": "FeatureMatching", "FEATURE_MATCHING": "Precomputed", "DATASET": {"ESTIMATED_DEPTH": depth},
                         "MATCHES_FILE_PATH": "{scene_root}/correspondences_" + matcher + ".npz", **solver})
    return cfg


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True).strip()
    except Exception as e:
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def timed(step):
    """pairs/s of `step` (one batch per call): the batch count that fills SECONDS is estimated from a short run, then run
    back to back between two CUDA events, the closing one after a device synchronise."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def window(n):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            step()
        torch.cuda.synchronize()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    window(3)
    n = max(5, int(np.ceil(SECONDS * 1e3 / (window(5) / 5) * 1.1)))
    return n * B / window(n) * 1e3


def pose_errors(R, t, scene):
    """Median rotation error [deg] and translation error [m] of the finite poses of one batch, and how many were finite."""
    rot, tra = [], []
    for b, q in enumerate(scene["queries"][:B]):
        Rb, tb = R[b].double().numpy(), t[b].double().numpy().ravel()
        if not (np.isfinite(Rb).all() and np.isfinite(tb).all()):
            continue
        c = (np.trace(Rb @ np.asarray(q["R_gt"]).T) - 1.0) / 2.0
        rot.append(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))
        tra.append(np.linalg.norm(tb - np.asarray(q["t_gt"]).ravel()))
    return (float(np.median(rot)) if rot else float("nan"), float(np.median(tra)) if tra else float("nan"), len(rot))


def main():
    print("card (name, power limit, SM clock, max SM clock):", card(), flush=True)
    scene = synth.make_scene(7, B, h=H, w=W)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    u8 = lambda img: synth.rgb_to_gray_u8(img)
    images = {torch.float32: (dev(scene["gray0"]), dev(np.stack([q["gray1"] for q in scene["queries"]]))),
              torch.uint8: (dev(u8(scene["image0"])), dev(np.stack([u8(q["image1"]) for q in scene["queries"]])))}
    d0, K0 = dev(scene["depth0"]), dev(scene["K_color0"])
    d1 = dev(np.stack([q["depth1"] for q in scene["queries"]]))
    K1 = dev(np.stack([q["K_color1"] for q in scene["queries"]]))
    D0, KK0 = d0[None].expand(B, H, W).contiguous(), K0[None].expand(B, 3, 3).contiguous()
    if build_ref.available():
        sg_weights, sg_kind = build_ref.weights_dir(), "real indoor"
    else:
        sg_weights, sg_kind = spsg.synthetic_state_dicts(0), "synthetic"
    weights = {"LoFTR": loftr.functional_state_dict(), "SG": sg_weights, "SIFT": None}
    results, by_spec = {}, {}
    for name in sorted(METHODS):
        cfg = method_cfg(name)
        spec = resolve_method(cfg)
        if spec in by_spec:
            results[name] = dict(by_spec[spec], same_as=by_spec[spec]["config"])
            continue
        pipe = from_cfg(cfg, B, weights=weights[spec.matcher], precision=PRECISION)
        eng = pipe.eng
        g0, g1 = images[eng.input_dtype]
        G0 = g0[None].expand(B, H, W).contiguous()
        pipe.set_map(g0, d0, K0)

        def paired():
            return pipe.submit_device(G0, g1, D0, d1, KK0, K1)

        def shared():
            return pipe.submit_device_queries(g1, d1, K1)

        res = {}
        for arm, step in (("paired", paired), ("shared", shared)):
            pipe.reset()
            step()
            res[arm] = pipe.drain()
        assert all(torch.equal(a, b) for a, b in zip(res["paired"], res["shared"])), f"{name}: shared arm differs"
        rot, tra, ok = pose_errors(res["paired"][0], res["paired"][1], scene)
        rates = {"paired": [], "shared": []}
        for _ in range(ROUNDS):
            for arm, step in (("paired", paired), ("shared", shared)):
                pipe.reset()
                rates[arm].append(timed(step))
        pipe.reset()
        r = {"config": name, "matcher": spec.matcher, "solver": spec.solver, "stage": type(pipe.solver).__name__,
             "frame": [spec.height, spec.width], "batch": B, "num_hyp": spec.num_hyp,
             "paired_pairs_s": float(np.median(rates["paired"])), "shared_pairs_s": float(np.median(rates["shared"])),
             "rounds": rates, "median_rot_err_deg": rot, "median_t_err_m": tra, "finite_poses": ok,
             "median_inliers": int(res["paired"][2].median())}
        if spec.matcher == "SG":
            r["weights"] = sg_kind
        if spec.matcher != "SIFT":
            r["precision"] = PRECISION
        by_spec[spec] = results[name] = r
        print(f"{name:24s} {r['stage']:16s} paired {r['paired_pairs_s']:8.1f}  shared {r['shared_pairs_s']:8.1f} pairs/s  "
              f"rot {rot:6.3f} deg  t {tra:6.3f} m  ({ok}/{B} finite, median inliers {r['median_inliers']})", flush=True)
        eng.close(); pipe.be.close()
        del pipe, eng
        torch.cuda.empty_cache()
    for name in sorted(results):
        if "same_as" in results[name]:
            r = results[name]
            print(f"{name:24s} = {r['same_as']}", flush=True)
    out = os.environ.get("OUT")
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            json.dump({"card": card(), "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
