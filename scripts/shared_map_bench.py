"""Shared map frame against the paired path, on one synthetic Map-free-style scene (synth.make_scene: one map frame and
B query frames rendered from it), 540x720 source frames, in one process.

  python scripts/shared_map_bench.py            # SECONDS=2 ROUNDS=3 B=16 SPSG_B=8

LoFTR (bf16, 720x544 engine frame, functional_state_dict(noise=1e-3), the weights bench.py times) + 5-point RANSAC +
scale from depth through mfr_b200.pipeline.RelocPipeline, device-resident inputs:
  paired: submit_device(map repeated B times, queries, ...)   shared: set_map once, then submit_device_queries(queries, ...)
SuperPoint + SuperGlue (bf16, SPSG_B pairs, up to 1024 keypoints; the real weights when oracle/build_ref.py has staged
them, else synthetic) + PnP from the map depth, as bench.py's C3 does:
  paired: forward_async(map repeated, queries)                shared: set_map once, then forward_shared_async(queries)

The arms alternate ROUNDS times; each timed window lasts at least SECONDS (CUDA events). Before timing, both arms'
poses and inlier counts are checked to be identical. The card name and its power limit are printed first."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import mfr_b200
from mfr_b200 import loftr, pose_solver, spsg, synth
from mfr_b200.pipeline import RelocPipeline
from oracle import build_ref

SECONDS = float(os.environ.get("SECONDS", 2.0))
ROUNDS = int(os.environ.get("ROUNDS", 3))
B, SPSG_B = int(os.environ.get("B", 16)), int(os.environ.get("SPSG_B", 8))
H, W, HP, WP = 720, 540, 720, 544
PIX_THR, SCALE_THR, HYP = 2.0, 0.1, 1024     # bench.py's pose back end settings


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception as e:   # the card name still comes from torch
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def timed(step, n_pairs):
    """pairs/s of `step` (one batch per call): the number of batches that fills SECONDS is estimated from a short run,
    then run back to back between two CUDA events on an idle device (the closing one after a device synchronise, since
    the batches run on the engines' own streams)."""
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
    return n * n_pairs / window(n) * 1e3


def alternate(name, arms, n_pairs):
    for r in range(ROUNDS):
        for arm, step in arms:
            print(f"[{name}] round {r}: {arm:6s} {timed(step, n_pairs):8.1f} pairs/s", flush=True)


print("card:", card(), flush=True)
scene = synth.make_scene(7, max(B, SPSG_B), h=H, w=W)
g0 = torch.from_numpy(scene["gray0"]).cuda()
d0 = torch.from_numpy(scene["depth0"]).cuda()
K0 = torch.from_numpy(scene["K_color0"]).cuda()
qs = scene["queries"]
g1 = torch.from_numpy(np.stack([q["gray1"] for q in qs])).cuda()
d1 = torch.from_numpy(np.stack([q["depth1"] for q in qs])).cuda()
K1 = torch.from_numpy(np.stack([q["K_color1"] for q in qs])).cuda()

# ---------------------------------------------------------------- LoFTR + 5-point + scale
eng = loftr.LoFTR(loftr.functional_state_dict(noise=1e-3), batch=B, height=HP, width=WP, cfg={"thr": 0.2}, graph=True,
                  precision="bf16", pipelined=True)
be = pose_solver.PoseBackend(max_pairs=B, max_pts=(HP // 8) * (WP // 8), max_hyp=HYP)
pipe = RelocPipeline([eng], be, PIX_THR, SCALE_THR, HYP)
G0, D0, KK0 = (x[None].expand(B, *x.shape).contiguous() for x in (g0, d0, K0))
G1, D1, KK1 = g1[:B].contiguous(), d1[:B].contiguous(), K1[:B].contiguous()
pipe.set_map(g0, d0, K0)


def loftr_paired():
    return pipe.submit_device(G0, G1, D0, D1, KK0, KK1)


def loftr_shared():
    return pipe.submit_device_queries(G1, D1, KK1)


def loftr_result(step):
    pipe.reset()
    step()
    return pipe.drain()


a, b = loftr_result(loftr_paired), loftr_result(loftr_shared)
assert all(torch.equal(x, y) for x, y in zip(a, b)), "LoFTR: the shared arm's poses differ from the paired arm's"
print(f"[loftr] B={B}, bf16, {HP}x{WP}: both arms give identical R, t and inliers (median inliers {int(a[2].median())}, "
      f"launches per paired batch {eng.num_launches()})", flush=True)
pipe.reset()
alternate("loftr", [("paired", loftr_paired), ("shared", loftr_shared)], B)
pipe.reset()
eng.close()
be.close()
del eng, be, pipe
torch.cuda.empty_cache()

# ---------------------------------------------------------------- SuperPoint + SuperGlue + PnP
if build_ref.available():
    sp = torch.load(build_ref.weights_dir() + "/superpoint_v1.pth", map_location="cpu")
    sg = torch.load(build_ref.weights_dir() + "/superglue_indoor.pth", map_location="cpu")
    weights = "real"
else:
    (sp, sg), weights = spsg.synthetic_state_dicts(0), "synthetic"
seng = spsg.SuperPointSuperGlue(sp, sg, batch=SPSG_B, height=H, width=W, graph=True, precision="bf16")
sbe = pose_solver.PoseBackend(max_pairs=SPSG_B, max_pts=1024, max_hyp=1024)
outs = seng.device_outputs()
S0, SD0, SK0 = (x[None].expand(SPSG_B, *x.shape).contiguous() for x in (g0, d0, K0))
S1, SK1 = g1[:SPSG_B].contiguous(), K1[:SPSG_B].contiguous()
seng.set_map(g0)


def pnp():
    with torch.cuda.stream(seng.stream):
        return sbe.pnp(outs["mkpts0"], outs["mkpts1"], outs["m_offsets"], SK0, SK1, SD0, 3.0, 1000)


def spsg_paired():
    seng.forward_async(S0, S1)
    return pnp()


def spsg_shared():
    seng.forward_shared_async(S1)
    return pnp()


def spsg_result(step):
    r = step()[:3]
    torch.cuda.synchronize()
    return [x.clone() for x in r]


a, b = spsg_result(spsg_paired), spsg_result(spsg_shared)
assert all(torch.equal(x, y) for x, y in zip(a, b)), "SP+SG: the shared arm's poses differ from the paired arm's"
print(f"[spsg] B={SPSG_B}, bf16, {H}x{W}, {weights} weights: both arms give identical R, t and inliers "
      f"(median inliers {int(a[2].median())})", flush=True)
alternate("spsg", [("paired", spsg_paired), ("shared", spsg_shared)], SPSG_B)
seng.close()
sbe.close()
