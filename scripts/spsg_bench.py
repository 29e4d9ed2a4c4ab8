"""BASELINE config C3 timing: SuperPoint + SuperGlue + PnP-from-depth, 540x720, up to 1024 keypoints, B pairs per step.

  PRECISION=tf32,bf16 ROUNDS=3 B=8 WEIGHTS=real python scripts/spsg_bench.py

WEIGHTS=real (the default when oracle/build_ref.py has staged them) runs the reference's in-tree SuperPoint and indoor
SuperGlue weights, whose matches give a meaningful pose error; WEIGHTS=synthetic runs seeded random weights, on which
SuperPoint fires on all 1024 keypoints per image (the full-size SuperGlue workload) but SuperGlue finds no match above
the 0.2 threshold, so the pose errors are infinite.

PRECISION lists the engine precisions to time (tf32, bf16, fp32x3; default tf32). With more than one, one engine per
precision is built up front and the modes are timed in turn, ROUNDS times (default 3), so that they share the card's
state. Each line gives the step time, pairs/s and the median rotation (deg) and translation (m) error of the PnP pose
against the synthetic ground truth. The card name and its power limit are printed first."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import mfr_b200
from mfr_b200 import spsg, synth, pose_solver
from oracle import build_ref


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception as e:   # the card name still comes from torch
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


B = int(os.environ.get("B", 8)); H, W = 720, 540
modes = [m.strip() for m in os.environ.get("PRECISION", "tf32").split(",") if m.strip()]
rounds = int(os.environ.get("ROUNDS", 3 if len(modes) > 1 else 1))
print("card:", card(), flush=True)
weights = os.environ.get("WEIGHTS", "real" if build_ref.available() else "synthetic")
if weights == "real":
    sp = torch.load(build_ref.weights_dir() + "/superpoint_v1.pth", map_location="cpu")
    sg = torch.load(build_ref.weights_dir() + "/superglue_indoor.pth", map_location="cpu")
else:
    sp, sg = spsg.synthetic_state_dicts(0)
print("weights:", weights, flush=True)
engines = {m: spsg.SuperPointSuperGlue(sp, sg, batch=B, height=H, width=W, graph=True, precision=m) for m in modes}
be = pose_solver.PoseBackend(max_pairs=B, max_pts=1024, max_hyp=1024)
ps = [synth.make_pair(1000 + b) for b in range(B)]
g0 = torch.from_numpy(np.stack([synth.rgb_to_gray_u8(p["image0"]).astype(np.float32) / 255.0 for p in ps])).cuda()
g1 = torch.from_numpy(np.stack([synth.rgb_to_gray_u8(p["image1"]).astype(np.float32) / 255.0 for p in ps])).cuda()
d0 = torch.from_numpy(np.stack([p["depth0"] for p in ps]).astype(np.float32)).cuda()
K = torch.from_numpy(np.stack([p["K_color0"] for p in ps]).astype(np.float32)).cuda().contiguous()


def step(eng, outs):
    eng.forward_async(g0, g1)
    with torch.cuda.stream(eng.stream):
        return be.pnp(outs["mkpts0"], outs["mkpts1"], outs["m_offsets"], K, K, d0, 3.0, 1000)


def pose_errors(R, t):
    R = R.reshape(B, 3, 3).double().cpu().numpy(); t = t.reshape(B, 3).double().cpu().numpy()
    rot, tra = [], []
    for b, p in enumerate(ps):
        c = (np.trace(R[b] @ np.asarray(p["R_gt"], np.float64).T) - 1.0) / 2.0
        rot.append(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))) if np.isfinite(c) else np.inf)
        e = np.linalg.norm(t[b] - np.asarray(p["t_gt"], np.float64).ravel())
        tra.append(e if np.isfinite(e) else np.inf)
    return float(np.median(rot)), float(np.median(tra))


def run(mode):
    eng = engines[mode]
    outs = eng.device_outputs()
    for _ in range(3):
        step(eng, outs)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 20
    with torch.cuda.stream(eng.stream):
        e0.record()
    for _ in range(n):
        R, t, inl, mask = step(eng, outs)
    with torch.cuda.stream(eng.stream):
        e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    rot, tra = pose_errors(R, t)
    print(f"[{mode}] SuperPoint+SuperGlue+PnP: B={B} pairs/step, {ms:.3f} ms/step, {B / ms * 1e3:.1f} pairs/s, "
          f"kernels/step {eng.num_launches()}, keypoints/image {outs['counts'].float().mean().item():.0f}, "
          f"matches/pair {(outs['m_offsets'][1:] - outs['m_offsets'][:-1]).float().mean().item():.0f}, "
          f"median pose error {rot:.3f} deg / {tra:.4f} m", flush=True)


for r in range(rounds):
    for m in modes:
        run(m)
