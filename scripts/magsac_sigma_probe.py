"""Which sigma_max does cv2.findEssentialMat(USAC_MAGSAC) use for the threshold the reference passes (pose_solver.py:43)?
CPU only (cv2 + scipy).

  python scripts/magsac_sigma_probe.py

For 16 synthetic cells (synth.make_correspondences, N in {500, 2000}, inlier ratio 0.2 .. 0.8, 0.5 px noise), cv2's
pose is polished by IRLS on the MAGSAC++ loss (tests/magsac_oracle.py) once with sigma_max = thr and once with
sigma_max = thr / k. The reading under which cv2's output is nearer a fixed point of the loss is the one cv2 minimises:
the script prints, per reading, how far the polish moves R and t and how much it lowers the sum of rho (relative)."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
import numpy as np  # noqa: E402

import magsac_oracle as mo  # noqa: E402
import mfr_b200  # noqa: E402,F401
from mfr_b200 import synth  # noqa: E402
from oracle import pose_solver_oracle as po  # noqa: E402


def main():
    rows = []
    for n, ratio in ((500, 0.3), (2000, 0.2), (2000, 0.5), (2000, 0.8)):
        for seed in range(4):
            c = synth.make_correspondences(1000 + seed, n=n, inlier_ratio=ratio, noise_px=0.5)
            R, t, _, _ = po.essential_matrix_solver(c["kpts0"], c["kpts1"], c["K_color0"], c["K_color1"], 2.0, 0.9999)
            k0, k1, thr = mo.normalised(c["kpts0"], c["kpts1"], c["K_color0"], c["K_color1"], 2.0)
            row = []
            for sigma in (thr, thr / mo.K):
                Rp, tp = mo.irls_polish(R, t, k0, k1, sigma)
                before = mo.rho(po.sampson_residuals(R, t, k0, k1), sigma).sum()
                after = mo.rho(po.sampson_residuals(Rp, tp, k0, k1), sigma).sum()
                row.append((po.rotation_angle(R, Rp), po.vector_angle(t, tp), 1.0 - after / before))
            rows.append(row)
            print(f"N={n} ratio={ratio} seed={seed}  " + "  |  ".join(
                f"{name}: dR {a:.2e} dt {b:.2e} drho {d:.2e}" for name, (a, b, d) in zip(("thr", "thr/k"), row)))
    a = np.array(rows)             # [cell][reading][dR, dt, drho]
    med = np.median(a, axis=0)
    for i, name in enumerate(("sigma_max = thr", "sigma_max = thr/k")):
        print(f"{name}: median dR {med[i, 0]:.2e} rad, dt {med[i, 1]:.2e} rad, relative sum-rho decrease {med[i, 2]:.2e}")
    print(f"cells where thr leaves the smaller relative decrease: {int((a[:, 0, 2] < a[:, 1, 2]).sum())} of {len(a)}")


if __name__ == "__main__":
    main()
