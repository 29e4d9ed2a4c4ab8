"""The float64 stage restatements of oracle/pose_stages_oracle.py pinned to the reference-side oracle
(oracle/pose_solver_oracle.py, OpenCV) on the CPU, so that tests/test_pose_stages_gpu.py compares the kernels with
something that is itself checked where no device exists."""
import cv2
import numpy as np
import pytest

from helpers import rot_angle, synth, vec_angle
from oracle import pose_solver_oracle as po
from oracle import pose_stages_oracle as so


@pytest.mark.parametrize("seed,n,ratio,noise", [(201, 800, 0.6, 0.3), (202, 1500, 0.5, 0.5)])
def test_hard_refit_reaches_polished_fixed_point(seed, n, ratio, noise):
    """The truncated least-squares LM rounds of emat_final_kernel (lo & 2) end on the fixed point that
    polish_essential_fixed_point reaches from the same start: the Sampson least-squares optimum of its own inlier set."""
    c = synth.make_correspondences(seed, n=n, inlier_ratio=ratio, noise_px=noise)
    pts = so.normalise(c["kpts0"], c["kpts1"], c["K_color0"], c["K_color1"])
    thr = float(so.emat_threshold(2.0, c["K_color0"], c["K_color1"])[0])
    R0, t0 = c["R_gt"], c["t_gt"] / np.linalg.norm(c["t_gt"])
    Rf, tf, _, _ = po.polish_essential_fixed_point(R0, t0, c["kpts0"], c["kpts1"], c["K_color0"], c["K_color1"], 2.0)
    R, t = R0.copy(), t0.copy()
    for _ in range(12):
        R, t = so.lm_round(R, t, pts, thr * thr, 1, True, 8)
    assert rot_angle(R, Rf) < 1e-6 and vec_angle(t, tf) < 1e-6, (rot_angle(R, Rf), vec_angle(t, tf))


@pytest.mark.parametrize("seed", [211, 212])
def test_pnp_prepare_matches_reference_lift(seed):
    """pnp_prepare's valid set is the reference's (depth > depth0.min() at the int32-truncated keypoint) and its lift
    is backproject_3d's to a few float64 ulp (the float32 inverse of K: LAPACK there, the rounded adjugate here)."""
    c = synth.make_correspondences(seed, n=700, inlier_ratio=0.6, noise_px=0.3)
    d0 = c["depth0"].copy()
    ik = np.int32(c["kpts0"])
    d0[ik[::5, 1], ik[::5, 0]] = 0.0
    vidx, X, uv = so.pnp_prepare(c["kpts0"], c["kpts1"], d0, c["K_color0"], so.depth_min(d0))
    dp = d0[ik[:, 1], ik[:, 0]]
    valid = dp > d0.min()
    assert np.array_equal(vidx, np.nonzero(valid)[0])
    Xr = po.backproject_3d(ik[valid], dp[valid], c["K_color0"])
    assert np.abs(X - Xr).max() <= 8 * np.spacing(np.abs(Xr).max())
    assert np.array_equal(uv, c["kpts1"][valid])


@pytest.mark.parametrize("seed,n,ratio,noise", [(221, 1000, 0.6, 0.3), (222, 2000, 0.5, 0.5)])
def test_scale_restatement_equals_reference(seed, n, ratio, noise):
    c = synth.make_correspondences(seed, n=n, inlier_ratio=ratio, noise_px=noise)
    Ro, to, no, mo = po.essential_matrix_solver(c["kpts0"], c["kpts1"], c["K_color0"], c["K_color1"], 2.0, 0.9999)
    Rm, tm, nm = po.scale_from_depth(Ro, to, mo, c["kpts0"], c["kpts1"], c["depth0"], c["depth1"], c["K_color0"],
                                     c["K_color1"], 0.1)
    R, t, cnt = so.scale_consensus(Ro, np.ravel(to), mo.ravel() == 1, c["kpts0"], c["kpts1"], c["depth0"], c["depth1"],
                                   c["K_color0"], c["K_color1"], 0.1)
    assert cnt == nm
    assert np.abs(t - tm.ravel()).max() < 1e-12


@pytest.mark.parametrize("seed", [231, 232])
def test_pnp_lm_equals_opencv(seed):
    """pnp_final's LM (20 steps on a fixed inlier set) ends where cv2.solvePnPGeneric(SOLVEPNP_ITERATIVE) does."""
    c = synth.make_correspondences(seed, n=400, inlier_ratio=1.0, noise_px=0.5)
    vidx, X, uv = so.pnp_prepare(c["kpts0"], c["kpts1"], c["depth0"], c["K_color0"], so.depth_min(c["depth0"]))
    rng = np.random.default_rng(seed)
    R0 = synth.rodrigues(rng.normal(0, 0.01, 3)) @ c["R_gt"]
    t0 = c["t_gt"] + rng.normal(0, 0.01, 3)
    R, t = so.pnp_lm(R0, t0, X, uv, c["K_color1"])
    rv, _ = cv2.Rodrigues(R0)
    _, rvs, tvs, _ = cv2.solvePnPGeneric(X, uv.astype(np.float64), c["K_color1"].astype(np.float64), None,
                                         useExtrinsicGuess=True, rvec=rv, tvec=t0.reshape(3, 1),
                                         flags=cv2.SOLVEPNP_ITERATIVE)
    Rc, _ = cv2.Rodrigues(rvs[0])
    assert rot_angle(R, Rc) < 1e-7 and np.abs(t - tvs[0].ravel()).max() < 1e-7


@pytest.mark.parametrize("seed", [241, 242])
def test_procrustes_stages_match_reference_solver(seed):
    """procrustes_prepare's valid set and lift are procrustes_solver's (depth > depth.min() on both sides at the
    int32-truncated keypoints, backproject_3d), and the hypotheses + refit, chained, reach its pose and inlier count."""
    c = synth.make_correspondences(seed, n=800, inlier_ratio=0.6, noise_px=0.2)
    d0, d1 = c["depth0"].copy(), c["depth1"].copy()
    ik0, ik1 = np.int32(c["kpts0"]), np.int32(c["kpts1"])
    d0[ik0[::7, 1], ik0[::7, 0]] = 0.0
    d1[ik1[::5, 1], ik1[::5, 0]] = d1.min()
    vidx, X0, X1 = so.procrustes_prepare(c["kpts0"], c["kpts1"], d0, d1, c["K_color0"], c["K_color1"],
                                         so.depth_min(d0), so.depth_min(d1))
    z0, z1 = d0[ik0[:, 1], ik0[:, 0]], d1[ik1[:, 1], ik1[:, 0]]
    valid = (z0 > d0.min()) & (z1 > d1.min())
    assert np.array_equal(vidx, np.nonzero(valid)[0])
    for X, Xr in ((X0, po.backproject_3d(ik0[valid], z0[valid], c["K_color0"])),
                  (X1, po.backproject_3d(ik1[valid], z1[valid], c["K_color1"]))):
        assert np.abs(X - Xr).max() <= 8 * np.spacing(np.abs(Xr).max())
    blocks = so.procrustes_hypotheses(X0, X1, 256, 7, 0)
    res = np.zeros(len(blocks), so.HYP_DTYPE)
    for b, cands in enumerate(blocks):     # a block winner: the most inliers (float64 count stands in for the kernel's)
        cnt = [int((np.linalg.norm(X0 @ R.T + t - X1, axis=1) < 0.05).sum()) for _, _, R, t in cands]
        k = int(np.argmax(cnt))
        res[b]["valid"], res[b]["cost"], res[b]["count"] = 1, -cnt[k], cnt[k]
        res[b]["model"][:9], res[b]["model"][9:] = cands[k][2].ravel(), cands[k][3]
    fin = so.procrustes_final(res, X0, X1, 0.05)
    Ro, to, no = po.procrustes_solver(c["kpts0"], c["kpts1"], d0, d1, c["K_color0"], c["K_color1"], 0.05, iters=256)
    assert not fin["failed"] and fin["near"] == 0
    assert rot_angle(fin["R"], Ro) < 1e-6 and np.abs(fin["t"] - to.ravel()).max() < 1e-6 and abs(fin["n"] - no) <= 2


@pytest.mark.parametrize("seed", [3, 8])
def test_icp_stages_match_reference_loop(seed):
    """icp_assoc + icp_update, chained by icp_loop, follow icp_point_to_point (the k-d tree restatement of Open3D's
    registration_icp) on the same clouds from the same start: same stop, pose and fitness."""
    p = synth.make_pair(seed, h=120, w=160, K=np.array([[150.0, 0, 79.5], [0, 150.0, 59.5], [0, 0, 1]]))
    rng = np.random.default_rng(seed)
    R0 = synth.rodrigues(rng.normal(0, 0.01, 3)) @ p["R_gt"]
    t0 = p["t_gt"] + rng.normal(0, 0.02, 3)
    X0, X1 = so.icp_clouds(p["depth0"], p["depth1"], p["K_color0"], p["K_color1"])
    R, t, fit, rmse, stop, conv = so.icp_loop(X0, X1, R0, t0, 0.05)
    T0 = np.eye(4); T0[:3, :3] = R0; T0[:3, 3] = t0
    T, fo, ro = po.icp_point_to_point(X0, X1, T0, float(np.float32(0.05)))
    assert conv and stop < 30
    assert np.abs(R - T[:3, :3]).max() < 1e-9 and np.abs(t - T[:3, 3]).max() < 1e-9
    assert fit == fo and abs(rmse - ro) <= 1e-12 * ro
