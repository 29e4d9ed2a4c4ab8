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
