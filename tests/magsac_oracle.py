"""ORACLE (test infrastructure only — never imported by the product path).

MAGSAC++ loss of the essential-matrix RANSAC (Barath et al., CVPR 2020, the objective of OpenCV's USAC_MAGSAC) for a
residual with nu = 4 degrees of freedom, here the Sampson distance r of normalised correspondences, computed from
scipy.special's regularised incomplete gamma functions. sigma = sigma_max = the normalised RANSAC threshold
(pose_solver.py:43; DESIGN §3.4 records the probe that confirms this reading):

    x = r^2 / (2 sigma^2),  x_k = k^2 / 2,  G_k = Gamma(1.5, x_k)
    rho(r) = (C 2^2.5 / sigma) [ sigma^2 / 2 gamma(2.5, x) + r^2 / 4 (Gamma(1.5, x) - G_k) ]    r < k sigma
           = rho(k sigma)                                                                        beyond
    w(r)   = rho'(r) / r = (C 2^1.5 / sigma) (Gamma(1.5, x) - G_k)   r < k sigma, else 0
"""
import numpy as np
from scipy import special

from oracle import pose_solver_oracle as po

NU = 4
C = 1.0 / (2.0 ** (NU / 2) * special.gamma(NU / 2))      # 0.25
K = 3.64                                                  # 0.99 quantile of chi_4, as OpenCV's USAC carries it


def upper_gamma(a, x):
    """Gamma(a, x), not regularised."""
    return special.gammaincc(a, x) * special.gamma(a)


def lower_gamma(a, x):
    """gamma(a, x), not regularised."""
    return special.gammainc(a, x) * special.gamma(a)


G_K = upper_gamma(1.5, K * K / 2)


def rho(r, sigma):
    r = np.abs(np.asarray(r, np.float64))
    x = np.minimum(r, K * sigma) ** 2 / (2 * sigma * sigma)
    rc = np.minimum(r, K * sigma)
    return (C * 2 ** 2.5 / sigma) * (sigma * sigma / 2 * lower_gamma(2.5, x) + rc * rc / 4 * (upper_gamma(1.5, x) - G_K))


def weight(r, sigma):
    r = np.abs(np.asarray(r, np.float64))
    x = r * r / (2 * sigma * sigma)
    return np.where(r < K * sigma, (C * 2 ** 1.5 / sigma) * (upper_gamma(1.5, x) - G_K), 0.0)


def normalised(kpts0, kpts1, K0, K1, pix_threshold):
    """Normalised correspondences (fp64) and the normalised threshold sigma_max of pose_solver.py:39-43."""
    K0 = np.asarray(K0, np.float64); K1 = np.asarray(K1, np.float64)
    k0, k1 = po.normalise_kpts(np.asarray(kpts0, np.float64), np.asarray(kpts1, np.float64), K0, K1)
    return k0, k1, po.ransac_threshold(pix_threshold, K0, K1)


def sum_rho_E(E, k0, k1, sigma):
    """Sum of rho over normalised correspondences under an essential matrix E (row-major 3x3)."""
    r = np.sqrt(po.sampson_sq(np.asarray(E, np.float64).reshape(3, 3), k0, k1))
    return float(rho(r, sigma).sum())


def sum_rho(R, t, kpts0, kpts1, K0, K1, pix_threshold, sigma_scale=1.0):
    """Sum of rho of the pose (R, t) over pixel correspondences, sigma = sigma_scale * the normalised threshold."""
    k0, k1, thr = normalised(kpts0, kpts1, K0, K1, pix_threshold)
    return float(rho(po.sampson_residuals(R, t, k0, k1), thr * sigma_scale).sum())


def irls_polish(R, t, k0, k1, sigma, iters=100):
    """sigma-consensus++ polish of (R, unit t): iteratively reweighted least squares on the Sampson residuals with the
    weights w(r) of the current model, parameters = rotation increment + 2 tangent coordinates of t. Returns (R, t)."""
    from scipy.optimize import least_squares
    Rc, tc = np.asarray(R, np.float64), np.asarray(t, np.float64).ravel()
    tc = tc / np.linalg.norm(tc)
    for _ in range(iters):
        sw = np.sqrt(weight(po.sampson_residuals(Rc, tc, k0, k1), sigma))
        a = np.eye(3)[np.argmin(np.abs(tc))]
        b1 = np.cross(tc, a); b1 /= np.linalg.norm(b1)
        b2 = np.cross(tc, b1)
        R0, t0 = Rc, tc

        def unpack(p):
            tt = t0 + p[3] * b1 + p[4] * b2
            return po._expm_so3(p[:3]) @ R0, tt / np.linalg.norm(tt)

        sol = least_squares(lambda p: sw * po.sampson_residuals(*unpack(p), k0, k1), np.zeros(5), method="lm",
                            xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=200)
        Rc, tc = unpack(sol.x)
        if np.linalg.norm(sol.x) < 1e-13:
            break
    return Rc, tc
