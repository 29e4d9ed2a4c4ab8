"""CPU unit tests of the minimal solvers that run inside the RANSAC kernels (same __host__ __device__
code through the host test hooks)."""
import ctypes

import cv2
import numpy as np

from helpers import synth
from mfr_b200 import lib

L = lib.load()


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def test_poly_real_roots():
    rng = np.random.default_rng(0)
    for _ in range(500):
        deg = int(rng.integers(1, 11))
        nreal = int(rng.integers(0, deg + 1))
        roots = list(rng.uniform(-3, 3, nreal))
        coef = np.array([1.0])
        for r in roots:
            coef = np.convolve(coef, [-r, 1.0])
        while len(coef) - 1 < deg:
            if deg - (len(coef) - 1) >= 2:
                a, b = rng.uniform(-2, 2), rng.uniform(0.3, 2)
                coef = np.convolve(coef, [a * a + b * b, -2 * a, 1.0])
            else:
                r = rng.uniform(-3, 3); roots.append(r); coef = np.convolve(coef, [-r, 1.0])
        coef = np.ascontiguousarray(coef * rng.uniform(0.1, 10))
        out = np.zeros(10)
        n = L.mfr_host_poly_real_roots(P(coef), deg, P(out))
        rt = np.sort(roots)
        assert n == len(rt)
        if n:
            assert np.abs(out[:n] - rt).max() < 1e-5


def _essential(R, t):
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    E = (tx @ R).ravel()
    return E / np.linalg.norm(E)


def test_five_point_contains_ground_truth_and_agrees_with_opencv():
    rng = np.random.default_rng(1)
    hits = 0
    trials = 200
    cv_total = cv_matched = 0
    for _ in range(trials):
        R, t = synth.random_pose(rng)
        X = np.c_[rng.uniform(-2, 2, 5), rng.uniform(-2, 2, 5), rng.uniform(2, 8, 5)]
        X1 = X @ R.T + t
        x0 = np.ascontiguousarray(X[:, :2] / X[:, 2:]); x1 = np.ascontiguousarray(X1[:, :2] / X1[:, 2:])
        E = np.zeros((10, 9))
        n = L.mfr_host_five_point(P(x0), P(x1), P(E))
        assert 0 <= n <= 10
        Et = _essential(R, t)
        h0 = np.c_[x0, np.ones(5)]; h1 = np.c_[x1, np.ones(5)]
        for i in range(n):   # every returned model satisfies the five epipolar constraints
            assert np.abs(np.einsum("ni,ij,nj->n", h1, E[i].reshape(3, 3), h0)).max() < 1e-8
            s = np.linalg.svd(E[i].reshape(3, 3), compute_uv=False)
            assert abs(s[0] - s[1]) < 1e-3 * s[0] and s[2] < 1e-3 * s[0]   # essential-matrix structure (ill-conditioned samples are looser)
        if n and min(min(np.abs(E[i] - Et).max(), np.abs(E[i] + Et).max()) for i in range(n)) < 1e-5:
            hits += 1
        # the reference's minimal solver (OpenCV five-point) returns the same candidate set
        Ecv, _ = cv2.findEssentialMat(x0, x1, np.eye(3), method=cv2.RANSAC, threshold=1e-3, prob=0.5)
        if Ecv is not None and n:
            for Ek in np.split(Ecv, len(Ecv) // 3):
                ek = Ek.ravel() / np.linalg.norm(Ek)
                d = min(min(np.abs(E[i] - ek).max(), np.abs(E[i] + ek).max()) for i in range(n))
                cv_total += 1
                cv_matched += d < 1e-4
                assert d < 1e-2
    assert hits >= 0.97 * trials
    assert cv_matched >= 0.97 * cv_total   # ill-conditioned samples differ in the 4th digit


def test_p3p_contains_ground_truth():
    rng = np.random.default_rng(2)
    hits = 0
    for _ in range(300):
        R, t = synth.random_pose(rng)
        X = np.ascontiguousarray(np.c_[rng.uniform(-2, 2, 3), rng.uniform(-2, 2, 3), rng.uniform(2, 8, 3)])
        Y = X @ R.T + t
        f = np.ascontiguousarray(Y / np.linalg.norm(Y, axis=1, keepdims=True))
        Ro = np.zeros((4, 9)); to = np.zeros((4, 3))
        n = L.mfr_host_p3p(P(X), P(f), P(Ro), P(to))
        for i in range(n):
            Ri = Ro[i].reshape(3, 3)
            assert np.abs(Ri @ Ri.T - np.eye(3)).max() < 1e-9 and np.linalg.det(Ri) > 0
            Yi = X @ Ri.T + to[i]
            fi = Yi / np.linalg.norm(Yi, axis=1, keepdims=True)
            assert np.abs(fi - f).max() < 1e-6      # every solution reprojects onto the bearings
        if any(np.abs(Ro[i].reshape(3, 3) - R).max() < 1e-6 and np.abs(to[i] - t).max() < 1e-6 for i in range(n)):
            hits += 1
    assert hits >= 295


def test_decompose_essential():
    rng = np.random.default_rng(3)
    for _ in range(50):
        R, t = synth.random_pose(rng)
        E = np.ascontiguousarray(_essential(R, t).reshape(3, 3) * rng.uniform(0.1, 5))
        R1 = np.zeros(9); R2 = np.zeros(9); tt = np.zeros(3)
        L.mfr_host_decompose_essential(P(E), P(R1), P(R2), P(tt))
        tn = t / np.linalg.norm(t)
        assert min(np.abs(R1.reshape(3, 3) - R).max(), np.abs(R2.reshape(3, 3) - R).max()) < 1e-9
        assert min(np.abs(tt - tn).max(), np.abs(tt + tn).max()) < 1e-9
        assert abs(np.linalg.det(R1.reshape(3, 3)) - 1) < 1e-9 and abs(np.linalg.det(R2.reshape(3, 3)) - 1) < 1e-9


def _kabsch(p, q):
    """mfr_host_kabsch on the moment sums of p, q [n, 3]: (ok, R, t)."""
    sp, sq = np.ascontiguousarray(p.sum(0)), np.ascontiguousarray(q.sum(0))
    spq = np.ascontiguousarray((p[:, :, None] * q[:, None, :]).sum(0).ravel())
    R, t = np.zeros(9), np.zeros(3)
    ok = L.mfr_host_kabsch(float(len(p)), P(sp), P(sq), P(spq), P(R), P(t))
    return ok, R.reshape(3, 3), t


def _kabsch_bar(p, q):
    """Error bound of a rotation from the moment sums: the sums carry a rounding error of a few ulps of their scale
    (n |pb| |qb| for a cloud far from the origin), which moves the singular vectors by that over the gap between the
    second and third singular values of the centred H."""
    pb, qb = p.mean(0), q.mean(0)
    spq = (p[:, :, None] * q[:, None, :]).sum(0)
    scale = len(p) * np.linalg.norm(pb) * np.linalg.norm(qb) + np.linalg.norm(spq)
    s = np.linalg.svd((p - pb).T @ (q - qb), compute_uv=False)
    return 16 * np.finfo(float).eps * scale / (s[1] - s[2])


def test_kabsch_matches_svd_where_htH_is_weakest():
    """kabsch_from_sums (the Procrustes hypotheses and refit, every ICP update) against SVD-based Kabsch
    (pose_solver_oracle.kabsch) on the inputs that break an eigen-decomposition of H^T H: exactly three points,
    near-collinear samples, a cloud 80 m away with a 5 cm spread, a reflection optimum."""
    from oracle import pose_solver_oracle as po
    rng = np.random.default_rng(4)
    cases = []
    for off, spread, n in [(0.0, 1.0, 3), (3.0, 0.5, 3), (80.0, 0.05, 3), (80.0, 0.05, 10), (80.0, 0.05, 1000),
                           (0.0, 1.0, 1000)]:
        cases += [(f"cloud {off} m / {spread} m / n {n}", rng.normal(0, spread, (n, 3)) + [0.0, 0.0, off])]
    for off in (0.0, 3.0, 80.0):
        for eps in (1e-3, 1e-4):
            d = rng.normal(0, 1, 3)
            cases += [(f"near-collinear {off} m / {eps}", np.outer(rng.normal(0, 1, 6), d) + [0.0, 0.0, off] +
                       rng.normal(0, eps, (6, 3)))]
    for name, p in cases:
        R0, t0 = synth.random_pose(rng)
        q = p @ R0.T + t0
        ok, R, t = _kabsch(p, q)
        Ro, to = po.kabsch(p, q)
        bar = _kabsch_bar(p, q)
        assert ok == 1, name
        assert np.abs(R @ R.T - np.eye(3)).max() < 1e-14 and np.linalg.det(R) > 0, name
        assert np.abs(R - Ro).max() <= bar, (name, np.abs(R - Ro).max(), bar)
        assert np.abs(t - to).max() <= bar * (1 + np.abs(p).max()) + 1e-14 * np.abs(to).max(), name
    # the least-squares optimum over O(3) is a reflection: both return the rotation that flips the weakest direction
    p = rng.normal(0, 1, (8, 3)) * [3.0, 2.0, 0.5]
    q = p * [1.0, 1.0, -1.0] + rng.normal(0, 0.01, (8, 3))
    ok, R, t = _kabsch(p, q)
    Ro, to = po.kabsch(p, q)
    assert ok == 1 and abs(np.linalg.det(R) - 1) < 1e-14 and np.abs(R - Ro).max() <= _kabsch_bar(p, q)


def test_kabsch_rejects_degenerate_sums():
    """Coincident points (at any distance from the origin, where the centred sums are rounding noise of a large
    scale), exactly collinear points and fewer than three points give false."""
    rng = np.random.default_rng(5)
    for off in (0.0, 0.5, 3.0, 80.0, 1000.0):
        R0, t0 = synth.random_pose(rng)
        p = np.tile(rng.normal(0, 1, 3) + [0.0, 0.0, off], (5, 1))
        assert _kabsch(p, p @ R0.T + t0)[0] == 0, ("coincident", off)
        p = np.outer(rng.normal(0, 1, 7), rng.normal(0, 1, 3)) + [0.0, 0.0, off]
        assert _kabsch(p, p @ R0.T + t0)[0] == 0, ("collinear", off)
    p = rng.normal(0, 1, (2, 3))
    assert _kabsch(p, p)[0] == 0
