"""The metrics oracle (oracle/metrics_oracle.py) against the reference's OWN tests for this code
(benchmark/test_metrics.py: properties of trans_err / rot_err / reproj_err and the known-answer vectors of
test_projection, replayed here with seeded randomness), and against the outputs of the reference module itself on seeded random poses,
stored in tests/golden/metrics_reference.npz."""
import sys
import types

import numpy as np
import pytest

from helpers import ROOT  # noqa: F401
from oracle import metrics_oracle as mo, ref_import

K0 = np.array([[590.0, 0, 270.0], [0, 590.0, 360.0], [0, 0, 1]])


def _rq(rng):
    return mo.euler2quat(*rng.uniform(0, 2 * np.pi, 3))


def test_reference_test_vectors_projection():            # benchmark/test_metrics.py:188-199
    xyz = np.array(((10, 20, 30), (10, 30, 50), (-20, -15, 5), (-20, -50, 10)), dtype=np.float32)
    uv = np.array(((1 / 3, 2 / 3), (1 / 5, 3 / 5), (-4, -3), (-2, -5)), dtype=np.float32)
    assert np.allclose(uv, mo.project(xyz, np.eye(3)))
    uv = np.array(((1 / 3, 2 / 3), (1 / 5, 3 / 5), (0, 0), (0, 0)), dtype=np.float32)
    assert np.allclose(uv, mo.project(xyz, np.eye(3), img_size=(5, 5)))


def test_reference_properties():
    rng = np.random.default_rng(0)
    for _ in range(50):
        t0, d = rng.normal(5, 10, 3), rng.normal(5, 10, 3)          # test_t_err_tinvariance
        q = _rq(rng)
        m = mo.pose_metrics(q, t0, q, t0 + d, K0, 540, 720)
        assert np.isclose(m["trans_err"], np.linalg.norm(d))
        axis = rng.uniform(-1, 1, 3); ang = rng.uniform(-np.pi, np.pi)      # test_rot_err_raxis
        qres = mo.axangle2quat(axis, ang)
        assert np.isclose(mo.quat_angle_error(label=mo.qmult(q, qres), pred=q), abs(np.degrees(ang)), rtol=1e-5, atol=1e-8)
        q1 = _rq(rng)                                                       # test_r_err_mat
        Rres = mo.quat2mat(q1) @ mo.quat2mat(q).T
        assert np.isclose(np.degrees(np.arccos(np.clip((np.trace(Rres) - 1) / 2, -1, 1))), mo.quat_angle_error(label=q1, pred=q))
    q, t = _rq(rng), rng.normal(0, 10, 3)                                   # test_reproj_error_identity
    assert np.isclose(mo.reprojection_error(q, t, q, t, np.eye(3), 1, 1), 0)
    for scale in np.logspace(-1, -9, 9):                                    # test_r_err_small
        q = _rq(rng); ang = rng.uniform(-np.pi, np.pi) * scale
        e = mo.quat_angle_error(label=mo.qmult(q, mo.axangle2quat(rng.uniform(-1, 1, 3), ang)), pred=q)
        assert np.isclose(e, abs(np.degrees(ang)), rtol=0.1 * scale, atol=0.1 * scale)


def test_precision_recall_small_case():
    # 4 estimates + 1 failure; confidences 9, 7, 7, 2; true positives 1, 0, 1, 1
    prec, rec, ap = mo.precision_recall([7, 9, 2, 7], [0, 1, 1, 1], 1)
    assert np.allclose(rec, [0.8, 0.6, 0.2, 0.0]) and np.allclose(prec, [0.75, 2 / 3, 1.0, 1.0])
    assert np.isclose(ap, 0.2 * 0.75 + 0.4 * 2 / 3 + 0.2 * 1.0)


def _cases():
    """40 seeded (q_gt, t_gt, q_est, t_est, confidence) cases around a ground-truth pose."""
    rng = np.random.default_rng(1)
    out = []
    for _ in range(40):
        qg = _rq(rng)
        qe = mo.qmult(qg, mo.axangle2quat(rng.uniform(-1, 1, 3), rng.uniform(0, 0.3)))
        tg = rng.normal(0, 1, 3); te_ = tg + rng.normal(0, 0.2, 3)
        out.append((qg, tg, qe, te_, float(rng.integers(0, 50))))
    return out


def _tp(trans_err, rot_err):
    return (np.array(trans_err) < 0.25) * (np.array(rot_err) < 5)


def reference_outputs():
    """The reference's MetricManager and precision_recall (benchmark/metrics.py, benchmark/utils.py) on _cases(), imported
    from the unmodified reference tree (tests/golden/make_golden.py stores the result in metrics_reference.npz);
    transforms3d, which the reference imports, is stood in for by the oracle's restatement of its quaternion helpers."""
    t3d = types.ModuleType("transforms3d"); tq = types.ModuleType("transforms3d.quaternions"); te = types.ModuleType("transforms3d.euler")
    for n in ("quat2mat", "qmult", "qinverse", "rotate_vector", "axangle2quat"):
        setattr(tq, n, getattr(mo, n))
    te.euler2quat = mo.euler2quat
    t3d.quaternions, t3d.euler = tq, te
    saved = {k: sys.modules.get(k) for k in ("transforms3d", "transforms3d.quaternions", "transforms3d.euler")}
    sys.modules.update({"transforms3d": t3d, "transforms3d.quaternions": tq, "transforms3d.euler": te})
    sys.path.insert(0, ref_import.REF)
    try:
        from benchmark.metrics import Inputs, MetricManager
        from benchmark.utils import precision_recall
        res = {"trans_err": [], "rot_err": [], "reproj_err": [], "confidence": []}
        mm = MetricManager()
        for qg, tg, qe, te_, conf in _cases():
            mm(Inputs(q_gt=qg, t_gt=tg, q_est=qe, t_est=te_, confidence=conf, K=K0, W=540, H=720), res)
        prec, rec, ap = precision_recall(res["confidence"], _tp(res["trans_err"], res["rot_err"]), 3)
        out = {k: np.asarray(v, dtype=np.float64) for k, v in res.items()}
        out.update(pr_precision=np.asarray(prec, dtype=np.float64), pr_recall=np.asarray(rec, dtype=np.float64),
                   pr_ap=np.float64(ap))
        return out
    finally:
        sys.path.remove(ref_import.REF)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k == "benchmark" or k.startswith("benchmark.")]:
            sys.modules.pop(k)


def test_oracle_equals_reference_module():
    """The oracle against the reference module's outputs on the same 40 cases (tests/golden/metrics_reference.npz)."""
    import os
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics_reference.npz"))
    ours = {k: [] for k in ("trans_err", "rot_err", "reproj_err", "confidence")}
    for qg, tg, qe, te_, conf in _cases():
        m = mo.pose_metrics(qg, tg, qe, te_, K0, 540, 720)
        for k in ("trans_err", "rot_err", "reproj_err"):
            ours[k].append(m[k])
        ours["confidence"].append(conf)
    for k in ours:
        assert np.allclose(G[k], ours[k], rtol=1e-10, atol=1e-10), k
    prec, rec, ap = mo.precision_recall(ours["confidence"], _tp(ours["trans_err"], ours["rot_err"]), 3)
    assert np.allclose(G["pr_precision"], prec) and np.allclose(G["pr_recall"], rec) and np.isclose(G["pr_ap"], ap)
