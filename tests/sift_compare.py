"""Keypoint-set comparison shared by the SIFT tests: pairs keypoints of two detectors by position, size and angle, and
explains every unpaired keypoint with the margin of the closest threshold decision (oracle.sift_oracle.decision_margins)."""
import numpy as np
from scipy.spatial import cKDTree


def as_rows(kp):
    """dict of arrays (sift_oracle layout) -> float64 [n, 5] (x, y, size, angle, response), int [n] octave."""
    return np.stack([kp["x"], kp["y"], kp["size"], kp["angle"], kp["response"]], 1).astype(np.float64), np.asarray(kp["octave"])


def cv_rows(kps):
    return (np.array([[k.pt[0], k.pt[1], k.size, k.angle, k.response] for k in kps], np.float64).reshape(-1, 5),
            np.array([k.octave for k in kps], np.int64))


def pair(a, b, pt_tol=1e-2, size_rel=1e-3, angle_tol=1.0):
    """Greedy one-to-one pairing of rows of a with rows of b -> index array into b (-1 = unpaired)."""
    out = np.full(len(a), -1)
    if len(a) == 0 or len(b) == 0:
        return out
    tree = cKDTree(b[:, :2])
    used = np.zeros(len(b), bool)
    k = min(16, len(b))
    dist, idx = tree.query(a[:, :2], k=k)
    dist = dist.reshape(len(a), k); idx = idx.reshape(len(a), k)
    for i in range(len(a)):
        best, bj = None, -1
        for d, j in zip(dist[i], idx[i]):
            if d > pt_tol or used[j]:
                continue
            da = abs(a[i, 3] - b[j, 3]); da = min(da, 360 - da)
            if abs(a[i, 2] - b[j, 2]) > size_rel * a[i, 2] or da > angle_tol:
                continue
            score = d + da * 1e-3
            if best is None or score < best:
                best, bj = score, j
        if bj >= 0:
            used[bj] = True; out[i] = bj
    return out


def errors(a, b, m):
    """Max abs errors of paired rows: pt (px), size (relative), angle (deg), response (relative)."""
    sel = m >= 0
    if not sel.any():
        return {"pt": 0.0, "size": 0.0, "angle": 0.0, "response": 0.0}
    x, y = a[sel], b[m[sel]]
    da = np.abs(x[:, 3] - y[:, 3]); da = np.minimum(da, 360 - da)
    return {"pt": float(np.abs(x[:, :2] - y[:, :2]).max()), "size": float((np.abs(x[:, 2] - y[:, 2]) / x[:, 2]).max()),
            "angle": float(da.max()), "response": float((np.abs(x[:, 4] - y[:, 4]) / x[:, 4]).max())}


def explain(so, gauss, dog, row, octave, cut=None):
    """Smallest relative decision margin for an input-pixel keypoint (row, packed octave field) on a pyramid; with
    `cut` (the retainBest response), the relative distance of its response to the cut is a decision too."""
    o = int(octave) & 255
    o = o - 256 if o >= 128 else o
    oi, layer = o + 1, (int(octave) >> 8) & 255
    r = int(round(row[1] * 2 / 2 ** oi)); c = int(round(row[0] * 2 / 2 ** oi))
    m = so.decision_margins(gauss, dog, oi, layer, r, c, row[3])
    if cut is not None:
        m["retain_best"] = abs(row[4] - cut) / cut
    return min(m.values()), m
