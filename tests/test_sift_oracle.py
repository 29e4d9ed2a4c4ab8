"""The numpy SIFT oracle (oracle/sift_oracle.py) against cv2.SIFT_create on synthetic frames (no GPU).

Every keypoint that only one side has must sit at a near-threshold decision (26-neighbour test, convergence of the
refinement, contrast, edge ratio, 0.8 orientation peak, retainBest cut); paired keypoints agree in every field and
descriptors agree component by component. Bars are at most 4x the maxima measured with OpenCV 4.13 on these frames."""
import cv2
import numpy as np
import pytest

from helpers import synth
from oracle import sift_oracle as so
from sift_compare import as_rows, cv_rows, errors, explain, pair

# measured maxima over the cases below (OpenCV 4.13): every keypoint paired; pt 3.1e-5 px, size 2.1e-7 rel,
# angle 1.6e-4 deg, response 1.2e-7 rel, descriptor 1 (of 255). A keypoint that only one side keeps must sit within
# MARGIN_BAR of a threshold (convergence margins of 2e-5..7e-5 were seen while the oracle's blur sigmas were off).
BARS = {"pt": 1.2e-4, "size": 8.4e-7, "angle": 6.4e-4, "response": 4.8e-7}
DESC_BAR = 2
MARGIN_BAR = 1e-4


def _frame(case):
    kind, i = case
    g = synth.rgb_to_gray_u8(synth.make_pair(i)["image0"])
    return np.ascontiguousarray(g[100:303, 50:207]) if kind == "crop" else g


@pytest.mark.parametrize("case,nfeatures", [(("full", 3), 0), (("full", 0), 2048), (("full", 1), 2048), (("crop", 5), 0)])
def test_oracle_matches_opencv(case, nfeatures):
    g = _frame(case)
    kps, des = cv2.SIFT_create(nfeatures).detectAndCompute(g, None)
    ok, od = so.detect_and_compute(g, nfeatures)
    a, aoct = cv_rows(kps)
    b, boct = as_rows(ok)
    m = pair(a, b)
    err = errors(a, b, m)
    gauss, dog = so.build_pyramid(g)
    cut = None
    if nfeatures and len(b) >= nfeatures:
        cut = float(np.sort(b[:, 4])[::-1][nfeatures - 1])
    worst = 0.0
    only_cv = np.nonzero(m < 0)[0]
    only_or = np.setdiff1d(np.arange(len(b)), m[m >= 0])
    for i in only_cv:
        mg, d = explain(so, gauss, dog, a[i], aoct[i], cut)
        print("cv2 only", a[i], d)
        worst = max(worst, mg)
    for j in only_or:
        mg, d = explain(so, gauss, dog, b[j], boct[j], cut)
        print("oracle only", b[j], d)
        worst = max(worst, mg)
    sel = m >= 0
    dd = np.abs(des[sel] - od[m[sel]]).max() if sel.any() else 0.0
    print(f"{case} n={nfeatures}: cv2 {len(a)} oracle {len(b)} paired {sel.sum()}; errors {err}; desc {dd}; "
          f"worst unexplained margin {worst:.2e}")
    assert sel.sum() >= 0.99 * max(len(a), len(b))
    for k, v in BARS.items():
        assert err[k] <= v, (k, err[k])
    assert dd <= DESC_BAR
    assert worst <= MARGIN_BAR
    # the octave field: octave and layer bytes exact, the sub-layer byte within one step
    x, y = aoct[sel], boct[m[sel]]
    assert np.array_equal(x & 0xFFFF, y & 0xFFFF)
    assert np.abs((x >> 16) - (y >> 16)).max() <= 1
    assert np.array_equal(np.sort(des[sel], axis=None).round(), np.sort(des[sel], axis=None))   # integer-valued


def test_oracle_edge_cases():
    flat = np.full((64, 80), 128, np.uint8)
    kp, d = so.detect_and_compute(flat, 0)
    assert len(kp["x"]) == 0 and d.shape == (0, 128)
    assert so.n_octaves(540, 720) == int(np.rint(np.log2(1080) - 2)) + 1
