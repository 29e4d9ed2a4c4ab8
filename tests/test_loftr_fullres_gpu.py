"""LoFTR CUDA engine at the BASELINE configuration (540x720 frames -> 720x544 engine frame, L = 6120 coarse cells,
B = 2) against vectors of the UNMODIFIED reference LoFTR on CPU fp32 (tests/golden/loftr_fullres_reference.npz), for
the three engine precisions and three weight sets:
  dense             seeded random weights, coarse threshold 0 (numerics through all 40+ layers at full size; the match
                    set itself is tiny: a random network has almost no mutual nearest neighbours)
  functional        the hand-constructed matcher weights of the benchmark's accuracy block, reference threshold 0.2
  functional_dense  the same + dense Gaussian perturbation = the weights of the throughput benchmark
Bars per precision: DESIGN.md §4."""
import pytest

from helpers import FULLRES_CASES, fullres_compare

pytestmark = pytest.mark.gpu

# precision -> (min match-set IoU on the functional weights, max |mkpts1_f| difference in px on common matches,
#               max relative error of the coarse tokens, max abs error of the sampled confidence matrix)
BARS = {"fp32x3": (0.995, 0.02, 5e-4, 1e-4), "tf32": (0.93, 0.3, 3e-2, 0.5), "bf16": (0.75, 2.0, 0.12, 1.0)}


@pytest.mark.parametrize("precision", ["fp32x3", "tf32", "bf16"])
@pytest.mark.parametrize("kind,thr", FULLRES_CASES)
def test_fullres_vs_reference(kind, thr, precision):
    iou_min, px_max, tok_max, conf_max = BARS[precision]
    for r in fullres_compare(kind, thr, precision, graph=(precision == "bf16")):
        assert r["tok_rel"] < tok_max, r
        assert r["conf_max_abs"] < conf_max, r
        if kind != "dense":
            assert r["M_ref"] > 500 and r["iou"] >= iou_min, r
            assert r["mkpts1_max_px"] < px_max, r
        elif precision == "fp32x3":
            assert r["iou"] == 1.0, r           # the handful of mutual nearest neighbours of the random network: identical
