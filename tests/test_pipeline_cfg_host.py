"""resolve_method maps each of the reference's 13 Map-free method configs (config/matching/mapfree/*.yaml, merged over
config/mapfree.yaml) to the streaming matcher, pose stage, thresholds and RANSAC settings (no GPU needed). The configs'
keys are restated here."""
import pytest

from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)
from mfr_b200 import config, pose_solver
from mfr_b200.pipeline import (EMatMetricStage, EMatStage, PnPStage, ProcrustesStage, resolve_method)

DATASET = {"DATA_SOURCE": "MapFree", "HEIGHT": 720, "WIDTH": 540}     # config/mapfree.yaml
EMAT = lambda pix: {"POSE_SOLVER": "EssentialMatrixMetric",
                    "EMAT_RANSAC": {"PIX_THRESHOLD": pix, "SCALE_THRESHOLD": 0.1, "CONFIDENCE": 0.9999}}
PNP = {"POSE_SOLVER": "PNP", "PNP": {"RANSAC_ITER": 1000, "REPROJECTION_INLIER_THRESHOLD": 3, "CONFIDENCE": 0.9999}}
PROC = {"POSE_SOLVER": "Procrustes", "PROCRUSTES": {"MAX_CORR_DIST": 0.05}}
CONFIGS = {
    "loftr_emat_dptkitti": ("LoFTR", "dptkitti", EMAT(2.0)), "loftr_emat_dptnyu": ("LoFTR", "dptnyu", EMAT(2.0)),
    "loftr_pnp_dptkitti": ("LoFTR", "dptkitti", PNP), "loftr_pnp_dptnyu": ("LoFTR", "dptnyu", PNP),
    "sg_emat_dptkitti": ("SG", "dptkitti", EMAT(2.0)), "sg_emat_dptnyu": ("SG", "dptnyu", EMAT(2.0)),
    "sg_pnp_dptkitti": ("SG", "dptkitti", PNP), "sg_pnp_dptnyu": ("SG", "dptnyu", PNP),
    "sg_procrustes_dptkitti": ("SG", "dptkitti", PROC),
    "sift_emat_dptkitti": ("SIFT", "dptkitti", EMAT(3.0)), "sift_emat_dptnyu": ("SIFT", "dptnyu", EMAT(3.0)),
    "sift_pnp_dptkitti": ("SIFT", "dptkitti", PNP), "sift_pnp_dptnyu": ("SIFT", "dptnyu", PNP),
}
# name -> matcher, solver, (height, width), thresholds, first budget
EXPECTED = {
    "emat2": ("EssentialMatrixMetric", {"pix_thr": 2.0, "scale_thr": 0.1}, 2048),
    "emat3": ("EssentialMatrixMetric", {"pix_thr": 3.0, "scale_thr": 0.1}, 2048),
    "pnp": ("PNP", {"reproj_thr": 3.0}, 1024),
    "proc": ("Procrustes", {"max_corr_dist": 0.05, "refine": False}, 2048),
}


def _cfg(name, extra=None):
    matcher, depth, solver = CONFIGS[name]
    cfg = config.get_default_cfg()
    cfg.merge_from_dict({"DATASET": DATASET})
    cfg.merge_from_dict({"MODEL": "FeatureMatching", "FEATURE_MATCHING": "Precomputed", "DATASET": {"ESTIMATED_DEPTH": depth},
                         "MATCHES_FILE_PATH": "{scene_root}/correspondences_" + matcher + ".npz", **solver})
    if extra:
        cfg.merge_from_dict(extra)
    return cfg


def _expected(name):
    kind = name.split("_")[1]
    return EXPECTED["emat3" if name.startswith("sift_emat") else {"emat": "emat2", "pnp": "pnp", "procrustes": "proc"}[kind]]


def test_thirteen_configs():
    assert len(CONFIGS) == 13


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_resolve_method(name):
    spec = resolve_method(_cfg(name))
    matcher = CONFIGS[name][0]
    solver, thr, budget = _expected(name)
    assert (spec.matcher, spec.solver, spec.num_hyp, spec.seed) == (matcher, solver, budget, pose_solver.DEFAULT_SEED)
    assert (spec.height, spec.width) == ((720, 544) if matcher == "LoFTR" else (720, 540))
    for k, v in thr.items():
        assert getattr(spec, k) == v, k
    assert spec.lo == pose_solver.LO_LSQ                      # LOCAL_OPTIMISATION on, FINAL_REFIT lsq by default
    if matcher == "SIFT":
        assert (spec.sift_features, spec.sift_ratio) == (2048, 0.8)
    else:
        assert spec.sift_features is None
    stage = spec.stage()
    cls = {"EssentialMatrixMetric": EMatMetricStage, "PNP": PnPStage, "Procrustes": ProcrustesStage}[solver]
    assert type(stage) is cls and stage.num_hyp == budget and stage.seed == spec.seed


def test_budget_matches_single_pair_plugins():
    """The stream's budget is the first launch budget of the single-pair plugins (pose_solver._SolverBase / PnPSolver)."""
    over = {"GPU_RANSAC": {"NUM_HYPOTHESES": 512, "SEED": 7, "LOCAL_OPTIMISATION": True, "FINAL_REFIT": "tukey"}}
    spec = resolve_method(_cfg("sg_emat_dptnyu", over))
    assert (spec.num_hyp, spec.seed, spec.lo) == (512, 7, pose_solver.LO_TUKEY)
    spec = resolve_method(_cfg("sift_pnp_dptkitti", {"GPU_RANSAC": {"LOCAL_OPTIMISATION": False}, "PNP": {"RANSAC_ITER": 300}}))
    assert (spec.num_hyp, spec.lo) == (384, 0)
    spec = resolve_method(_cfg("sg_procrustes_dptkitti", {"PROCRUSTES": {"REFINE": True}}))
    assert spec.refine and spec.stage().refine


def test_other_entry_points():
    """FEATURE_MATCHING 'LoFTR' / 'SIFT' select the matcher without a matches file; EssentialMatrix is the scale-free
    stage; SIFT keys and the frame come from the config."""
    cfg = config.get_default_cfg()
    cfg.merge_from_dict({"FEATURE_MATCHING": "SIFT", "POSE_SOLVER": "EssentialMatrix",
                         "SIFT": {"NUM_FEATURES": 1000, "RATIO_THRESHOLD": 0.7},
                         "EMAT_RANSAC": {"PIX_THRESHOLD": 1.5}, "DATASET": {"HEIGHT": 480, "WIDTH": 640}})
    spec = resolve_method(cfg)
    assert (spec.matcher, spec.solver, spec.height, spec.width) == ("SIFT", "EssentialMatrix", 480, 640)
    assert (spec.sift_features, spec.sift_ratio, spec.pix_thr) == (1000, 0.7, 1.5)
    assert type(spec.stage()) is EMatStage
    cfg.merge_from_dict({"FEATURE_MATCHING": "LoFTR", "DATASET": {"HEIGHT": 720, "WIDTH": 540}})
    assert (resolve_method(cfg).matcher, resolve_method(cfg).width) == ("LoFTR", 544)


@pytest.mark.parametrize("over", [{"FEATURE_MATCHING": "ORB"}, {"FEATURE_MATCHING": None, "MATCHES_FILE_PATH": None},
                                  {"MATCHES_FILE_PATH": "{scene_root}/correspondences_ORB.npz"},
                                  {"POSE_SOLVER": "Homography"}, {"POSE_SOLVER": None}])
def test_unknown_names_raise(over):
    with pytest.raises(NotImplementedError):
        resolve_method(_cfg("sg_emat_dptkitti", over))
