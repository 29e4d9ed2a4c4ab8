"""Config surface of the estimator (reference: config/default.py:1-116, config/matching/**/*.yaml,
config/mapfree.yaml). The reference uses a global yacs CfgNode; yacs is not a dependency here, so
this is a small attribute-dict with the same keys, the same layered ``merge_from_file`` semantics
(dataset yaml first, method yaml second, submission.py:70-71) and the same rule that only
pre-declared keys may be set. The reference's yaml files load unchanged.

Additive keys (not in the reference): FEATURE_MATCHING may also be 'LoFTR' (fused on-GPU matcher),
LOFTR.{WEIGHTS, THR, BORDER_RM, TEMPERATURE, BATCH}, GPU_RANSAC.{NUM_HYPOTHESES, MAX_HYPOTHESES, SEED,
LOCAL_OPTIMISATION, FINAL_REFIT, SCORING}, SIFT.GPU_DETECTOR (False: OpenCV's host SIFT as in the reference; True: the CUDA
SIFT engine detects, describes and ratio-matches on the device).
"""
import copy

import yaml


class CfgNode(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v

    def clone(self):
        return copy.deepcopy(self)

    def merge_from_dict(self, d, _path=""):
        for k, v in d.items():
            if k not in self:
                raise KeyError(f"Non-existent config key: {_path}{k}")
            if isinstance(self[k], CfgNode):
                if not isinstance(v, dict):
                    raise ValueError(f"{_path}{k} must be a mapping")
                self[k].merge_from_dict(v, _path + k + ".")
            else:
                # the reference's yamls spell None as the string 'None' (config/mapfree.yaml:4-6)
                self[k] = None if v == "None" else v
        return self

    def merge_from_file(self, path):
        with open(path) as f:
            d = yaml.safe_load(f) or {}
        return self.merge_from_dict(d)


def _node(d):
    n = CfgNode()
    for k, v in d.items():
        n[k] = _node(v) if isinstance(v, dict) else v
    return n


def get_default_cfg():
    """Keys of config/default.py that the feature-matching path reads (+ the additive GPU keys)."""
    return _node({
        "MODEL": None, "DEBUG": False,
        "FEATURE_MATCHING": None, "POSE_SOLVER": None,
        "SIFT": {"NUM_FEATURES": None, "RATIO_THRESHOLD": None, "GPU_DETECTOR": False},
        "MATCHES_FILE_PATH": None,
        "EMAT_RANSAC": {"PIX_THRESHOLD": None, "SCALE_THRESHOLD": None, "CONFIDENCE": None},
        "PROCRUSTES": {"MAX_CORR_DIST": None, "REFINE": False},
        "PNP": {"RANSAC_ITER": None, "REPROJECTION_INLIER_THRESHOLD": None, "CONFIDENCE": None},
        "DATASET": {"DATA_SOURCE": None, "SCENES": None, "DATA_ROOT": None, "NPZ_ROOT": None,
                    "MIN_OVERLAP_SCORE": None, "MAX_OVERLAP_SCORE": None, "AUGMENTATION_TYPE": None,
                    "BLACK_WHITE": False, "PAIRS_TXT": {"TRAIN": None, "VAL": None, "TEST": None, "ONE_NN": False},
                    "HEIGHT": None, "WIDTH": None, "ESTIMATED_DEPTH": None, "QUERY_FRAME_COUNT": 1},
        "TRAINING": {"BATCH_SIZE": None, "NUM_WORKERS": None, "SAMPLER": None, "N_SAMPLES_SCENE": None,
                     "SAMPLE_WITH_REPLACEMENT": None, "LR": None, "LR_STEP_INTERVAL": None,
                     "LR_STEP_GAMMA": None, "VAL_INTERVAL": None, "VAL_BATCHES": None, "LOG_INTERVAL": None,
                     "EPOCHS": None, "GRAD_CLIP": 0.0, "ROT_LOSS": "rot_frobenius_loss",
                     "TRANS_LOSS": "trans_l2_loss", "LAMBDA": 1.0},
        # regression-model keys are declared (so the reference's yamls merge) but unused here
        "ENCODER": {"TYPE": None, "NUM_BLOCKS": None, "BLOCK_TYPE": None, "NOT_CONCAT": None, "NUM_OUT_LAYERS": None},
        "AGGREGATOR": {"TYPE": None, "POSITION_ENCODER": None, "POSITION_ENCODER_IM1": None,
                       "MAX_SCORE_CHANNEL": None, "NORMALISE_DOT": False, "RESIDUAL_ATT": False,
                       "CV_OUTLAYERS": 0, "CV_HALF_CHANNELS": False, "UPSAMPLE_POS_ENC": 0, "DUSTBIN": False},
        "HEAD": {"TYPE": None, "ADD_BASIS": False, "NUM_PTS": 6, "AVG_POOL": False, "BATCH_NORM": True,
                 "SEPARATE_SCALE": True},
        "BACKPROJECT_ANCHORS": None,
        # additive
        "LOFTR": {"WEIGHTS": None, "THR": 0.2, "BORDER_RM": 2, "TEMPERATURE": 0.1, "BATCH": 1},
        # NUM_HYPOTHESES None = the solver's default (E-mat 2048; PnP: PNP.RANSAC_ITER rounded up to 128);
        # MAX_HYPOTHESES bounds the CONFIDENCE-driven escalation of the solver plugins (pose_solver._SolverBase) and of
        # the stream when it is asked to escalate (pipeline.from_cfg(..., escalate=True), decided per pair on the device)
        # SCORING: objective of the E-mat RANSAC, 'msac' (MSAC + Tukey LO, as LOCAL_OPTIMISATION / FINAL_REFIT say) or
        # 'magsac' (MAGSAC++ scoring with sigma-consensus++, the estimator of the reference's USAC_MAGSAC; LO keys at
        # their defaults)
        "GPU_RANSAC": {"NUM_HYPOTHESES": None, "MAX_HYPOTHESES": 32768, "SEED": 0x5EED, "LOCAL_OPTIMISATION": True,
                       "FINAL_REFIT": "lsq", "SCORING": "msac"},
    })


def load_cfg(*yaml_paths, overrides=None):
    cfg = get_default_cfg()
    for p in yaml_paths:
        cfg.merge_from_file(p)
    if overrides:
        cfg.merge_from_dict(overrides)
    return cfg
