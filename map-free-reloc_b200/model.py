"""Estimator shell with the reference's plugin surface (lib/models/matching/model.py:7-40,
lib/models/builder.py:8-10, lib/models/matching/feature_matching.py:5-50).

``FeatureMatchingModel(cfg).forward(data) -> (R float32 [1,3,3], t float32 [1,1,3])`` with the side
effect ``data['inliers']``; failure = NaN pose. Matchers implement ``get_correspondences(data)``,
solvers ``estimate_pose(kpts0, kpts1, data)``. All geometry runs in the CUDA back end.
"""
import numpy as np
import torch

from .pose_solver import EssentialMatrixMetricSolver, EssentialMatrixSolver, PnPSolver, ProcrustesSolver


class PrecomputedMatching:
    """Correspondences from the npz written by the offline matcher driver
    (feature_matching.py:5-50): float64 [Npairs, maxN, 4] NaN-padded, cast to float32 on load."""

    def __init__(self, cfg):
        self.correspondences = None
        self.debug = cfg.DEBUG
        if "{" in cfg.MATCHES_FILE_PATH:
            self.matches_file_path = cfg.MATCHES_FILE_PATH
            self.scene_id = None
            self.pairs_txt = cfg.DATASET.PAIRS_TXT.TEST
        else:
            self.load_correspondences(cfg.MATCHES_FILE_PATH)

    def load_correspondences(self, file_path):
        data = np.load(file_path, allow_pickle=True)
        self.correspondences = data["correspondences"].astype(np.float32)

    def get_correspondences(self, data):
        if hasattr(self, "scene_id"):
            if self.scene_id != data["scene_id"][0]:
                self.scene_id = data["scene_id"][0]
                self.load_correspondences(self.matches_file_path.format(
                    scene_root=data["scene_root"][0], pairs_txt=self.pairs_txt))
        pair_id = int(torch.as_tensor(data["pair_id"]).item())
        corr = self.correspondences[pair_id]
        corr = corr[~np.isnan(corr)].reshape(-1, 4)
        if len(corr) > 0:
            return corr[:, :2], corr[:, 2:]
        return np.array([]), np.array([])


def root_sift(descs):
    """Hellinger kernel: L1-normalise, square root (feature_matching.py:67-73)."""
    eps = 1e-7
    descs = descs / (descs.sum(axis=1, keepdims=True) + eps)
    return np.sqrt(descs)


def knn2_gpu(des0, des1):
    """Exact 2-NN of every row of des0 among des1 on the GPU -> (idx1, dist1, idx2, dist2) numpy."""
    from . import lib as _lib
    l = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    a = torch.as_tensor(np.ascontiguousarray(des0, dtype=np.float32)).to(dev)
    b = torch.as_tensor(np.ascontiguousarray(des1, dtype=np.float32)).to(dev)
    n = a.shape[0]
    i1 = torch.empty(n, dtype=torch.int32, device=dev); i2 = torch.empty(n, dtype=torch.int32, device=dev)
    d1 = torch.empty(n, device=dev); d2 = torch.empty(n, device=dev)
    _lib.check(l.mfr_knn2_l2(_lib.ptr(a), n, _lib.ptr(b), b.shape[0], a.shape[1], _lib.ptr(i1), _lib.ptr(d1),
                             _lib.ptr(i2), _lib.ptr(d2), _lib.cur_stream()), "mfr_knn2_l2")
    return i1.cpu().numpy(), d1.cpu().numpy(), i2.cpu().numpy(), d2.cpu().numpy()


def sift_matches_host(sift, img0, img1, ratio):
    """Matches of two uint8 gray images with OpenCV's detector ``sift`` (a cv2.SIFT), RootSIFT, the exact 2-NN on the GPU
    and Lowe's ratio test (feature_matching.py:75-118) -> (pts0, pts1) float32 [N, 2]."""
    kp0, des0 = sift.detectAndCompute(img0, None)
    kp1, des1 = sift.detectAndCompute(img1, None)
    if des0 is None or des1 is None or len(des1) < 2:
        return np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32)
    i1, d1, _, d2 = knn2_gpu(root_sift(des0), root_sift(des1))
    good = d1 < ratio * d2          # Lowe's ratio test (feature_matching.py:97-99)
    pts0 = np.float32([kp0[i].pt for i in np.where(good)[0]]).reshape(-1, 2)
    pts1 = np.float32([kp1[j].pt for j in i1[good]]).reshape(-1, 2)
    return pts0, pts1


def sift_matches_gpu(engines, img0, img1, nfeatures, ratio):
    """The same with detection, description and matching on the CUDA SIFT engine (mfr_b200.sift); ``engines`` caches
    one engine per frame shape. img0 and img1 (uint8 arrays or tensors) have the same shape."""
    from . import sift
    if img0.shape not in engines:
        engines[img0.shape] = sift.SIFT(2, img0.shape[0], img0.shape[1], nfeatures=nfeatures, root_sift=True)
    eng = engines[img0.shape]
    imgs = torch.stack([img0, img1]) if isinstance(img0, torch.Tensor) else torch.from_numpy(np.stack([img0, img1]))
    eng.detect(imgs.to(eng.device))
    k0, k1, _ = eng.match_pairs(ratio)
    return k0.cpu().numpy(), k1.cpu().numpy()


class SIFTMatching:
    """SIFT + RootSIFT + 2-NN ratio test (feature_matching.py:53-118). By default detection/description
    stays on OpenCV's CPU SIFT exactly as in the reference; with SIFT.GPU_DETECTOR the CUDA SIFT engine
    (mfr_b200.sift, one engine per frame size) detects, describes and matches on the device. The
    descriptor search runs on the GPU as an EXACT brute-force 2-NN instead of the reference's
    approximate, non-deterministic FLANN kd-tree."""

    def __init__(self, cfg):
        import cv2 as cv
        self.cv = cv
        self.ratio_threshold = cfg.SIFT.RATIO_THRESHOLD
        self.num_features = cfg.SIFT.NUM_FEATURES
        self.sift = cv.SIFT_create(cfg.SIFT.NUM_FEATURES)
        self.gpu_detector = bool(cfg.SIFT.get("GPU_DETECTOR", False))
        self.engines = {}
        self.debug = cfg.DEBUG

    def transform_grayscale(self, img):
        img = torch.as_tensor(img).permute(1, 2, 0).numpy()
        return self.cv.cvtColor((255 * img).astype(np.uint8), self.cv.COLOR_RGB2GRAY)

    def get_correspondences(self, data):
        img0 = self.transform_grayscale(torch.as_tensor(data["image0"]).squeeze(0))
        img1 = self.transform_grayscale(torch.as_tensor(data["image1"]).squeeze(0))
        if self.gpu_detector and img0.shape == img1.shape:
            return sift_matches_gpu(self.engines, img0, img1, self.num_features, self.ratio_threshold)
        return sift_matches_host(self.sift, img0, img1, self.ratio_threshold)


class LoFTRMatching:
    """Additive online matcher: runs the CUDA LoFTR engine on data['image0'/'image1'] (RGB float
    [1,3,H,W] in [0,1]) instead of reading a precomputed npz. Grayscale = the uint8 BT.601 conversion
    the reference's SIFT plugin applies (feature_matching.py:61-65), /255."""

    def __init__(self, cfg):
        from . import loftr, synth
        self._gray = synth.rgb_to_gray_u8
        h, w = loftr.engine_frame(int(cfg.DATASET.HEIGHT), int(cfg.DATASET.WIDTH))
        self.engine = loftr.LoFTR(loftr.load_weights(cfg.LOFTR.WEIGHTS), batch=1, height=h, width=w,
                                  cfg=loftr.engine_cfg(cfg))

    def get_correspondences(self, data):
        g0 = self._gray(torch.as_tensor(data["image0"]).squeeze(0).numpy()).astype(np.float32) / 255.0
        g1 = self._gray(torch.as_tensor(data["image1"]).squeeze(0).numpy()).astype(np.float32) / 255.0
        dev = self.engine.device
        out = self.engine.forward(torch.from_numpy(g0)[None].to(dev), torch.from_numpy(g1)[None].to(dev))
        if out["M"] == 0:
            return np.array([]), np.array([])
        return out["mkpts0_f"].cpu().numpy(), out["mkpts1_f"].cpu().numpy()


class FeatureMatchingModel(torch.nn.Module):
    def __init__(self, cfg):
        super().__init__()
        if cfg.FEATURE_MATCHING == "Precomputed":
            self.feature_matching = PrecomputedMatching(cfg)
        elif cfg.FEATURE_MATCHING == "LoFTR":
            self.feature_matching = LoFTRMatching(cfg)
        elif cfg.FEATURE_MATCHING == "SIFT":
            self.feature_matching = SIFTMatching(cfg)
        else:
            raise NotImplementedError("Invalid feature matching")
        if cfg.POSE_SOLVER == "EssentialMatrix":
            self.pose_solver = EssentialMatrixSolver(cfg)
        elif cfg.POSE_SOLVER == "EssentialMatrixMetric":
            self.pose_solver = EssentialMatrixMetricSolver(cfg)
        elif cfg.POSE_SOLVER == "PNP":
            self.pose_solver = PnPSolver(cfg)
        elif cfg.POSE_SOLVER == "Procrustes":
            self.pose_solver = ProcrustesSolver(cfg)
        else:
            raise NotImplementedError("Invalid pose solver")

    def forward(self, data):
        assert torch.as_tensor(data["depth0"]).shape[0] == 1, "Baseline models require batch size of 1"
        pts1, pts2 = self.feature_matching.get_correspondences(data)
        d = {k: (torch.as_tensor(v).squeeze(0) if k in ("K_color0", "K_color1", "depth0", "depth1") else v)
             for k, v in data.items()}
        R, t, inliers = self.pose_solver.estimate_pose(pts1, pts2, d)
        data["inliers"] = inliers
        R = torch.from_numpy(np.asarray(R, dtype=np.float64).copy()).unsqueeze(0).float()
        t = torch.from_numpy(np.asarray(t, dtype=np.float64).copy()).view(1, 3).unsqueeze(0).float()
        return R, t


def build_model(cfg, checkpoint=""):
    if cfg.MODEL == "FeatureMatching":
        return FeatureMatchingModel(cfg)
    raise NotImplementedError("only MODEL: 'FeatureMatching' is in scope (lib/models/builder.py:8-26)")
