"""Offline matcher plugins + registry with the reference's interface
(etc/feature_matching_baselines/matchers.py, compute.py:10): ``X_matcher(resize, outdoor)`` with
``match((path0, path1)) -> float [N,4] (x0,y0,x1,y1)`` or ``np.full((1,4), nan)``; ``stack_pts``
packs a scene's pairs into the NaN-padded [Npairs, maxN, 4] float64 array the online
``PrecomputedMatching`` plugin reads (etc/feature_matching_baselines/utils.py:59-69)."""
import numpy as np

from .loftr import LoFTR_matcher
from .model import knn2_gpu, root_sift
from .spsg import SuperGlue_matcher


class SIFT_matcher:
    """matchers.py:123-188: 2048 SIFT features, RootSIFT, 2-NN + ratio 0.8 (exact NN on the GPU).
    gpu_detector=True: detection, description and matching run on the CUDA SIFT engine (mfr_b200.sift)."""

    def __init__(self, resize, outdoor=False, gpu_detector=False):
        self.resize = resize
        self.gpu_detector = gpu_detector
        self.engines = {}

    def match(self, pair_path):
        import cv2
        img0 = cv2.resize(cv2.imread(pair_path[0], 0), self.resize)
        img1 = cv2.resize(cv2.imread(pair_path[1], 0), self.resize)
        if self.gpu_detector and img0.shape == img1.shape:
            return self.match_arrays_gpu(img0, img1)
        sift = cv2.SIFT_create(2048)
        return self.match_arrays(sift, img0, img1)

    def match_arrays_gpu(self, img0, img1, ratio=0.8):
        import torch
        from . import sift
        key = img0.shape
        if key not in self.engines:
            self.engines[key] = sift.SIFT(2, key[0], key[1], nfeatures=2048, root_sift=True)
        eng = self.engines[key]
        eng.detect(torch.from_numpy(np.stack([img0, img1])).to(eng.device))
        k0, k1, _ = eng.match_pairs(ratio)
        if k0.shape[0] == 0:
            return np.full((1, 4), np.nan)
        return torch.cat([k0, k1], 1).cpu().numpy()

    @staticmethod
    def match_arrays(sift, img0, img1, ratio=0.8):
        kp0, des0 = sift.detectAndCompute(img0, None)
        kp1, des1 = sift.detectAndCompute(img1, None)
        if des0 is None or des1 is None or len(des1) < 2:
            return np.full((1, 4), np.nan)
        i1, d1, _, d2 = knn2_gpu(root_sift(des0), root_sift(des1))
        good = d1 < ratio * d2
        if not good.any():
            return np.full((1, 4), np.nan)
        pts1 = np.float32([kp0[i].pt for i in np.where(good)[0]]).reshape(-1, 2)
        pts2 = np.float32([kp1[j].pt for j in i1[good]]).reshape(-1, 2)
        return np.concatenate([pts1, pts2], axis=1)


MATCHERS = {"LoFTR": LoFTR_matcher, "SG": SuperGlue_matcher, "SIFT": SIFT_matcher}


def stack_pts(pts_list):
    assert len(pts_list) > 0, "list must not be empty"
    n, m, d = len(pts_list), max(p.shape[0] for p in pts_list), pts_list[0].shape[1]
    out = np.full((n, m, d), np.nan)
    for i, p in enumerate(pts_list):
        out[i, : p.shape[0]] = p
    return out
