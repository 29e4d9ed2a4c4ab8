"""Offline matcher plugins + registry with the reference's interface
(etc/feature_matching_baselines/matchers.py, compute.py:10): ``X_matcher(resize, outdoor)`` with
``match((path0, path1)) -> float [N,4] (x0,y0,x1,y1)`` or ``np.full((1,4), nan)``; ``stack_pts``
packs a scene's pairs into the NaN-padded [Npairs, maxN, 4] float64 array the online
``PrecomputedMatching`` plugin reads (etc/feature_matching_baselines/utils.py:59-69)."""
import numpy as np

from . import image_io
from .loftr import LoFTR_matcher
from .model import sift_matches_gpu, sift_matches_host
from .spsg import SuperGlue_matcher


class SIFT_matcher:
    """matchers.py:123-188: 2048 SIFT features, RootSIFT, 2-NN + ratio 0.8 (exact NN on the GPU).
    gpu_detector=True: detection, description and matching run on the CUDA SIFT engine (mfr_b200.sift); JPEG frames whose
    size equals ``resize`` are also decoded on the GPU (image_io.decode_jpegs, cv2.imread's pixels)."""

    def __init__(self, resize, outdoor=False, gpu_detector=False):
        self.resize = resize
        self.gpu_detector = gpu_detector
        self.engines = {}

    def match(self, pair_path):
        import cv2
        if self.gpu_detector and all(image_io.jpeg_size(p) == tuple(self.resize) for p in pair_path):
            # resize = the image size (Map-free frames: cv2.resize is a copy): decode on the GPU, cv2's exact pixels;
            # other sizes keep cv2.resize on the host, whose dispatched uint8 path the GPU resize does not restate
            img0, img1 = image_io.decode_jpegs(list(pair_path))
            if img0 is not None and img1 is not None:
                return self.match_arrays_gpu(img0, img1)
        img0 = cv2.resize(cv2.imread(pair_path[0], 0), self.resize)
        img1 = cv2.resize(cv2.imread(pair_path[1], 0), self.resize)
        if self.gpu_detector and img0.shape == img1.shape:
            return self.match_arrays_gpu(img0, img1)
        sift = cv2.SIFT_create(2048)
        return self.match_arrays(sift, img0, img1)

    def match_arrays_gpu(self, img0, img1, ratio=0.8):
        return _rows(*sift_matches_gpu(self.engines, img0, img1, 2048, ratio))

    @staticmethod
    def match_arrays(sift, img0, img1, ratio=0.8):
        return _rows(*sift_matches_host(sift, img0, img1, ratio))


def _rows(pts0, pts1):
    """The plugins' result: [N, 4] rows (x0, y0, x1, y1), or np.full((1, 4), nan) when there is no match."""
    if len(pts0) == 0:
        return np.full((1, 4), np.nan)
    return np.concatenate([pts0, pts1], axis=1)


MATCHERS = {"LoFTR": LoFTR_matcher, "SG": SuperGlue_matcher, "SIFT": SIFT_matcher}


def stack_pts(pts_list):
    assert len(pts_list) > 0, "list must not be empty"
    n, m, d = len(pts_list), max(p.shape[0] for p in pts_list), pts_list[0].shape[1]
    out = np.full((n, m, d), np.nan)
    for i, p in enumerate(pts_list):
        out[i, : p.shape[0]] = p
    return out
