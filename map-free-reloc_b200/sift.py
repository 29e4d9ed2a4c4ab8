"""Host side of the CUDA SIFT engine: ``SIFT(batch, height, width)`` detects, describes and ratio-matches keypoints
of uint8 gray images on the device, as cv2.SIFT_create(nfeatures).detectAndCompute + exact 2-NN + Lowe's ratio test
do on the host in the reference's SIFT plugins (lib/models/matching/feature_matching.py:53-118,
etc/feature_matching_baselines/matchers.py:123-188). ``SIFTPairs(batch, height, width)`` is the same engine as a pair
engine for ``pipeline.RelocPipeline``. All arithmetic runs in libmfr_b200.so; torch is used for device memory and
streams only. No CPU fallback."""
import ctypes

import numpy as np
import torch

from . import lib as _lib


class SIFT(_lib.Engine):
    """Engine for ``batch`` images of ``height`` x ``width`` on the current device, running on the caller's stream.
    ``nfeatures`` = 0 keeps every keypoint; otherwise OpenCV's retainBest (all keypoints whose response is >= the N-th
    largest). ``root_sift`` makes the descriptors RootSIFT rows. ``max_candidates`` bounds the refined extrema and the
    oriented keypoints per image; ``detect`` raises when an image has more."""

    def __init__(self, batch, height, width, nfeatures=2048, root_sift=False, max_candidates=32768, graph=True):
        self.B, self.H, self.W = int(batch), int(height), int(width)
        super().__init__("sift", "mfr_sift_create", (self.B, self.H, self.W, int(nfeatures), int(max_candidates),
                                                     int(bool(root_sift))), stream=False)
        self._l.mfr_sift_set_graph(self._h, int(bool(graph)))
        o = self._get_outputs(self._l.mfr_sift_get_outputs, _lib.SiftOutputs)
        self.cap = o.capacity
        B, cap = self.B, self.cap
        self._counts = self.view(o.extrema_counts, (3, B), torch.int32)   # rows: extrema, oriented, selected
        self._kp = self.view(o.keypoints, (B, cap, 5), torch.float32)
        self._oct = self.view(o.octaves, (B, cap), torch.int32)
        self._desc = self.view(o.descriptors, (B, cap, 128), torch.float32)

    @property
    def l(self):
        """The library, with ``h`` the handle: for calling mfr_sift_* directly, e.g. with caller-owned buffers."""
        return self._l

    @property
    def h(self):
        return self._h

    def octave_shapes(self):
        """(h, w) of every octave's levels, octave 0 = the doubled image."""
        shapes, h, w = [], 2 * self.H, 2 * self.W
        n = int(np.rint(np.log(min(h, w)) / np.log(2.0) - 2)) + 1
        for _ in range(n):
            shapes.append((h, w)); h //= 2; w //= 2
        return shapes

    def detect(self, imgs):
        """imgs: uint8 [B, H, W] CUDA tensor -> dict of device tensors: counts int32 [B], keypoints float32
        [B, cap, 5] (x, y, size, angle, response), octaves int32 [B, cap], descriptors float32 [B, cap, 128]; rows past
        counts[b] are unused. Also raw_counts / extrema_counts (before selection / orientation)."""
        if imgs.dtype != torch.uint8 or tuple(imgs.shape) != (self.B, self.H, self.W) or not imgs.is_cuda:
            raise ValueError(f"expected a uint8 CUDA tensor of shape {(self.B, self.H, self.W)}")
        imgs = imgs.contiguous()
        _lib.check(self._l.mfr_sift_detect(self._h, _lib.ptr(imgs), _lib.cur_stream()), "mfr_sift_detect")
        c = self._counts.cpu()
        if int(c[:2].max()) > self.cap:
            raise _lib.MfrError(f"SIFT candidates exceed max_candidates={self.cap}: extrema {c[0].tolist()}, "
                                f"oriented {c[1].tolist()}")
        return {"counts": self._counts[2], "raw_counts": self._counts[1], "extrema_counts": self._counts[0],
                "keypoints": self._kp, "octaves": self._oct, "descriptors": self._desc}

    def match_pairs(self, ratio):
        """Ratio-test matches of the last detect for pairs (2p, 2p + 1) -> (kpts0, kpts1 float32 [total, 2], offsets
        int32 [P + 1]) on the device, in query order: the pose back end's layout."""
        P = self.B // 2
        if P < 1 or self.B % 2:
            raise ValueError("match_pairs needs an even batch (pairs of images 2p, 2p + 1)")
        k0 = torch.empty(P * self.cap, 2, device=self.device); k1 = torch.empty_like(k0)
        off = torch.empty(P + 1, dtype=torch.int32, device=self.device)
        _lib.check(self._l.mfr_sift_match_pairs(self._h, float(ratio), _lib.ptr(k0), _lib.ptr(k1), _lib.ptr(off),
                                                _lib.cur_stream()), "mfr_sift_match_pairs")
        n = int(off[-1])
        return k0[:n], k1[:n], off

    def profile(self, imgs):
        """Eager detect with events between the stages -> dict of milliseconds."""
        ms = (ctypes.c_float * 5)()
        _lib.check(self._l.mfr_sift_profile(self._h, _lib.ptr(imgs.contiguous()), ms, _lib.cur_stream()),
                   "mfr_sift_profile")
        return dict(zip(("pyramid", "extrema", "orientation", "selection", "descriptors"), list(ms)))


class SIFTPairs(_lib.Engine):
    """Pair engine for ``batch`` pairs of ``height`` x ``width`` uint8 gray images (the bytes the reference's SIFT_matcher
    hands to cv2: ``imread(path, 0)`` then ``cv2.resize`` on uint8): detection, 2-NN and the ratio test of both images of
    every pair in one CUDA graph with no host synchronisation, matches in engine-owned buffers. Bit-identical to
    ``SIFT(2 * batch, ...).detect(interleaved)`` + ``match_pairs(ratio)``. ``root_sift=True`` is what the reference's
    SIFT plugins match on. When an image has more than ``max_candidates`` refined extrema or oriented keypoints, the
    pair's flag in ``overflow`` is set on the device (nothing is read on the host here)."""

    input_dtype = torch.uint8

    def __init__(self, batch, height, width, nfeatures=2048, ratio=0.8, root_sift=True, max_candidates=32768, device=0,
                 graph=True):
        self.B, self.H, self.W = int(batch), int(height), int(width)
        super().__init__("sift_pairs", "mfr_sift_pairs_create",
                         (self.B, self.H, self.W, int(nfeatures), int(max_candidates), int(bool(root_sift)), float(ratio)),
                         device)
        self._l.mfr_sift_pairs_set_graph(self._h, int(bool(graph)))
        o = self._get_outputs(self._l.mfr_sift_get_pair_outputs, _lib.SiftPairOutputs)
        self.capacity, self.max_pts_per_pair = o.capacity, o.max_pts_per_pair
        self._k0 = self.view(o.kpts0, (self.capacity, 2), torch.float32)
        self._k1 = self.view(o.kpts1, (self.capacity, 2), torch.float32)
        self._off = self.view(o.offsets, (self.B + 1,), torch.int32)
        self.overflow = self.view(o.overflow, (self.B,), torch.int32)

    def forward_async(self, img0, img1):
        """Enqueues one batch of pairs (uint8 CUDA [B,(1,)H,W] each) on the engine stream."""
        self._call(self._l.mfr_sift_forward_pairs, self._images(img0, self.B, self.H, self.W),
                   self._images(img1, self.B, self.H, self.W))

    def set_map(self, img0):
        """Detects and describes the map image img0 (uint8 CUDA [(1,)(1,)H,W]) once, eagerly, on the engine stream. Until
        the next set_map, ``forward_shared_async(img1)`` gives the bits ``forward_async`` gives with img0 repeated for every
        pair; a paired forward in between does not disturb the map."""
        self._call(self._l.mfr_sift_set_map, self._images(img0, self.H, self.W))

    def forward_shared_async(self, img1):
        """Enqueues one batch of B query images (uint8 CUDA [B,(1,)H,W]) against the map of ``set_map``."""
        self._call(self._l.mfr_sift_forward_shared, self._images(img1, self.B, self.H, self.W))

    def pose_inputs(self):
        """(kpts0 [capacity, 2], kpts1 [capacity, 2], offsets [B + 1]): device views of the last forward's matches."""
        return self._k0, self._k1, self._off
