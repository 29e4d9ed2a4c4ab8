"""Input path of the matcher plugins on the GPU (SURVEY §8(f) rank 1): JPEG decode with nvJPEG and the reference's
resize + normalise steps as CUDA kernels (libmfr_b200.so: mfr_jpeg_decode, mfr_resize_linear).

  read_image(path, resize, resize_float)   = SuperGlue/models/utils.py:263-285 (gray, cv2.resize, / 255) -> CUDA [h, w]
  read_color_image(path, resize)           = lib/datasets/utils.py:58-75 (RGB, uint8 cv2.resize, / 255)   -> CUDA [3, h, w]
  PairMatcher                              = match / match_scene / match_arrays of the LoFTR and SuperGlue plugins

JPEG files are decoded on the GPU (luma plane = OpenCV's IMREAD_GRAYSCALE of a JPEG, up to the +-1 level differences
between two IDCT implementations); other formats are decoded by OpenCV on the host and uploaded as uint8. The resize
kernels restate cv2.resize(INTER_LINEAR) for both of its arithmetic paths (tests/test_image_io_gpu.py: float path
within 1e-6 of cv2, uint8 path bit-exact)."""
import ctypes
import os

import numpy as np
import torch

from . import lib as _lib

MODE_F32, MODE_U8_AS_F32, MODE_U8_FIXED = 0, 1, 2


def _device(device):
    if not torch.cuda.is_available():
        raise _lib.MfrError("mfr_b200.image_io needs a CUDA device (no CPU fallback)")
    if isinstance(device, torch.device):
        return device
    return torch.device("cuda", torch.cuda.current_device() if device is None else int(device))


def decode_jpeg(data, rgb=False, device=None):
    """JPEG bytes (or a path) -> CUDA uint8 tensor [h, w] (luma) or [h, w, 3] (RGB)."""
    dev = _device(device)
    if not isinstance(data, (bytes, bytearray)):
        with open(data, "rb") as f:
            data = f.read()
    l = _lib.load()
    buf = (ctypes.c_ubyte * len(data)).from_buffer_copy(data)
    w, h, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(l.mfr_jpeg_info(buf, len(data), ctypes.byref(w), ctypes.byref(h), ctypes.byref(c)), "mfr_jpeg_info")
    out = torch.empty((h.value, w.value, 3) if rgb else (h.value, w.value), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(l.mfr_jpeg_decode(buf, len(data), int(rgb), _lib.ptr(out), w.value, h.value, _lib.cur_stream()), "mfr_jpeg_decode")
        torch.cuda.current_stream().synchronize()          # `buf` (host) must outlive the decode
    return out


def resize_linear(img, size, mode, out_scale=1.0, chw=False):
    """cv2.resize(img, size=(w, h), INTER_LINEAR) * out_scale on the device. img: CUDA uint8 / float32 [h, w] or [h, w, c]."""
    assert img.is_cuda and img.dtype in (torch.uint8, torch.float32)
    img = img.contiguous()
    sh, sw = img.shape[:2]
    c = 1 if img.dim() == 2 else img.shape[2]
    dw, dh = int(size[0]), int(size[1])
    shape = (c, dh, dw) if chw else ((dh, dw) if img.dim() == 2 else (dh, dw, c))
    out = torch.empty(shape, dtype=torch.float32, device=img.device)
    l = _lib.load()
    with torch.cuda.device(img.device):
        _lib.check(l.mfr_resize_linear(_lib.ptr(img), int(img.dtype == torch.uint8), sw, sh, sw * c, c, _lib.ptr(out), dw, dh, int(mode),
                                       float(out_scale), int(chw), _lib.cur_stream()), "mfr_resize_linear")
    return out


def _load_u8(path, rgb, device):
    p = str(path)
    if not os.path.isfile(p):
        return None                                  # cv2.imread's convention for unreadable files (utils.py:265-266)
    if p.lower().endswith((".jpg", ".jpeg")):
        try:
            return decode_jpeg(p, rgb=rgb, device=device)
        except _lib.MfrError:
            pass                                     # e.g. progressive / CMYK files nvJPEG's simple API rejects: decode on the host
    import cv2
    im = cv2.imread(p, cv2.IMREAD_COLOR if rgb else cv2.IMREAD_GRAYSCALE)
    if im is None:
        return None
    if rgb:
        im = np.ascontiguousarray(im[:, :, ::-1])    # lib/datasets/utils.py:7-17: BGR -> RGB
    return torch.from_numpy(im).to(_device(device))


def read_image(path, resize, resize_float=True, device=None):
    """Gray image, resized to resize = (w, h), in [0, 1]: CUDA float32 [h, w]; None if the file cannot be read
    (SuperGlue/models/utils.py:263-285 with rotation 0; `resize` given as the two-element form the FMB plugins use)."""
    im = _load_u8(path, False, device)
    if im is None:
        return None
    return resize_linear(im, resize, MODE_U8_AS_F32 if resize_float else MODE_U8_FIXED, 1.0 / 255.0)


class PairMatcher:
    """Body of the image-pair matcher plugins (loftr.LoFTR_matcher, spsg.SuperGlue_matcher) over a batch-1 pair engine:
    images read with ``read_image(path, resize, True)`` on the engine's device, results as the reference's plugins give
    them, float [N, 4] (x0, y0, x1, y1) or ``np.full((1, 4), nan)``. A subclass builds the engine and reads the matched
    keypoints of an engine output in ``_matches(out) -> (kpts0, kpts1)``."""

    def __init__(self, resize, engine):
        self.resize, self.engine = resize, engine

    def match(self, pair_path):
        """matchers.py:24-59 / 93-120; images decoded (JPEG: nvJPEG) and resized on the GPU."""
        return self._result(self.engine.forward(self._read(pair_path[0]), self._read(pair_path[1])))

    def match_scene(self, ref_path, query_paths):
        """``[self.match((ref_path, q)) for q in query_paths]``, array for array, with the reference image decoded and
        encoded once (Map-free: every pair of a scene shares its first image)."""
        self.engine.set_map(self._read(ref_path))
        return [self._result(self.engine.forward_shared(self._read(q))) for q in query_paths]

    def match_arrays(self, im0, im1):
        """``match`` on two gray float [h, w] arrays in [0, 1]."""
        dev = self.engine.device
        t0 = torch.from_numpy(np.ascontiguousarray(im0, dtype=np.float32))[None].to(dev)
        t1 = torch.from_numpy(np.ascontiguousarray(im1, dtype=np.float32))[None].to(dev)
        return self._result(self.engine.forward(t0, t1))

    def _read(self, path):
        return read_image(path, self.resize, True, self.engine.device)[None]

    def _result(self, out):
        kpts0, kpts1 = self._matches(out)
        if len(kpts0) > 0:
            return torch.cat([kpts0, kpts1], 1).cpu().numpy()
        return np.full((1, 4), np.nan)


def read_color_image(path, resize=(640, 480), device=None):
    """lib/datasets/utils.py:58-75: RGB, cv2.resize on uint8, (3, h, w) float in [0, 1]."""
    im = _load_u8(path, True, device)
    if im is None:
        return None
    return resize_linear(im, resize, MODE_U8_FIXED, 1.0 / 255.0, chw=True)
