"""Input path of the matcher plugins on the GPU (SURVEY §8(f) rank 1): JPEG decode and the reference's resize +
normalise steps as CUDA kernels (libmfr_b200.so: mfr_jpeg_decode_batch / mfr_jpeg_decode, mfr_png_decode_batch,
mfr_resize_linear).

  decode_jpegs(items, rgb)                 = [cv2.imread(p, GRAYSCALE or COLOR) for p in items], one batched GPU decode
  decode_pngs(items)                       = [cv2.imread(p, IMREAD_UNCHANGED) for p in items], one batched GPU decode
  read_depth_image(path) / read_depth_images(paths)
                                           = lib/datasets/utils.py:77-81 (IMREAD_UNCHANGED / 1000, .float()) -> CUDA [h, w] / [B, h, w]
  read_image(path, resize, resize_float)   = SuperGlue/models/utils.py:263-285 (gray, cv2.resize, / 255) -> CUDA [h, w]
  read_color_image(path, resize)           = lib/datasets/utils.py:58-75 (RGB, uint8 cv2.resize, / 255)   -> CUDA [3, h, w]
  PairMatcher                              = match / match_scene / match_arrays of the LoFTR and SuperGlue plugins

JPEG files are decoded on the GPU with libjpeg's arithmetic (csrc/jpeg.cuh): the bytes equal cv2.imread's (Exif
orientation included) for baseline / extended-sequential Huffman files, gray or YCbCr 4:4:4 / 4:2:2 / 4:2:0. Other files
(progressive, 4:1:1, CMYK, ... and other formats) are decoded by OpenCV on the host and uploaded as uint8, so every
loader returns cv2's pixels. Gray 8- / 16-bit PNGs (the depth maps) are inflated, unfiltered and converted on the GPU
(csrc/png.cuh); other PNGs, and files the device rejects (bad CRC, deflate data or Adler-32), go to OpenCV on the host.
The resize kernels restate cv2.resize(INTER_LINEAR) for both of its arithmetic paths
(tests/test_image_io_gpu.py: float path within 1e-6 of cv2, uint8 path bit-exact)."""
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


def _bytes(item):
    if isinstance(item, (bytes, bytearray, memoryview)):
        return bytes(item)
    with open(item, "rb") as f:
        return f.read()


def decode_jpeg(data, rgb=False, device=None):
    """JPEG bytes (or a path) -> CUDA uint8 tensor [h, w] (gray) or [h, w, 3] (RGB): cv2.imread's pixels. Raises
    MfrError for a file the GPU decoder does not take (mfr_jpeg_info's status) or whose data fails to decode."""
    dev = _device(device)
    data = _bytes(data)
    l = _lib.load()
    w, h, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(l.mfr_jpeg_info(data, len(data), ctypes.byref(w), ctypes.byref(h), ctypes.byref(c)), "mfr_jpeg_info")
    out = torch.empty((h.value, w.value, 3) if rgb else (h.value, w.value), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):     # returns once decoded: the bytes need not outlive the call
        _lib.check(l.mfr_jpeg_decode(data, len(data), int(rgb), _lib.ptr(out), w.value, h.value, _lib.cur_stream()), "mfr_jpeg_decode")
    return out


class _Decoder:
    """A batch decoder handle (mfr_jpeg_decoder_create / mfr_png_decoder_create) and its capacity."""

    def __init__(self, fmt, images, nbytes, pixels):
        self.fmt, self.caps = fmt, (images, nbytes, pixels)
        h = ctypes.c_void_p()
        _lib.check(getattr(_lib.load(), f"mfr_{fmt}_decoder_create")(images, nbytes, pixels, ctypes.byref(h)),
                   f"mfr_{fmt}_decoder_create")
        self.h = h

    def fits(self, images, nbytes, pixels):
        return all(a <= b for a, b in zip((images, nbytes, pixels), self.caps))

    def __del__(self):
        try:
            if getattr(self, "h", None):
                getattr(_lib.load(), f"mfr_{self.fmt}_decoder_destroy")(self.h)  # waits for the decoder's last batch
                self.h = None
        except Exception:
            pass                                          # interpreter shutdown: the module may be gone


_DECODERS = {}


def _decoder(fmt, dev, images, nbytes, pixels):
    """The decoder of format `fmt` ("jpeg" or "png") on `dev`, one per (format, device), grown on demand."""
    key = (fmt, dev.index)
    d = _DECODERS.get(key)
    if d is None or not d.fits(images, nbytes, pixels):
        old = d.caps if d is not None else (0, 0, 0)
        _DECODERS.pop(key, None)
        with torch.cuda.device(dev):
            d = _DECODERS[key] = _Decoder(fmt, max(images, old[0], 16), max(nbytes, old[1], 1 << 22),
                                          max(pixels, old[2], 1 << 22))
    return d


def _host_decode(item, rgb, dev):
    """cv2's decode of a file or bytes, uploaded (None if OpenCV cannot read it)."""
    import cv2
    flag = cv2.IMREAD_COLOR if rgb else cv2.IMREAD_GRAYSCALE
    if isinstance(item, (bytes, bytearray, memoryview)):
        im = cv2.imdecode(np.frombuffer(bytes(item), np.uint8), flag)
    else:
        im = cv2.imread(str(item), flag)
    if im is None:
        return None
    if rgb:
        im = np.ascontiguousarray(im[:, :, ::-1])    # lib/datasets/utils.py:7-17: BGR -> RGB
    return torch.from_numpy(im).to(dev)


def decode_jpegs(items, rgb=False, device=None):
    """JPEG files (bytes or paths) -> list of CUDA uint8 tensors [h, w] / [h, w, 3], cv2.imread's pixels, in one decoder
    call on the current stream. Files the GPU decoder does not take, or whose data it rejects, are decoded by OpenCV on
    the host in their place in the list (None where OpenCV cannot read them either). The per-image statuses are read
    back once for the batch."""
    dev = _device(device)
    datas = [_bytes(x) for x in items]
    n = len(datas)
    if n == 0:
        return []
    l = _lib.load()
    ptrs = (ctypes.c_char_p * n)(*datas)
    lens = (ctypes.c_longlong * n)(*[len(d) for d in datas])
    w, h, st = (ctypes.c_int * n)(), (ctypes.c_int * n)(), (ctypes.c_int * n)()
    _lib.check(l.mfr_jpeg_batch_info(ptrs, lens, n, w, h, st), "mfr_jpeg_batch_info")
    outs = [None] * n
    dst = (ctypes.c_void_p * n)()
    nbytes = pixels = 0
    for i in range(n):
        if st[i] == 0:
            outs[i] = torch.empty((h[i], w[i], 3) if rgb else (h[i], w[i]), dtype=torch.uint8, device=dev)
            dst[i] = outs[i].data_ptr()
            nbytes += len(datas[i])
            pixels += -(-w[i] // 16) * 16 * (-(-h[i] // 16) * 16)
    if nbytes:
        status = torch.empty(n, dtype=torch.int32, device=dev)
        dec = _decoder("jpeg", dev, n, nbytes, pixels)
        with torch.cuda.device(dev):
            _lib.check(l.mfr_jpeg_decode_batch(dec.h, ptrs, lens, n, int(rgb), dst, _lib.ptr(status), _lib.cur_stream()),
                       "mfr_jpeg_decode_batch")
        ok = status.cpu().tolist()
    else:
        ok = [1] * n
    for i in range(n):
        if ok[i] != 0:
            outs[i] = _host_decode(items[i], rgb, dev)
    return outs


def _png_batch(datas, kind, dev, dst_of):
    """One mfr_png_decode_batch call over the files `datas` (bytes). dst_of(i, w, h, depth) returns the CUDA tensor file
    i is decoded into (or None to skip it). Returns (tensors, per-file status: 0 where the GPU decoded the file)."""
    n = len(datas)
    l = _lib.load()
    ptrs = (ctypes.c_char_p * n)(*datas)
    lens = (ctypes.c_longlong * n)(*[len(d) for d in datas])
    w, h, bd, st = (ctypes.c_int * n)(), (ctypes.c_int * n)(), (ctypes.c_int * n)(), (ctypes.c_int * n)()
    _lib.check(l.mfr_png_batch_info(ptrs, lens, n, w, h, bd, st), "mfr_png_batch_info")
    outs = [None] * n
    dst = (ctypes.c_void_p * n)()
    nbytes = pixels = 0
    for i in range(n):
        if st[i] == 0:
            outs[i] = dst_of(i, w[i], h[i], bd[i])
        if outs[i] is not None:
            dst[i] = outs[i].data_ptr()
            nbytes += len(datas[i])
            pixels += w[i] * h[i]
        else:
            st[i] = 1
    if not nbytes:
        return outs, [1] * n
    status = torch.empty(n, dtype=torch.int32, device=dev)
    dec = _decoder("png", dev, n, nbytes, pixels)
    with torch.cuda.device(dev):
        _lib.check(l.mfr_png_decode_batch(dec.h, ptrs, lens, n, kind, dst, _lib.ptr(status), _lib.cur_stream()),
                   "mfr_png_decode_batch")
    return outs, status.cpu().tolist()


def _host_png(item, dev, depth_kind):
    """cv2.imread(IMREAD_UNCHANGED) of a file or bytes, uploaded (None if OpenCV cannot read it); with depth_kind,
    read_depth_image's float32 v / 1000."""
    import cv2
    if isinstance(item, (bytes, bytearray, memoryview)):
        im = cv2.imdecode(np.frombuffer(bytes(item), np.uint8), cv2.IMREAD_UNCHANGED)
    else:
        im = cv2.imread(str(item), cv2.IMREAD_UNCHANGED)
    if im is None:
        return None
    t = torch.from_numpy(im / 1000).float() if depth_kind else torch.from_numpy(np.ascontiguousarray(im))
    return t.to(dev)


def _readable(items):
    """(bytes or None per item): a path that does not exist reads as None, as cv2.imread returns None for it."""
    out = []
    for x in items:
        try:
            out.append(_bytes(x))
        except OSError:
            out.append(None)
    return out


def decode_pngs(items, device=None):
    """PNG files (bytes or paths) -> list of CUDA tensors, each cv2.imread(p, IMREAD_UNCHANGED) (torch.uint16 or uint8
    [h, w] for the gray 8- / 16-bit files the GPU decoder takes), from one decoder call on the current stream. Other
    files, and files the device rejects, are decoded by OpenCV on the host in their place in the list (None where
    OpenCV cannot read them either)."""
    dev = _device(device)
    datas = _readable(items)
    ok_idx = [i for i, d in enumerate(datas) if d]
    outs = [None] * len(items)
    if ok_idx:
        def alloc(i, w, h, depth):
            return torch.empty((h, w), dtype=torch.uint16 if depth == 16 else torch.uint8, device=dev)
        got, st = _png_batch([datas[i] for i in ok_idx], 0, dev, alloc)
        for i, g, s in zip(ok_idx, got, st):
            outs[i] = g if s == 0 else None
    for i in range(len(items)):
        if outs[i] is None and datas[i]:
            outs[i] = _host_png(datas[i], dev, False)
    return outs


def read_depth_image(path, device=None):
    """lib/datasets/utils.py:77-81: torch.from_numpy(cv2.imread(path, IMREAD_UNCHANGED) / 1000).float() as a CUDA
    float32 [h, w], bit for bit, or None if the file cannot be read. Gray 8- / 16-bit PNGs decode on the GPU; other
    files, and files the device rejects, are read by OpenCV on the host with that same expression."""
    out = read_depth_images([path], device)
    return None if out is None else out[0]


def read_depth_images(paths, device=None):
    """[read_depth_image(p) for p in paths] stacked into one CUDA float32 [B, h, w], from one decoder call whose kernels
    write each map straight into its slice (the form RelocPipeline.set_map / submit_device_queries take). The maps
    must share one size; None if any file cannot be read."""
    dev = _device(device)
    datas = _readable(paths)
    if not datas or any(d is None for d in datas):
        return None
    l = _lib.load()
    shapes = []
    for d in datas:
        w, h, bd = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        rc = l.mfr_png_info(d, len(d), ctypes.byref(w), ctypes.byref(h), ctypes.byref(bd))
        shapes.append((h.value, w.value) if rc == 0 else None)
    known = [s for s in shapes if s]
    out = None
    if known:
        hw = known[0]
        out = torch.empty((len(datas), *hw), dtype=torch.float32, device=dev)
        _, st = _png_batch(datas, 1, dev, lambda i, w, h, depth: out[i] if (h, w) == hw else None)
    else:
        st = [1] * len(datas)
    for i, s in enumerate(st):
        if s != 0:
            im = _host_png(datas[i], dev, True)
            if im is None:
                return None
            if out is None:
                out = torch.empty((len(datas), *im.shape), dtype=torch.float32, device=dev)
            if tuple(im.shape) != tuple(out.shape[1:]):
                raise ValueError(f"read_depth_images: depth map {i} is {tuple(im.shape)}, not {tuple(out.shape[1:])}")
            out[i] = im
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


def _is_jpeg(path):
    return str(path).lower().endswith((".jpg", ".jpeg"))


def _load_u8(path, rgb, device):
    p = str(path)
    if not os.path.isfile(p):
        return None                                  # cv2.imread's convention for unreadable files (utils.py:265-266)
    if _is_jpeg(p):
        try:
            return decode_jpeg(p, rgb=rgb, device=device)
        except _lib.MfrError:
            pass                                     # a file the GPU decoder does not take: OpenCV on the host
    return _host_decode(p, rgb, _device(device))


def _load_u8_many(paths, rgb, device):
    """[_load_u8(p, rgb, device) for p in paths] with every existing JPEG decoded in one decode_jpegs call."""
    out = [None] * len(paths)
    jpg = [i for i, p in enumerate(paths) if _is_jpeg(p) and os.path.isfile(str(p))]
    for i, im in zip(jpg, decode_jpegs([str(paths[i]) for i in jpg], rgb, device)):
        out[i] = im
    for i in set(range(len(paths))) - set(jpg):
        out[i] = _load_u8(paths[i], rgb, device)
    return out


def _gray_input(im, resize, resize_float):
    if im is None:
        return None
    return resize_linear(im, resize, MODE_U8_AS_F32 if resize_float else MODE_U8_FIXED, 1.0 / 255.0)


def read_image(path, resize, resize_float=True, device=None):
    """Gray image, resized to resize = (w, h), in [0, 1]: CUDA float32 [h, w]; None if the file cannot be read
    (SuperGlue/models/utils.py:263-285 with rotation 0; `resize` given as the two-element form the FMB plugins use)."""
    return _gray_input(_load_u8(path, False, device), resize, resize_float)


class PairMatcher:
    """Body of the image-pair matcher plugins (loftr.LoFTR_matcher, spsg.SuperGlue_matcher) over a batch-1 pair engine:
    images read with ``read_image(path, resize, True)`` on the engine's device, results as the reference's plugins give
    them, float [N, 4] (x0, y0, x1, y1) or ``np.full((1, 4), nan)``. A subclass builds the engine and reads the matched
    keypoints of an engine output in ``_matches(out) -> (kpts0, kpts1)``."""

    def __init__(self, resize, engine):
        self.resize, self.engine = resize, engine

    def match(self, pair_path):
        """matchers.py:24-59 / 93-120; images decoded and resized on the GPU."""
        return self._result(self.engine.forward(self._read(pair_path[0]), self._read(pair_path[1])))

    def match_scene(self, ref_path, query_paths):
        """``[self.match((ref_path, q)) for q in query_paths]``, array for array, with the reference image decoded and
        encoded once (Map-free: every pair of a scene shares its first image) and the query JPEGs decoded in one batch."""
        self.engine.set_map(self._read(ref_path))
        ims = _load_u8_many(list(query_paths), False, self.engine.device)
        return [self._result(self.engine.forward_shared(_gray_input(im, self.resize, True)[None])) for im in ims]

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


def jpeg_size(path):
    """(width, height) cv2.imread would return for a JPEG file the GPU decoder takes (orientation applied), else None."""
    try:
        data = _bytes(path)
    except OSError:
        return None
    w, h, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    if _lib.load().mfr_jpeg_info(data, len(data), ctypes.byref(w), ctypes.byref(h), ctypes.byref(c)) != 0:
        return None
    return w.value, h.value
