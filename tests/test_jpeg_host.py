"""The JPEG decoder's arithmetic without a GPU: mfr_host_jpeg_decode runs the same __host__ __device__ code as the
kernels (csrc/jpeg.cuh) serially, and must equal cv2.imread byte for byte on every generated file; unsupported files are
reported as such and malformed ones as errors."""
import ctypes

import numpy as np
import pytest

import jpeg_cases as jc
from mfr_b200 import lib

MFR_OK, MFR_ERR_ARG, MFR_ERR_UNSUPPORTED = 0, 2, 3


def info(data):
    l = lib.load()
    w, h, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = l.mfr_jpeg_info(data, len(data), ctypes.byref(w), ctypes.byref(h), ctypes.byref(c))
    return rc, w.value, h.value


def host_decode(data, rgb, w=None, h=None):
    """(status, image) of the host hook; w, h default to the oriented size mfr_jpeg_info reports."""
    if w is None:
        rc, w, h = info(data)
        if rc != MFR_OK:
            return rc, None
    out = np.zeros((h, w, 3) if rgb else (h, w), np.uint8)
    rc = lib.load().mfr_host_jpeg_decode(data, len(data), int(rgb), out.ctypes.data_as(ctypes.c_void_p), w, h)
    return rc, out


MATRIX = jc.matrix() + jc.orientation_cases()


@pytest.mark.parametrize("rgb", [False, True])
def test_host_decode_equals_cv2(rgb):
    bad = []
    for name, data in MATRIX:
        rc, got = host_decode(data, rgb)
        ref = jc.cv2_decode(data, rgb)
        if rc != MFR_OK or got.shape != ref.shape or not np.array_equal(got, ref):
            diff = None if rc != MFR_OK or got.shape != ref.shape else int(np.abs(got.astype(int) - ref).max())
            bad.append((name, rc, None if got is None else got.shape, ref.shape, diff))
    assert not bad, bad


def test_orientation_swaps_shape():
    for name, data in jc.orientation_cases():
        o = int(name[6])
        rc, w, h = info(data)
        assert rc == MFR_OK and (w, h) == ((37, 50) if o >= 5 else (50, 37)), name


def test_unsupported_files_are_reported():
    for name, data in jc.unsupported_cases():
        assert info(data)[0] == MFR_ERR_UNSUPPORTED, name
        for rgb in (False, True):
            assert host_decode(data, rgb, 56, 40)[0] == MFR_ERR_UNSUPPORTED, name


def _segment(data, marker):
    """Offset of the first segment with ``marker`` (the FF byte)."""
    i = 2
    while data[i + 1] != marker:
        i += 2 + int.from_bytes(data[i + 2:i + 4], "big")
    return i


def test_malformed_files_are_errors():
    data = jc.encode(jc.content("texture", 64, 48), [])
    assert host_decode(data, True)[0] == MFR_OK
    # truncated entropy-coded data: the headers parse, the data ends before the last block
    rc, w, h = info(data[: len(data) * 3 // 5])
    assert rc == MFR_OK
    assert host_decode(data[: len(data) * 3 // 5], True, w, h)[0] == MFR_ERR_ARG
    # a DHT segment whose code counts promise more symbols than it holds
    i = _segment(data, 0xC4)
    n = sum(data[i + 5:i + 21])
    bad = bytearray(data)
    bad[i + 5 + 15] += 1                                   # one more 16-bit code, no symbol for it in the segment
    assert n + 1 > int.from_bytes(data[i + 2:i + 4], "big") - 19
    assert host_decode(bytes(bad), True, 48, 64)[0] == MFR_ERR_ARG
    assert info(bytes(bad))[0] == MFR_ERR_ARG
    # a zero-length buffer
    assert lib.load().mfr_host_jpeg_decode(b"", 0, 1, ctypes.c_void_p(1), 1, 1) == MFR_ERR_ARG
    assert info(b"\xff\xd8")[0] == MFR_ERR_ARG
    # a SOF whose height promises more rows than the data holds
    i = _segment(data, 0xC0)
    bad = bytearray(data)
    bad[i + 5:i + 7] = (128).to_bytes(2, "big")
    assert info(bytes(bad))[:3] == (MFR_OK, 48, 128)
    assert host_decode(bytes(bad), False, 48, 128)[0] == MFR_ERR_ARG
    # a destination of another size than the oriented image
    assert host_decode(data, False, 64, 48)[0] == MFR_ERR_ARG
