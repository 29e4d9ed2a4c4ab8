"""The depth-PNG decoder's arithmetic without a GPU: mfr_host_png_decode runs the same __host__ __device__ code as the
kernels (csrc/png.cuh) serially, and must equal cv2.imdecode(IMREAD_UNCHANGED) byte for byte on every generated file;
unsupported files are reported as such and malformed ones as errors."""
import ctypes

import numpy as np
import pytest
import torch

import png_cases as pc
from mfr_b200 import lib

MFR_OK, MFR_ERR_ARG, MFR_ERR_UNSUPPORTED = 0, 2, 3


def info(data):
    w, h, d = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = lib.load().mfr_png_info(data, len(data), ctypes.byref(w), ctypes.byref(h), ctypes.byref(d))
    return rc, w.value, h.value, d.value


def host_decode(data, kind=0, w=None, h=None):
    """(status, image) of the host hook; w, h default to mfr_png_info's."""
    rc, iw, ih, depth = info(data)
    if w is None:
        if rc != MFR_OK:
            return rc, None
        w, h = iw, ih
    dtype = np.float32 if kind == 1 else (np.uint8 if depth == 8 else np.uint16)
    out = np.zeros((h, w), dtype)
    rc = lib.load().mfr_host_png_decode(data, len(data), kind, out.ctypes.data_as(ctypes.c_void_p), w, h)
    return rc, out


@pytest.fixture(scope="module")
def matrix():
    return pc.matrix()


def test_host_decode_equals_cv2(matrix):
    bad = []
    for name, data in matrix:
        rc, got = host_decode(data)
        ref = pc.cv2_decode(data)
        if rc != MFR_OK or ref is None or got.dtype != ref.dtype or not np.array_equal(got, ref):
            bad.append((name, rc, None if ref is None else ref.dtype))
    assert not bad, bad


def test_depth_kind_is_read_depth_image(matrix):
    """out_kind 1 = torch.from_numpy(cv2.imread(p, IMREAD_UNCHANGED) / 1000).float() bitwise, on every 16-bit value and
    on 8-bit files."""
    for name, data in [c for c in matrix if c[0].startswith(("all-values", "17x33-depth"))]:
        rc, got = host_decode(data, 1)
        ref = torch.from_numpy(pc.cv2_decode(data) / 1000).float().numpy()
        assert rc == MFR_OK and np.array_equal(got.view(np.uint32), ref.view(np.uint32)), name
    rc, got = host_decode(pc.cv2_png(pc.all_values()), 1)
    assert np.unique(got).size == 65536


def test_unsupported_files_are_reported():
    for name, data in pc.unsupported_cases():
        assert info(data)[0] == MFR_ERR_UNSUPPORTED, name
        assert host_decode(data, 0, 24, 20)[0] == MFR_ERR_UNSUPPORTED, name


def test_malformed_files_are_errors():
    for name, data, where in pc.malformed_cases():
        rc = info(data)[0]
        if where == "header":
            assert rc == MFR_ERR_ARG, name
        else:
            assert rc == MFR_OK, name
            assert host_decode(data)[0] == MFR_ERR_ARG, name
    assert lib.load().mfr_host_png_decode(b"", 0, 0, ctypes.c_void_p(1), 1, 1) == MFR_ERR_ARG
    data = pc.cv2_png(pc.content("depth", 9, 8))
    assert host_decode(data, 0, 9, 8)[0] == MFR_ERR_ARG          # a destination of another size
    assert host_decode(data, 2)[0] == MFR_ERR_ARG                # an output kind outside {0, 1}


def test_malformed_files_are_refused_by_cv2():
    """The device rejects what libpng rejects, so the host fallback reproduces cv2's None."""
    for name, data, where in pc.malformed_cases():
        if name in ("beyond-window", "payload-bit", "adler", "truncated-stream", "truncated-file", "idat-crc", "filter5", "block-type3",
                    "too-far", "signature", "ihdr-crc", "no-iend"):
            assert pc.cv2_decode(data) is None, name
