"""The GPU JPEG decoder (image_io.decode_jpeg / decode_jpegs, csrc/jpeg.cuh kernels) against cv2.imread and the host hook,
byte for byte, and the loaders and plugins that read files through it."""
import cv2
import numpy as np
import pytest
import torch

import jpeg_cases as jc
from oracle import build_ref
from test_jpeg_host import host_decode

pytestmark = pytest.mark.gpu

MATRIX = jc.matrix() + jc.orientation_cases()


@pytest.mark.parametrize("rgb", [False, True])
def test_decode_jpeg_equals_cv2_and_host(rgb):
    from mfr_b200 import image_io
    bad = []
    for name, data in MATRIX:
        got = image_io.decode_jpeg(data, rgb=rgb).cpu().numpy()
        ref = jc.cv2_decode(data, rgb)
        rc, host = host_decode(data, rgb)
        if rc != 0 or got.shape != ref.shape or not np.array_equal(got, ref) or not np.array_equal(got, host):
            bad.append(name)
    assert not bad, bad


@pytest.mark.parametrize("rgb", [False, True])
def test_decode_jpegs_batch_mixed(rgb):
    """One batch mixing sizes, sampling modes, restart intervals, orientations and unsupported files (decoded by the
    host fallback in place); a file's bytes do not depend on its batch or its position in it."""
    from mfr_b200 import image_io
    items = MATRIX + jc.unsupported_cases()
    rng = np.random.default_rng(3)
    order = rng.permutation(len(items))
    batch = [items[i] for i in order]
    outs = image_io.decode_jpegs([d for _, d in batch], rgb=rgb)
    torch.cuda.synchronize()
    assert len(outs) == len(batch)
    for (name, data), got in zip(batch, outs):
        assert got.is_cuda and got.dtype == torch.uint8
        assert np.array_equal(got.cpu().numpy(), jc.cv2_decode(data, rgb)), name
    # the same files again in other batches: a batch of one, and a reversed sub-batch on another stream
    s = torch.cuda.Stream()
    sub = batch[::-7]
    with torch.cuda.stream(s):
        outs2 = image_io.decode_jpegs([d for _, d in sub], rgb=rgb)
    s.synchronize()
    first = {name: o for (name, _), o in zip(batch, outs)}
    for (name, data), got in zip(sub, outs2):
        assert torch.equal(got, first[name]), name
        assert torch.equal(image_io.decode_jpegs([data], rgb=rgb)[0], first[name]), name


def test_loaders_on_files(tmp_path):
    """read_image / read_color_image = cv2.resize of cv2.imread within the resize tests' tolerances (the float path to
    fp32 round-off of OpenCV's generic code path, cv2.setUseOptimized(False))."""
    from mfr_b200 import image_io
    cases = [c for c in MATRIX if c[0].startswith(("720x540", "333x250", "orient6"))]
    for name, data in cases:
        p = str(tmp_path / f"{name}.jpg")
        open(p, "wb").write(data)
        gray = cv2.imread(p, cv2.IMREAD_GRAYSCALE)
        col = cv2.imread(p, cv2.IMREAD_COLOR)[:, :, ::-1]
        for size in ((270, 360), (640, 480)):
            got = image_io.read_image(p, size, True).cpu().numpy()
            ref = cv2.resize(gray.astype("float32"), size) / 255.0
            np.testing.assert_allclose(got, ref.astype(np.float32), rtol=0, atol=5e-3 / 255, err_msg=name)
            got8 = image_io.read_image(p, size, False).cpu().numpy() * 255.0
            d = np.abs(np.round(got8) - cv2.resize(gray, size))
            assert d.max() <= 1 and (d > 0).mean() < 3e-3, name
            gc = image_io.read_color_image(p, size).cpu().numpy()
            dc = np.abs(np.round(gc.transpose(1, 2, 0) * 255.0) - cv2.resize(np.ascontiguousarray(col), size))
            assert dc.max() <= 1 and (dc > 0).mean() < 3e-3, name
            cv2.setUseOptimized(False)
            try:
                ref_g = cv2.resize(gray.astype("float32"), size) / 255.0
                ref_c = cv2.resize(np.ascontiguousarray(col), size)
            finally:
                cv2.setUseOptimized(True)
            np.testing.assert_allclose(got, ref_g.astype(np.float32), rtol=0, atol=2e-5 / 255 + 1e-7, err_msg=name)
            # the uint8 path: OpenCV's vectorised fixed-point code also runs without the optimised (IPP) dispatch, so
            # the resize tests' one-level tolerance applies here too
            dg = np.abs(np.round(gc.transpose(1, 2, 0) * 255.0) - ref_c)
            assert dg.max() <= 1 and (dg > 0).mean() < 3e-3, name


@pytest.mark.skipif(not build_ref.available(), reason="oracle/_ref assets not staged")
def test_readme_pair_decodes_like_cv2():
    from mfr_b200 import image_io
    paths = [build_ref.data_dir() + "/" + n for n in ("scene0711_00_frame-001680.jpg", "scene0711_00_frame-001995.jpg")]
    for rgb in (False, True):
        outs = image_io.decode_jpegs(paths, rgb=rgb)
        for p, got in zip(paths, outs):
            ref = cv2.imread(p, cv2.IMREAD_COLOR if rgb else cv2.IMREAD_GRAYSCALE)
            ref = ref[:, :, ::-1] if rgb else ref
            assert np.array_equal(got.cpu().numpy(), ref), p
            assert np.array_equal(image_io.decode_jpeg(p, rgb=rgb).cpu().numpy(), ref), p


def _frames(tmp_path, n):
    rgb = jc.content("texture", 720, 540, 11)
    paths = []
    for i in range(n):
        p = str(tmp_path / f"f{i}.jpg")
        cv2.imwrite(p, np.roll(rgb, (4 * i, 6 * i), (0, 1))[:, :, ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
        paths.append(p)
    return paths


def test_sift_matcher_gpu_decode(tmp_path):
    from mfr_b200 import matchers
    p0, p1 = _frames(tmp_path, 2)
    m = matchers.SIFT_matcher((540, 720), gpu_detector=True)
    got = m.match((p0, p1))
    ref = m.match_arrays_gpu(cv2.imread(p0, 0), cv2.imread(p1, 0))
    assert got.shape == ref.shape and got.shape[1] == 4 and np.array_equal(got, ref)


def test_loftr_match_scene_equals_match(tmp_path):
    from mfr_b200 import loftr
    paths = _frames(tmp_path, 4)
    paths.append(str(tmp_path / "q.png"))
    cv2.imwrite(paths[-1], cv2.imread(paths[2]))                      # a non-JPEG query: host decode
    m = loftr.LoFTR_matcher((272, 360), weights=loftr.functional_state_dict(), cfg={"thr": 0.2})
    scene = m.match_scene(paths[0], paths[1:])
    single = [m.match((paths[0], q)) for q in paths[1:]]
    assert len(scene) == len(single)
    for a, b in zip(scene, single):
        assert a.shape == b.shape and np.array_equal(a, b, equal_nan=True)
