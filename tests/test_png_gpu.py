"""The GPU depth-PNG decoder (image_io.decode_pngs / read_depth_image / read_depth_images, csrc/png.cuh kernels) against
cv2.imdecode(IMREAD_UNCHANGED) and the host hook, byte for byte, and a RelocPipeline fed from its depth maps."""
import cv2
import numpy as np
import pytest
import torch

import png_cases as pc
from helpers import synth
from test_png_host import host_decode

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def matrix():
    return pc.matrix()


def _same(got, ref):
    return got is not None and ref is not None and got.is_cuda and got.cpu().numpy().dtype == ref.dtype and \
        np.array_equal(got.cpu().numpy(), ref)


def test_decode_pngs_equals_cv2_and_host(matrix):
    from mfr_b200 import image_io
    batch = image_io.decode_pngs([d for _, d in matrix])
    bad = []
    for (name, data), got in zip(matrix, batch):
        ref = pc.cv2_decode(data)
        rc, host = host_decode(data)
        single = image_io.decode_pngs([data])[0]
        if not (_same(got, ref) and _same(single, ref) and rc == 0 and np.array_equal(host, ref)):
            bad.append(name)
    assert not bad, bad


def test_batch_independence(matrix):
    """The same bytes alone and at every position of a batch of 64 give the same tensor."""
    from mfr_b200 import image_io
    pick = [d for n, d in matrix if n.startswith(("540x720-depth-16", "17x33", "filter-mix", "split7-16"))]
    target = pick[0]
    alone = image_io.decode_pngs([target])[0]
    others = [pick[1 + i % (len(pick) - 1)] for i in range(63)]
    for pos in range(64):
        outs = image_io.decode_pngs(others[:pos] + [target] + others[pos:])
        assert torch.equal(outs[pos], alone), pos


def test_mixed_batch_falls_back_to_cv2(matrix, tmp_path):
    """Supported, unsupported, corrupt files and a missing path: cv2's answer for every entry, None included."""
    from mfr_b200 import image_io
    items = [d for _, d in matrix[::9]] + [d for _, d in pc.unsupported_cases()] + [d for _, d, _ in pc.malformed_cases()]
    names = list(range(len(items)))
    p = tmp_path / "d.png"
    p.write_bytes(matrix[3][1])
    items += [str(p), str(tmp_path / "missing.png")]
    rng = np.random.default_rng(1)
    order = rng.permutation(len(items))
    outs = image_io.decode_pngs([items[i] for i in order])
    for i, got in zip(order, outs):
        item = items[i]
        ref = cv2.imread(item, cv2.IMREAD_UNCHANGED) if isinstance(item, str) else pc.cv2_decode(item)
        if ref is None:
            assert got is None, i
        else:
            assert got is not None and np.array_equal(got.cpu().numpy(), ref), (i, names[i] if i < len(names) else item)


def test_decoder_growth_and_two_streams(matrix):
    from mfr_b200 import image_io
    small = [d for n, d in matrix if n.startswith("17x33")]
    large = [d for n, d in matrix if n.startswith(("1080x1920", "540x720-depth", "720x540-noise"))]
    a = image_io.decode_pngs(small)
    b = image_io.decode_pngs(large * 3)                     # grows the per-device decoder
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        c = image_io.decode_pngs(small)
    with torch.cuda.stream(s2):
        d = image_io.decode_pngs(large * 3)
    torch.cuda.synchronize()
    for x, y, src in zip(a + b, c + d, small + large * 3):
        assert torch.equal(x, y) and np.array_equal(y.cpu().numpy(), pc.cv2_decode(src))


def test_read_depth_image_is_the_reference_expression(tmp_path):
    from mfr_b200 import image_io
    rng = np.random.default_rng(4)
    paths, refs = [], []
    for i in range(5):
        mm = np.round(synth.make_depth(rng, 60, 80).astype(np.float64) * 1000).astype(np.uint16)
        if i == 4:
            mm = pc.all_values()[:60, :80] * 0 + np.arange(60 * 80, dtype=np.uint16).reshape(60, 80) * 13
        p = str(tmp_path / f"d{i}.png")
        cv2.imwrite(p, mm)
        paths.append(p)
        refs.append(torch.from_numpy(cv2.imread(p, cv2.IMREAD_UNCHANGED) / 1000).float())
    for p, r in zip(paths, refs):
        assert torch.equal(image_io.read_depth_image(p).cpu(), r)
    stacked = image_io.read_depth_images(paths)
    assert stacked.shape == (5, 60, 80) and torch.equal(stacked.cpu(), torch.stack(refs))
    av = str(tmp_path / "all.png")
    cv2.imwrite(av, pc.all_values())
    assert torch.equal(image_io.read_depth_image(av).cpu(), torch.from_numpy(pc.all_values() / 1000).float())
    col = str(tmp_path / "c.png")                            # a colour PNG: the host fallback, same expression
    cv2.imwrite(col, np.dstack([refs[0].numpy().astype(np.uint16)] * 3))
    ref = torch.from_numpy(cv2.imread(col, cv2.IMREAD_UNCHANGED) / 1000).float()
    assert torch.equal(image_io.read_depth_image(col).cpu(), ref)
    assert image_io.read_depth_image(str(tmp_path / "missing.png")) is None


@pytest.mark.parametrize("matcher", ["loftr", "spsg"])
def test_pipeline_from_depth_files(tmp_path, matcher):
    """One RelocPipeline fed twice: depths from read_depth_images, and from host cv2; identical R, t and inliers."""
    from mfr_b200 import image_io, loftr, pose_solver, spsg
    from mfr_b200.pipeline import EMatMetricStage, ProcrustesStage, RelocPipeline
    H, W, B, N = 240, 320, 2, 4
    K = np.array([[300.0, 0, 159.5], [0, 300.0, 119.5], [0, 0, 1]])
    s = synth.make_scene(71, N, h=H, w=W, K=K)
    frames = [(s["image0"], s["depth0"])] + [(q["image1"], q["depth1"]) for q in s["queries"]]
    jpgs, pngs = [], []
    for i, (im, dep) in enumerate(frames):
        jpgs.append(str(tmp_path / f"f{i}.jpg"))
        pngs.append(str(tmp_path / f"f{i}.png"))
        cv2.imwrite(jpgs[-1], synth.rgb_to_gray_u8(im), [cv2.IMWRITE_JPEG_QUALITY, 95])
        cv2.imwrite(pngs[-1], np.round(dep.astype(np.float64) * 1000).astype(np.uint16))
    if matcher == "loftr":
        eng = loftr.LoFTR(loftr.functional_state_dict(), batch=B, height=H, width=W, cfg={"thr": 0.2}, graph=True)
    else:
        sp, sg = spsg.synthetic_state_dicts(0)
        eng = spsg.SuperPointSuperGlue(sp, sg, batch=B, height=H, width=W, cfg={"max_keypoints": 512, "match_threshold": 0.0},
                                       graph=True)
    be = pose_solver.PoseBackend(max_pairs=B, max_pts=min(eng.max_pts_per_pair, pose_solver.MAX_PTS_LIMIT), max_hyp=512)
    grays = image_io.decode_jpegs(jpgs)
    g = torch.stack(grays) if eng.input_dtype == torch.uint8 else torch.stack(grays).float() / 255.0
    Ks = torch.from_numpy(K).float()[None].expand(N, 3, 3).contiguous().cuda()
    gpu_d = image_io.read_depth_images(pngs)
    host_d = torch.stack([torch.from_numpy(cv2.imread(p, cv2.IMREAD_UNCHANGED) / 1000).float() for p in pngs]).cuda()
    assert torch.equal(gpu_d, host_d)
    for stage in (EMatMetricStage(2.0, 0.3, 512), ProcrustesStage(0.05, 512)):
        res = []
        for depths in (image_io.read_depth_images(pngs), host_d):
            pipe = RelocPipeline(eng, be, solver=stage)
            pipe.set_map(g[0], depths[0], Ks[0])
            got = [pipe.submit_device_queries(g[1 + k:1 + k + B], depths[1 + k:1 + k + B], Ks[k:k + B]) for k in range(0, N, B)]
            got.append(pipe.drain())
            res.append([torch.cat([r[j] for r in got[1:]]).cpu() for j in range(3)])
        (R0, t0, n0), (R1, t1, n1) = res
        assert int(n0.max()) > 8
        assert torch.equal(n0, n1) and torch.equal(R0.nan_to_num(), R1.nan_to_num()) and torch.equal(t0.nan_to_num(), t1.nan_to_num())
    eng.close(); be.close()
