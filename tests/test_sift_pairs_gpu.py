"""SIFT pair engine (mfr_b200.sift.SIFTPairs): forward_pairs must give the bits of SIFT.detect on the pair-interleaved
batch + match_pairs, as a graph and eagerly; set_map + forward_shared the bits of forward_pairs with the map repeated;
an image with more candidates than max_candidates sets its pair's overflow flag, and RelocPipeline refuses that batch."""
import numpy as np
import pytest
import torch

from helpers import synth

pytestmark = pytest.mark.gpu
K_SMALL = np.array([[300.0, 0, 159.5], [0, 300.0, 119.5], [0, 0, 1]])
SIZES = [(240, 320, K_SMALL, 3), (720, 540, synth.K_DEFAULT, 2)]


def _u8(img_chw):
    return torch.from_numpy(synth.rgb_to_gray_u8(img_chw))


def _pairs(seed, P, h, w, K):
    ps = [synth.make_pair(seed + i, h=h, w=w, K=K) for i in range(P)]
    return (torch.stack([_u8(p["image0"]) for p in ps]).cuda(), torch.stack([_u8(p["image1"]) for p in ps]).cuda())


def _scene(seed, P, h, w, K):
    s = synth.make_scene(seed, P, h=h, w=w, K=K)
    return _u8(s["image0"]).cuda(), torch.stack([_u8(q["image1"]) for q in s["queries"]]).cuda()


def _state(eng):
    k0, k1, off = eng.pose_inputs()
    eng.stream.synchronize()
    n = int(off[-1])
    return {"kpts0": k0[:n].clone(), "kpts1": k1[:n].clone(), "offsets": off.clone(), "overflow": eng.overflow.clone()}


def _pairs_run(eng, a, b):
    eng.forward_async(a, b)
    return _state(eng)


def _shared_run(eng, q):
    eng.forward_shared_async(q)
    return _state(eng)


def _equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("h,w,K,P", SIZES, ids=["240x320", "720x540"])
def test_forward_pairs_equals_detect_and_match(h, w, K, P):
    from mfr_b200 import sift
    a, b = _pairs(70, P, h, w, K)
    ref_eng = sift.SIFT(2 * P, h, w, nfeatures=2048, root_sift=True)
    ref_eng.detect(torch.stack([a, b], 1).reshape(2 * P, h, w).contiguous())
    k0, k1, off = ref_eng.match_pairs(0.8)
    ref = {"kpts0": k0, "kpts1": k1, "offsets": off, "overflow": torch.zeros(P, dtype=torch.int32, device="cuda")}
    eng = sift.SIFTPairs(P, h, w, nfeatures=2048, ratio=0.8, root_sift=True)
    got = _pairs_run(eng, a, b)                     # first call: eager run + capture
    assert int(off[-1]) > 8 * P, "the synthetic pairs should give matches"
    _equal(got, ref)
    _equal(_pairs_run(eng, a, b), ref)             # graph replay
    eager = sift.SIFTPairs(P, h, w, nfeatures=2048, ratio=0.8, root_sift=True, graph=False)
    _equal(_pairs_run(eager, a, b), ref)
    print(f"{h}x{w}: matches per pair {torch.diff(off).tolist()}")
    ref_eng.close(); eng.close(); eager.close()


@pytest.mark.parametrize("h,w,K,P", SIZES, ids=["240x320", "720x540"])
def test_shared_map_equals_paired(h, w, K, P):
    from mfr_b200 import sift
    from mfr_b200.lib import MfrError
    m, q = _scene(80, P, h, w, K)
    m2, q2 = _scene(81, P, h, w, K)
    eng = sift.SIFTPairs(P, h, w)
    with pytest.raises(MfrError):
        eng.forward_shared_async(q)
    eng.set_map(m)
    got = _shared_run(eng, q)
    ref = _pairs_run(eng, m.expand(P, h, w), q)
    assert ref["kpts0"].shape[0] > 8 * P
    _equal(got, ref)
    _equal(_shared_run(eng, q), ref)               # graph replay, a paired forward in between
    eng.set_map(m2)
    _pairs_run(eng, m.expand(P, h, w), q)           # a paired call must not disturb the map
    _equal(_shared_run(eng, q2), _pairs_run(eng, m2.expand(P, h, w), q2))
    eng.close()


def test_overflow_flag_and_pipeline_refusal():
    """A capacity check: an image past max_candidates flags exactly its own pair, on the paired and the shared path, and
    RelocPipeline raises when it hands out that batch."""
    from mfr_b200 import pose_solver, sift
    from mfr_b200.lib import MfrError
    from mfr_b200.pipeline import RelocPipeline
    h, w, P = 240, 320, 2
    noise = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (h, w), dtype=np.uint8)).cuda()
    flat = torch.full((h, w), 77, dtype=torch.uint8, device="cuda")
    eng = sift.SIFTPairs(P, h, w, nfeatures=0, max_candidates=256)
    got = _pairs_run(eng, torch.stack([flat, flat]), torch.stack([flat, noise]))
    assert got["overflow"].tolist() == [0, 1] and got["offsets"].tolist() == [0, 0, 0]
    assert _pairs_run(eng, torch.stack([noise, flat]), torch.stack([flat, flat]))["overflow"].tolist() == [1, 0]
    eng.set_map(flat)
    assert _shared_run(eng, torch.stack([noise, flat]))["overflow"].tolist() == [1, 0]
    eng.set_map(noise)
    assert _shared_run(eng, torch.stack([flat, flat]))["overflow"].tolist() == [1, 1]
    be = pose_solver.PoseBackend(max_pairs=P, max_pts=256, max_hyp=256)
    pipe = RelocPipeline(eng, be, 2.0, 0.3, 256)
    K = torch.from_numpy(np.stack([K_SMALL] * P).astype(np.float32)).cuda()
    d = torch.ones(P, h, w, device="cuda")
    assert pipe.submit_device(torch.stack([flat, flat]), torch.stack([flat, flat]), d, d, K) is None
    R, t, n = pipe.submit_device(torch.stack([flat, flat]), torch.stack([noise, flat]), d, d, K)   # batch 0: fine
    with pytest.raises(MfrError, match="batch 1"):
        pipe.drain()
    eng.close(); be.close()
