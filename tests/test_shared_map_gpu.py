"""Shared map frame: set_map(map) + forward_shared(queries) must give exactly the bits of forward(map repeated, queries)
on the same engine, in every precision, for the LoFTR and SuperPoint + SuperGlue engines, through RelocPipeline and
through the offline matcher plugins."""
import numpy as np
import pytest
import torch

from helpers import synth

pytestmark = pytest.mark.gpu
H, W = 240, 320
K_SMALL = np.array([[300.0, 0, 159.5], [0, 300.0, 119.5], [0, 0, 1]])
LOFTR_KEYS = ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_f", "mkpts1_f", "mkpts1_c", "expec_f")


def _scene(seed, n, h=H, w=W, K=K_SMALL):
    s = synth.make_scene(seed, n, h=h, w=w, K=K)
    m = torch.from_numpy(s["gray0"]).cuda()
    q = torch.from_numpy(np.stack([x["gray1"] for x in s["queries"]])).cuda()
    return s, m, q


def _loftr_state(eng, B):
    """Every output of the last forward (live region) plus the final coarse tokens and the query half of feat_f."""
    d = eng.device_outputs()
    M = int(d["m_total"][0])
    st = {k: d[k][:M].clone() for k in LOFTR_KEYS}
    st["m_total"] = d["m_total"].clone()
    st["m_offsets"] = d["m_offsets"].clone()
    L = (eng.H // 8) * (eng.W // 8)
    st["tok"] = eng.debug_tensor("tok", (2 * B, L, 512)).clone()
    st["feat_f1"] = eng.debug_tensor("feat_f", (2 * B, eng.H // 2, eng.W // 2, 128))[B:].clone()
    return st, M


def _equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k


def _loftr_pair(eng, m, q):
    eng.forward_async(m.expand(q.shape[0], -1, -1), q)
    eng.stream.synchronize()
    return _loftr_state(eng, q.shape[0])


def _loftr_shared(eng, q):
    eng.forward_shared_async(q)
    eng.stream.synchronize()
    return _loftr_state(eng, q.shape[0])


@pytest.mark.parametrize("precision", ["tf32", "bf16", "fp32x3"])
@pytest.mark.parametrize("thr", [0.2, 0.0])
def test_loftr_shared_equals_paired(precision, thr):
    from mfr_b200 import loftr
    B = 3
    _, m, q = _scene(11, B)
    _, m2, q2 = _scene(12, B)
    eng = loftr.LoFTR(loftr.functional_state_dict(), batch=B, height=H, width=W, cfg={"thr": thr}, graph=True,
                      precision=precision)
    n_launches = eng.num_launches()
    eng.set_map(m)
    got, M = _loftr_shared(eng, q)
    ref, _ = _loftr_pair(eng, m, q)
    assert M > 0
    _equal(got, ref)
    got, _ = _loftr_shared(eng, q)                  # second replay of the shared graph (the paired one ran in between)
    _equal(got, ref)
    eng.set_map(m2)                                 # a new scene
    _equal(_loftr_shared(eng, q2)[0], _loftr_pair(eng, m2, q2)[0])
    eng.set_map(m)                                  # back to the first map, with paired forwards in between
    ref, _ = _loftr_pair(eng, m, q)
    eng.forward_async(m2.expand(B, -1, -1), q2)
    _equal(_loftr_shared(eng, q)[0], ref)
    assert eng.num_launches() == n_launches
    eng.close()


def test_loftr_shared_full_size():
    from mfr_b200 import loftr
    B = 2
    _, m, q = _scene(21, B, h=720, w=540, K=synth.K_DEFAULT)
    eng = loftr.LoFTR(loftr.functional_state_dict(), batch=B, height=720, width=544, cfg={"thr": 0.2}, graph=True,
                      precision="bf16")
    eng.set_map(m)
    got, M = _loftr_shared(eng, q)
    ref, _ = _loftr_pair(eng, m, q)
    assert M > 0
    _equal(got, ref)
    eng.close()


def test_loftr_shared_errors_and_padding():
    """forward_shared before set_map and with a source size other than the map's are rejected; a source smaller than
    the engine frame is zero-padded as in forward."""
    from mfr_b200 import loftr
    from mfr_b200.lib import MfrError
    B = 2
    _, m, q = _scene(31, B)
    eng = loftr.LoFTR(loftr.functional_state_dict(), batch=B, height=H + 8, width=W, cfg={"thr": 0.2}, graph=True)
    with pytest.raises(MfrError):
        eng.forward_shared_async(q)
    eng.set_map(m)
    with pytest.raises(MfrError):
        eng.forward_shared_async(q[:, :H - 8].contiguous())
    got, M = _loftr_shared(eng, q)
    ref, _ = _loftr_pair(eng, m, q)
    assert M > 0
    _equal(got, ref)
    eng.close()


SPSG_KEYS = ("counts", "keypoints", "scores", "descriptors", "matches0", "matching_scores0", "m_offsets")


def _spsg_state(eng):
    d = eng.device_outputs()
    st = {k: d[k].clone() for k in SPSG_KEYS}
    n = int(d["m_offsets"][-1])
    st["mkpts0"], st["mkpts1"] = d["mkpts0"][:n].clone(), d["mkpts1"][:n].clone()
    return st, n


def _spsg_shared(eng, q):
    eng.forward_shared(q)
    return _spsg_state(eng)


def _spsg_pair(eng, m, q):
    eng.forward(m.expand(q.shape[0], -1, -1), q)
    return _spsg_state(eng)


def _spsg_check(eng, m, q, m2, q2):
    eng.set_map(m)
    got, n = _spsg_shared(eng, q)
    ref, _ = _spsg_pair(eng, m, q)
    assert n > 0
    _equal(got, ref)
    _equal(_spsg_shared(eng, q)[0], ref)            # second replay of the shared graph
    eng.set_map(m2)
    _spsg_pair(eng, m, q)                           # a paired forward must not disturb the map
    got = _spsg_shared(eng, q2)[0]
    _equal(got, _spsg_pair(eng, m2, q2)[0])


@pytest.mark.parametrize("precision", ["tf32", "bf16", "fp32x3"])
def test_spsg_shared_equals_paired(precision):
    from mfr_b200 import spsg
    from mfr_b200.lib import MfrError
    B = 2
    _, m, q = _scene(41, B)
    _, m2, q2 = _scene(42, B)
    sp, sg = spsg.synthetic_state_dicts(0)
    # match_threshold 0: the synthetic SuperGlue weights give no match above the default 0.2
    eng = spsg.SuperPointSuperGlue(sp, sg, batch=B, height=H, width=W, cfg={"max_keypoints": 256, "match_threshold": 0.0},
                                   graph=True, precision=precision)
    with pytest.raises(MfrError):
        eng.forward_shared_async(q)
    n_launches = eng.num_launches()
    _spsg_check(eng, m, q, m2, q2)
    assert eng.num_launches() == n_launches
    eng.close()


def test_spsg_shared_real_weights():
    from oracle import build_ref
    if not build_ref.available():
        pytest.skip("oracle/_ref assets not staged (python oracle/build_ref.py)")
    from mfr_b200 import spsg
    w = build_ref.weights_dir()
    sp = torch.load(w + "/superpoint_v1.pth", map_location="cpu")
    sg = torch.load(w + "/superglue_indoor.pth", map_location="cpu")
    B = 2
    _, m, q = _scene(43, B, h=720, w=540, K=synth.K_DEFAULT)
    _, m2, q2 = _scene(44, B, h=720, w=540, K=synth.K_DEFAULT)
    eng = spsg.SuperPointSuperGlue(sp, sg, batch=B, height=720, width=540, graph=True, precision="bf16")
    _spsg_check(eng, m, q, m2, q2)
    eng.close()


def _pinned_scene(s):
    g1 = torch.from_numpy(np.stack([x["gray1"] for x in s["queries"]])).pin_memory()
    d1 = torch.from_numpy(np.stack([x["depth1"] for x in s["queries"]])).pin_memory()
    K1 = torch.from_numpy(np.stack([x["K_color1"] for x in s["queries"]])).pin_memory()
    return g1, d1, K1


def test_pipeline_shared_map_equals_paired():
    """Two scenes (7 and 4 queries, B = 2: the first ends in a ragged batch) through parallel.run_stream: set_map +
    submit_host_queries gives the record table of submit_host with the map frame repeated for every pair. Then the
    same scenes as one continuous stream, the second set_map issued while the first scene's last batches are still in
    flight, through submit_device_queries."""
    from mfr_b200 import loftr, parallel, pose_solver
    from mfr_b200.pipeline import RelocPipeline
    B = 2
    scenes = [synth.make_scene(51, 7, h=H, w=W, K=K_SMALL), synth.make_scene(52, 4, h=H, w=W, K=K_SMALL)]
    eng = loftr.LoFTR(loftr.functional_state_dict(), batch=B, height=H, width=W, cfg={"thr": 0.2}, graph=True,
                      pipelined=True)
    be = pose_solver.PoseBackend(max_pairs=B, max_pts=(H // 8) * (W // 8), max_hyp=512)
    pipe = RelocPipeline(eng, be, 2.0, 0.3, 512, depth_hw=(H, W))
    paired, shared = [], []
    for s in scenes:
        g1, d1, K1 = _pinned_scene(s)
        n = g1.shape[0]
        g0 = torch.from_numpy(s["gray0"])[None].expand(n, H, W).contiguous().pin_memory()
        d0 = torch.from_numpy(s["depth0"])[None].expand(n, H, W).contiguous().pin_memory()
        K0 = torch.from_numpy(s["K_color0"])[None].expand(n, 3, 3).contiguous().pin_memory()
        pipe.reset()
        paired.append(parallel.run_stream(n, B, lambda ids: pipe.submit_host(g0[ids], g1[ids], d0[ids], d1[ids], K0[ids], K1[ids]),
                                          pipe.drain))
        pipe.reset()
        pipe.set_map(torch.from_numpy(s["gray0"]), torch.from_numpy(s["depth0"]), torch.from_numpy(s["K_color0"]))
        shared.append(parallel.run_stream(n, B, lambda ids: pipe.submit_host_queries(g1[ids], d1[ids], K1[ids]), pipe.drain))
    for a, b in zip(paired, shared):
        assert int(a[:, 1].min()) > 20, "the synthetic scenes should give solvable poses"
        assert torch.equal(a, b)
    # one continuous stream over both scenes: results arrive one batch late, across the scene change
    pipe.reset()
    got = []
    for s in scenes:
        g1, d1, K1 = (x.cuda() for x in _pinned_scene(s))
        pipe.set_map(torch.from_numpy(s["gray0"]).cuda(), torch.from_numpy(s["depth0"]).cuda(),
                     torch.from_numpy(s["K_color0"]).cuda())
        n = g1.shape[0]
        for k in range(0, n, B):
            ids = [min(j, n - 1) for j in range(k, k + B)]
            r = pipe.submit_device_queries(g1[ids], d1[ids], K1[ids])
            if r is not None:
                got.append(r)
    got.append(pipe.drain())
    rows = [(table, k, min(B, table.shape[0] - k)) for table in shared for k in range(0, table.shape[0], B)]
    assert len(got) == len(rows)
    for (R, t, inl), (table, k, m) in zip(got, rows):
        assert torch.equal(inl[:m].to(torch.float64), table[k:k + m, 1])
        assert torch.equal(R[:m].reshape(m, 9).to(torch.float64), table[k:k + m, 2:11])
        assert torch.equal(t[:m].to(torch.float64), table[k:k + m, 11:14])
    eng.close(); be.close()


@pytest.mark.parametrize("matcher", ["loftr", "superglue"])
def test_plugin_match_scene(matcher, tmp_path):
    import cv2
    from mfr_b200 import loftr, spsg
    s = synth.make_scene(61, 3, h=H, w=W, K=K_SMALL)
    paths = []
    for i, g in enumerate([s["gray0"]] + [q["gray1"] for q in s["queries"]]):
        p = str(tmp_path / f"frame_{i:05d}.jpg")
        assert cv2.imwrite(p, np.round(g * 255.0).astype(np.uint8))
        paths.append(p)
    if matcher == "loftr":
        mt = loftr.LoFTR_matcher((W, H), weights=loftr.functional_state_dict(), cfg={"thr": 0.2})
    else:
        sp, sg = spsg.synthetic_state_dicts(0)
        mt = spsg.SuperGlue_matcher((W, H), state_dicts=(sp, sg))
        mt.engine = spsg.SuperPointSuperGlue(sp, sg, batch=1, height=H, width=W, cfg={"match_threshold": 0.0})
    ref = [mt.match((paths[0], p)) for p in paths[1:]]
    got = mt.match_scene(paths[0], paths[1:])
    assert len(got) == len(ref)
    assert any(r.shape[0] > 1 for r in ref), "the synthetic scene should give matches"
    for a, b in zip(got, ref):
        assert a.shape == b.shape and np.array_equal(a, b, equal_nan=True)
