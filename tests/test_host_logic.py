"""Host-side logic that needs no GPU: BN folding / weight layout, the yaml config surface, the
submission format, the npz correspondence format, the position encoding quirk."""
import io
import zipfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import ROOT
from mfr_b200 import config, loftr, model, submission


def test_bn_folding_matches_conv_bn():
    sd = loftr.synthetic_state_dict(1)
    w = loftr.prepare_weights(sd, 6, 5)
    x = torch.randn(1, 128, 9, 7)
    p = "backbone.layer1.0"
    ref = F.batch_norm(F.conv2d(x, sd[p + ".conv1.weight"], None, 1, 1), sd[p + ".bn1.running_mean"],
                       sd[p + ".bn1.running_var"], sd[p + ".bn1.weight"], sd[p + ".bn1.bias"], False, 0.0, 1e-5)
    wf = torch.from_numpy(w["layer1.0.conv1.w"]).reshape(128, 3, 3, 128).permute(0, 3, 1, 2)   # [Cout][RS][Cin] -> OIHW
    got = F.conv2d(x, wf, torch.from_numpy(w["layer1.0.conv1.b"]), 1, 1)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)
    assert w["coarse.0.qkv.w"].shape == (768, 256) and w["fine.1.mlp0.w"].shape == (256, 256)
    assert w["pos_enc"].shape == (6, 5, 256)


def test_position_encoding_buggy_divisor():
    pe = loftr.position_encoding(256, 4, 3)
    # temp_bug_fix=False: div_term = exp(-2k) (position_encoding.py:28); channel 4 uses k = 2 -> exp(-2)
    assert pe[0, 0, 0].item() == pytest.approx(np.sin(1.0), rel=1e-6)
    assert pe[0, 2, 4].item() == pytest.approx(np.sin(3.0 * np.exp(-2.0)), rel=1e-5)
    assert pe[1, 0, 6].item() == pytest.approx(np.sin(2.0 * np.exp(-2.0)), rel=1e-5)   # y position 2


def test_pad_to_8_quirk():
    assert loftr.pad_to_8(torch.zeros(1, 1, 720, 540)).shape == (1, 1, 720, 544)     # 540 % 8 = 4 -> +4
    assert loftr.pad_to_8(torch.zeros(1, 1, 721, 542)).shape == (1, 1, 722, 548)     # the reference's remainder rule


def test_config_loads_reference_yaml_layers(tmp_path):
    ds = tmp_path / "mapfree.yaml"
    ds.write_text("DATASET:\n  DATA_SOURCE: 'MapFree'\n  SCENES: None\n  HEIGHT: 720\n  WIDTH: 540\n")
    me = tmp_path / "method.yaml"
    me.write_text("MODEL: 'FeatureMatching'\nFEATURE_MATCHING: 'Precomputed'\nPOSE_SOLVER: 'PNP'\n"
                  "MATCHES_FILE_PATH: '{scene_root}/correspondences_SG.npz'\n"
                  "PNP:\n  RANSAC_ITER: 1000\n  REPROJECTION_INLIER_THRESHOLD: 3\n  CONFIDENCE: 0.9999\n")
    cfg = config.load_cfg(str(ds), str(me))
    assert cfg.POSE_SOLVER == "PNP" and cfg.PNP.RANSAC_ITER == 1000 and cfg.DATASET.SCENES is None
    assert cfg.DATASET.HEIGHT == 720 and cfg.GPU_RANSAC.NUM_HYPOTHESES is None and cfg.GPU_RANSAC.FINAL_REFIT == "lsq"
    bad = tmp_path / "bad.yaml"
    bad.write_text("NOT_A_KEY: 1\n")
    with pytest.raises(KeyError):
        config.load_cfg(str(bad))


def test_precomputed_matching_npz_format(tmp_path):
    corr = np.full((3, 5, 4), np.nan)
    corr[1, :3] = np.arange(12).reshape(3, 4)
    path = tmp_path / "correspondences_X.npz"
    np.savez_compressed(path, correspondences=corr)
    cfg = config.load_cfg(overrides={"DEBUG": False, "MATCHES_FILE_PATH": str(path)})
    pm = model.PrecomputedMatching(cfg)
    a, b = pm.get_correspondences({"pair_id": torch.tensor([1])})
    assert a.dtype == np.float32 and a.shape == (3, 2) and np.array_equal(b[2], [10, 11])
    a, b = pm.get_correspondences({"pair_id": torch.tensor([0])})
    assert len(a) == 0 and len(b) == 0


def test_submission_format_and_mat2quat(tmp_path):
    from mfr_b200 import synth
    R = synth.rodrigues([0.3, -0.2, 0.5])
    q = submission.mat2quat(R)
    assert q[0] > 0 and abs(np.linalg.norm(q) - 1) < 1e-12
    w, x, y, z = q
    Rq = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                   [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                   [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    assert np.abs(Rq - R).max() < 1e-12
    p = submission.Pose("seq1/frame_00005.jpg", q, np.array([0.1, -0.25, 1.0]), 57)
    parts = str(p).split(" ")
    assert parts[0] == "seq1/frame_00005.jpg" and len(parts) == 9 and parts[-1] == "57"
    assert all(len(s.split(".")[1]) == 6 for s in parts[1:8])
    out = tmp_path / "submission.zip"
    submission.save_submission({"s00460": [p, p]}, out)
    with zipfile.ZipFile(out) as z:
        assert z.namelist() == ["pose_s00460.txt"]
        assert z.read("pose_s00460.txt").decode().count("\n") == 1


def test_model_rejects_unknown_plugins():
    cfg = config.load_cfg(overrides={"MODEL": "FeatureMatching", "FEATURE_MATCHING": "nope", "POSE_SOLVER": "PNP"})
    with pytest.raises(NotImplementedError):
        model.FeatureMatchingModel(cfg)
    cfg.MODEL = "Regression"
    with pytest.raises(NotImplementedError):
        model.build_model(cfg)


def test_linear_attention_stage_reference_matches_oracle():
    """The fp64 restatement the GPU stage test (tests/test_loftr_gpu.py::test_linear_attention_stage) checks the kernels
    against is the oracle's LinearAttention (linear_attention.py:31-45) with the feature map applied outside and the
    v / S ... * S pair cancelled."""
    import torch
    from oracle import loftr_oracle as lo
    from test_loftr_gpu import _lin_att_ref
    g = torch.Generator().manual_seed(5)
    n, L, S, H, D = 2, 37, 53, 8, 32
    q = torch.randn(n, L, H * D, generator=g); k = torch.randn(n, S, H * D, generator=g); v = torch.randn(n, S, H * D, generator=g)
    want = lo.linear_attention(q.view(n, L, H, D), k.view(n, S, H, D), v.view(n, S, H, D)).reshape(n, L, H * D)
    got = _lin_att_ref(torch.nn.functional.elu(q) + 1, torch.nn.functional.elu(k) + 1, v, H)
    assert torch.allclose(got.float(), want, rtol=1e-4, atol=1e-5)


def test_launch_summary_of_committed_profile(tmp_path):
    """profiles tooling: an ncu launch list (warm-up pass, then one step starting at its stem launch) summarises to the
    per-kernel totals of the last step."""
    import os, subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    rows = ['"ID","Kernel Name","Metric Name","Metric Unit","Metric Value"']
    step = [("stem_mma_kernel", "usecond", "10.5")] + [("conv_gemm_kernel<128, 1>", "nsecond", "2,000")] * 94 + \
           [("layernorm_kernel", "usecond", "1")] * 91
    for i, (k, u, v) in enumerate(step[:40] + step):              # a partial warm-up pass before the step
        rows.append(f'"{i}","{k}(params)","gpu__time_duration.sum","{u}","{v}"')
    csv_path = tmp_path / "launches.csv"
    csv_path.write_text("\n".join(rows) + "\n")
    out = subprocess.run([sys.executable, os.path.join(root, "scripts", "summarize_launches.py"), str(csv_path)],
                         capture_output=True, text=True, check=True).stdout
    first = out.splitlines()[0]
    assert first.startswith("186 launches, 289.5 us total"), first
    conv = next(l for l in out.splitlines() if l.startswith("conv_gemm_kernel"))
    assert int(conv.split("x")[1].split()[0]) == 94
