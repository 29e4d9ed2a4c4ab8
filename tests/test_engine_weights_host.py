"""The weight loaders and the LoFTR frame rule that the matcher plugins, the estimator shell and pipeline.from_cfg share
(no GPU needed)."""
import numpy as np
import pytest
import torch

from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)
from mfr_b200 import config, loftr, spsg
from mfr_b200.pipeline import resolve_method


@pytest.fixture(scope="module")
def loftr_sd():
    return loftr.synthetic_state_dict(0)


def _loftr_cfg(height, width, **loftr_keys):
    cfg = config.get_default_cfg()
    cfg.merge_from_dict({"FEATURE_MATCHING": "LoFTR", "POSE_SOLVER": "EssentialMatrix",
                         "DATASET": {"HEIGHT": height, "WIDTH": width}, "LOFTR": loftr_keys})
    return cfg


def test_loftr_weights_every_form(loftr_sd, tmp_path):
    """A bare state dict, a Lightning checkpoint (keys under "matcher."), and a saved file of each: one engine table."""
    ckpt = {"state_dict": {"matcher." + k: v for k, v in loftr_sd.items()}, "epoch": 3}
    torch.save(loftr_sd, tmp_path / "bare.pt")
    torch.save(ckpt, tmp_path / "lightning.ckpt")
    ref = loftr.prepare_weights(loftr_sd, 4, 4)
    for w in (loftr_sd, ckpt, str(tmp_path / "bare.pt"), str(tmp_path / "lightning.ckpt")):
        got = loftr.prepare_weights(loftr.load_weights(w), 4, 4)
        assert got.keys() == ref.keys()
        assert all(np.array_equal(got[k], ref[k]) for k in ref)


@pytest.mark.parametrize("hw, frame", [((720, 540), (720, 544)), ((720, 720), (720, 720)), ((540, 720), (544, 720))])
def test_loftr_frame(hw, frame):
    assert loftr.engine_frame(*hw) == frame
    spec = resolve_method(_loftr_cfg(*hw))
    assert (spec.height, spec.width) == frame


@pytest.mark.parametrize("hw", [(721, 540), (720, 542)])
def test_loftr_frame_not_a_multiple_of_8(hw):
    """721 % 8 = 1 pads to 722, 542 % 8 = 6 to 548: neither is a multiple of 8."""
    with pytest.raises(ValueError):
        loftr.engine_frame(*hw)
    with pytest.raises(ValueError):
        resolve_method(_loftr_cfg(*hw))


def test_loftr_engine_cfg():
    assert loftr.engine_cfg(_loftr_cfg(720, 540)) == loftr.DEFAULT_CFG
    got = loftr.engine_cfg(_loftr_cfg(720, 540, THR=0.5, BORDER_RM=3, TEMPERATURE=None))
    assert got == {"thr": 0.5, "border_rm": 3, "temperature": loftr.DEFAULT_CFG["temperature"]}
    assert loftr.engine_cfg({}) == loftr.DEFAULT_CFG


@pytest.mark.parametrize("outdoor", [False, True])
def test_spsg_weights_pair_or_directory(tmp_path, outdoor):
    sp, sg = spsg.synthetic_state_dicts(0)
    sg_other = {k: v + 1 for k, v in sg.items()}
    torch.save(sp, tmp_path / "superpoint_v1.pth")
    torch.save(sg_other if outdoor else sg, tmp_path / "superglue_indoor.pth")
    torch.save(sg if outdoor else sg_other, tmp_path / "superglue_outdoor.pth")
    for got_sp, got_sg in (spsg.load_weights((sp, sg), outdoor), spsg.load_weights(str(tmp_path), outdoor)):
        assert got_sp.keys() == sp.keys() and all(torch.equal(got_sp[k], sp[k]) for k in sp)
        assert got_sg.keys() == sg.keys() and all(torch.equal(got_sg[k], sg[k]) for k in sg)
