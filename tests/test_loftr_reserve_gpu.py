"""reserved_sms of mfr_loftr_create, which LoFTR(pipelined=True) sets to 8: the first conv launches of a forward run on
fewer SMs, so that the pose back end of the previous batch finds room next to them. Fewer CTAs change which CTA
computes a tile, never how a tile is computed, so the matches must be bit-identical to those of an engine that uses
every SM."""
import ctypes

import pytest
import torch

from helpers import fullres_inputs

pytestmark = pytest.mark.gpu

KEYS = ("b_ids", "i_ids", "j_ids", "mkpts0_f", "mkpts1_f", "mconf")


def test_pipelined_engine_bit_identical():
    """bf16 engines with pipelined=True and False on one 720x540 pair in the 720x544 frame: there the first conv
    launches have far more tiles than SMs, so the SM limit takes effect (a 160x120 frame has fewer tiles than SMs)."""
    from mfr_b200 import loftr
    i0, i1 = fullres_inputs()
    i0, i1 = i0[:1].cuda(), i1[:1].cuda()
    sd = loftr.functional_state_dict()
    outs = []
    for pipelined in (False, True):
        eng = loftr.LoFTR(sd, batch=1, height=720, width=544, precision="bf16", pipelined=pipelined)
        out = eng.forward(i0, i1)
        outs.append({k: out[k].clone() for k in KEYS})
        eng.close()
    assert outs[0]["b_ids"].numel() > 0
    for k in KEYS:
        assert torch.equal(outs[0][k], outs[1][k]), f"{k} differs with reserved SMs"
    torch.cuda.empty_cache()


def test_reserved_sms_range(mfr):
    """0 <= reserved_sms < SM count: -1 and the SM count are rejected with MFR_ERR_ARG and no engine; SM count - 1 is
    accepted."""
    lib = mfr.load()
    n = lib.mfr_device_sm_count()
    assert n > 1
    for reserved, rc_want in ((-1, 2), (n, 2), (n - 1, 0)):
        h = ctypes.c_void_p()
        rc = lib.mfr_loftr_create(1, 160, 120, 0.2, 2, 0.1, 1, reserved, ctypes.byref(h))
        assert rc == rc_want, (reserved, rc)
        if rc == 0:
            lib.mfr_loftr_destroy(h)
        else:
            assert not h.value
