"""Rules every engine shares through its host-side core (csrc/engine_core.cuh), checked through the C ABI: a forward is
refused until every weight tensor has been uploaded, and debug buffers report their size in 4-byte words."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
B, H, W, K = 1, 96, 128, 256
MFR_ERR_ARG = 2


def _create(l, engine, precision=0):
    h = ctypes.c_void_p()
    if engine == "loftr":
        rc = l.mfr_loftr_create(B, H, W, 0.2, 2, 0.1, precision, 0, ctypes.byref(h))
    elif engine == "spsg":
        rc = l.mfr_spsg_create_ex(B, H, W, K, 4, 0.005, 4, 20, 0.2, precision, ctypes.byref(h))
    else:
        rc = l.mfr_sift_create(B, H, W, 0, 1024, 0, ctypes.byref(h))
    assert rc == 0
    return h


def _words(l, engine, h, name):
    p, n = ctypes.c_void_p(), ctypes.c_longlong()
    assert getattr(l, f"mfr_{engine}_debug_tensor")(h, name.encode(), ctypes.byref(p), ctypes.byref(n)) == 0
    return n.value


@pytest.mark.parametrize("engine", ["loftr", "spsg"])
def test_forward_refused_until_every_weight_is_uploaded(mfr, engine):
    from mfr_b200 import loftr, spsg
    l = mfr.load()
    h = _create(l, engine)
    st = torch.cuda.Stream()
    sp = ctypes.c_void_p(st.cuda_stream)
    img = torch.rand(B, H, W, device="cuda")
    if engine == "loftr":
        w = loftr.prepare_weights(loftr.synthetic_state_dict(0), H // 8, W // 8)
        forward = lambda: l.mfr_loftr_forward(h, mfr.ptr(img), mfr.ptr(img), H, W, sp)
    else:
        w = spsg.prepare_weights(*spsg.synthetic_state_dicts(0))
        forward = lambda: l.mfr_spsg_forward(h, mfr.ptr(img), mfr.ptr(img), sp)
    try:
        getattr(l, f"mfr_{engine}_set_graph")(h, 0)
        torch.cuda.synchronize()

        def upload(i):
            a = w[getattr(l, f"mfr_{engine}_weight_name")(h, i).decode()].reshape(-1)
            assert getattr(l, f"mfr_{engine}_set_weight")(h, i, a.ctypes.data_as(ctypes.c_void_p), a.size, sp) == 0

        n = getattr(l, f"mfr_{engine}_num_weights")(h)
        for i in range(1, n):   # every tensor but the first, the last one included
            upload(i)
        assert forward() == MFR_ERR_ARG
        upload(0)
        assert forward() == 0
        st.synchronize()
    finally:
        getattr(l, f"mfr_{engine}_destroy")(h)


def test_debug_sizes_are_words(mfr):
    l = mfr.load()
    px2 = 2 * B * (H // 2) * (W // 2)
    for precision, words in ((0, px2 * 128), (1, px2 * 128 // 2)):   # "a0" holds fp32 in tf32 mode, bf16 in bf16 mode
        h = _create(l, "loftr", precision)
        try:
            assert _words(l, "loftr", h, "a0") == words
        finally:
            l.mfr_loftr_destroy(h)
    h = _create(l, "spsg", 1)   # bf16 q|k|v
    try:
        assert _words(l, "spsg", h, "qkv") == 2 * B * K * 768 // 2
    finally:
        l.mfr_spsg_destroy(h)
    h = _create(l, "sift")
    try:
        assert _words(l, "sift", h, "extrema_f") == B * 1024 * 4
    finally:
        l.mfr_sift_destroy(h)
