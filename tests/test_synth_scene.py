"""synth.make_scene: one map frame and its query frames, drawn in make_pair's order and with its conventions."""
import numpy as np

from helpers import synth


def test_make_scene_shapes():
    K = np.array([[300.0, 0, 159.5], [0, 300.0, 119.5], [0, 0, 1]])
    s = synth.make_scene(7, 3, h=120, w=160, K=K)
    assert s["image0"].shape == (3, 120, 160) and s["image0"].dtype == np.float32
    assert s["gray0"].shape == (120, 160) and s["gray0"].dtype == np.float32
    assert 0.0 <= s["gray0"].min() and s["gray0"].max() <= 1.0
    assert s["depth0"].shape == (120, 160) and s["depth0"].dtype == np.float32
    assert np.array_equal(s["K_color0"], K.astype(np.float32))
    assert len(s["queries"]) == 3
    for q in s["queries"]:
        assert q["image1"].shape == (3, 120, 160) and q["gray1"].shape == (120, 160) and q["depth1"].shape == (120, 160)
        assert np.array_equal(q["K_color1"], K.astype(np.float32))
        assert np.allclose(q["R_gt"] @ q["R_gt"].T, np.eye(3), atol=1e-12) and q["t_gt"].shape == (3,)
    poses = [(q["R_gt"], q["t_gt"]) for q in s["queries"]]
    assert not np.allclose(poses[0][1], poses[1][1]), "every query has its own pose"
    assert np.array_equal(s["gray0"], synth.rgb_to_gray_u8(s["image0"]).astype(np.float32) / 255.0)


def test_make_scene_agrees_with_make_pair():
    h, w = 96, 128
    for i in (0, 3):
        p = synth.make_pair(i, h=h, w=w)
        s = synth.make_scene(1000 + i, 2, h=h, w=w)
        q = s["queries"][0]
        for a, b in ((s["image0"], p["image0"]), (s["depth0"], p["depth0"]), (s["K_color0"], p["K_color0"]),
                     (q["image1"], p["image1"]), (q["depth1"], p["depth1"]), (q["K_color1"], p["K_color1"]),
                     (q["R_gt"], p["R_gt"]), (q["t_gt"], p["t_gt"])):
            assert a.dtype == b.dtype and np.array_equal(a, b)
