"""MAGSAC++ scoring without a GPU: the fp64 loss the LO / polish kernels run (mfr_host_magsac_loss, the __host__ __device__
function itself) against the scipy oracle, its constants and derivative, and the GPU_RANSAC.SCORING config key."""
import ctypes

import numpy as np
import pytest
from scipy import special, stats

import magsac_oracle as mo
from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)
from mfr_b200 import config, lib, pose_solver
from mfr_b200.pipeline import EMatMetricStage, EMatStage, resolve_method
from test_pipeline_cfg_host import CONFIGS, _cfg

SIGMAS = (1e-4, 2.7e-3, 4e-3, 0.05, 1.0)


def _loss(r, sigma):
    l = lib.load()
    rho, w = ctypes.c_double(), ctypes.c_double()
    assert l.mfr_host_magsac_loss(float(r), float(sigma), ctypes.byref(rho), ctypes.byref(w)) == 0
    return rho.value, w.value


def _grid(sigma, n=2001):
    return np.linspace(0.0, 1.2 * mo.K * sigma, n)


def test_constants():
    assert mo.C == 0.25 and special.gamma(2) == 1.0
    assert abs(stats.chi.ppf(0.99, 4) - 3.6437) < 1e-4 and round(stats.chi.ppf(0.99, 4), 2) == mo.K
    xk = mo.K * mo.K / 2
    assert abs(mo.upper_gamma(1.5, xk) - 0.0036573) < 5e-8
    assert abs(mo.lower_gamma(2.5, xk) - 1.3012) < 5e-5
    # the closed forms the kernels use
    for x in (1e-6, 0.3, 1.0, 2.5, xk):
        sx = np.sqrt(x)
        assert np.isclose(sx * np.exp(-x) + np.sqrt(np.pi) / 2 * special.erfc(sx), mo.upper_gamma(1.5, x), rtol=1e-13)
        assert np.isclose(3 * np.sqrt(np.pi) / 4 * special.erf(sx) - sx * np.exp(-x) * (x + 1.5), mo.lower_gamma(2.5, x),
                          rtol=1e-8)
    # rho at the cut-off, from the device code: C 2^1.5 sigma gamma(2.5, x_k)
    assert np.isclose(_loss(10.0, 1.0)[0], 0.25 * 2 ** 1.5 * mo.lower_gamma(2.5, xk), rtol=1e-14)


@pytest.mark.parametrize("sigma", SIGMAS)
def test_loss_against_oracle(sigma):
    r = _grid(sigma)
    got = np.array([_loss(x, sigma) for x in r])
    rho, w = mo.rho(r, sigma), mo.weight(r, sigma)
    np.testing.assert_allclose(got[:, 0], rho, rtol=1e-12, atol=1e-300)
    # w -> 0 at the cut-off, where Gamma(1.5, x) - G_k cancels: relative 1e-12 of w(0) there
    np.testing.assert_allclose(got[:, 1], w, rtol=1e-12, atol=1e-12 * w[0])


@pytest.mark.parametrize("sigma", SIGMAS)
def test_weight_is_derivative(sigma):
    """w = rho' / r: central difference of the device rho away from 0 and from the cut-off."""
    for r in np.linspace(0.02, 0.98, 25) * mo.K * sigma:
        h = 1e-5 * sigma
        d = (_loss(r + h, sigma)[0] - _loss(r - h, sigma)[0]) / (2 * h)
        assert np.isclose(d / r, _loss(r, sigma)[1], rtol=1e-6), (r, sigma)


@pytest.mark.parametrize("sigma", SIGMAS)
def test_continuous_and_constant_past_cutoff(sigma):
    kc = mo.K * sigma
    below, above = _loss(kc * (1 - 1e-9), sigma), _loss(kc * (1 + 1e-12), sigma)
    assert np.isclose(below[0], above[0], rtol=1e-12) and abs(below[1]) < 1e-6 * _loss(0.0, sigma)[1] and above[1] == 0.0
    rho = np.array([_loss(r, sigma)[0] for r in _grid(sigma)])
    assert np.all(np.diff(rho) >= 0.0)                      # non-decreasing, rho(0) = 0
    assert rho[0] == 0.0
    past = [_loss(kc * f, sigma) for f in (1 + 1e-12, 1.01, 2.0, 1e3)]
    assert all(p == above for p in past)


def test_bad_sigma_rejected():
    l = lib.load()
    rho, w = ctypes.c_double(), ctypes.c_double()
    for s in (0.0, -1.0, float("nan")):
        assert l.mfr_host_magsac_loss(0.1, s, ctypes.byref(rho), ctypes.byref(w)) != 0


# ------------------------------------------------------------------------------------------------ GPU_RANSAC.SCORING
def test_default_is_msac():
    assert config.get_default_cfg().GPU_RANSAC.SCORING == "msac"
    assert pose_solver.ransac_scoring(config.get_default_cfg()) == "msac"
    assert pose_solver.ransac_scoring({}) == "msac"


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_shipped_configs_resolve_to_msac(name):
    """Every shipped method config keeps MSAC and the stage it had: same type, lo flags and budget."""
    spec = resolve_method(_cfg(name))
    assert spec.scoring == "msac"
    stage = spec.stage()
    if spec.solver.startswith("EssentialMatrix"):
        assert stage.scoring == "msac" and stage.lo == pose_solver.LO_LSQ == spec.lo
    assert not hasattr(stage, "scoring") or stage.scoring == "msac"


@pytest.mark.parametrize("name", ["loftr_emat_dptkitti", "sift_emat_dptnyu"])
def test_magsac_reaches_the_stage(name):
    spec = resolve_method(_cfg(name, {"GPU_RANSAC": {"SCORING": "MAGSAC"}}))
    assert spec.scoring == "magsac"
    for esc in (False, True):
        stage = spec.stage(escalate=esc)
        assert type(stage) is EMatMetricStage and stage.scoring == "magsac" and stage.lo is True
    cfg = config.get_default_cfg()
    cfg.merge_from_dict({"FEATURE_MATCHING": "SIFT", "POSE_SOLVER": "EssentialMatrix", "EMAT_RANSAC": {"PIX_THRESHOLD": 2.0},
                         "GPU_RANSAC": {"SCORING": "magsac"}})
    stage = resolve_method(cfg).stage()
    assert type(stage) is EMatStage and stage.scoring == "magsac"


def test_pnp_and_procrustes_ignore_scoring():
    """SCORING is an E-mat key: the PnP and Procrustes specs keep the default."""
    for name in ("sg_pnp_dptkitti", "sg_procrustes_dptkitti"):
        assert resolve_method(_cfg(name, {"GPU_RANSAC": {"SCORING": "magsac"}})).scoring == "msac"


@pytest.mark.parametrize("over", [
    {"SCORING": "ransac"}, {"SCORING": "prosac"}, {"SCORING": ""},
    {"SCORING": "magsac", "LOCAL_OPTIMISATION": False},
    {"SCORING": "magsac", "FINAL_REFIT": "tukey"},
])
def test_invalid_values_raise(over):
    cfg = _cfg("sg_emat_dptkitti", {"GPU_RANSAC": over})
    with pytest.raises(ValueError):
        pose_solver.ransac_scoring(cfg)
    with pytest.raises(ValueError):
        resolve_method(cfg)


def test_msac_with_lo_keys_still_valid():
    cfg = _cfg("sg_emat_dptkitti", {"GPU_RANSAC": {"SCORING": "msac", "LOCAL_OPTIMISATION": False, "FINAL_REFIT": "tukey"}})
    assert pose_solver.ransac_scoring(cfg) == "msac" and resolve_method(cfg).lo == 0
