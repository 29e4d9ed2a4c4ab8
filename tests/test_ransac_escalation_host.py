"""The CONFIDENCE escalation without a GPU: the device's stopping rule (mfr_host_ransac_satisfied, the __host__
__device__ function the escalate kernel runs) against the solver plugins' host rule (pose_solver._SolverBase._satisfied
and required_hypotheses), and the method configs' confidence and cap reaching the stream's pose stages."""
import pytest

from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)
from mfr_b200 import lib, pose_solver
from mfr_b200.pipeline import EMatMetricStage, PnPStage, ProcrustesStage, resolve_method
from test_pipeline_cfg_host import CONFIGS, _cfg

CONFIDENCES = (0.9, 0.99, 0.9999, 0.999999, 1.0)
POINTS = (5, 37, 2000, 8192)
BUDGETS = (128, 512, 2048, 8192, 32768)
CAP = 32768


def _plugin_rule(sample_size):
    """A _SolverBase with the cap and sample size set, without a backend (its _satisfied reads nothing else)."""
    s = object.__new__(pose_solver._SolverBase)
    s.max_hyp, s.SAMPLE_SIZE = CAP, sample_size
    return s


def _inlier_counts(N):
    if N <= 64:
        return range(0, N + 1)
    return sorted(set(range(0, N + 1, 7)) | set(range(0, 40)) | set(range(N - 40, N + 1)))


def _branch(n, N, s):
    w = min(max(n / N, 0.0), 1.0) ** s
    return "n0" if n <= 0 else "w1" if w >= 1.0 - 1e-12 else "w15" if w < 1e-15 else "w8" if w < 1e-8 else "log1p"


@pytest.mark.parametrize("sample_size", [4, 5])
def test_device_rule_matches_plugin_rule(sample_size):
    l = lib.load()
    rule = _plugin_rule(sample_size)
    seen, decisions = set(), set()
    for c in CONFIDENCES:
        for N in POINTS:
            for n in _inlier_counts(N):
                seen.add(_branch(n, N, sample_size))
                for h in BUDGETS:
                    want = rule._satisfied(c, n, N, h)
                    got = l.mfr_host_ransac_satisfied(c, n, N, h, CAP, sample_size)
                    assert got == int(want), (c, n, N, h, sample_size)
                    decisions.add(want)
    assert seen == {"n0", "w1", "w15", "w8", "log1p"}, seen
    assert decisions == {True, False}
    # no correspondences: satisfied at once; correspondences but no inlier: only at the cap
    assert l.mfr_host_ransac_satisfied(0.9999, 0, 0, 128, CAP, sample_size) == 1
    assert [l.mfr_host_ransac_satisfied(0.9999, 0, 2000, h, CAP, sample_size) for h in BUDGETS] == [0, 0, 0, 0, 1]


def test_required_hypotheses_table():
    """The budgets of the escalation's motivating table (confidence 0.9999, E-mat sample of 5)."""
    req = [pose_solver.required_hypotheses(0.9999, r, 5) for r in (0.5, 0.3, 0.2)]
    assert 280 <= req[0] <= 300 and 3700 <= req[1] <= 3900 and 28000 <= req[2] <= 29500, req
    l = lib.load()
    for r, first_ok in zip((0.5, 0.3, 0.2), (2048, 8192, 32768)):
        n = int(round(r * 2000))
        got = [h for h in (2048, 8192, 32768) if l.mfr_host_ransac_satisfied(0.9999, n, 2000, h, CAP, 5)]
        assert got[0] == first_ok, (r, got)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_resolve_method_escalation(name):
    spec = resolve_method(_cfg(name))
    proc = spec.solver == "Procrustes"
    assert spec.confidence == (None if proc else 0.9999)
    assert spec.max_hyp == 32768                      # GPU_RANSAC.MAX_HYPOTHESES default
    plain, esc = spec.stage(), spec.stage(escalate=True)
    cls = {"EssentialMatrixMetric": EMatMetricStage, "PNP": PnPStage, "Procrustes": ProcrustesStage}[spec.solver]
    assert type(plain) is cls and type(esc) is cls
    assert vars(spec.stage(escalate=False)) == vars(plain)
    if proc:
        assert vars(esc) == vars(plain)               # the Procrustes plugin does not escalate
        return
    assert (plain.confidence, plain.max_hyp) == (None, None)
    assert (esc.confidence, esc.max_hyp) == (0.9999, 32768)
    assert {k: v for k, v in vars(esc).items() if k not in ("confidence", "max_hyp")} == \
        {k: v for k, v in vars(plain).items() if k not in ("confidence", "max_hyp")}


def test_escalation_settings_follow_the_plugins():
    """Cap and confidence come from the same keys the plugins read: MAX_HYPOTHESES below the first budget is raised
    to it, an unset CONFIDENCE leaves the stage at one budget even when asked to escalate."""
    spec = resolve_method(_cfg("sift_pnp_dptkitti", {"GPU_RANSAC": {"MAX_HYPOTHESES": 4096}, "PNP": {"CONFIDENCE": 0.99}}))
    assert (spec.num_hyp, spec.max_hyp, spec.confidence) == (1024, 4096, 0.99)
    spec = resolve_method(_cfg("sg_emat_dptnyu", {"GPU_RANSAC": {"NUM_HYPOTHESES": 4096, "MAX_HYPOTHESES": 1000}}))
    assert (spec.num_hyp, spec.max_hyp) == (4096, 4096)
    spec = resolve_method(_cfg("loftr_emat_dptkitti", {"EMAT_RANSAC": {"CONFIDENCE": None}}))
    assert spec.confidence is None and spec.stage(escalate=True).confidence is None
