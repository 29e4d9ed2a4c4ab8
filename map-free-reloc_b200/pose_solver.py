"""Host side of the pose back end. Mirrors the reference's solver plugins
(lib/models/matching/pose_solver.py): classes with ``__init__(cfg)`` and
``estimate_pose(kpts0, kpts1, data) -> (R[3,3], t, inliers)``, NaN-filled on failure, while the
arithmetic runs in the batched-hypothesis CUDA kernels of libmfr_b200.so. ``PoseBackend`` is the
batched device-resident interface the fused matcher+solver pipeline and the benchmark use.
"""
import ctypes
import math
import warnings

import numpy as np
import torch

from . import lib as _lib

DEFAULT_NUM_HYP = 2048
DEFAULT_SEED = 0x5EED
LO_TUKEY, LO_LSQ = 1, 3       # mfr_emat_ransac lo_enabled flags: bit 0 local optimisation, bit 1 final least-squares refit
DEFAULT_FINAL_REFIT = "lsq"
SCORINGS = ("msac", "magsac")  # GPU_RANSAC.SCORING: E-mat RANSAC objective (mfr_emat_ransac* / mfr_emat_magsac)
MAX_PTS_LIMIT = 8192          # correspondences per pair the RANSAC kernels can hold (shared memory)


def _cfg_get(cfg, path, default=None):
    cur = cfg
    for k in path.split("."):
        try:
            cur = cur[k] if isinstance(cur, dict) else getattr(cur, k)
        except (KeyError, AttributeError):
            return default
    return default if cur is None else cur


class PoseBackend(_lib.Engine):
    """Batched GPU pose solver for up to ``max_pairs`` pairs per call, on the caller's current stream."""

    def __init__(self, max_pairs=1, max_pts=8192, max_hyp=8192, device=0):
        if not 8 <= int(max_pts) <= MAX_PTS_LIMIT:
            raise ValueError(f"PoseBackend: max_pts must be in [8, {MAX_PTS_LIMIT}] (correspondences of a pair are staged "
                             f"in shared memory), got {max_pts}")
        super().__init__("pose_solver", "mfr_pose_solver_create", (int(max_pairs), int(max_pts), int(max_hyp)), device,
                         stream=False)
        self.max_pairs, self.max_pts, self.max_hyp = int(max_pairs), int(max_pts), int(max_hyp)

    def _outs(self, P, total):
        dev = self.device
        return (torch.empty(P, 3, 3, device=dev), torch.empty(P, 3, device=dev),
                torch.empty(P, dtype=torch.int32, device=dev), torch.empty(max(total, 1), dtype=torch.uint8, device=dev))

    @staticmethod
    def _prep(kpts0, kpts1, offsets, K0, K1):
        assert kpts0.is_cuda and kpts0.dtype == torch.float32 and kpts0.is_contiguous()
        assert kpts1.is_cuda and kpts1.dtype == torch.float32 and kpts1.is_contiguous()
        assert offsets.is_cuda and offsets.dtype == torch.int32
        assert K0.is_cuda and K0.dtype == torch.float32 and K0.is_contiguous()
        assert K1.is_cuda and K1.dtype == torch.float32 and K1.is_contiguous()
        return offsets.numel() - 1

    def _escalation(self, P, num_hyp, max_hyp, budgets):
        """(cap, budgets pointer) of an escalating call: the cap defaults to the handle's max_hyp."""
        cap = self.max_hyp if max_hyp is None else int(max_hyp)
        if cap < int(num_hyp):
            raise ValueError(f"max_hyp {cap} is below the first budget {num_hyp}")
        if budgets is not None:
            assert budgets.is_cuda and budgets.dtype == torch.int32 and budgets.is_contiguous() and budgets.numel() >= P
        return cap, _lib.ptr(budgets)

    def emat(self, kpts0, kpts1, offsets, K0, K1, pix_thr, num_hyp=DEFAULT_NUM_HYP, seed=DEFAULT_SEED,
             lo=True, total=None, confidence=None, max_hyp=None, budgets=None, scoring="msac"):
        """EssentialMatrixSolver for P pairs. Returns R [P,3,3], t [P,3] (unit), n [P], mask [total].
        lo: False / 0 = raw RANSAC winner; True / 1 = local optimisation (LO_TUKEY); 3 = LO + the final truncated
        least-squares refit on the model's own inlier set (LO_LSQ, the reference-equivalent optimum).
        confidence: None = one solve at num_hyp; else EMAT_RANSAC.CONFIDENCE, escalated per pair on the device as the
        plugins do (x4 per round up to max_hyp, default the handle's max_hyp; mfr_emat_ransac_escalate). budgets: optional
        int32 [P] CUDA tensor that receives the budget each pair's result comes from (0: fewer than 5 correspondences).
        scoring: "msac" (the above) or "magsac", the estimator of the reference's cv.USAC_MAGSAC (mfr_emat_magsac:
        MAGSAC++ scoring, sigma-consensus++ LO and polish); ``lo`` must then stay at its default."""
        if scoring not in SCORINGS:
            raise ValueError(f"scoring must be one of {SCORINGS}, got {scoring!r}")
        if scoring == "magsac" and lo is not True:
            raise ValueError("scoring='magsac' has its own local optimisation: leave lo at its default")
        P = self._prep(kpts0, kpts1, offsets, K0, K1)
        total = kpts0.shape[0] if total is None else total
        R, t, n, mask = self._outs(P, total)
        head = (self._h, _lib.ptr(kpts0), _lib.ptr(kpts1), _lib.ptr(offsets), P, _lib.ptr(K0), _lib.ptr(K1), float(pix_thr),
                int(num_hyp), ctypes.c_ulonglong(seed))
        outs = (_lib.ptr(R), _lib.ptr(t), _lib.ptr(n), _lib.ptr(mask))
        if scoring == "magsac":
            cap, b = (int(num_hyp), _lib.ptr(budgets)) if confidence is None else self._escalation(P, num_hyp, max_hyp, budgets)
            _lib.check(self._l.mfr_emat_magsac(*head, *outs, 0.0 if confidence is None else float(confidence), cap, b,
                                               _lib.cur_stream()), "mfr_emat_magsac")
            return R, t, n, mask
        args = (*head, int(lo), *outs)
        if confidence is None:
            _lib.check(self._l.mfr_emat_ransac(*args, _lib.cur_stream()), "mfr_emat_ransac")
        else:
            cap, b = self._escalation(P, num_hyp, max_hyp, budgets)
            _lib.check(self._l.mfr_emat_ransac_escalate(*args, float(confidence), cap, b, _lib.cur_stream()),
                       "mfr_emat_ransac_escalate")
        return R, t, n, mask

    def scale(self, kpts0, kpts1, offsets, K0, K1, mask, depth0, depth1, scale_thr, Rd=None, td=None):
        """Scale-from-depth step of EssentialMatrixMetricSolver (uses the pose kept by ``emat`` when
        Rd/td are None). depth0/depth1: [P,H,W] float32 CUDA."""
        P = self._prep(kpts0, kpts1, offsets, K0, K1)
        H, W = depth0.shape[-2:]
        R = torch.empty(P, 3, 3, device=self.device)
        t = torch.empty(P, 3, device=self.device)
        n = torch.empty(P, dtype=torch.int32, device=self.device)
        _lib.check(self._l.mfr_scale_from_depth(
            self._h, _lib.ptr(kpts0), _lib.ptr(kpts1), _lib.ptr(offsets), P, _lib.ptr(K0), _lib.ptr(K1),
            _lib.ptr(mask), _lib.ptr(Rd), _lib.ptr(td), _lib.ptr(depth0.contiguous()),
            _lib.ptr(depth1.contiguous()), int(H), int(W), float(scale_thr), _lib.ptr(R), _lib.ptr(t),
            _lib.ptr(n), _lib.cur_stream()), "mfr_scale_from_depth")
        return R, t, n

    def emat_metric(self, kpts0, kpts1, offsets, K0, K1, depth0, depth1, pix_thr, scale_thr,
                    num_hyp=DEFAULT_NUM_HYP, seed=DEFAULT_SEED, lo=True, confidence=None, max_hyp=None, budgets=None,
                    scoring="msac"):
        """EssentialMatrixMetricSolver for P pairs: R [P,3,3], t [P,3] metres, inliers [P]. confidence / max_hyp /
        budgets / scoring: the E-mat escalation and objective of ``emat`` (the escalation is driven by the E-mat inlier
        count); the scale runs once, on the final pose."""
        _, _, _, mask = self.emat(kpts0, kpts1, offsets, K0, K1, pix_thr, num_hyp, seed, lo, confidence=confidence,
                                  max_hyp=max_hyp, budgets=budgets, scoring=scoring)
        return self.scale(kpts0, kpts1, offsets, K0, K1, mask, depth0, depth1, scale_thr)

    def pnp(self, kpts0, kpts1, offsets, K0, K1, depth0, reproj_thr, num_hyp=DEFAULT_NUM_HYP,
            seed=DEFAULT_SEED, confidence=None, max_hyp=None, budgets=None):
        """PnPSolver for P pairs: R [P,3,3], t [P,3], inliers [P], mask [total]. confidence / max_hyp / budgets: the
        PNP.CONFIDENCE escalation, as in ``emat`` (budget 0: fewer than 4 correspondences)."""
        P = self._prep(kpts0, kpts1, offsets, K0, K1)
        H, W = depth0.shape[-2:]
        R, t, n, mask = self._outs(P, kpts0.shape[0])
        depth0 = depth0.contiguous()
        args = (self._h, _lib.ptr(kpts0), _lib.ptr(kpts1), _lib.ptr(offsets), P, _lib.ptr(K0), _lib.ptr(K1),
                _lib.ptr(depth0), int(H), int(W), int(num_hyp), float(reproj_thr), ctypes.c_ulonglong(seed),
                _lib.ptr(R), _lib.ptr(t), _lib.ptr(n), _lib.ptr(mask))
        if confidence is None:
            _lib.check(self._l.mfr_pnp_ransac(*args, _lib.cur_stream()), "mfr_pnp_ransac")
        else:
            cap, b = self._escalation(P, num_hyp, max_hyp, budgets)
            _lib.check(self._l.mfr_pnp_ransac_escalate(*args, float(confidence), cap, b, _lib.cur_stream()),
                       "mfr_pnp_ransac_escalate")
        return R, t, n, mask

    def procrustes(self, kpts0, kpts1, offsets, K0, K1, depth0, depth1, max_corr_dist,
                   num_hyp=DEFAULT_NUM_HYP, seed=DEFAULT_SEED):
        """ProcrustesSolver (REFINE=False) for P pairs: R [P,3,3], t [P,3], inliers [P]."""
        P = self._prep(kpts0, kpts1, offsets, K0, K1)
        H, W = depth0.shape[-2:]
        R = torch.empty(P, 3, 3, device=self.device); t = torch.empty(P, 3, device=self.device)
        n = torch.empty(P, dtype=torch.int32, device=self.device)
        _lib.check(self._l.mfr_procrustes_ransac(
            self._h, _lib.ptr(kpts0), _lib.ptr(kpts1), _lib.ptr(offsets), P, _lib.ptr(K0), _lib.ptr(K1),
            _lib.ptr(depth0.contiguous()), _lib.ptr(depth1.contiguous()), int(H), int(W), int(num_hyp),
            float(max_corr_dist), ctypes.c_ulonglong(seed), _lib.ptr(R), _lib.ptr(t), _lib.ptr(n),
            _lib.cur_stream()), "mfr_procrustes_ransac")
        return R, t, n

    def icp(self, R_in, t_in, K0, K1, depth0, depth1, max_corr_dist, max_iter=30, rel_fitness=1e-4, rel_rmse=1e-4):
        """ICP refinement of ProcrustesSolver (REFINE=True) over the full depth clouds: R [P,3,3], t [P,3], inliers [P]."""
        P = R_in.shape[0]
        H, W = depth0.shape[-2:]
        R = torch.empty(P, 3, 3, device=self.device); t = torch.empty(P, 3, device=self.device)
        n = torch.empty(P, dtype=torch.int32, device=self.device)
        _lib.check(self._l.mfr_icp_refine(self._h, _lib.ptr(depth0.contiguous()), _lib.ptr(depth1.contiguous()), int(H), int(W), P,
                                          _lib.ptr(K0), _lib.ptr(K1), _lib.ptr(R_in.contiguous()), _lib.ptr(t_in.contiguous()),
                                          float(max_corr_dist), int(max_iter), float(rel_fitness), float(rel_rmse),
                                          _lib.ptr(R), _lib.ptr(t), _lib.ptr(n), _lib.cur_stream()), "mfr_icp_refine")
        return R, t, n


# ------------------------------------------------------------------------------------------------
# reference-shaped plugins (one pair per call, host arrays in / host arrays out)
# ------------------------------------------------------------------------------------------------
def required_hypotheses(confidence, inlier_ratio, sample_size):
    """RANSAC stopping rule (what cv2's `confidence` / `prob` argument drives): the number of minimal samples after
    which an all-inlier sample has been drawn with probability `confidence`, given the inlier ratio found."""
    w = min(max(float(inlier_ratio), 0.0), 1.0) ** sample_size
    if w >= 1.0 - 1e-12:
        return 1
    c = min(max(float(confidence), 0.0), 1.0 - 1e-12)
    if w < 1e-15:                      # no consensus at all: no finite budget reaches the confidence
        return 2 ** 31 - 1
    return int(min(2 ** 31 - 1, math.ceil(math.log(1.0 - c) / -w if w < 1e-8 else math.log(1.0 - c) / math.log1p(-w))))


def ransac_settings(cfg, default_hyp=DEFAULT_NUM_HYP):
    """GPU_RANSAC keys -> (first hypothesis budget, escalation cap, seed, lo flags of mfr_emat_ransac), as every solver
    plugin reads them; ``default_hyp`` is the solver's budget when NUM_HYPOTHESES is unset."""
    num_hyp = int(_cfg_get(cfg, "GPU_RANSAC.NUM_HYPOTHESES", default_hyp))
    max_hyp = max(num_hyp, int(_cfg_get(cfg, "GPU_RANSAC.MAX_HYPOTHESES", 32768)))
    seed = int(_cfg_get(cfg, "GPU_RANSAC.SEED", DEFAULT_SEED))
    lo = bool(_cfg_get(cfg, "GPU_RANSAC.LOCAL_OPTIMISATION", True))
    refit = str(_cfg_get(cfg, "GPU_RANSAC.FINAL_REFIT", DEFAULT_FINAL_REFIT)).lower()
    if refit not in ("lsq", "tukey"):
        raise ValueError("GPU_RANSAC.FINAL_REFIT must be 'lsq' or 'tukey'")
    return num_hyp, max_hyp, seed, (LO_LSQ if refit == "lsq" else LO_TUKEY) if lo else 0


def ransac_scoring(cfg):
    """GPU_RANSAC.SCORING -> "msac" (the default) or "magsac" (the MAGSAC++ estimator of the reference's USAC_MAGSAC).
    Anything else raises ValueError, and so does "magsac" with a non-default GPU_RANSAC.LOCAL_OPTIMISATION or FINAL_REFIT:
    MAGSAC++ has its own LO, so those keys would be ignored."""
    scoring = str(_cfg_get(cfg, "GPU_RANSAC.SCORING", "msac")).lower()
    if scoring not in SCORINGS:
        raise ValueError("GPU_RANSAC.SCORING must be 'msac' or 'magsac'")
    if scoring == "magsac" and (_cfg_get(cfg, "GPU_RANSAC.LOCAL_OPTIMISATION", True) is not True or
                                str(_cfg_get(cfg, "GPU_RANSAC.FINAL_REFIT", DEFAULT_FINAL_REFIT)).lower() != DEFAULT_FINAL_REFIT):
        raise ValueError("GPU_RANSAC.SCORING 'magsac' has its own local optimisation: leave GPU_RANSAC.LOCAL_OPTIMISATION "
                         "and GPU_RANSAC.FINAL_REFIT at their defaults")
    return scoring


def pnp_default_hyp(cfg):
    """PnPSolver's budget when GPU_RANSAC.NUM_HYPOTHESES is unset: PNP.RANSAC_ITER (the reference's iteration cap of
    cv2.solvePnPRansac) rounded up to a multiple of 128, at least 128."""
    iters = _cfg_get(cfg, "PNP.RANSAC_ITER")
    iters = int(iters) if iters else DEFAULT_NUM_HYP
    return max(128, (iters + 127) // 128 * 128)


class _SolverBase:
    """The GPU solvers run a fixed hypothesis budget per launch instead of OpenCV's sequential loop with an early
    exit. The reference's `CONFIDENCE` is honoured as an escalation rule: when the inlier ratio a launch found says
    that its budget was too small for the requested confidence (``required_hypotheses``), the launch is repeated with
    a larger budget (x4 per round, up to ``GPU_RANSAC.MAX_HYPOTHESES``)."""
    SAMPLE_SIZE = 5

    def __init__(self, cfg, default_hyp=DEFAULT_NUM_HYP):
        self.num_hyp, self.max_hyp, self.seed, self.lo = ransac_settings(cfg, default_hyp)
        self.backend = PoseBackend(max_pairs=1, max_hyp=max(self.max_hyp, 128))
        self.dev = self.backend.device
        self.last_num_hyp = 0       # budget of the launch whose result was returned

    def _budgets(self, confidence):
        """Hypothesis budgets to try in order; the caller stops at the first one that satisfies `confidence`."""
        h = self.num_hyp
        yield h
        if confidence is None:
            return
        while h < self.max_hyp:
            h = min(self.max_hyp, 4 * h)
            yield h

    def _satisfied(self, confidence, n_inliers, n_points, budget):
        if confidence is None or n_points <= 0 or n_inliers <= 0:    # nothing found: a larger budget is tried only when
            return confidence is None or n_points <= 0 or budget >= self.max_hyp   # some remains (and then the NaN pose stands)
        return budget >= required_hypotheses(confidence, n_inliers / float(n_points), self.SAMPLE_SIZE)

    def _upload(self, kpts0, kpts1, data):
        if len(kpts0) > MAX_PTS_LIMIT:    # the reference has no limit; no matcher on this path produces this many
            warnings.warn(f"{type(self).__name__}: {len(kpts0)} correspondences, the GPU solver takes the first "
                          f"{MAX_PTS_LIMIT}", RuntimeWarning, stacklevel=3)
            kpts0, kpts1 = kpts0[:MAX_PTS_LIMIT], kpts1[:MAX_PTS_LIMIT]
        k0 = torch.as_tensor(np.ascontiguousarray(kpts0, dtype=np.float32)).to(self.dev).reshape(-1, 2)
        k1 = torch.as_tensor(np.ascontiguousarray(kpts1, dtype=np.float32)).to(self.dev).reshape(-1, 2)
        off = torch.tensor([0, k0.shape[0]], dtype=torch.int32, device=self.dev)
        K0 = torch.as_tensor(data["K_color0"]).float().reshape(1, 3, 3).to(self.dev).contiguous()
        K1 = torch.as_tensor(data["K_color1"]).float().reshape(1, 3, 3).to(self.dev).contiguous()
        return k0, k1, off, K0, K1

    @staticmethod
    def _nan():
        return np.full((3, 3), np.nan), np.full((3, 1), np.nan), 0


class EssentialMatrixSolver(_SolverBase):
    """Relative pose up to scale from 2D-2D correspondences (pose_solver.py:20-61)."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.ransac_pix_threshold = float(_cfg_get(cfg, "EMAT_RANSAC.PIX_THRESHOLD"))
        self.ransac_confidence = _cfg_get(cfg, "EMAT_RANSAC.CONFIDENCE")  # escalation rule, see _SolverBase
        self.scoring = ransac_scoring(cfg)
        self.mask = None

    def estimate_pose(self, kpts0, kpts1, data):
        if len(kpts0) < 5:
            return self._nan()
        k0, k1, off, K0, K1 = self._upload(kpts0, kpts1, data)
        for budget in self._budgets(self.ransac_confidence):
            if self.scoring == "magsac":
                R, t, n, mask = self.backend.emat(k0, k1, off, K0, K1, self.ransac_pix_threshold, budget, self.seed,
                                                  scoring="magsac")
            else:
                R, t, n, mask = self.backend.emat(k0, k1, off, K0, K1, self.ransac_pix_threshold, budget,
                                                  self.seed, self.lo)
            n = int(n.item())
            self.last_num_hyp = budget
            if self._satisfied(self.ransac_confidence, n, k0.shape[0], budget):
                break
        self.mask = mask.cpu().numpy().reshape(-1, 1)
        self._dev = (k0, k1, off, K0, K1, mask)
        if n == 0:
            return self._nan()
        return R[0].double().cpu().numpy(), t[0].double().cpu().numpy(), n


class EssentialMatrixMetricSolver(EssentialMatrixSolver):
    """E-mat decomposition + scale from depth at the inliers (pose_solver.py:115-172)."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.ransac_scale_threshold = float(_cfg_get(cfg, "EMAT_RANSAC.SCALE_THRESHOLD"))

    def estimate_pose(self, kpts0, kpts1, data):
        R, t, inliers = super().estimate_pose(kpts0, kpts1, data)
        if inliers == 0:
            return R, t, inliers
        k0, k1, off, K0, K1, mask = self._dev
        d0 = torch.as_tensor(data["depth0"]).float().reshape(1, *torch.as_tensor(data["depth0"]).shape[-2:]).to(self.dev)
        d1 = torch.as_tensor(data["depth1"]).float().reshape(1, *torch.as_tensor(data["depth1"]).shape[-2:]).to(self.dev)
        R, t, n = self.backend.scale(k0, k1, off, K0, K1, mask, d0, d1, self.ransac_scale_threshold)
        n = int(n.item())
        if n == 0:
            return self._nan()
        return R[0].double().cpu().numpy(), t[0].double().cpu().numpy().reshape(3, 1), n


class PnPSolver(_SolverBase):
    """Metric relative pose from 2D-3D correspondences (pose_solver.py:175-235)."""

    SAMPLE_SIZE = 4   # P3P + the disambiguating 4th point

    def __init__(self, cfg):
        # PNP.RANSAC_ITER (reference: the iteration cap of cv2.solvePnPRansac) is the first launch's hypothesis
        # budget unless GPU_RANSAC.NUM_HYPOTHESES overrides it; PNP.CONFIDENCE escalates it (see _SolverBase)
        self.ransac_iterations = _cfg_get(cfg, "PNP.RANSAC_ITER")
        super().__init__(cfg, default_hyp=pnp_default_hyp(cfg))
        self.reprojection_inlier_threshold = float(_cfg_get(cfg, "PNP.REPROJECTION_INLIER_THRESHOLD"))
        self.confidence = _cfg_get(cfg, "PNP.CONFIDENCE")

    def estimate_pose(self, pts0, pts1, data):
        if len(pts0) < 4:
            return self._nan()
        k0, k1, off, K0, K1 = self._upload(pts0, pts1, data)
        d0 = torch.as_tensor(data["depth0"]).float()
        d0 = d0.reshape(1, *d0.shape[-2:]).to(self.dev)
        for budget in self._budgets(self.confidence):
            R, t, n, _ = self.backend.pnp(k0, k1, off, K0, K1, d0, self.reprojection_inlier_threshold,
                                          budget, self.seed)
            n = int(n.item())
            self.last_num_hyp = budget
            if self._satisfied(self.confidence, n, k0.shape[0], budget):
                break
        if n == 0:
            return self._nan()
        return R[0].double().cpu().numpy(), t[0].double().cpu().numpy().reshape(3, 1), n


class ProcrustesSolver(_SolverBase):
    """Metric relative pose from 3D-3D correspondences (pose_solver.py:238-320): RANSAC over 3-point Kabsch alignments,
    and with PROCRUSTES.REFINE the point-to-point ICP over the full depth clouds (pose_solver.py:289-315)."""
    SAMPLE_SIZE = 3

    def __init__(self, cfg):
        super().__init__(cfg)
        self.ransac_max_corr_distance = float(_cfg_get(cfg, "PROCRUSTES.MAX_CORR_DIST"))
        self.refine = bool(_cfg_get(cfg, "PROCRUSTES.REFINE", False))

    def estimate_pose(self, pts0, pts1, data):
        if len(pts0) < 3:
            return self._nan()
        k0, k1, off, K0, K1 = self._upload(pts0, pts1, data)
        d0 = torch.as_tensor(data["depth0"]).float(); d0 = d0.reshape(1, *d0.shape[-2:]).to(self.dev)
        d1 = torch.as_tensor(data["depth1"]).float(); d1 = d1.reshape(1, *d1.shape[-2:]).to(self.dev)
        R, t, n = self.backend.procrustes(k0, k1, off, K0, K1, d0, d1, self.ransac_max_corr_distance,
                                          self.num_hyp, self.seed)
        n = int(n.item())
        if n == 0:
            return self._nan()
        if self.refine:          # pose_solver.py:289-319: ICP over all valid depth pixels, starting from the RANSAC pose
            R, t, n = self.backend.icp(R, t, K0, K1, d0, d1, self.ransac_max_corr_distance)
            n = int(n.item())
        return R[0].double().cpu().numpy(), t[0].double().cpu().numpy().reshape(3, 1), n
