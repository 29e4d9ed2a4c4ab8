"""Streaming front end of the hot path: a three-stage software pipeline over batches of image pairs.

The reference processes one pair at a time (``FeatureMatchingModel.forward``, lib/models/matching/model.py:23-40:
matcher -> solver, synchronously). On the GPU the two halves have opposite characters — the matcher is
tensor-core bound and fills every SM, the RANSAC back end is a handful of latency-bound fp64 blocks — so for
a *stream* of pairs they are overlapped:

    copy stream   : host (pinned) -> device of batch i+1
    engine stream : LoFTR forward of batch i          (then a device copy of its matches into slot i % 2)
    solver stream : essential-matrix RANSAC + scale-from-depth of batch i-1 (reads slot (i-1) % 2)

``submit()`` enqueues a batch and returns the finished result of the batch submitted one call earlier
(None on the first call); ``drain()`` returns the last one.

The matcher is any pair engine: ``loftr.LoFTR``, ``spsg.SuperPointSuperGlue`` or ``sift.SIFTPairs``. The pipeline uses
their common members: ``B``, ``device``, ``stream``, ``capacity`` (match rows of a batch), ``max_pts_per_pair``,
``input_dtype`` (of the images), ``forward_async``, ``set_map``, ``forward_shared_async`` and ``pose_inputs()``. The
solver is a pose stage (``EMatMetricStage``, ``EMatStage``, ``PnPStage``, ``ProcrustesStage``); ``from_cfg`` builds
engine, back end and stage from one of the reference's method configs (config/matching/mapfree/*.yaml).

Map-free scenes match every query against one map frame. ``set_map(g0, d0, K0)`` encodes that frame once on every
engine; ``submit_host_queries`` / ``submit_device_queries`` then copy and match only the query side, with results
bit-identical to submitting the map frame with every pair. Results are ``(R [B,3,3], t [B,3], inliers [B])``
float32 / int32 tensors in pinned host memory, written by an asynchronous device->host copy that is
complete when they are handed out.
"""
import dataclasses
import os

import torch

from . import lib as _lib
from . import loftr, sift, spsg
from . import pose_solver as _ps


# ------------------------------------------------------------------------------------------------ pose stages
# Each runs on the solver stream: (be, kpts0, kpts1, offsets, K0, K1, depth0, depth1) -> R [B,3,3], t [B,3], inliers [B].
# By default a stage runs one fixed hypothesis budget per batch. With ``confidence`` (EMAT_RANSAC.CONFIDENCE /
# PNP.CONFIDENCE) and ``max_hyp`` (GPU_RANSAC.MAX_HYPOTHESES) the E-mat and PnP stages escalate each pair's budget as
# the single-pair plugins (pose_solver._SolverBase) do, x4 per round up to max_hyp, decided per pair on the device
# with no host round trip; each pair's result is then that of the fixed-budget call at the budget where it stopped.
# The E-mat stages take ``scoring`` (GPU_RANSAC.SCORING): "msac", or "magsac" for the MAGSAC++ estimator of the
# reference's USAC_MAGSAC (PoseBackend.emat), which leaves ``lo`` at its default.
class EMatMetricStage:
    """EssentialMatrixMetricSolver: E-mat RANSAC, then the metric scale from depth at its inliers."""

    def __init__(self, pix_thr, scale_thr, num_hyp=_ps.DEFAULT_NUM_HYP, seed=_ps.DEFAULT_SEED, lo=True, confidence=None,
                 max_hyp=None, scoring="msac"):
        self.pix_thr, self.scale_thr, self.num_hyp, self.seed, self.lo = float(pix_thr), float(scale_thr), int(num_hyp), seed, lo
        self.confidence, self.max_hyp, self.scoring = confidence, max_hyp, scoring

    def __call__(self, be, k0, k1, off, K0, K1, d0, d1):
        return be.emat_metric(k0, k1, off, K0, K1, d0, d1, self.pix_thr, self.scale_thr, self.num_hyp, self.seed, self.lo,
                              confidence=self.confidence, max_hyp=self.max_hyp, scoring=self.scoring)


class EMatStage:
    """EssentialMatrixSolver: the pose up to scale, t of unit norm."""

    def __init__(self, pix_thr, num_hyp=_ps.DEFAULT_NUM_HYP, seed=_ps.DEFAULT_SEED, lo=True, confidence=None, max_hyp=None,
                 scoring="msac"):
        self.pix_thr, self.num_hyp, self.seed, self.lo = float(pix_thr), int(num_hyp), seed, lo
        self.confidence, self.max_hyp, self.scoring = confidence, max_hyp, scoring

    def __call__(self, be, k0, k1, off, K0, K1, d0, d1):
        R, t, n, _ = be.emat(k0, k1, off, K0, K1, self.pix_thr, self.num_hyp, self.seed, self.lo,
                             confidence=self.confidence, max_hyp=self.max_hyp, scoring=self.scoring)
        return R, t, n


class PnPStage:
    """PnPSolver: 2D-3D RANSAC with the map frame's depth (depth1 is not read)."""

    def __init__(self, reproj_thr, num_hyp=_ps.DEFAULT_NUM_HYP, seed=_ps.DEFAULT_SEED, confidence=None, max_hyp=None):
        self.reproj_thr, self.num_hyp, self.seed = float(reproj_thr), int(num_hyp), seed
        self.confidence, self.max_hyp = confidence, max_hyp

    def __call__(self, be, k0, k1, off, K0, K1, d0, d1):
        R, t, n, _ = be.pnp(k0, k1, off, K0, K1, d0, self.reproj_thr, self.num_hyp, self.seed,
                            confidence=self.confidence, max_hyp=self.max_hyp)
        return R, t, n


class ProcrustesStage:
    """ProcrustesSolver: 3D-3D RANSAC; with ``refine`` the ICP over the full depth clouds continues from its pose."""

    def __init__(self, max_corr_dist, num_hyp=_ps.DEFAULT_NUM_HYP, seed=_ps.DEFAULT_SEED, refine=False):
        self.max_corr_dist, self.num_hyp, self.seed, self.refine = float(max_corr_dist), int(num_hyp), seed, bool(refine)

    def __call__(self, be, k0, k1, off, K0, K1, d0, d1):
        R, t, n = be.procrustes(k0, k1, off, K0, K1, d0, d1, self.max_corr_dist, self.num_hyp, self.seed)
        if self.refine:
            R, t, n = be.icp(R, t, K0, K1, d0, d1, self.max_corr_dist)
        return R, t, n


class RelocPipeline:
    def __init__(self, engine, backend, pix_thr=None, scale_thr=None, num_hyp=_ps.DEFAULT_NUM_HYP, depth_hw=None,
                 solver=None):
        # solver=None: EMatMetricStage(pix_thr, scale_thr, num_hyp), i.e. emat_metric(..., lo=True)
        # `engine` may be a list of identical engines: consecutive batches then alternate between them, each on
        # its own stream, so that the HBM-bound kernels of one batch (attention, LayerNorm, dual softmax, token
        # GEMMs) share the SMs with the tensor-core-bound convolutions of the next.
        self.engines = list(engine) if isinstance(engine, (list, tuple)) else [engine]
        engine = self.engines[0]
        self.eng, self.be = engine, backend
        self.solver = EMatMetricStage(pix_thr, scale_thr, num_hyp) if solver is None else solver
        dev = engine.device
        self.dev = dev
        self.s_copy = torch.cuda.Stream(device=dev)
        self.s_solve = torch.cuda.Stream(device=dev)
        B, cap = engine.B, engine.capacity
        self.slots = []
        for _ in range(2):
            self.slots.append({
                "k0": torch.empty(cap, 2, device=dev), "k1": torch.empty(cap, 2, device=dev),
                "off": torch.empty(B + 1, dtype=torch.int32, device=dev),
                "rec": torch.empty(B, 13, device=dev),
                "rec_host": torch.zeros(B, 13).pin_memory(),
                "ev_fwd": torch.cuda.Event(), "ev_solved": torch.cuda.Event(), "ev_in": torch.cuda.Event(),
                "inputs": None, "busy": False,
            })
        self.has_overflow = getattr(engine, "overflow", None) is not None   # SIFTPairs: per-pair capacity flags
        if self.has_overflow:
            for slot in self.slots:
                slot["ovf"] = torch.zeros(B, dtype=torch.int32, device=dev)
                slot["ovf_host"] = torch.zeros(B, dtype=torch.int32).pin_memory()
        self.stage = None
        if depth_hw is not None:                      # device staging for host inputs (two slots)
            h, w = depth_hw
            gd = engine.input_dtype
            self.stage = [{"g0": torch.empty(B, h, w, device=dev, dtype=gd), "g1": torch.empty(B, h, w, device=dev, dtype=gd),
                           "d0": torch.empty(B, h, w, device=dev), "d1": torch.empty(B, h, w, device=dev),
                           "K0": torch.empty(B, 3, 3, device=dev), "K1": torch.empty(B, 3, 3, device=dev)}
                          for _ in range(2)]
        self.i = 0
        self._outs_all = [e.pose_inputs() for e in self.engines]
        # shared map frame: its depth / intrinsics, a generation counter bumped by set_map, and per slot the [B,...]
        # copies the solver reads, refilled when the slot's generation is behind (the slot's last batch must be solved)
        self.map_gen, self.map_d0, self.map_K0 = 0, None, None
        self.ev_map = torch.cuda.Event()
        self.map_slots = [{"d0": None, "K0": None, "gen": 0} for _ in range(2)]

    # ---------------------------------------------------------------- stages
    def _enqueue(self, g0, g1, d0, d1, K0, K1):
        """g0/g1/d0/d1/K0/K1: device tensors of this batch (already ordered after whatever produced them on the
        current stream or on self.s_copy via slot['ev_in']). K0 / K1 are the intrinsics of the reference and the
        query frame: Map-free frames have per-frame intrinsics (lib/datasets/mapfree.py:39-54) and the solver
        normalises each image's points with its own K (pose_solver.py:39-43, 150-151)."""
        eng, slot = self.engines[self.i % len(self.engines)], self.slots[self.i % 2]
        outs = self._outs_all[self.i % len(self.engines)]
        if slot["busy"]:                              # the solver of batch i-2 must be done with this slot
            eng.stream.wait_event(slot["ev_solved"])
        if g0 is None:
            eng.forward_shared_async(g1)
        else:
            eng.forward_async(g0, g1)
        with torch.cuda.stream(eng.stream):
            slot["k0"].copy_(outs[0], non_blocking=True)
            slot["k1"].copy_(outs[1], non_blocking=True)
            slot["off"].copy_(outs[2], non_blocking=True)
            if self.has_overflow:
                slot["ovf"].copy_(eng.overflow, non_blocking=True)
            slot["ev_fwd"].record(eng.stream)
        with torch.cuda.stream(self.s_solve):
            self.s_solve.wait_event(slot["ev_fwd"])
            R, t, n = self.solver(self.be, slot["k0"], slot["k1"], slot["off"], K0, K1, d0, d1)
            B = eng.B
            slot["rec"][:, :9] = R.reshape(B, 9)
            slot["rec"][:, 9:12] = t.reshape(B, 3)
            slot["rec"][:, 12] = n.to(torch.float32)
            slot["rec_host"].copy_(slot["rec"], non_blocking=True)
            if self.has_overflow:
                slot["ovf_host"].copy_(slot["ovf"], non_blocking=True)
            slot["ev_solved"].record(self.s_solve)
        for x in (d0, d1, K0, K1):
            x.record_stream(self.s_solve)
        slot["inputs"] = (g0, g1, d0, d1, K0, K1)     # keep alive until the slot is reused
        slot["busy"] = True

    def _collect(self, j):
        slot = self.slots[j % 2]
        slot["ev_solved"].synchronize()
        rec = slot["rec_host"]
        B = self.eng.B
        if self.has_overflow and bool(slot["ovf_host"].any()):
            pairs = torch.nonzero(slot["ovf_host"]).flatten().tolist()
            raise _lib.MfrError(f"batch {j}: pairs {pairs} had more SIFT candidates than the engine's max_candidates; "
                                f"their matches are incomplete")
        return rec[:, :9].reshape(B, 3, 3).clone(), rec[:, 9:12].clone(), rec[:, 12].to(torch.int32)

    def _submit(self, g0, g1, d0, d1, K0, K1):
        self._enqueue(g0, g1, d0, d1, K0, K1)
        self.i += 1
        return self._collect(self.i - 2) if self.i >= 2 else None

    def _stage_copy(self, st, items):
        for k, src in items:
            if isinstance(src, (list, tuple)):    # one pinned tensor per pair
                for j, row in enumerate(src):
                    st[k][j].copy_(row, non_blocking=True)
            else:
                st[k].copy_(src, non_blocking=True)

    def _map_inputs(self, stream):
        """The map depth / intrinsics of this batch's slot as [B,h,w] / [B,3,3], refilled on `stream` when set_map ran
        since the slot was last filled. `stream` must already wait for the slot's previous solve."""
        assert self.map_d0 is not None, "call set_map before submitting queries"
        ms = self.map_slots[self.i % 2]
        if ms["gen"] != self.map_gen:
            B, (h, w) = self.eng.B, self.map_d0.shape
            if ms["d0"] is None or ms["d0"].shape[1:] != (h, w):
                ms["d0"] = torch.empty(B, h, w, device=self.dev)
                ms["K0"] = torch.empty(B, 3, 3, device=self.dev)
            with torch.cuda.stream(stream):
                stream.wait_event(self.ev_map)
                ms["d0"].copy_(self.map_d0.expand(B, h, w), non_blocking=True)
                ms["K0"].copy_(self.map_K0.expand(B, 3, 3), non_blocking=True)
            for x in (self.map_d0, self.map_K0, ms["d0"], ms["K0"]):
                x.record_stream(stream)
            ms["gen"] = self.map_gen
        return ms["d0"], ms["K0"]

    # ---------------------------------------------------------------- public
    def submit_device(self, g0, g1, d0, d1, K0, K1=None):
        """Batch already resident on the device ([B,3,3] float32 intrinsics per image; K1=None: both frames share
        K0). Returns the result of the previous batch (or None)."""
        return self._submit(g0, g1, d0, d1, K0, K0 if K1 is None else K1)

    def set_map(self, g0, d0, K0):
        """Map frame of the batches submitted from now on: gray image g0 [(1,)h,w] (of the engine's input_dtype), depth
        d0 [(1,)h,w] and intrinsics K0 [(1,)3,3] float32, on the host or the device. g0 is encoded once on every engine;
        batches already submitted keep the map they were submitted with."""
        cur = torch.cuda.current_stream(self.dev)
        h, w = g0.shape[-2:]
        g0 = g0.reshape(h, w).to(self.dev, self.eng.input_dtype)
        self.map_d0 = torch.empty(d0.shape[-2:], device=self.dev)
        self.map_d0.copy_(d0.reshape(self.map_d0.shape))
        self.map_K0 = torch.empty(3, 3, device=self.dev)
        self.map_K0.copy_(K0.reshape(3, 3))
        for e in self.engines:
            e.set_map(g0)
        self.ev_map.record(cur)
        self.map_gen += 1

    def submit_device_queries(self, g1, d1, K1):
        """Query side of a batch already resident on the device (g1, d1 [B,h,w], K1 [B,3,3]), matched against the map
        of the last set_map. Returns the result of the previous batch (or None)."""
        slot = self.slots[self.i % 2]
        cur = torch.cuda.current_stream(self.dev)
        if slot["busy"]:                              # the slot's map copies are read by the solver of batch i-2
            cur.wait_event(slot["ev_solved"])
        d0, K0 = self._map_inputs(cur)
        return self._submit(None, g1, d0, d1, K0, K1)

    def submit_host_queries(self, g1, d1, K1):
        """Query side of a batch in pinned host memory (as in submit_host), matched against the map of the last
        set_map: only the queries are copied to the device."""
        assert self.stage is not None, "construct the pipeline with depth_hw=(h, w) to feed host batches"
        st, slot = self.stage[self.i % 2], self.slots[self.i % 2]
        with torch.cuda.stream(self.s_copy):
            if slot["busy"]:                          # staging tensors of batch i-2 are read by its solver
                self.s_copy.wait_event(slot["ev_solved"])
            self._stage_copy(st, (("g1", g1), ("d1", d1), ("K1", K1)))
            d0, K0 = self._map_inputs(self.s_copy)
            slot["ev_in"].record(self.s_copy)
        self.engines[self.i % len(self.engines)].stream.wait_event(slot["ev_in"])
        self.s_solve.wait_event(slot["ev_in"])
        return self._submit(None, st["g1"], d0, st["d1"], K0, st["K1"])

    def submit_host(self, g0, g1, d0, d1, K0, K1=None):
        """Batch in pinned host memory ([B,h,w] images of the engine's input_dtype, float32 depths, [B,3,3] intrinsics of
        each frame; K1=None: both frames share K0): the copy to the device runs on its own stream, overlapping the forward
        of the previous batch."""
        assert self.stage is not None, "construct the pipeline with depth_hw=(h, w) to feed host batches"
        st, slot = self.stage[self.i % 2], self.slots[self.i % 2]
        with torch.cuda.stream(self.s_copy):
            if slot["busy"]:                          # staging tensors of batch i-2 are read by its solver
                self.s_copy.wait_event(slot["ev_solved"])
            self._stage_copy(st, (("g0", g0), ("g1", g1), ("d0", d0), ("d1", d1), ("K0", K0),
                                  ("K1", K0 if K1 is None else K1)))
            slot["ev_in"].record(self.s_copy)
        self.engines[self.i % len(self.engines)].stream.wait_event(slot["ev_in"])
        self.s_solve.wait_event(slot["ev_in"])
        return self.submit_device(st["g0"], st["g1"], st["d0"], st["d1"], st["K0"], st["K1"])

    def drain(self):
        """Result of the last submitted batch (blocks until it is done)."""
        return self._collect(self.i - 1) if self.i >= 1 else None

    def reset(self):
        """Waits for everything in flight and forgets it: the next submit starts a new stream (returns None)."""
        for e in self.engines:
            e.stream.synchronize()
        self.s_copy.synchronize(); self.s_solve.synchronize()
        for slot in self.slots:
            slot["busy"] = False
            slot["inputs"] = None
        self.i = 0


# ------------------------------------------------------------------------------------------------ method configs
MATCHERS = ("LoFTR", "SG", "SIFT")      # etc/feature_matching_baselines/compute.py:10, the correspondences_<key>.npz names
SOLVERS = ("EssentialMatrix", "EssentialMatrixMetric", "PNP", "Procrustes")   # lib/models/matching/model.py:18-27
SIFT_NUM_FEATURES, SIFT_RATIO = 2048, 0.8                                     # matchers.py:145-146


@dataclasses.dataclass(frozen=True)
class MethodSpec:
    """What one Map-free method config asks of the stream: the matcher, the solver with its thresholds, the RANSAC
    settings and the engine frame."""
    matcher: str                    # "LoFTR" | "SG" | "SIFT"
    solver: str                     # "EssentialMatrix" | "EssentialMatrixMetric" | "PNP" | "Procrustes"
    height: int                     # engine frame: DATASET.HEIGHT / WIDTH, for LoFTR padded by loftr.engine_frame
    width: int
    num_hyp: int
    seed: int
    lo: int                         # mfr_emat_ransac lo flags (E-mat solvers with MSAC scoring)
    pix_thr: float = None           # EMAT_RANSAC.PIX_THRESHOLD
    scale_thr: float = None         # EMAT_RANSAC.SCALE_THRESHOLD (metric solver)
    reproj_thr: float = None        # PNP.REPROJECTION_INLIER_THRESHOLD
    max_corr_dist: float = None     # PROCRUSTES.MAX_CORR_DIST [m]
    refine: bool = False            # PROCRUSTES.REFINE
    sift_features: int = None       # SIFT.NUM_FEATURES
    sift_ratio: float = None        # SIFT.RATIO_THRESHOLD
    confidence: float = None        # EMAT_RANSAC.CONFIDENCE / PNP.CONFIDENCE (None: Procrustes, or the key unset)
    max_hyp: int = None             # GPU_RANSAC.MAX_HYPOTHESES, at least num_hyp: the escalation's cap
    scoring: str = "msac"           # GPU_RANSAC.SCORING: E-mat objective, "msac" or "magsac" (MAGSAC++)

    def stage(self, escalate=False):
        """The pose stage of this method: the first hypothesis budget only, or with ``escalate`` the CONFIDENCE
        escalation up to max_hyp (E-mat and PnP; the Procrustes plugin does not escalate). The E-mat stages score with
        ``scoring``; MAGSAC++ brings its own LO, so ``lo`` is not passed to it."""
        esc = {"confidence": self.confidence, "max_hyp": self.max_hyp} if escalate else {}
        if self.solver.startswith("EssentialMatrix"):
            esc["scoring"] = self.scoring
            lo = True if self.scoring == "magsac" else self.lo
        if self.solver == "EssentialMatrixMetric":
            return EMatMetricStage(self.pix_thr, self.scale_thr, self.num_hyp, self.seed, lo, **esc)
        if self.solver == "EssentialMatrix":
            return EMatStage(self.pix_thr, self.num_hyp, self.seed, lo, **esc)
        if self.solver == "PNP":
            return PnPStage(self.reproj_thr, self.num_hyp, self.seed, **esc)
        return ProcrustesStage(self.max_corr_dist, self.num_hyp, self.seed, self.refine)


def _matcher_name(cfg):
    path = _ps._cfg_get(cfg, "MATCHES_FILE_PATH")
    fm = _ps._cfg_get(cfg, "FEATURE_MATCHING")
    if fm == "Precomputed" or (fm is None and path):
        base = os.path.basename(str(path or ""))
        for m in MATCHERS:
            if base == f"correspondences_{m}.npz":
                return m
        raise NotImplementedError(f"Invalid feature matching: no streaming matcher for MATCHES_FILE_PATH {path!r}")
    if fm in ("LoFTR", "SIFT"):
        return fm
    raise NotImplementedError(f"Invalid feature matching {fm!r}")


def resolve_method(cfg):
    """Reference method config (a config.CfgNode or nested dict, e.g. config/mapfree.yaml + a
    config/matching/mapfree/*.yaml) -> MethodSpec. Unknown matchers or solvers raise NotImplementedError as the
    reference's FeatureMatchingModel does. Budget, escalation cap, confidence, seed, LO flags and the E-mat scoring
    follow the single-pair plugins (pose_solver); the stage escalates on the confidence only when asked to
    (``MethodSpec.stage``)."""
    g = lambda k, d=None: _ps._cfg_get(cfg, k, d)
    matcher = _matcher_name(cfg)
    solver = g("POSE_SOLVER")
    if solver not in SOLVERS:
        raise NotImplementedError(f"Invalid pose solver {solver!r}")
    num_hyp, max_hyp, seed, lo = _ps.ransac_settings(cfg, _ps.pnp_default_hyp(cfg) if solver == "PNP" else _ps.DEFAULT_NUM_HYP)
    h, w = int(g("DATASET.HEIGHT", 720)), int(g("DATASET.WIDTH", 540))   # Map-free's frame (config/mapfree.yaml)
    if matcher == "LoFTR":
        h, w = loftr.engine_frame(h, w)
    f = lambda k: None if g(k) is None else float(g(k))
    kw = {}
    if solver.startswith("EssentialMatrix"):
        kw["scoring"] = _ps.ransac_scoring(cfg)
        kw["pix_thr"] = f("EMAT_RANSAC.PIX_THRESHOLD")
        kw["confidence"] = f("EMAT_RANSAC.CONFIDENCE")
        if solver == "EssentialMatrixMetric":
            kw["scale_thr"] = f("EMAT_RANSAC.SCALE_THRESHOLD")
    elif solver == "PNP":
        kw["reproj_thr"] = f("PNP.REPROJECTION_INLIER_THRESHOLD")
        kw["confidence"] = f("PNP.CONFIDENCE")
    else:
        kw["max_corr_dist"] = f("PROCRUSTES.MAX_CORR_DIST")
        kw["refine"] = bool(g("PROCRUSTES.REFINE", False))
    if matcher == "SIFT":
        kw["sift_features"] = int(g("SIFT.NUM_FEATURES", SIFT_NUM_FEATURES))
        kw["sift_ratio"] = float(g("SIFT.RATIO_THRESHOLD", SIFT_RATIO))
    return MethodSpec(matcher=matcher, solver=solver, height=h, width=w, num_hyp=num_hyp, seed=seed, lo=lo,
                      max_hyp=max_hyp, **kw)


def from_cfg(cfg, batch, weights=None, precision="tf32", depth_hw=None, outdoor=False, device=0, graph=True,
             escalate=False):
    """Engine + PoseBackend + RelocPipeline for the method of ``cfg`` (see resolve_method), ``batch`` pairs per engine
    call. ``weights``: LoFTR, what loftr.load_weights takes (a state dict, a {'state_dict': ...} checkpoint or a path to
    either); SG, what spsg.load_weights takes (a (superpoint, superglue) pair of state dicts or the directory holding
    superpoint_v1.pth and superglue_{indoor,outdoor}.pth, indoor unless ``outdoor``); SIFT, none.
    ``precision`` applies to LoFTR and SG. ``escalate``: the E-mat / PnP stage escalates on the config's CONFIDENCE up
    to GPU_RANSAC.MAX_HYPOTHESES, as the single-pair plugins do (default: the first budget only). The method is at
    ``pipeline.method``."""
    spec = resolve_method(cfg)
    if spec.matcher == "LoFTR":
        if weights is None:
            raise ValueError("LoFTR needs a state dict")
        eng = loftr.LoFTR(loftr.load_weights(weights), batch=batch, height=spec.height, width=spec.width,
                          cfg=loftr.engine_cfg(cfg), device=device, graph=graph, precision=precision)
    elif spec.matcher == "SG":
        if weights is None:
            raise ValueError("SuperPoint + SuperGlue needs state dicts or their directory")
        sp, sg = spsg.load_weights(weights, outdoor)
        eng = spsg.SuperPointSuperGlue(sp, sg, batch=batch, height=spec.height, width=spec.width, device=device,
                                       graph=graph, precision=precision)
    else:
        eng = sift.SIFTPairs(batch, spec.height, spec.width, nfeatures=spec.sift_features, ratio=spec.sift_ratio,
                             root_sift=True, device=device, graph=graph)
    be = _ps.PoseBackend(max_pairs=batch, max_pts=max(8, min(eng.max_pts_per_pair, _ps.MAX_PTS_LIMIT)),
                         max_hyp=max(spec.max_hyp if escalate else spec.num_hyp, 128), device=device)
    pipe = RelocPipeline(eng, be, depth_hw=depth_hw, solver=spec.stage(escalate))
    pipe.method = spec
    return pipe
