"""ctypes binding of libmfr_b200.so, and ``Engine``, the host side that every engine class shares. There is NO CPU
fallback: if the library is missing or a CUDA device is absent, compute entry points raise."""
import ctypes
import math
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmfr_b200.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "mfr_b200.h")

_lib = None

c_f32p = ctypes.c_void_p
c_ll = ctypes.c_longlong
c_int = ctypes.c_int
c_float = ctypes.c_float
c_vp = ctypes.c_void_p

class LoftrOutputs(ctypes.Structure):
    """mfr_loftr_outputs of include/mfr_b200.h."""
    _fields_ = [("m_total", c_vp), ("m_offsets", c_vp), ("b_ids", c_vp), ("i_ids", c_vp),
                ("j_ids", c_vp), ("mconf", c_vp), ("mkpts0_f", c_vp), ("mkpts1_f", c_vp),
                ("mkpts1_c", c_vp), ("expec_f", c_vp), ("capacity", c_int)]


class SpsgOutputs(ctypes.Structure):
    """mfr_spsg_outputs of include/mfr_b200.h."""
    _fields_ = [("counts", c_vp), ("keypoints", c_vp), ("scores", c_vp), ("descriptors", c_vp),
                ("desc_ld", c_int), ("matches0", c_vp), ("matching_scores0", c_vp), ("m_offsets", c_vp),
                ("mkpts0", c_vp), ("mkpts1", c_vp), ("max_keypoints", c_int)]


class SiftOutputs(ctypes.Structure):
    """mfr_sift_outputs of include/mfr_b200.h."""
    _fields_ = [("counts", c_vp), ("raw_counts", c_vp), ("extrema_counts", c_vp), ("keypoints", c_vp),
                ("octaves", c_vp), ("descriptors", c_vp), ("capacity", c_int)]


class SiftPairOutputs(ctypes.Structure):
    """mfr_sift_pair_outputs of include/mfr_b200.h."""
    _fields_ = [("kpts0", c_vp), ("kpts1", c_vp), ("offsets", c_vp), ("overflow", c_vp), ("capacity", c_int),
                ("max_pts_per_pair", c_int)]


c_pp = ctypes.POINTER(ctypes.c_void_p)

# name -> (restype, argtypes); mirrors include/mfr_b200.h one to one
SIGNATURES = {
    "mfr_version": (c_int, []),
    "mfr_device_sm_count": (c_int, []),
    "mfr_conv2d_nhwc_tf32": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_ll, c_vp, c_int, c_int,
                                     c_int, c_int, c_int, c_int, c_vp, c_vp, c_ll, c_int, c_float,
                                     c_vp, c_ll, c_vp]),
    "mfr_conv2d_nhwc_bf16": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_ll, c_vp, c_ll, c_int, c_int, c_int,
                                     c_int, c_int, c_vp, c_vp, c_ll, c_int, c_float, c_vp, c_ll, c_int, c_vp]),
    "mfr_token_gemm_dyn_rows": (c_int, [c_vp, c_int, c_int, c_int, c_ll, c_vp, c_ll, c_int, c_int, c_vp, c_int, c_vp,
                                        c_ll, c_int, c_vp, c_vp]),
    "mfr_loftr_create": (c_int, [c_int, c_int, c_int, c_float, c_int, c_float, c_int, c_int, c_pp]),
    "mfr_loftr_destroy": (None, [c_vp]),
    "mfr_loftr_num_weights": (c_int, [c_vp]),
    "mfr_loftr_weight_name": (ctypes.c_char_p, [c_vp, c_int]),
    "mfr_loftr_weight_numel": (c_ll, [c_vp, c_int]),
    "mfr_loftr_set_weight": (c_int, [c_vp, c_int, c_vp, c_ll, c_vp]),
    "mfr_loftr_forward": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "mfr_loftr_set_map": (c_int, [c_vp, c_vp, c_int, c_int, c_vp]),
    "mfr_loftr_forward_shared": (c_int, [c_vp, c_vp, c_int, c_int, c_vp]),
    "mfr_loftr_set_graph": (None, [c_vp, c_int]),
    "mfr_loftr_get_outputs": (c_int, [c_vp, ctypes.POINTER(LoftrOutputs)]),
    "mfr_loftr_debug_tensor": (c_int, [c_vp, ctypes.c_char_p, c_pp, ctypes.POINTER(c_ll)]),
    "mfr_loftr_num_kernels": (c_int, [c_vp]),
    "mfr_loftr_num_launches": (c_int, [c_vp]),
    "mfr_loftr_profile": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_int, c_vp, c_vp, c_vp, c_vp]),
    "mfr_loftr_step_name": (ctypes.c_char_p, [c_vp, c_int]),
    "mfr_loftr_run_steps": (c_int, [c_vp, c_int, c_int, c_vp]),
    "mfr_spsg_create": (c_int, [c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_int, c_float, c_pp]),
    "mfr_spsg_create_ex": (c_int, [c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_int, c_float, c_int, c_pp]),
    "mfr_spsg_destroy": (None, [c_vp]),
    "mfr_spsg_num_weights": (c_int, [c_vp]),
    "mfr_spsg_weight_name": (ctypes.c_char_p, [c_vp, c_int]),
    "mfr_spsg_weight_numel": (c_ll, [c_vp, c_int]),
    "mfr_spsg_set_weight": (c_int, [c_vp, c_int, c_vp, c_ll, c_vp]),
    "mfr_spsg_forward": (c_int, [c_vp, c_vp, c_vp, c_vp]),
    "mfr_spsg_set_map": (c_int, [c_vp, c_vp, c_vp]),
    "mfr_spsg_forward_shared": (c_int, [c_vp, c_vp, c_vp]),
    "mfr_spsg_set_graph": (None, [c_vp, c_int]),
    "mfr_spsg_get_outputs": (c_int, [c_vp, ctypes.POINTER(SpsgOutputs)]),
    "mfr_spsg_debug_tensor": (c_int, [c_vp, ctypes.c_char_p, c_pp, ctypes.POINTER(c_ll)]),
    "mfr_spsg_num_launches": (c_int, [c_vp]),
    "mfr_spsg_forward_superglue": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mfr_coarse_match": (c_int, [c_vp, c_int, c_int, c_int, c_float, c_int, c_float, c_int, c_vp, c_vp,
                                 c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mfr_knn2_l2": (c_int, [c_vp, c_int, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mfr_sift_create": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_pp]),
    "mfr_sift_destroy": (None, [c_vp]),
    "mfr_sift_detect": (c_int, [c_vp, c_vp, c_vp]),
    "mfr_sift_set_graph": (None, [c_vp, c_int]),
    "mfr_sift_get_outputs": (c_int, [c_vp, ctypes.POINTER(SiftOutputs)]),
    "mfr_sift_match_pairs": (c_int, [c_vp, c_float, c_vp, c_vp, c_vp, c_vp]),
    "mfr_sift_debug_tensor": (c_int, [c_vp, ctypes.c_char_p, c_pp, ctypes.POINTER(c_ll)]),
    "mfr_sift_profile": (c_int, [c_vp, c_vp, c_vp, c_vp]),
    "mfr_sift_pairs_create": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_pp]),
    "mfr_sift_pairs_destroy": (None, [c_vp]),
    "mfr_sift_pairs_set_graph": (None, [c_vp, c_int]),
    "mfr_sift_forward_pairs": (c_int, [c_vp, c_vp, c_vp, c_vp]),
    "mfr_sift_set_map": (c_int, [c_vp, c_vp, c_vp]),
    "mfr_sift_forward_shared": (c_int, [c_vp, c_vp, c_vp]),
    "mfr_sift_get_pair_outputs": (c_int, [c_vp, ctypes.POINTER(SiftPairOutputs)]),
    "mfr_pose_solver_create": (c_int, [c_int, c_int, c_int, c_pp]),
    "mfr_pose_solver_destroy": (None, [c_vp]),
    "mfr_pose_solver_debug_tensor": (c_int, [c_vp, ctypes.c_char_p, c_pp, ctypes.POINTER(c_ll)]),
    "mfr_emat_ransac": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_float, c_int,
                                ctypes.c_ulonglong, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mfr_scale_from_depth": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp,
                                     c_vp, c_vp, c_int, c_int, c_float, c_vp, c_vp, c_vp, c_vp]),
    "mfr_pnp_ransac": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int,
                               c_float, ctypes.c_ulonglong, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mfr_emat_ransac_escalate": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_float, c_int, ctypes.c_ulonglong,
                                         c_int, c_vp, c_vp, c_vp, c_vp, ctypes.c_double, c_int, c_vp, c_vp]),
    "mfr_emat_magsac": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_float, c_int, ctypes.c_ulonglong, c_vp, c_vp,
                                c_vp, c_vp, ctypes.c_double, c_int, c_vp, c_vp]),
    "mfr_pnp_ransac_escalate": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_float,
                                        ctypes.c_ulonglong, c_vp, c_vp, c_vp, c_vp, ctypes.c_double, c_int, c_vp, c_vp]),
    "mfr_linear_attention": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "mfr_superglue_attention": (c_int, [c_vp, c_ll, c_vp, c_int, c_int, c_int, c_vp, c_ll, c_vp]),
    "mfr_stem_conv7x7": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "mfr_icp_refine": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_float, c_int, c_float, c_float,
                               c_vp, c_vp, c_vp, c_vp]),
    "mfr_jpeg_info": (c_int, [c_vp, c_ll, c_vp, c_vp, c_vp]),
    "mfr_jpeg_decode": (c_int, [c_vp, c_ll, c_int, c_vp, c_int, c_int, c_vp]),
    "mfr_jpeg_decoder_create": (c_int, [c_int, c_ll, c_ll, c_pp]),
    "mfr_jpeg_decoder_destroy": (None, [c_vp]),
    "mfr_jpeg_batch_info": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp]),
    "mfr_jpeg_decode_batch": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp]),
    "mfr_png_info": (c_int, [c_vp, c_ll, c_vp, c_vp, c_vp]),
    "mfr_png_decoder_create": (c_int, [c_int, c_ll, c_ll, c_pp]),
    "mfr_png_decoder_destroy": (None, [c_vp]),
    "mfr_png_batch_info": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp]),
    "mfr_debug_png_kernel_ms": (c_int, [c_vp, c_vp]),
    "mfr_png_decode_batch": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp]),
    "mfr_resize_linear": (c_int, [c_vp, c_int, c_int, c_int, c_ll, c_int, c_vp, c_int, c_int, c_int, c_float, c_int, c_vp]),
    "mfr_pose_metrics": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp]),
    "mfr_encoder_tail": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_ll, c_vp, c_int, c_vp]),
    "mfr_debug_time_conv": (c_float, [c_vp, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_vp, c_int, c_int, c_vp]),
    "mfr_procrustes_ransac": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int,
                                      c_float, ctypes.c_ulonglong, c_vp, c_vp, c_vp, c_vp]),
    "mfr_host_five_point": (c_int, [c_vp, c_vp, c_vp]),
    "mfr_host_p3p": (c_int, [c_vp, c_vp, c_vp, c_vp]),
    "mfr_host_kabsch": (c_int, [ctypes.c_double, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mfr_host_poly_real_roots": (c_int, [c_vp, c_int, c_vp]),
    "mfr_host_decompose_essential": (c_int, [c_vp, c_vp, c_vp, c_vp]),
    "mfr_host_ransac_satisfied": (c_int, [ctypes.c_double, c_int, c_int, c_int, c_int, c_int]),
    "mfr_host_magsac_loss": (c_int, [ctypes.c_double, ctypes.c_double, c_vp, c_vp]),
    "mfr_host_jpeg_decode": (c_int, [c_vp, c_ll, c_int, c_vp, c_int, c_int]),
    "mfr_host_png_decode": (c_int, [c_vp, c_ll, c_int, c_vp, c_int, c_int]),
}


class MfrError(RuntimeError):
    pass


def load():
    """Loads the shared library (building is done by ``build.py`` / ``__graft_entry__.build``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MfrError(
            f"{LIB_PATH} not found: run `python map-free-reloc_b200/build.py` "
            "(there is no CPU fallback for the CUDA path)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        raise MfrError(f"libmfr_b200 call failed rc={rc} {what}")


def ptr(t):
    """Device (or host) pointer of a torch tensor / None."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def cur_stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class Engine:
    """Host side of one engine handle of the library (its ``mfr_<name>_*`` functions): the handle, the device and, for
    the pair engines, the stream the engine runs on. ``close`` (also run by ``__del__``) waits for the engine's work and
    destroys the handle."""

    def __init__(self, name, create, args, device=None, stream=True):
        """Creates the handle with ``create(*args, &handle)`` (the name of an mfr_* function) on cuda:``device`` (None:
        the current device). ``stream``: whether the engine runs on a stream of its own (``_call``) rather than on the
        caller's current stream."""
        if not torch.cuda.is_available():
            raise MfrError(f"{type(self).__name__} needs a CUDA device (there is no CPU fallback)")
        self._l, self._name = load(), name
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        torch.cuda.set_device(self.device)
        self.stream = torch.cuda.Stream(device=self.device) if stream else None
        h = ctypes.c_void_p()
        check(getattr(self._l, create)(*args, ctypes.byref(h)), create)
        self._h = h

    def _get_outputs(self, fn, struct):
        """The engine's table of output buffers: ``fn`` is its mfr_*_get_outputs function, ``struct`` the table's type."""
        o = struct()
        check(fn(self._h, ctypes.byref(o)), fn.__name__)
        return o

    def _upload_weights(self, weights):
        """Uploads ``weights`` ({name: float32 ndarray}) on the engine stream in the engine's order; a tensor the engine
        expects that is missing or of another size raises MfrError naming it."""
        l, h, stream = self._l, self._h, ctypes.c_void_p(self.stream.cuda_stream)
        for i in range(getattr(l, f"mfr_{self._name}_num_weights")(h)):
            name = getattr(l, f"mfr_{self._name}_weight_name")(h, i).decode()
            numel = getattr(l, f"mfr_{self._name}_weight_numel")(h, i)
            if name not in weights:
                raise MfrError(f"missing weight tensor {name}")
            a = weights[name].reshape(-1)
            if a.size != numel:
                raise MfrError(f"weight {name}: {a.size} elements, engine expects {numel}")
            check(getattr(l, f"mfr_{self._name}_set_weight")(h, i, a.ctypes.data_as(ctypes.c_void_p), numel, stream),
                  f"set_weight {name}")

    def _images(self, imgs, *shape):
        """``imgs`` as a contiguous tensor of ``shape``; ValueError unless it is a CUDA tensor of the engine's
        ``input_dtype``."""
        if not imgs.is_cuda or imgs.dtype != self.input_dtype:
            raise ValueError(f"expected {self.input_dtype} CUDA images of shape {list(shape)}")
        return imgs.reshape(shape).contiguous()

    def _call(self, fn, *args):
        """Runs ``fn(handle, *args, engine stream)`` on the engine stream, after the work queued so far on the caller's
        current stream. Tensor arguments are passed as pointers and kept alive until the engine stream is done with
        them."""
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            check(fn(self._h, *[ptr(a) if isinstance(a, torch.Tensor) else a for a in args],
                     ctypes.c_void_p(self.stream.cuda_stream)), fn.__name__)
        for a in args:
            if isinstance(a, torch.Tensor):
                a.record_stream(self.stream)

    def view(self, addr, shape, dtype):
        """Zero-copy torch view (float32, float64, int32 or bfloat16) of an engine-owned device buffer, valid while the
        engine lives."""
        class _A:   # __cuda_array_interface__ carrier
            pass
        a = _A()
        typestr = {torch.float32: "<f4", torch.float64: "<f8", torch.int32: "<i4", torch.bfloat16: "<i2"}[dtype]
        a.__cuda_array_interface__ = {"shape": (int(math.prod(shape)),), "typestr": typestr, "data": (int(addr), False),
                                      "version": 2}
        t = torch.as_tensor(a, device=self.device)
        return (t.view(torch.bfloat16) if dtype == torch.bfloat16 else t).view(*shape)

    def debug_tensor(self, name, shape, dtype=torch.float32):
        """View of the engine's named intermediate buffer (listed at mfr_<name>_debug_tensor in include/mfr_b200.h, which
        reports its size in 4-byte words); ``shape`` must fit in it. It shows what the last call that wrote the buffer
        left there."""
        p, n = ctypes.c_void_p(), ctypes.c_longlong()
        fn = getattr(self._l, f"mfr_{self._name}_debug_tensor")
        check(fn(self._h, name.encode(), ctypes.byref(p), ctypes.byref(n)), f"debug tensor {name}")
        assert math.prod(shape) * torch.empty((), dtype=dtype).element_size() <= 4 * n.value, (name, shape, n.value)
        return self.view(p.value, shape, dtype)

    def close(self):
        """Waits for the engine's work (its stream's, or the device's for an engine without one), then destroys the
        handle. Later calls do nothing."""
        if getattr(self, "_h", None):
            if self.stream is None:
                torch.cuda.synchronize(self.device)
            else:
                self.stream.synchronize()
            getattr(self._l, f"mfr_{self._name}_destroy")(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
