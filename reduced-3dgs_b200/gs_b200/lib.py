"""ctypes binding of libgs_b200.so (C ABI: include/gs_b200.h).

This is the only bridge between the Python host side and the CUDA library.  There is NO fallback: if the
library is missing or no CUDA device is present, calls raise.  PyTorch is used for device memory and streams only.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import threading
from typing import Optional

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "libgs_b200.so")

ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)


class GsbQuant(C.Structure):
    _fields_ = [("ids_dc", C.c_void_p), ("ids_rest", C.c_void_p), ("ids_opacity", C.c_void_p),
                ("ids_scaling", C.c_void_p), ("ids_rot", C.c_void_p), ("centers", C.c_void_p)]


class GsbScene(C.Structure):
    _fields_ = [("P", C.c_int32), ("M", C.c_int32), ("means3D", C.c_void_p), ("opacities", C.c_void_p),
                ("scales", C.c_void_p), ("rotations", C.c_void_p), ("cov3D_precomp", C.c_void_p), ("shs", C.c_void_p),
                ("colors_precomp", C.c_void_p), ("degrees", C.c_void_p), ("scale_modifier", C.c_float),
                ("sh_packed", C.c_int32), ("band_count", C.c_int32 * 4), ("prune_mask", C.c_void_p),
                ("filter_3D", C.c_void_p), ("quant", C.POINTER(GsbQuant))]


class GsbCamera(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("tan_fovx", C.c_float), ("tan_fovy", C.c_float),
                ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p),
                ("background", C.c_void_p), ("prefiltered", C.c_int32)]


class GsbDebug(C.Structure):
    _fields_ = [("depths", C.c_void_p), ("means2D", C.c_void_p), ("cov3D", C.c_void_p), ("conic_opacity", C.c_void_p),
                ("rgb", C.c_void_p), ("tiles_touched", C.c_void_p), ("clamped", C.c_void_p)]


class GsbGrads(C.Structure):
    _fields_ = [("dL_dmeans2D", C.c_void_p), ("dL_dcolors", C.c_void_p), ("dL_dopacity", C.c_void_p),
                ("dL_dmeans3D", C.c_void_p), ("dL_dcov3D", C.c_void_p), ("dL_dsh", C.c_void_p),
                ("dL_dscales", C.c_void_p), ("dL_drotations", C.c_void_p), ("dL_dconic", C.c_void_p),
                ("accumulate", C.c_int32), ("dL_dmeans2D_view", C.c_void_p)]


class GsbRawParams(C.Structure):
    _fields_ = [("features_dc", C.c_void_p), ("features_rest", C.c_void_p), ("C", C.c_int32), ("scaling", C.c_void_p),
                ("rotation", C.c_void_p)]


class GsbRawGrads(C.Structure):
    _fields_ = [("dL_dfeatures_dc", C.c_void_p), ("dL_dfeatures_rest", C.c_void_p), ("dL_dscaling", C.c_void_p),
                ("dL_drotation", C.c_void_p)]


class GsbFeatures(C.Structure):
    _fields_ = [("F", C.c_int32), ("features", C.c_void_p), ("out", C.c_void_p), ("dL_dout", C.c_void_p), ("dL_dfeatures", C.c_void_p)]


FEATURES_MAX = 256             # GSB_FEATURES_MAX


class GsbForwardRequest(C.Structure):
    _fields_ = [("scene", C.POINTER(GsbScene)), ("cam", C.POINTER(GsbCamera)), ("geom_alloc", ALLOC_FN), ("geom_user", C.c_void_p),
                ("binning_alloc", ALLOC_FN), ("binning_user", C.c_void_p), ("image_alloc", ALLOC_FN), ("image_user", C.c_void_p),
                ("out_color", C.c_void_p), ("radii", C.c_void_p), ("num_rendered", C.POINTER(C.c_int64)),
                ("debug", C.POINTER(GsbDebug)), ("out_invdepth", C.c_void_p), ("out_alpha", C.c_void_p), ("antialiasing", C.c_int32),
                ("raw", C.POINTER(GsbRawParams)), ("touched_pixels", C.c_void_p), ("transmittance_sum", C.c_void_p),
                ("deterministic", C.c_int32), ("workspace", C.c_void_p), ("features", C.POINTER(GsbFeatures)), ("stream", C.c_void_p)]


class GsbBackwardRequest(C.Structure):
    _fields_ = [("scene", C.POINTER(GsbScene)), ("cam", C.POINTER(GsbCamera)), ("num_rendered", C.c_int64), ("radii", C.c_void_p),
                ("geom_blob", C.c_void_p), ("binning_blob", C.c_void_p), ("image_blob", C.c_void_p), ("dL_dout_color", C.c_void_p),
                ("grads", C.POINTER(GsbGrads)), ("dL_dinvdepth", C.c_void_p), ("dL_dalpha", C.c_void_p),
                ("lambda_sh_sparsity", C.c_float), ("dL_dviewmatrix", C.c_void_p), ("dL_dprojmatrix", C.c_void_p),
                ("dL_dcampos", C.c_void_p), ("camera_workspace", C.c_void_p), ("antialiasing", C.c_int32),
                ("raw", C.POINTER(GsbRawParams)), ("raw_grads", C.POINTER(GsbRawGrads)), ("deterministic", C.c_int32),
                ("det_workspace", C.c_void_p), ("features", C.POINTER(GsbFeatures)), ("dL_dmeans2D_abs", C.c_void_p),
                ("stream", C.c_void_p)]


class GsbAdamTensor(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("numel", C.c_int64), ("row_width", C.c_int32), ("sh_offset", C.c_int32), ("one_minus_beta1", C.c_float),
                ("beta2", C.c_float), ("one_minus_beta2", C.c_float), ("eps", C.c_float), ("bc2_sqrt", C.c_float),
                ("step_size", C.c_float)]


ADAM_MAX_TENSORS = 16          # GSB_ADAM_MAX_TENSORS


class GsbDensifyTensor(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("exp_avg_src", C.c_void_p), ("exp_avg_dst", C.c_void_p),
                ("exp_avg_sq_src", C.c_void_p), ("exp_avg_sq_dst", C.c_void_p), ("grad_src", C.c_void_p), ("grad_dst", C.c_void_p),
                ("row_width", C.c_int32), ("kind", C.c_int32)]


DENSIFY_MAX_TENSORS = 16       # GSB_DENSIFY_MAX_TENSORS
DENSIFY_COUNTS = 8             # GSB_DENSIFY_COUNTS
DENSIFY_CLONE_SPLIT, DENSIFY_PRUNE, DENSIFY_PRUNE_MASK = 0, 1, 2
DENSIFY_COPY, DENSIFY_XYZ, DENSIFY_SCALING = 0, 1, 2
MCMC_RELOCATE, MCMC_ADD, MCMC_COUNTS = 0, 1, 4
MCMC_OPACITY, MCMC_FRESH = 3, 4
MERCY_REDUNDANCY_OPACITY, MERCY_REDUNDANCY_RANDOM, MERCY_OPACITY, MERCY_REDUNDANCY_OPACITY_OPACITY, MERCY_REDUNDANCY = 0, 1, 2, 3, 4


# Every exported function: name -> (restype, argtypes), in the order of include/gs_b200.h.  lib() applies the table, so a symbol
# cannot be declared without its signature.
_V, _I32, _I64, _F, _SZ = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_size_t
SIGNATURES = {
    "gsb_geom_bytes": (_SZ, [_I32]),
    "gsb_image_bytes": (_SZ, [_I32, _I32]),
    "gsb_image_bytes_for": (_SZ, [_I32, _I32, _I32, _I32]),
    "gsb_binning_bytes": (_SZ, [_I64]),
    "gsb_forward": (C.c_int, [C.POINTER(GsbForwardRequest)]),
    "gsb_statistics_workspace_bytes": (_SZ, [_I32]),
    "gsb_backward": (C.c_int, [C.POINTER(GsbBackwardRequest)]),
    "gsb_camera_grad_workspace_bytes": (_SZ, [_I32]),
    "gsb_deterministic_workspace_bytes": (_SZ, [_I32, _I64, _I32]),
    "gsb_mark_visible": (C.c_int, [_I32, _V, _V, _V, _V, _V]),
    "gsb_export_binning": (C.c_int, [_V, _I32, _V, _I64, _V, _I32, _I32, _V, _V, _V]),
    "gsb_export_image": (C.c_int, [_V, _I32, _I32, _V, _V, _V, _V]),
    "gsb_contributions_workspace_bytes": (_SZ, [_I32]),
    "gsb_contributions": (C.c_int, [_V, _I32, _V, _I64, _V, _I32, _I32] + [_V] * 7),
    "gsb_debug_dequant": (C.c_int, [C.POINTER(GsbQuant), _I32, _V, _V, _V]),
    "gsb_sh_statistics_update": (C.c_int, [_I32, _I32] + [_V] * 13),
    "gsb_min_projected_pixel_size": (C.c_int, [_I32, _V, _I32, _V, _V, _V, _V, _V, _V]),
    "gsb_filter_3d_workspace_bytes": (_SZ, []),
    "gsb_filter_3d": (C.c_int, [_I32, _V, _I32, _V, _V, _V, _V, _V, _V]),
    "gsb_sphere_ellipsoid_intersection": (C.c_int, [_I32, _V, _V, _V, _V, _V, _I32, _V, _V, _V]),
    "gsb_min_redundancy_value": (C.c_int, [_I32, _V, _V, _V, _I32, _V, _V]),
    "gsb_kmeans_workspace_bytes": (_SZ, [_I64, _I32, _I32]),
    "gsb_kmeans": (C.c_int, [_V, _I64, _V, _I32, _F, _I32, _I32, _V, _V, _V, _V]),
    "gsb_knn_workspace_bytes": (_SZ, [_I32, _I32]),
    "gsb_knn": (C.c_int, [_V, _I32, _I32, _V, _I32, _V, _I32, _V, _V, _V, _V, _V]),
    "gsb_l1_ssim_blocks": (C.c_int64, [_I32, _I32, _I32]),
    "gsb_l1_ssim_forward": (C.c_int, [_V, _V, _I32, _I32, _I32, _V, _V, _V]),
    "gsb_l1_ssim_backward": (C.c_int, [_V, _V, _I32, _I32, _I32, _V, _F, _V, _F, _V, _V, _V]),
    "gsb_adam_step": (C.c_int, [C.POINTER(GsbAdamTensor), _I32, _I32, _V, _V, _V]),
    "gsb_densify_stats": (C.c_int, [_I32, _V, _I32, _V, _I32] + [_V] * 7),
    "gsb_densify_workspace_bytes": (_SZ, [_I32]),
    "gsb_densify_split_std_offset": (_SZ, [_I32]),
    "gsb_densify_plan": (C.c_int, [_I32, _I32] + [_V] * 7 + [_F] * 4 + [_I32] + [_F] * 3 + [_V] * 3),
    "gsb_densify_emit": (C.c_int, [C.POINTER(GsbDensifyTensor), _I32, _I32, _V] + [_I64] * 4 + [_V, _V, _F, _V]),
    "gsb_redundancy_workspace_bytes": (_SZ, [_I32, _I32]),
    "gsb_redundancy_score": (C.c_int, [_I32, _V, _V, _V, _I32, _V, _V, _V, _V, _F, _I32, _V, _V, _V, _V]),
    "gsb_mercy_workspace_bytes": (_SZ, [_I32]),
    "gsb_mercy_plan": (C.c_int, [_I32, _V, _V, _I32, _F, C.c_double, _F, _V, _I64, _V, _V, _V, _V, _V]),
    "gsb_mcmc_noise": (C.c_int, [_I32] + [_V] * 5 + [_F, _F, _V]),
    "gsb_mcmc_workspace_bytes": (_SZ, [_I32]),
    "gsb_mcmc_plan": (C.c_int, [_I32, _I32, _V, _V, _V, _F, _I64, _V, _V, _V, _V]),
    "gsb_mcmc_emit": (C.c_int, [C.POINTER(GsbDensifyTensor), _I32, _I32, _I32, _I64, _V, _V]),
    "gsb_launch_count": (C.c_uint64, []),
    "gsb_profile_enable": (None, [C.c_int]),
    "gsb_profile_read": (C.c_int, [C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "gsb_last_error": (C.c_char_p, []),
    "gsb_version": (C.c_char_p, []),
}
EXPORTED_SYMBOLS = list(SIGNATURES)

_lib = None


def ensure_built() -> str:
    """Compile the library if it is absent or stale (needs nvcc; without it an existing build is used)."""
    src_dir = os.path.join(os.path.dirname(HERE), "csrc")
    if os.path.isfile(os.path.join(src_dir, "build.py")):
        import importlib.util
        spec = importlib.util.spec_from_file_location("gsb_build", os.path.join(src_dir, "build.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        try:
            return mod.build()
        except (RuntimeError, FileNotFoundError):
            if os.path.isfile(SO_PATH):
                return SO_PATH
            raise
    return SO_PATH


def lib():
    global _lib
    if _lib is None:
        path = ensure_built()
        if not os.path.isfile(path):
            raise RuntimeError(f"gs_b200: CUDA library {path} is missing — build it with reduced-3dgs_b200/csrc/build.py "
                               "(there is no CPU / PyTorch fallback)")
        L = C.CDLL(path)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = L
    return _lib


def profile_enable(on: bool):
    lib().gsb_profile_enable(1 if on else 0)


def profile_read() -> dict:
    """{kernel name: (total ms, launches)} since the previous read (waits for the recorded events)."""
    n = 32
    names = (C.c_char_p * n)()
    ms = (C.c_double * n)()
    cnt = (C.c_uint64 * n)()
    k = lib().gsb_profile_read(n, names, ms, cnt)
    return {names[i].decode(): (float(ms[i]), int(cnt[i])) for i in range(k)}


def check(status: int):
    if status != 0:
        raise RuntimeError("gs_b200: " + lib().gsb_last_error().decode())


def launch_count() -> int:
    return int(lib().gsb_launch_count())


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    """Device pointer of a tensor; None / empty tensors are the reference's "absent" (NULL)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def aligned16(t: torch.Tensor) -> torch.Tensor:
    """`t`, or a copy of it when its data does not start on a 16-byte boundary.  The kernels read rotation rows (and, where
    aligned, SH rows) with 128-bit loads; a contiguous view may start at any float of its storage."""
    return t if t.data_ptr() % 16 == 0 else t.clone()


def f32(t: Optional[torch.Tensor], device) -> Optional[torch.Tensor]:
    """Reference L1 contract: fp32, contiguous, on the CUDA device (rasterize_points.cu:197-217 .contiguous()), and 16-byte
    aligned (aligned16).  For inputs only: a tensor the library writes must be passed as it is."""
    if t is None or t.numel() == 0:
        return None
    if t.dtype != torch.float32 or t.device != device or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.float32).contiguous()
    return aligned16(t)


class BlobAllocator:
    """Python side of gsb_alloc_fn: allocates a torch uint8 tensor (the reference's resizeFunctional,
    rasterize_points.cu:33-41) and keeps it so it can be returned to the caller.

    The three ctypes callbacks (geometry / binning / image) are created ONCE per host thread and reused by every forward:
    building a CFUNCTYPE thunk costs ~10-15 us, three of them per call were a tenth of the host time of a step.  A callback
    closes over this per-thread object only; the tensors of the current call live in `held` and are handed to the caller by
    `take()`, so nothing keeps a blob alive after the call (no reference cycle through the thunk)."""

    # High-water mark of the sizes requested per (device, blob kind).  The instance count R — and with it the binning blob —
    # changes from view to view; requests of slightly different sizes make the caching allocator split / mismatch its cached
    # blocks and fall back to cudaMalloc (1-40 ms, inside a training step) every now and then.  Asking for the largest size
    # seen so far makes every request after the first pass over the views identical, so a freed block always fits.
    _hwm = {}
    _tls = threading.local()
    KINDS = ("geom", "binning", "image")

    def __init__(self):
        self.device = None
        self.held = {k: None for k in self.KINDS}
        self.cb = {k: ALLOC_FN(self._make(k)) for k in self.KINDS}

    @classmethod
    def for_device(cls, device) -> "BlobAllocator":
        a = getattr(cls._tls, "alloc", None)
        if a is None:
            a = cls._tls.alloc = cls()
        a.device = device
        for k in cls.KINDS:
            a.held[k] = None
        return a

    def _make(self, kind):
        hwm = BlobAllocator._hwm

        def alloc(_user, nbytes):
            # round up to 1/16 of the next power of two, then to the high-water mark (unless that is over twice the request:
            # a much smaller workload has started, restart the mark)
            nbytes = int(nbytes)
            if nbytes > (1 << 20):
                q = 1 << (nbytes.bit_length() - 5)
                nbytes = (nbytes + q - 1) // q * q
                key = (self.device, kind)
                top = hwm.get(key, 0)
                if nbytes <= top <= 2 * nbytes:
                    nbytes = top
                else:
                    hwm[key] = nbytes
            t = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self.held[kind] = t                     # a second request of the same kind in one call supersedes the first
            return t.data_ptr()
        return alloc

    def take(self, kind):
        """The blob of `kind` allocated during the call just finished (an empty tensor if the library asked for none)."""
        t, self.held[kind] = self.held[kind], None
        return t if t is not None else torch.empty(0, dtype=torch.uint8, device=self.device)


def on_device(device):
    """Context that makes `device` current for the C-ABI call; free when it already is (the usual case: one process per GPU)."""
    if torch.cuda.current_device() == device.index:
        return contextlib.nullcontext()
    return torch.cuda.device(device)


def current_stream(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream
