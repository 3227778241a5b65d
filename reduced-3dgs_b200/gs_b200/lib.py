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
                ("quant", C.POINTER(GsbQuant))]


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
        L.gsb_geom_bytes.restype = C.c_size_t
        L.gsb_geom_bytes.argtypes = [C.c_int32]
        L.gsb_image_bytes.restype = C.c_size_t
        L.gsb_image_bytes.argtypes = [C.c_int32, C.c_int32]
        L.gsb_image_bytes_for.restype = C.c_size_t
        L.gsb_image_bytes_for.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
        L.gsb_binning_bytes.restype = C.c_size_t
        L.gsb_binning_bytes.argtypes = [C.c_int64]
        L.gsb_launch_count.restype = C.c_uint64
        L.gsb_last_error.restype = C.c_char_p
        L.gsb_version.restype = C.c_char_p
        L.gsb_forward.restype = C.c_int
        L.gsb_forward.argtypes = [C.POINTER(GsbScene), C.POINTER(GsbCamera), ALLOC_FN, C.c_void_p, ALLOC_FN, C.c_void_p,
                                  ALLOC_FN, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64),
                                  C.POINTER(GsbDebug), C.c_void_p]
        L.gsb_forward_statistics.restype = C.c_int
        L.gsb_forward_statistics.argtypes = [C.POINTER(GsbScene), C.POINTER(GsbCamera), ALLOC_FN, C.c_void_p, ALLOC_FN, C.c_void_p,
                                             ALLOC_FN, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64),
                                             C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_sh_statistics_update.restype = C.c_int
        L.gsb_sh_statistics_update.argtypes = [C.c_int32, C.c_int32] + [C.c_void_p] * 13
        L.gsb_min_projected_pixel_size.restype = C.c_int
        L.gsb_min_projected_pixel_size.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]
        L.gsb_sphere_ellipsoid_intersection.restype = C.c_int
        L.gsb_sphere_ellipsoid_intersection.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                                        C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_min_redundancy_value.restype = C.c_int
        L.gsb_min_redundancy_value.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        L.gsb_kmeans_workspace_bytes.restype = C.c_size_t
        L.gsb_kmeans_workspace_bytes.argtypes = [C.c_int64, C.c_int32]
        L.gsb_kmeans.restype = C.c_int
        L.gsb_kmeans.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_float, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]
        L.gsb_knn_workspace_bytes.restype = C.c_size_t
        L.gsb_knn_workspace_bytes.argtypes = [C.c_int32, C.c_int32]
        L.gsb_knn.restype = C.c_int
        L.gsb_knn.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_l1_ssim_blocks.restype = C.c_int64
        L.gsb_l1_ssim_blocks.argtypes = [C.c_int32, C.c_int32, C.c_int32]
        L.gsb_l1_ssim_forward.restype = C.c_int
        L.gsb_l1_ssim_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_l1_ssim_backward.restype = C.c_int
        L.gsb_l1_ssim_backward.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_float, C.c_void_p,
                                           C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_backward.restype = C.c_int
        L.gsb_backward.argtypes = [C.POINTER(GsbScene), C.POINTER(GsbCamera), C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.POINTER(GsbGrads), C.c_float, C.c_void_p]
        L.gsb_mark_visible.restype = C.c_int
        L.gsb_mark_visible.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_export_binning.restype = C.c_int
        L.gsb_export_binning.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32,
                                         C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_export_image.restype = C.c_int
        L.gsb_export_image.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_debug_dequant.restype = C.c_int
        L.gsb_debug_dequant.argtypes = [C.POINTER(GsbQuant), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gsb_profile_enable.restype = None
        L.gsb_profile_enable.argtypes = [C.c_int]
        L.gsb_profile_read.restype = C.c_int
        L.gsb_profile_read.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


def profile_enable(on: bool):
    lib().gsb_profile_enable(1 if on else 0)


def profile_read() -> dict:
    """{kernel name: (total ms, launches)} since the previous read (waits for the recorded events)."""
    n = 16
    names = (C.c_char_p * n)()
    ms = (C.c_double * n)()
    cnt = (C.c_uint64 * n)()
    k = lib().gsb_profile_read(n, names, ms, cnt)
    return {names[i].decode(): (float(ms[i]), int(cnt[i])) for i in range(k)}


EXPORTED_SYMBOLS = ["gsb_geom_bytes", "gsb_image_bytes", "gsb_image_bytes_for", "gsb_binning_bytes", "gsb_forward", "gsb_backward",
                    "gsb_mark_visible", "gsb_export_binning", "gsb_export_image", "gsb_launch_count", "gsb_last_error",
                    "gsb_version", "gsb_profile_enable", "gsb_profile_read", "gsb_debug_dequant", "gsb_forward_statistics",
                    "gsb_sh_statistics_update", "gsb_min_projected_pixel_size", "gsb_sphere_ellipsoid_intersection",
                    "gsb_min_redundancy_value", "gsb_kmeans_workspace_bytes", "gsb_kmeans", "gsb_l1_ssim_blocks",
                    "gsb_l1_ssim_forward", "gsb_l1_ssim_backward", "gsb_knn_workspace_bytes", "gsb_knn"]


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


def f32(t: Optional[torch.Tensor], device) -> Optional[torch.Tensor]:
    """Reference L1 contract: fp32, contiguous, on the CUDA device (rasterize_points.cu:197-217 .contiguous())."""
    if t is None or t.numel() == 0:
        return None
    if t.dtype != torch.float32 or t.device != device or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.float32).contiguous()
    return t


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
