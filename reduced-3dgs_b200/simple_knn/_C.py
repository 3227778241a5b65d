"""Drop-in for the reference's pybind module `simple_knn._C` (submodules/simple-knn/ext.cpp:16-18), re-hosted on the C ABI
function gsb_knn (include/gs_b200.h) through ctypes.  Same names, positional signatures, flat return layout and dtypes as
spatial.cu:15-58:

    distCUDA2(points)                           -> float32 [P]: mean squared distance to the 3 nearest other points
    distIndex2(points, K)                       -> [dists float32 [P*K], indices int32 [P*K]]
    distIndexQ(points, q_indices, n_indices, K) -> [dists float32 [Q*K], indices int32 [Q*K]]: the K nearest of each query among
                                                   the points listed in the first min(N, P) entries of n_indices

Each row is sorted by (squared distance, index); missing neighbours are (FLT_MAX, -1).  The distances are bit-identical to the
reference's; the reference's slot order is an artefact of its visiting order, and of several neighbours tied at the K-th distance
it keeps the one it happened to visit first, where this module keeps the smallest index.  Differences, all additive: query ids
outside [0, P) give a row of (FLT_MAX, -1) and candidate ids outside [0, P) are ignored (the reference reads out of bounds);
K is limited to GSB_KNN_MAX_K = 64.  Runs on the tensors' device and its current stream; CPU tensors raise.
"""
from __future__ import annotations

import torch

from gs_b200 import lib as _lib
from gs_b200.lib import on_device, ptr


def _points(points: torch.Tensor):
    if not isinstance(points, torch.Tensor) or not points.is_cuda:
        raise RuntimeError("simple_knn: points must be a CUDA tensor (no CPU path exists)")
    if points.dtype != torch.float32:
        raise RuntimeError(f"simple_knn: points must be float32, got {points.dtype}")
    if points.ndimension() != 2 or points.size(1) != 3:
        raise RuntimeError(f"simple_knn: points must have shape (P, 3), got {tuple(points.shape)}")
    d = points.device
    return points.contiguous(), (d if d.index is not None else torch.device("cuda", torch.cuda.current_device()))


def _ids(t: torch.Tensor, device, what: str):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"simple_knn: {what} must be a CUDA tensor")
    if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
        raise RuntimeError(f"simple_knn: {what} must be an integer tensor, got {t.dtype}")
    return t.to(device=device, dtype=torch.int32).reshape(-1).contiguous()


def _knn(points, K, q=None, n=None, mean=False):
    pts, device = _points(points)
    K = int(K)
    if K < 0:
        raise RuntimeError(f"simple_knn: K must be >= 0, got {K}")
    P = int(pts.size(0))
    qi = None if q is None else _ids(q, device, "q_indices")
    ni = None if n is None else _ids(n, device, "n_indices")
    rows = P if qi is None else int(qi.numel())
    L = _lib.lib()
    with on_device(device):
        m = torch.empty((rows,), dtype=torch.float32, device=device) if mean else None
        d = torch.empty((0 if mean else rows * K,), dtype=torch.float32, device=device)
        i = torch.empty((0 if mean else rows * K,), dtype=torch.int32, device=device)
        ws = torch.empty((int(L.gsb_knn_workspace_bytes(P, -1 if qi is None else rows)),), dtype=torch.uint8, device=device)
        _lib.check(L.gsb_knn(ptr(pts), P, K, ptr(qi), -1 if qi is None else rows, ptr(ni), -1 if ni is None else int(ni.numel()),
                             ptr(m), ptr(d), ptr(i), ws.data_ptr(), _lib.current_stream(device)))
    return m if mean else [d, i]


def distCUDA2(points):
    """spatial.cu:15-26 -> float32 [P]: ((d0 + d1) + d2) / 3 of the three smallest squared distances (FLT_MAX where missing)."""
    return _knn(points, 3, mean=True)


def distIndex2(points, K):
    """spatial.cu:28-41 distCudaIndices2 -> [dists float32 [P*K], indices int32 [P*K]]."""
    return _knn(points, K)


def distIndexQ(points, q_indices, n_indices, K):
    """spatial.cu:43-58 distCudaIndicesQ -> [dists float32 [Q*K], indices int32 [Q*K]]."""
    return _knn(points, K, q_indices, n_indices)
