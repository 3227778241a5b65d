"""Mip-Splatting's 3D smoothing filter (Yu et al., "Mip-Splatting: Alias-free 3D Gaussian Splatting", CVPR 2024; DESIGN.md §5o).

    from gs_b200 import mip
    mip.compute_3D_filter(gaussians, scene.getTrainCameras())       # INTEGRATION.md section J
    render(camera, gaussians, pipe, bg)                              # render() forwards gaussians.filter_3D to the kernels

compute_3D_filter is Mip-Splatting's GaussianModel.compute_3D_filter in one native call (gsb_filter_3d): for every centre, the
smallest depth at which a training camera sees it, over the largest focal length, times sqrt(0.2).  The kernels then render with
scales sqrt(s^2 + f^2) and opacities sigmoid(logit) * c3.  Differences from Mip-Splatting's loop: the view transform is
world_view_transform (the rasterizer's own depth), and a model no camera sees gets a zero filter where Mip-Splatting raises.
"""
from __future__ import annotations

import math

import torch

from . import lib as gsl


def compute_3D_filter(model, cameras):
    """Sets model.filter_3D = f as fp32 [P, 1] on the model's device (Mip-Splatting's layout) from `cameras`, objects exposing
    world_view_transform (4 x 4, the transposed view matrix), FoVx, FoVy, image_width and image_height.  The camera table goes to the
    device in one copy; nothing is read back.  -> model.filter_3D."""
    xyz = model.get_xyz
    if not torch.is_tensor(xyz) or not xyz.is_cuda or xyz.dtype != torch.float32 or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise RuntimeError("mip: the model's get_xyz must be an fp32 CUDA tensor [P, 3]")
    dev, P, n = xyz.device, int(xyz.shape[0]), len(cameras)
    xyz = xyz.detach().contiguous()
    # one host table: [n, 16] view matrices, [n, 2] focal lengths (fp64 on the host, used as fp32), [n, 2] int32 (W, H)
    host = torch.empty(20 * n, dtype=torch.float32)
    views = [c.world_view_transform for c in cameras]
    on_host = all(not v.is_cuda for v in views)
    sizes = [(int(c.image_width), int(c.image_height)) for c in cameras]
    focals = [(W / (2.0 * math.tan(c.FoVx / 2.0)), H / (2.0 * math.tan(c.FoVy / 2.0))) for c, (W, H) in zip(cameras, sizes)]
    if n:
        host[16 * n:18 * n] = torch.tensor(focals, dtype=torch.float64).reshape(-1)      # rounded to fp32 once, here
        host[18 * n:].view(torch.int32)[:] = torch.tensor(sizes, dtype=torch.int32).reshape(-1)
    if n and on_host:
        host[:16 * n] = torch.stack([v.detach().to(torch.float32).reshape(16) for v in views]).reshape(-1)
    table = host.to(dev)
    if n and not on_host:
        table[:16 * n] = torch.stack([v.detach().to(device=dev, dtype=torch.float32).reshape(16) for v in views]).reshape(-1)
    out = torch.empty((P, 1), dtype=torch.float32, device=dev)
    L = gsl.lib()
    ws = torch.empty(int(L.gsb_filter_3d_workspace_bytes()), dtype=torch.uint8, device=dev)
    base = table.data_ptr() if n else None
    with gsl.on_device(dev):
        gsl.check(L.gsb_filter_3d(P, xyz.data_ptr() if P else None, n, base, base + 64 * n if n else None,
                                  base + 72 * n if n else None, out.data_ptr() if P else None, ws.data_ptr(), gsl.current_stream(dev)))
    model.filter_3D = out
    return out
