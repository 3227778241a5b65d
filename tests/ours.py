"""Run OUR CUDA path through the reference-facing `_C` API and return numpy dicts shaped like oracle outputs
(shared by the GPU parity tests, __graft_entry__.smoke and tools/), plus the tensor-level call helpers of the GPU feature tests."""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))

from diff_gaussian_rasterization import _C  # noqa: E402
from gs_b200 import synth  # noqa: E402

EMPTY = torch.Tensor([])


def forward_args(scene, cam, bg, extra=None, dev="cuda"):
    extra = extra or {}
    cov, col = extra.get("cov3D_precomp"), extra.get("colors_precomp")
    return (bg.to(dev), scene.means3D.to(dev), EMPTY if col is None else col.to(dev), scene.opacity.to(dev),
            EMPTY if cov is not None else scene.scales.to(dev), EMPTY if cov is not None else scene.rotations.to(dev), 1.0,
            EMPTY if cov is None else cov.to(dev), cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev),
            math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), cam.image_height, cam.image_width,
            EMPTY if col is not None else scene.sh.to(dev), scene.degrees.to(dev), cam.camera_center.to(dev), False, False)


def run_forward(scene, cam, bg, extra=None, prune_mask=None, quant=None, dev="cuda"):
    """-> (args, raw outputs, dict of numpy intermediates in reference layouts)."""
    args = forward_args(scene, cam, bg, extra, dev)
    dbg = {}
    out = _C.rasterize_gaussians(*args, prune_mask=None if prune_mask is None else prune_mask.to(dev),
                                 quant=None if quant is None else quant.to(dev), debug_out=dbg)
    R, color, radii, geomB, binB, imgB = out
    st = _C.export_state(geomB, binB, imgB, R, cam.image_width, cam.image_height, P=scene.means3D.shape[0])
    torch.cuda.synchronize()
    res = dict(num_rendered=R, color=color.cpu().numpy(), radii=radii.cpu().numpy(),
               depths=dbg["depths"].cpu().numpy(), means2D=dbg["means2D"].cpu().numpy(), cov3D=dbg["cov3D"].cpu().numpy(),
               conic_opacity=dbg["conic_opacity"].cpu().numpy(), rgb=dbg["rgb"].cpu().numpy(),
               tiles_touched=dbg["tiles_touched"].cpu().numpy().astype(np.uint32), clamped=dbg["clamped"].cpu().numpy(),
               keys=st["keys"].cpu().numpy().astype(np.uint64), point_list=st["point_list"].cpu().numpy().astype(np.uint32),
               ranges=st["ranges"].cpu().numpy().astype(np.uint32), final_T=st["final_T"].cpu().numpy(),
               n_contrib=st["n_contrib"].cpu().numpy().astype(np.uint32))
    return args, out, res


GRAD_NAMES = ["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations"]


def run_backward(args, out, dL, lam=0.0, prune_mask=None, quant=None):
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = args
    R, color, radii, geom, binning, img = out
    dev = means3D.device
    grads = _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, view, proj, tx, ty,
                                            dL.to(dev), sh, degrees, campos, geom, R, binning, img, lam, False,
                                            prune_mask=None if prune_mask is None else prune_mask.to(dev),
                                            quant=None if quant is None else quant.to(dev), want_conic=True)
    torch.cuda.synchronize()
    res = {n: g.cpu().numpy() for n, g in zip(GRAD_NAMES + ["dL_dconic"], grads)}
    return res


# ---- tensor-level helpers of the feature tests (maps, camera, anti-aliasing) ----------------------------------------------------

def yaw_cam(W, H, deg, dev="cuda"):
    """synth's default camera (4 units from the origin, looking at it) turned by `deg` degrees about the y axis."""
    th = math.radians(deg)
    Rc2w = np.array([[math.cos(th), 0, math.sin(th)], [0, 1, 0], [-math.sin(th), 0, math.cos(th)]])
    C = Rc2w @ np.array([0.0, 0.0, -4.0])
    return synth.make_camera(W, H, Rc2w, -Rc2w.T @ C).to(dev)


def device_kw(prune, quant, dev="cuda"):
    return dict(prune_mask=None if prune is None else prune.to(dev), quant=None if quant is None else quant.to(dev))


def forward(scene, cam, bg, prune=None, quant=None, colors=None, maps=False, dbg=None, aa=False, extra=None):
    """_C.rasterize_gaussians on forward_args; `colors` is short for extra={"colors_precomp": colors}.  -> (args, outputs)."""
    args = forward_args(scene, cam, bg, extra if colors is None else {"colors_precomp": colors})
    return args, _C.rasterize_gaussians(*args, return_maps=maps, debug_out=dbg, antialiasing=aa, **device_kw(prune, quant))


def backward(args, out, dL, prune=None, quant=None, aa=False, **extra):
    """_C.rasterize_gaussians_backward of a `forward` call; `extra` are its keyword arguments."""
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = args
    R, color, radii, geom, binning, img = out[:6]
    return _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, view, proj, tx, ty, dL.to("cuda"), sh,
                                           degrees, campos, geom, R, binning, img, 0.0, False, antialiasing=aa,
                                           **device_kw(prune, quant), **extra)


def state(out, cam, P):
    """The reference-layout binning and image state of a `forward` output (export_state)."""
    st = _C.export_state(out[3], out[4], out[5], out[0], cam.image_width, cam.image_height, P=P)
    torch.cuda.synchronize()
    return st


def bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def same(a, b):
    """Same shape and the same bytes."""
    return a.shape == b.shape and torch.equal(bits(a), bits(b))
