"""Run OUR CUDA path through the reference-facing `_C` API and return numpy dicts shaped like oracle outputs
(shared by the GPU parity tests, __graft_entry__.smoke and tools/), plus the tensor-level call helpers, scenes, cameras and model
of the GPU feature tests."""
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


def run_forward(scene, cam, bg, extra=None, prune_mask=None, quant=None, dev="cuda", aa=False):
    """-> (args, raw outputs, dict of numpy intermediates in reference layouts); `aa`: antialiasing=True."""
    args = forward_args(scene, cam, bg, extra, dev)
    dbg = {}
    out = _C.rasterize_gaussians(*args, prune_mask=None if prune_mask is None else prune_mask.to(dev),
                                 quant=None if quant is None else quant.to(dev), debug_out=dbg, antialiasing=aa)
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


def run_backward(args, out, dL, lam=0.0, prune_mask=None, quant=None, aa=False, deterministic=False):
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = args
    R, color, radii, geom, binning, img = out
    dev = means3D.device
    grads = _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, view, proj, tx, ty,
                                            dL.to(dev), sh, degrees, campos, geom, R, binning, img, lam, False,
                                            prune_mask=None if prune_mask is None else prune_mask.to(dev),
                                            quant=None if quant is None else quant.to(dev), want_conic=True, antialiasing=aa,
                                            deterministic=deterministic)
    torch.cuda.synchronize()
    res = {n: g.cpu().numpy() for n, g in zip(GRAD_NAMES + ["dL_dconic"], grads)}
    return res


# ---- tensor-level helpers of the feature tests (maps, camera, anti-aliasing) ----------------------------------------------------

def yaw_cam(W, H, deg=0.0, dev="cuda", grad=False):
    """synth's default camera (4 units from the origin, looking at it) turned by `deg` degrees about the y axis; with `grad` its
    view, projection and centre are fresh leaves that require grad."""
    th = math.radians(deg)
    Rc2w = np.array([[math.cos(th), 0, math.sin(th)], [0, 1, 0], [-math.sin(th), 0, math.cos(th)]])
    C = Rc2w @ np.array([0.0, 0.0, -4.0])
    cam = synth.make_camera(W, H, Rc2w, -Rc2w.T @ C).to(dev)
    if grad:
        for k in ("world_view_transform", "full_proj_transform", "camera_center"):
            setattr(cam, k, getattr(cam, k).detach().clone().requires_grad_())
    return cam


# One row per synthetic test scene: image W, H, count P, seed, SH degree or "mixed", log-scale mean (the box then follows the
# image's aspect) or None for synth's defaults, yaw of the camera in degrees or None for synth's default camera, prune-mask seed
# or None, quantised.  "c1" is config C1 for every option.
_SCENES = {
    ("camera", "sh3"): (320, 200, 20_000, 181, 3, 0.03, 8.0, None, False),
    ("camera", "mixed"): (320, 200, 20_000, 182, "mixed", 0.03, -5.0, None, False),
    ("camera", "quant"): (320, 200, 20_000, 183, "mixed", 0.03, 4.0, None, True),
    ("camera", "pruned"): (320, 200, 20_000, 184, 2, 0.03, -3.0, 185, False),
    ("aa", "mixed"): (320, 200, 20_000, 201, "mixed", 0.02, -5.0, None, False),
    ("aa", "quant"): (320, 200, 20_000, 202, "mixed", 0.02, 4.0, None, True),
    ("aa", "pruned"): (320, 200, 20_000, 203, 2, 0.02, -3.0, 204, False),
    ("maps", "hd"): (1920, 1080, 300_000, 81, "mixed", None, None, None, False),
    ("maps", "quant"): (320, 200, 20_000, 82, "mixed", 0.03, None, None, True),
    ("maps", "pruned"): (320, 200, 20_000, 83, 2, 0.03, None, 84, False),
}


def scene_config(option, name):
    """The test scene `name` of an option's GPU tests -> (scene, cam, prune_mask or None, quant or None), all on the CPU."""
    if name == "c1":
        return synth.config_scene("C1"), synth.make_camera(*synth.config_image("C1")), None, None
    W, H, P, seed, deg, ls, yaw, prune_seed, quantised = _SCENES[(option, name)]
    kw = dict(mixed_degrees=True) if deg == "mixed" else dict(sh_degree=deg)
    if ls is not None:
        kw.update(box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(ls))
    scene = synth.make_scene(P, seed, **kw)
    cam = synth.make_camera(W, H) if yaw is None else yaw_cam(W, H, yaw, dev="cpu")
    return (scene, cam, None if prune_seed is None else synth.prune_mask(scene.P, prune_seed),
            synth.quantise_scene(scene) if quantised else None)


def empty_and_culled_scenes(P=33):
    """(P = 0, P Gaussians all behind synth's default camera: every one is culled and R = 0), on the CPU."""
    empty = synth.Scene(torch.zeros(0, 3), torch.zeros(0, 1), torch.zeros(0, 3), torch.zeros(0, 4), torch.zeros(0, 1, 3),
                        torch.zeros(0, 1, dtype=torch.int32))
    means = torch.zeros(P, 3)
    means[:, 2] = -9.0
    culled = synth.Scene(means, torch.zeros(P, 1), torch.full((P, 3), 0.1), torch.tensor([[1.0, 0, 0, 0]]).repeat(P, 1),
                         torch.zeros(P, 1, 3), torch.zeros(P, 1, dtype=torch.int32))
    return empty, culled


class Model:
    """The attributes render() reads from the reference's GaussianModel, with the reference's activations
    (scene/gaussian_model.py:141-158: exp for scales, normalize for rotations; opacity stays a logit)."""

    def __init__(self, scene, dev):
        self._xyz = scene.means3D.to(dev).clone().requires_grad_(True)
        self._opacity = scene.opacity.to(dev).clone().requires_grad_(True)
        self._log_scaling = torch.log(scene.scales.to(dev)).requires_grad_(True)
        self._rotation = scene.rotations.to(dev).clone().requires_grad_(True)
        self._features = scene.sh.to(dev).clone().requires_grad_(True)
        self._degrees = scene.degrees.to(dev)
        self.active_sh_degree = self.max_sh_degree = 3
        self.per_band_count = [int((scene.degrees == d).sum()) for d in range(4)]

    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: torch.exp(s._log_scaling))
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rotation))
    get_features = property(lambda s: s._features)

    def params(self):
        return [self._xyz, self._opacity, self._log_scaling, self._rotation, self._features]


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
    """Both present, the same shape and the same bytes."""
    return a is not None and b is not None and a.shape == b.shape and torch.equal(bits(a), bits(b))
