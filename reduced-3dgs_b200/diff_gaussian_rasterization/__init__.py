"""Drop-in replacement for the reference Python package `diff_gaussian_rasterization`
(submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py): same
GaussianRasterizationSettings (:169-181), GaussianRasterizer (:183-234), rasterize_gaussians (:21-46) and
_RasterizeGaussians autograd op (:48-167), backed by the H100-native kernels through `_C`.

Differences, all additive: GaussianRasterizer.forward takes keyword-only `prune_mask` and `quant`
(fused resolution-aware prune mask / codebook de-quantisation, SURVEY §8(b)) and `return_maps` (differentiable inverse-depth
and alpha maps from the same pass: (color, radii, invdepth, alpha)); a raster_settings.viewmatrix / projmatrix / campos
that requires grad receives its gradient, where the reference silently treats the camera as a
constant; GaussianRasterizationSettings takes upstream 3DGS's trailing `antialiasing` argument (default False; the tuple keeps the
reference's 12 fields), which turns on the opacity-compensated 2D filter in the forward and the backward; the
forward no longer forces
debug=True (reference :85 hard-wires a device sync after every stage); gradients are allocated uninitialised
because the kernels write every element.  GaussianRasterizer.forward also takes keyword-only `raw_params`, the model's leaf
tensors (features_dc, features_rest, scaling, rotation) in place of shs / scales / rotations: exp, F.normalize and the SH
concatenation then run inside the kernels, and the gradients of the four tensors are the kernels' own outputs.
GaussianRasterizationSettings' keyword-only `deterministic` (default: torch's deterministic-algorithms
flag) selects the backward that sums each Gaussian's gradients in a fixed order (the same bytes on every run).
GaussianRasterizer.forward's keyword-only `features` ([P, F] fp32, 1 <= F <= 256) appends the [F, H, W] image of per-Gaussian
features composited over the colour pass with background 0; its gradient reaches the features and, through alpha, everything the
colour gradient reaches.  The feature gradient has no deterministic form: it is refused when the deterministic mode is on.
GaussianRasterizer.forward's keyword-only `means2D_abs` (a [P, 3] tensor that requires grad, e.g. a zeros leaf) receives as its
gradient the absolute screen-space gradient (sum_p |g_x|, sum_p |g_y|, 0) of AbsGS, the densification
statistic whose per-pixel terms cannot cancel; it has no feature form.
GaussianRasterizer.forward's keyword-only `filter_3D` ([P] or [P, 1] fp32, gs_b200.mip.compute_3D_filter) applies Mip-Splatting's
3D smoothing filter to the scales and the opacity inside the kernels; it is a constant (no gradient), as Mip-Splatting's buffer is.
GaussianRasterizer.forward's keyword-only `contributions=True` appends _C.Contributions(weight_sum [P], weight_max [P], pixels [P],
top_id [H, W]), the view's per-Gaussian blending-weight statistics from the forward's own blobs (no gradient); `pixel_weights`
([H, W] fp32) weights the sum.
Every option goes through the one autograd op, _RasterizeGaussians, each optional input in a slot of its own.
"""
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _C


def cpu_deep_copy_tuple(input_tuple):
    copied_tensors = [item.cpu().clone() if isinstance(item, torch.Tensor) else item for item in input_tuple]
    return tuple(copied_tensors)


def _call(fn, args, kw, dump, message):
    """fn(*args, **kw); in debug mode, a failure first saves a CPU copy of the arguments to `dump` (reference :90-97, 142-149)."""
    if not args[-1]:                                               # raster_settings.debug
        return fn(*args, **kw)
    cpu_args = cpu_deep_copy_tuple(args)   # Copy them before they can be corrupted
    try:
        return fn(*args, **kw)
    except Exception as ex:
        torch.save(cpu_args, dump)
        print(message)
        raise ex


# The autograd op's inputs, in the order of its forward's parameters: the reference's fourteen (means3D ... cov3Ds_precomp,
# raster_settings, lambda_sh_sparsity, prune_mask, quant, return_maps), then one slot per optional input.  A call that uses no
# optional input passes the first fourteen only.  The contributions request (a 1-tuple of the pixel weights, or None) comes last and
# only when it is made.
MEANS3D, MEANS2D, SH, DEGREES, COLORS, OPACITIES, SCALES, ROTATIONS, COV3D = range(9)
VIEWMATRIX, PROJMATRIX, CAMPOS, FEATURES, MEANS2D_ABS, FEATURES_DC, FEATURES_REST, SCALING, ROTATION, FILTER_3D, CONTRIBUTIONS = range(14, 25)
N_INPUTS = 25


def _deterministic(raster_settings):
    """The settings' `deterministic`: an explicit bool wins; None follows torch.are_deterministic_algorithms_enabled(), read when
    the backward runs."""
    d = getattr(raster_settings, "deterministic", None)
    return torch.are_deterministic_algorithms_enabled() if d is None else bool(d)


def rasterize_gaussians(means3D, means2D, sh, degrees, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings, lambda_sh_sparsity, prune_mask=None, quant=None, return_maps=False, features=None,
                        means2D_abs=None, raw_params=None, filter_3D=None, contributions=None):
    """`contributions`: None, or the request (pixel_weights or None,): the outputs then end with a _C.Contributions."""
    camera = (raster_settings.viewmatrix, raster_settings.projmatrix, raster_settings.campos)
    if not (torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in camera)):
        # a constant camera is read from raster_settings; a learnable one is also an input, so that its gradients have a destination
        camera = (None,) * 3
    optional = (*camera, features, means2D_abs, *(raw_params or (None,) * 4), filter_3D)
    if contributions is not None:
        optional += (contributions,)
    out = _RasterizeGaussians.apply(means3D, means2D, sh, degrees, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                    raster_settings, lambda_sh_sparsity, prune_mask, quant, return_maps,
                                    *(optional if any(t is not None for t in optional) else ()))
    return out if contributions is None else out[:-4] + (_C.Contributions(*out[-4:]),)


class _RasterizeGaussians(torch.autograd.Function):
    """The reference's op with the optional inputs above.  `viewmatrix` / `projmatrix` / `campos` are raster_settings' own tensors,
    given only when the camera is learnable.  `features_dc` [P,1,3], `features_rest` [P,C,3] (both None with colors_precomp),
    `scaling` [P,3] (log-scales) and `rotation` [P,4] (unnormalised) are the model's leaf tensors in place of sh, scales and rotations
    (then empty): the kernels apply get_features / get_scaling / get_rotation themselves and return the gradients of these four
    tensors directly, so the graph holds no Cat / Exp / Div node and no [P,16,3] copy or gradient exists.  `filter_3D` is
    Mip-Splatting's 3D filter, a constant: the backward gets it and the opacity logits, and it receives no gradient.
    `contributions` = (pixel_weights or None,) runs _C.contributions on the blobs this forward left.
    -> (color, radii), with return_maps (color, radii, invdepth, alpha); with `features` the feature image [F, H, W] comes next, and with
    `contributions` its four tensors (weight_sum, weight_max, pixels, top_id) last, non-differentiable."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, degrees, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                lambda_sh_sparsity, prune_mask=None, quant=None, return_maps=False, viewmatrix=None, projmatrix=None, campos=None,
                features=None, means2D_abs=None, features_dc=None, features_rest=None, scaling=None, rotation=None, filter_3D=None,
                contributions=None):
        rs = raster_settings
        args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix,
                rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh, degrees, rs.campos, rs.prefiltered, rs.debug)
        ctx.raw = scaling is not None
        kw = dict(raw=(features_dc, features_rest, scaling, rotation)) if ctx.raw else dict(quant=quant)
        kw.update(prune_mask=prune_mask, return_maps=return_maps, antialiasing=rs.antialiasing)
        if features is not None:
            kw.update(features=features)
        if filter_3D is not None:
            kw.update(filter_3D=filter_3D)
        out = _call(_C.rasterize_gaussians, args, kw,
                    "snapshot_fw.dump", "\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
        ctx.raster_settings, ctx.num_rendered, ctx.lambda_sh_sparsity = rs, out[0], lambda_sh_sparsity
        ctx.prune_mask, ctx.quant, ctx.return_maps, ctx.has_features = prune_mask, quant, return_maps, features is not None
        ctx.has_abs = means2D_abs is not None
        ctx.camera_meta = None if viewmatrix is None else [(t.shape, t.dtype) for t in (viewmatrix, projmatrix, campos)]
        contrib = ()
        if contributions is not None:
            contrib = tuple(_C.contributions(out[3], out[4], out[5], out[0], rs.image_width, rs.image_height, means3D.shape[0],
                                             pixel_weights=contributions[0]))
        ctx.mark_non_differentiable(out[2], *contrib)
        if return_maps or features is not None:
            # a loss on some outputs only: the others' gradients arrive as None and reach the kernels as NULL (zero), and a feature
            # image without a gradient leaves the backward exactly the call without features
            ctx.set_materialize_grads(False)
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, out[2], sh, out[3], out[4], out[5], degrees,
                              features, features_dc, features_rest, scaling, rotation, filter_3D,
                              opacities if filter_3D is not None else None)
        return (out[1], out[2]) + (out[6:8] if return_maps else ()) + (out[-1:] if features is not None else ()) + contrib

    @staticmethod
    def backward(ctx, grad_out_color, _, *grads):
        # after (color, radii): the maps' gradients with return_maps, then the feature image's when given (the contributions, last,
        # have none)
        grad_invdepth, grad_alpha = grads[:2] if ctx.return_maps else (None, None)
        grad_features = grads[2 if ctx.return_maps else 0] if ctx.has_features else None
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer, imgBuffer, degrees, features,
         features_dc, features_rest, scaling, rotation, filter_3D, opacities) = ctx.saved_tensors
        rs = ctx.raster_settings
        if grad_out_color is None:
            grad_out_color = torch.zeros((3, rs.image_height, rs.image_width), dtype=torch.float32, device=means3D.device)
        need = ctx.needs_input_grad + (False,) * (N_INPUTS - len(ctx.needs_input_grad))
        args = (rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix, rs.projmatrix,
                rs.tanfovx, rs.tanfovy, grad_out_color, sh, degrees, rs.campos, geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer,
                ctx.lambda_sh_sparsity, rs.debug)
        kw = dict(raw=(features_dc, features_rest, scaling, rotation)) if ctx.raw else dict(quant=ctx.quant)
        kw.update(prune_mask=ctx.prune_mask, dL_dinvdepth=grad_invdepth, dL_dalpha=grad_alpha,
                  camera_grads=any(need[VIEWMATRIX:CAMPOS + 1]), antialiasing=rs.antialiasing)
        if _deterministic(rs):
            kw.update(deterministic=True)
        if grad_features is not None:
            kw.update(features=features, dL_dfeatures_out=grad_features)
        if filter_3D is not None:
            kw.update(filter_3D=filter_3D, opacity=opacities)
        out = [None] * N_INPUTS
        if ctx.has_abs:
            out[MEANS2D_ABS] = torch.empty((means3D.shape[0], 3), dtype=torch.float32, device=means3D.device)
            kw.update(absgrad_out=out[MEANS2D_ABS])
        g = _call(_C.rasterize_gaussians_backward, args, kw,
                  "snapshot_bw.dump", "\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
        # the 8-tuple, or the raw 9-tuple; then the camera gradients (camera_grads) and dL_dfeatures (features)
        if ctx.raw:
            (out[MEANS2D], out[COLORS], out[OPACITIES], out[MEANS3D], _, out[FEATURES_DC], out[FEATURES_REST], out[SCALING],
             out[ROTATION]) = g[:9]
        else:
            out[MEANS2D], out[COLORS], out[OPACITIES], out[MEANS3D], out[COV3D], out[SH], out[SCALES], out[ROTATIONS] = g[:8]
        if kw["camera_grads"]:
            k = 9 if ctx.raw else 8
            for i, (t, (shape, dtype)) in enumerate(zip(g[k:k + 3], ctx.camera_meta)):
                out[VIEWMATRIX + i] = t.reshape(shape).to(dtype)
        if grad_features is not None:
            out[FEATURES] = g[-1]
        if ctx.quant is not None:
            # inputs were id planes: the per-Gaussian attribute gradients have no autograd destination; expose them with the
            # semantics of `.grad`: they accumulate over backward calls until the caller resets `quant.grads = None`
            new = dict(sh=out[SH], opacity=out[OPACITIES], scales=out[SCALES], rotations=out[ROTATIONS])
            old = getattr(ctx.quant, "grads", None)
            if old:
                for k, t in new.items():
                    old[k].add_(t)
            else:
                ctx.quant.grads = new
        return tuple(t if n else None for t, n in zip(out, need))


class _ReferenceSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class GaussianRasterizationSettings(_ReferenceSettings):
    """The reference's 12-field settings tuple (its `_fields`, length and positional layout are unchanged) plus upstream 3DGS's
    trailing `antialiasing` flag, given as a keyword or as a 13th positional argument; default False.
    `deterministic` (keyword only): True sums the backward's per-Gaussian gradients in a fixed order, so the same inputs give the
    same bytes on every run; False keeps the faster atomic summation; None (default) follows torch.use_deterministic_algorithms,
    read when the backward runs."""
    antialiasing = False
    deterministic = None

    def __new__(cls, *args, antialiasing=False, deterministic=None, **kwargs):
        if len(args) == len(_ReferenceSettings._fields) + 1:
            *args, antialiasing = args
        self = super().__new__(cls, *args, **kwargs)
        self.antialiasing = bool(antialiasing)
        self.deterministic = None if deterministic is None else bool(deterministic)
        return self

    def _replace(self, **kwargs):
        antialiasing = kwargs.pop("antialiasing", self.antialiasing)
        deterministic = kwargs.pop("deterministic", self.deterministic)
        return type(self)(*super()._replace(**kwargs), antialiasing=antialiasing, deterministic=deterministic)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        # Mark visible points (based on frustum culling for camera) with a boolean
        with torch.no_grad():
            raster_settings = self.raster_settings
            visible = _C.mark_visible(positions, raster_settings.viewmatrix, raster_settings.projmatrix)
        return visible

    def forward(self, means3D, means2D, opacities, shs=None, degrees=None, colors_precomp=None, scales=None,
                rotations=None, cov3D_precomp=None, lambda_sh_sparsity=0., *, prune_mask=None, quant=None, return_maps=False,
                raw_params=None, features=None, means2D_abs=None, filter_3D=None, contributions=False, pixel_weights=None):
        """-> (color, radii); with return_maps, (color, radii, invdepth [1,H,W], alpha [1,H,W]), all three differentiable.
        `raw_params`: (features_dc [P,1,3], features_rest [P,C,3], scaling [P,3], rotation [P,4]), the model's leaf tensors, in place
        of shs / scales / rotations (which must then be None, as must cov3D_precomp and quant); with colors_precomp the two
        feature tensors are None.  The kernels apply exp / F.normalize / the concatenation and return the four gradients.
        `features`: [P, F] fp32 on the device, 1 <= F <= 256; the outputs end with the [F, H, W] feature image (each channel composited
        like a colour channel with background 0), differentiable w.r.t. the features and, through alpha, the scene and the camera.
        A feature gradient under the deterministic mode is refused (here when `features` requires grad, else in the backward).
        `means2D_abs`: a [P, 3] tensor (a zeros leaf that requires grad); its gradient is the absolute screen-space gradient
        (sum_p |g_x|, sum_p |g_y|, 0), deterministic with the deterministic mode.  Not together with `features`.
        `filter_3D`: [P] or [P, 1] fp32 on the device, Mip-Splatting's 3D smoothing filter (a constant): the kernels render with
        scales sqrt(s^2 + f^2) and opacities sigmoid(logit) * c3, and chain the gradients through both.  Not with cov3D_precomp.
        `contributions`: the outputs end with _C.Contributions(weight_sum [P], weight_max [P], pixels [P], top_id [H, W]) of this view
        (DESIGN.md §5p), no gradient; `pixel_weights` ([H, W] or [1, H, W] fp32 on the device, clamped to [0, 1]) weights the sum."""
        raster_settings = self.raster_settings
        if pixel_weights is not None:
            if not contributions:
                raise RuntimeError("pixel_weights weights the contribution sums; it needs contributions=True")
            _C.check_pixel_weights(pixel_weights, int(raster_settings.image_height), int(raster_settings.image_width), means3D.device)
        if means2D_abs is not None:
            if features is not None:
                raise RuntimeError("means2D_abs: the absolute screen-space gradient has no feature form; render the features separately")
            if not isinstance(means2D_abs, torch.Tensor) or tuple(means2D_abs.shape) != (int(means3D.shape[0]), 3):
                raise RuntimeError(f"means2D_abs must be a [P, 3] tensor with P = {int(means3D.shape[0])}")
        if features is not None:
            refuse = getattr(features, "requires_grad", False) and torch.is_grad_enabled() and _deterministic(raster_settings)
            # a deterministic feature gradient is refused after the other checks but before the device is looked at
            _C.check_features(features, int(means3D.shape[0]), cuda=not refuse)
            if refuse:
                raise RuntimeError("features: the feature gradient has no deterministic form; detach the features or turn the "
                                   "deterministic mode off")
        if raw_params is not None:
            if quant is not None or any(t is not None for t in (shs, scales, rotations, cov3D_precomp)):
                raise Exception('raw_params replace shs, scales and rotations; leave those, cov3D_precomp and quant None')
            features_dc, features_rest, _, _ = raw_params
            # the SHs are the two feature tensors, and an empty colors_precomp counts as none (the raw op reads it so)
            sh, with_colors = (features_dc, features_rest), colors_precomp is not None and colors_precomp.numel() > 0
        else:
            sh, with_colors = (shs,), colors_precomp is not None
        if quant is None:
            if any(t is not None for t in sh) if with_colors else any(t is None for t in sh):
                raise Exception('Please provide excatly one of either SHs or precomputed colors!')
            if raw_params is None and (((scales is None or rotations is None) and cov3D_precomp is None) or
                                       ((scales is not None or rotations is not None) and cov3D_precomp is not None)):
                raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        empty = torch.Tensor([])
        e = lambda t: empty if t is None else t                                  # absent inputs travel as empty tensors
        return rasterize_gaussians(means3D, means2D, e(shs), degrees, e(colors_precomp), e(opacities), e(scales), e(rotations),
                                   e(cov3D_precomp), raster_settings, lambda_sh_sparsity, prune_mask, quant, return_maps, features,
                                   means2D_abs, raw_params, filter_3D, (pixel_weights,) if contributions else None)
