"""Drop-in replacement for the reference Python package `diff_gaussian_rasterization`
(submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py): same
GaussianRasterizationSettings (:169-181), GaussianRasterizer (:183-234), rasterize_gaussians (:21-46) and
_RasterizeGaussians autograd op (:48-167), backed by the H100-native kernels through `_C`.

Differences, all additive: GaussianRasterizer.forward takes keyword-only `prune_mask` and `quant`
(fused resolution-aware prune mask / codebook de-quantisation, SURVEY §8(b)) and `return_maps` (differentiable inverse-depth
and alpha maps from the same pass: (color, radii, invdepth, alpha)); a raster_settings.viewmatrix / projmatrix / campos
that requires grad receives its gradient (gsb_backward_camera), where the reference silently treats the camera as a
constant; GaussianRasterizationSettings takes upstream 3DGS's trailing `antialiasing` argument (default False; the tuple keeps the
reference's 12 fields), which turns on the opacity-compensated 2D filter in the forward and the backward; the
forward no longer forces
debug=True (reference :85 hard-wires a device sync after every stage); gradients are allocated uninitialised
because the kernels write every element.  GaussianRasterizer.forward also takes keyword-only `raw_params`, the model's leaf
tensors (features_dc, features_rest, scaling, rotation) in place of shs / scales / rotations: exp, F.normalize and the SH
concatenation then run inside the kernels, and the gradients of the four tensors are the kernels' own outputs
(_RasterizeGaussiansRaw).  GaussianRasterizationSettings' keyword-only `deterministic` (default: torch's deterministic-algorithms
flag) selects the backward that sums each Gaussian's gradients in a fixed order (the same bytes on every run).
GaussianRasterizer.forward's keyword-only `features` ([P, F] fp32, 1 <= F <= 256) appends the [F, H, W] image of per-Gaussian
features composited over the colour pass with background 0; its gradient reaches the features and, through alpha, everything the
colour gradient reaches.  The feature gradient has no deterministic form: it is refused when the deterministic mode is on.
GaussianRasterizer.forward's keyword-only `means2D_abs` (a [P, 3] tensor that requires grad, e.g. a zeros leaf) receives as its
gradient the absolute screen-space gradient (sum_p |g_x|, sum_p |g_y|, 0) of AbsGS (gsb_backward_absgrad), the densification
statistic whose per-pixel terms cannot cancel; it has no feature form.
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


def _apply(op, raster_settings, *args, features=None, means2D_abs=None):
    camera = (raster_settings.viewmatrix, raster_settings.projmatrix, raster_settings.campos)
    feat = () if features is None else (features,)
    if means2D_abs is not None:
        # means2D_abs is the op's last input, after the features' slot (None when absent)
        feat = (features, means2D_abs)
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in camera):
        # a learnable camera: the three tensors become inputs of the autograd op so that their gradients have a destination
        return op.apply(*args, *camera, *feat)
    # the features, when given, are the op's last input (after three absent camera slots)
    return op.apply(*args, *((None,) * 3 + feat if feat else ()))


def _forward(ctx, args, raster_settings, lambda_sh_sparsity, prune_mask, return_maps, camera, features=None, means2D_abs=None, **kw):
    """The forward both ops share: the _C call and the ctx state their backwards read.  `camera` is (viewmatrix, projmatrix,
    campos), raster_settings' own tensors, passed again as inputs only when the camera is learnable, else (None, None, None).
    -> (_C.rasterize_gaussians' tuple, the op's outputs: (color, radii) or, with return_maps, (color, radii, invdepth, alpha);
    with `features` the feature image [F, H, W] comes last)."""
    ctx.camera_meta = None if camera[0] is None else [(t.shape, t.dtype) for t in camera]
    ctx.return_maps, ctx.has_features, ctx.has_abs = return_maps, features is not None, means2D_abs is not None
    kw.update(prune_mask=prune_mask, return_maps=return_maps, antialiasing=raster_settings.antialiasing)
    if features is not None:
        kw.update(features=features)
    out = _call(_C.rasterize_gaussians, args, kw,
                "snapshot_fw.dump", "\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
    ctx.raster_settings = raster_settings
    ctx.num_rendered = out[0]
    ctx.lambda_sh_sparsity = lambda_sh_sparsity
    ctx.prune_mask = prune_mask
    ctx.mark_non_differentiable(out[2])
    feat = (out[-1],) if features is not None else ()
    if return_maps or features is not None:
        # a loss on some outputs only: the others' gradients arrive as None and reach the kernels as NULL (zero), and a feature
        # image without a gradient leaves the backward exactly the call without features
        ctx.set_materialize_grads(False)
    if return_maps:
        return out, (out[1], out[2], out[6], out[7]) + feat
    return out, (out[1], out[2]) + feat


def _split_grads(ctx, grads):
    """The incoming gradients after (color, radii) -> (grad_invdepth, grad_alpha, grad_features), None where absent."""
    grads = list(grads)
    maps = (grads.pop(0), grads.pop(0)) if ctx.return_maps else (None, None)
    return maps + (grads.pop(0) if ctx.has_features else None,)


def _deterministic(raster_settings):
    """The settings' `deterministic`: an explicit bool wins; None follows torch.are_deterministic_algorithms_enabled(), read when
    the backward runs."""
    d = getattr(raster_settings, "deterministic", None)
    return torch.are_deterministic_algorithms_enabled() if d is None else bool(d)


def _backward(ctx, grad_out_color, grad_invdepth, grad_alpha, means3D, radii, colors_precomp, scales, rotations, cov3Ds_precomp,
              sh, degrees, geomBuffer, binningBuffer, imgBuffer, features=None, grad_features=None, **kw):
    """The backward both ops share: the _C call from the saved state.  -> (its gradient tuple, the gradients of the camera
    inputs: () for a constant camera, else one per tensor, None where not needed, dL_dfeatures or None)."""
    rs = ctx.raster_settings
    if grad_out_color is None:
        grad_out_color = torch.zeros((3, rs.image_height, rs.image_width), dtype=torch.float32, device=means3D.device)
    # the camera tensors are the op's last three inputs when it has them (followed by the features when given, and by the
    # features' slot and means2D_abs with absgrad)
    n = len(ctx.needs_input_grad) - (2 if ctx.has_abs else 1 if ctx.has_features else 0)
    camera_need = ctx.needs_input_grad[n - 3:n] if ctx.camera_meta is not None else (False, False, False)
    args = (rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix, rs.projmatrix,
            rs.tanfovx, rs.tanfovy, grad_out_color, sh, degrees, rs.campos, geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer,
            ctx.lambda_sh_sparsity, rs.debug)
    kw.update(prune_mask=ctx.prune_mask, dL_dinvdepth=grad_invdepth, dL_dalpha=grad_alpha, camera_grads=any(camera_need),
              antialiasing=rs.antialiasing)
    if _deterministic(rs):
        kw.update(deterministic=True)
    if grad_features is not None:
        kw.update(features=features, dL_dfeatures_out=grad_features)
    dabs = None
    if ctx.has_abs:
        dabs = torch.empty((means3D.shape[0], 3), dtype=torch.float32, device=means3D.device)
        kw.update(absgrad_out=dabs)
    g = _call(_C.rasterize_gaussians_backward, args, kw,
              "snapshot_bw.dump", "\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
    dfeat = None
    if grad_features is not None:
        g, dfeat = g[:-1], g[-1]                                       # dL_dfeatures comes last
    ctx.grad_abs = dabs
    if ctx.camera_meta is None:
        # the features' gradient (and means2D_abs's) follows three absent camera slots
        return g, (None,) * 3 if ctx.has_features or ctx.has_abs else (), dfeat
    # with camera_grads the tuple ends with (dL_dviewmatrix, dL_dprojmatrix, dL_dcampos)
    return g, tuple(gc.reshape(shape).to(dtype) if n else None
                    for gc, n, (shape, dtype) in zip(g[-3:] if any(camera_need) else (None,) * 3, camera_need, ctx.camera_meta)), dfeat


def _tail(ctx, grad_feat):
    """The gradients of the op's inputs after the camera: the features (when given, or their absent slot before means2D_abs) and
    means2D_abs, whose gradient is the absolute screen-space gradient."""
    need = ctx.needs_input_grad
    if ctx.has_abs:
        return (grad_feat if ctx.has_features and need[-2] else None, ctx.grad_abs if need[-1] else None)
    return (grad_feat if need[-1] else None,) if ctx.has_features else ()


def rasterize_gaussians(means3D, means2D, sh, degrees, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings, lambda_sh_sparsity, prune_mask=None, quant=None, return_maps=False, features=None,
                        means2D_abs=None):
    return _apply(_RasterizeGaussians, raster_settings, means3D, means2D, sh, degrees, colors_precomp, opacities, scales, rotations,
                  cov3Ds_precomp, raster_settings, lambda_sh_sparsity, prune_mask, quant, return_maps, features=features,
                  means2D_abs=means2D_abs)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, degrees, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, lambda_sh_sparsity, prune_mask=None, quant=None, return_maps=False, viewmatrix=None,
                projmatrix=None, campos=None, features=None, means2D_abs=None):
        args = (raster_settings.bg, means3D, colors_precomp, opacities, scales, rotations, raster_settings.scale_modifier,
                cov3Ds_precomp, raster_settings.viewmatrix, raster_settings.projmatrix, raster_settings.tanfovx,
                raster_settings.tanfovy, raster_settings.image_height, raster_settings.image_width, sh, degrees,
                raster_settings.campos, raster_settings.prefiltered, raster_settings.debug)
        out, outputs = _forward(ctx, args, raster_settings, lambda_sh_sparsity, prune_mask, return_maps, (viewmatrix, projmatrix, campos),
                                features, means2D_abs, quant=quant)
        ctx.quant = quant
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, out[2], sh, out[3], out[4], out[5], degrees,
                              features)
        return outputs

    @staticmethod
    def backward(ctx, grad_out_color, _, *grads):
        grad_invdepth, grad_alpha, grad_features = _split_grads(ctx, grads)
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer, imgBuffer,
         degrees, features) = ctx.saved_tensors
        g, grad_camera, grad_feat = _backward(ctx, grad_out_color, grad_invdepth, grad_alpha, means3D, radii, colors_precomp, scales,
                                              rotations, cov3Ds_precomp, sh, degrees, geomBuffer, binningBuffer, imgBuffer, features,
                                              grad_features, quant=ctx.quant)
        (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh, grad_scales,
         grad_rotations) = g[:8]
        if ctx.quant is not None:
            # inputs were id planes: the per-Gaussian attribute gradients have no autograd destination; expose them with the
            # semantics of `.grad`: they accumulate over backward calls until the caller resets `quant.grads = None`
            new = dict(sh=grad_sh, opacity=grad_opacities, scales=grad_scales, rotations=grad_rotations)
            old = getattr(ctx.quant, "grads", None)
            if old:
                for k, t in new.items():
                    old[k].add_(t)
            else:
                ctx.quant.grads = new
        need = ctx.needs_input_grad
        return (grad_means3D, grad_means2D, grad_sh if need[2] else None, None,
                grad_colors_precomp if need[4] else None, grad_opacities if need[5] else None,
                grad_scales if need[6] else None, grad_rotations if need[7] else None,
                grad_cov3Ds_precomp if need[8] else None, None, None, None, None, None) + grad_camera + _tail(ctx, grad_feat)


def rasterize_gaussians_raw(means3D, means2D, features_dc, features_rest, degrees, colors_precomp, opacities, scaling, rotation,
                            raster_settings, lambda_sh_sparsity, prune_mask=None, return_maps=False, features=None, means2D_abs=None):
    """rasterize_gaussians on the model's raw parameters (see _RasterizeGaussiansRaw)."""
    return _apply(_RasterizeGaussiansRaw, raster_settings, means3D, means2D, features_dc, features_rest, degrees, colors_precomp,
                  opacities, scaling, rotation, raster_settings, lambda_sh_sparsity, prune_mask, return_maps, features=features,
                  means2D_abs=means2D_abs)


class _RasterizeGaussiansRaw(torch.autograd.Function):
    """_RasterizeGaussians with the model's leaf tensors as inputs: features_dc [P,1,3], features_rest [P,C,3] (empty with
    colors_precomp), scaling [P,3] (log-scales), rotation [P,4] (unnormalised).  The kernels apply get_features / get_scaling /
    get_rotation themselves and return the gradients of these four tensors directly, so the graph holds no Cat / Exp / Div node
    and no [P,16,3] copy or gradient exists.  Outputs, camera handling and `return_maps` as in _RasterizeGaussians."""

    @staticmethod
    def forward(ctx, means3D, means2D, features_dc, features_rest, degrees, colors_precomp, opacities, scaling, rotation,
                raster_settings, lambda_sh_sparsity, prune_mask=None, return_maps=False, viewmatrix=None, projmatrix=None, campos=None,
                features=None, means2D_abs=None):
        empty = torch.Tensor([])
        with_colors = colors_precomp.numel() > 0
        raw = (None, None, scaling, rotation) if with_colors else (features_dc, features_rest, scaling, rotation)
        args = (raster_settings.bg, means3D, colors_precomp, opacities, empty, empty, raster_settings.scale_modifier, empty,
                raster_settings.viewmatrix, raster_settings.projmatrix, raster_settings.tanfovx, raster_settings.tanfovy,
                raster_settings.image_height, raster_settings.image_width, empty, degrees, raster_settings.campos,
                raster_settings.prefiltered, raster_settings.debug)
        out, outputs = _forward(ctx, args, raster_settings, lambda_sh_sparsity, prune_mask, return_maps, (viewmatrix, projmatrix, campos),
                                features, means2D_abs, raw=raw)
        ctx.with_colors = with_colors
        ctx.save_for_backward(colors_precomp, means3D, features_dc, features_rest, scaling, rotation, out[2], out[3], out[4], out[5],
                              degrees, features)
        return outputs

    @staticmethod
    def backward(ctx, grad_out_color, _, *grads):
        grad_invdepth, grad_alpha, grad_features = _split_grads(ctx, grads)
        (colors_precomp, means3D, features_dc, features_rest, scaling, rotation, radii, geomBuffer, binningBuffer, imgBuffer,
         degrees, features) = ctx.saved_tensors
        empty = torch.Tensor([])
        raw = (None, None, scaling, rotation) if ctx.with_colors else (features_dc, features_rest, scaling, rotation)
        g, grad_camera, grad_feat = _backward(ctx, grad_out_color, grad_invdepth, grad_alpha, means3D, radii, colors_precomp, empty, empty,
                                              empty, empty, degrees, geomBuffer, binningBuffer, imgBuffer, features, grad_features, raw=raw)
        (grad_means2D, grad_colors, grad_opacities, grad_means3D, _, grad_dc, grad_rest, grad_scaling, grad_rotation) = g[:9]
        need = ctx.needs_input_grad
        return (grad_means3D, grad_means2D, grad_dc if need[2] else None, grad_rest if need[3] else None, None,
                grad_colors if need[5] else None, grad_opacities if need[6] else None, grad_scaling if need[7] else None,
                grad_rotation if need[8] else None, None, None, None, None) + grad_camera + _tail(ctx, grad_feat)


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
                raw_params=None, features=None, means2D_abs=None):
        """-> (color, radii); with return_maps, (color, radii, invdepth [1,H,W], alpha [1,H,W]), all three differentiable.
        `raw_params`: (features_dc [P,1,3], features_rest [P,C,3], scaling [P,3], rotation [P,4]), the model's leaf tensors, in place
        of shs / scales / rotations (which must then be None, as must cov3D_precomp and quant); with colors_precomp the two
        feature tensors are None.  The kernels apply exp / F.normalize / the concatenation and return the four gradients.
        `features`: [P, F] fp32 on the device, 1 <= F <= 256; the outputs end with the [F, H, W] feature image (each channel composited
        like a colour channel with background 0), differentiable w.r.t. the features and, through alpha, the scene and the camera.
        A feature gradient under the deterministic mode is refused (here when `features` requires grad, else in the backward).
        `means2D_abs`: a [P, 3] tensor (a zeros leaf that requires grad); its gradient is the absolute screen-space gradient
        (sum_p |g_x|, sum_p |g_y|, 0), deterministic with the deterministic mode.  Not together with `features`."""
        raster_settings = self.raster_settings
        if means2D_abs is not None:
            if features is not None:
                raise RuntimeError("means2D_abs: the absolute screen-space gradient has no feature form; render the features separately")
            if not isinstance(means2D_abs, torch.Tensor) or tuple(means2D_abs.shape) != (int(means3D.shape[0]), 3):
                raise RuntimeError(f"means2D_abs must be a [P, 3] tensor with P = {int(means3D.shape[0])}")
        if features is not None:
            _C.check_features(features, int(means3D.shape[0]), cuda=False)
            if features.requires_grad and torch.is_grad_enabled() and _deterministic(raster_settings):
                raise RuntimeError("features: the feature gradient has no deterministic form; detach the features or turn the "
                                   "deterministic mode off")
            _C.check_features(features, int(means3D.shape[0]))
        if raw_params is not None:
            if quant is not None or any(t is not None for t in (shs, scales, rotations, cov3D_precomp)):
                raise Exception('raw_params replace shs, scales and rotations; leave those, cov3D_precomp and quant None')
            features_dc, features_rest, scaling, rotation = raw_params
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
        if raw_params is not None:
            return rasterize_gaussians_raw(means3D, means2D, e(features_dc), e(features_rest), degrees, e(colors_precomp), e(opacities),
                                           scaling, rotation, raster_settings, lambda_sh_sparsity, prune_mask, return_maps, features,
                                           means2D_abs)
        return rasterize_gaussians(means3D, means2D, e(shs), degrees, e(colors_precomp), e(opacities), e(scales), e(rotations),
                                   e(cov3D_precomp), raster_settings, lambda_sh_sparsity, prune_mask, quant, return_maps, features,
                                   means2D_abs)
