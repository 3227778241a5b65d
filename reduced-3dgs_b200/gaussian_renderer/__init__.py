"""Drop-in for the reference `gaussian_renderer.render()` (gaussian_renderer/__init__.py:19-148): same signature and
return dict.  `pc` is duck-typed (anything exposing the GaussianModel properties the reference reads: get_xyz,
_opacity, _degrees, get_scaling, get_rotation, get_features, get_covariance, active_sh_degree, max_sh_degree,
per_band_count); `viewpoint_camera` likewise (FoVx, FoVy, image_height, image_width, world_view_transform,
full_proj_transform, camera_center).

Build-defined extras: `pc.prune_mask` (optional tensor) and `pc.quant` (optional QuantScene) are forwarded to the
fused kernels when present; `return_maps=True` adds the inverse-depth and alpha maps of the same pass to the dict
("invdepth", "alpha", [1,H,W] each; differentiable except on the variable-SH inference path).  `pipe.antialiasing` (upstream
3DGS's PipelineParams flag; absent = off, as in reduced-3dgs) renders with the opacity-compensated 2D filter, on every path.
`pipe.fused_activations` (absent = off) renders from the model's raw parameters `_features_dc`, `_features_rest`, `_scaling` and
`_rotation`: exp, F.normalize and the SH concatenation run inside the kernels, which write the four gradients directly
(DESIGN.md §5h).  It needs a GaussianModel-like `pc` whose scaling_activation is torch.exp and rotation_activation
torch.nn.functional.normalize; the variable-SH inference path ignores it.
`features` ([P, F] fp32 on the device, 1 <= F <= 256) adds pkg["features"], the [F, H, W] image of per-Gaussian features composited
over the colour pass with background 0 (semantic features, normals, per-Gaussian statistics such as the SH degree or the opacity).
It is differentiable w.r.t. the features and the scene on every path but the variable-SH inference one, which renders it forward only.
`absgrad=True` adds pkg["viewspace_points_abs"], a zeros leaf [P, 3] whose .grad after loss.backward() is the absolute screen-space
gradient (sum_p |g_x|, sum_p |g_y|, 0) of AbsGS, the split statistic of densify_and_prune(max_grad_abs=...) (DESIGN.md §5m).  It needs
a backward, so the variable-SH inference path refuses it, and it has no feature form.
`pc.filter_3D` (optional, [P] or [P, 1] fp32 on the device; gs_b200.mip.compute_3D_filter sets it) is Mip-Splatting's 3D smoothing
filter, applied in the kernels on every path (DESIGN.md §5o); it does not go with pipe.compute_cov3D_python.
`contributions=True` adds pkg["contributions"], the view's _C.Contributions(weight_sum [P], weight_max [P], pixels [P], top_id [H, W])
of the blending weights w = alpha * T (DESIGN.md §5p), on every path; `pixel_weights` ([H, W] fp32 on the device, clamped to [0, 1])
weights the sum (INTEGRATION.md K: importance pruning, error-weighted scores, per-pixel winners).  No gradient.

A learnable camera needs no argument: when world_view_transform, full_proj_transform or camera_center requires grad, the
rasterizer returns their gradients (the variable-SH inference path stays non-differentiable).  The rasterizer takes
full_proj_transform as its own input, so a camera that builds `full = view @ proj` (and `campos = inverse(view)[3, :3]`) in
torch gets the gradients of all three paths chained back to its parameters by autograd.
"""
import math
import pkgutil

import torch
import torch.nn.functional as F

# When this package shadows the reference's `gaussian_renderer` on sys.path, its sibling modules (network_gui, imported by
# train.py next to `render`) must stay importable: let submodule lookups continue into same-named packages further down the path.
__path__ = pkgutil.extend_path(__path__, __name__)

from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _C
from diff_gaussian_rasterization._C import rasterize_gaussians_variableSH_bands


def eval_sh(deg, sh, dirs):
    """utils/sh_utils.py:57-112 (degrees 0..3), used only by pipe.convert_SHs_python."""
    C0 = 0.28209479177387814
    C1 = 0.4886025119029199
    C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
    C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
          1.445305721320277, -0.5900435899266435]
    result = C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        result = (result - C1 * y * sh[..., 1] + C1 * z * sh[..., 2] - C1 * x * sh[..., 3])
        if deg > 1:
            xx, yy, zz = x * x, y * y, z * z
            xy, yz, xz = x * y, y * z, x * z
            result = (result + C2[0] * xy * sh[..., 4] + C2[1] * yz * sh[..., 5] + C2[2] * (2.0 * zz - xx - yy) * sh[..., 6] +
                      C2[3] * xz * sh[..., 7] + C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                result = (result + C3[0] * y * (3 * xx - yy) * sh[..., 9] + C3[1] * xy * z * sh[..., 10] +
                          C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12] +
                          C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + C3[5] * z * (xx - yy) * sh[..., 14] +
                          C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return result


def _raw_params(pc, pipe, override_color):
    """pipe.fused_activations: the leaf tensors of `pc` for GaussianRasterizer(raw_params=...), after the refusals (nothing runs
    before they are checked)."""
    if getattr(pc, "quant", None) is not None:
        raise RuntimeError("gaussian_renderer.render: pipe.fused_activations needs fp32 parameters; a quantised model is fused already")
    if pipe.compute_cov3D_python or pipe.convert_SHs_python:
        raise RuntimeError("gaussian_renderer.render: pipe.fused_activations replaces pipe.compute_cov3D_python / convert_SHs_python; "
                           "turn those off")
    if getattr(pc, "scaling_activation", None) is not torch.exp:
        raise RuntimeError("gaussian_renderer.render: pipe.fused_activations applies exp to pc._scaling; this model's "
                           "scaling_activation is not torch.exp")
    if getattr(pc, "rotation_activation", None) is not F.normalize:
        raise RuntimeError("gaussian_renderer.render: pipe.fused_activations applies F.normalize to pc._rotation; this model's "
                           "rotation_activation is not torch.nn.functional.normalize")
    if isinstance(pc._features_rest, (list, tuple)) or isinstance(pc._features_dc, (list, tuple)):
        raise RuntimeError("gaussian_renderer.render: pipe.fused_activations does not take the packed variable-SH layout")
    if override_color is not None:
        return (None, None, pc._scaling, pc._rotation)
    return (pc._features_dc, pc._features_rest, pc._scaling, pc._rotation)


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None,
           lambda_sh_sparsity=0., measure_fps=False, variable_sh_bands=False, return_maps=False, features=None, absgrad=False,
           contributions=False, pixel_weights=None):
    """
    Render the scene.

    Background tensor (bg_color) must be on GPU!
    """
    # Create zero tensor. We will use it to make pytorch return gradients of the 2D (screen-space) means.
    # (The reference adds 0 to make it a non-leaf and then calls retain_grad(), GR:27-31; a leaf keeps its .grad by itself and
    # saves an elementwise pass over [P,3].)
    if absgrad and variable_sh_bands:
        raise RuntimeError("gaussian_renderer.render: absgrad needs the backward; the variable-SH inference path renders forward only")
    if absgrad and features is not None:
        raise RuntimeError("gaussian_renderer.render: absgrad has no feature form; render the features in a call without absgrad")
    if pixel_weights is not None:
        if not contributions:
            raise RuntimeError("gaussian_renderer.render: pixel_weights weights the contribution sums; it needs contributions=True")
        _C.check_pixel_weights(pixel_weights, int(viewpoint_camera.image_height), int(viewpoint_camera.image_width), pc.get_xyz.device)
    filter_3D = getattr(pc, "filter_3D", None)
    if filter_3D is not None and pipe.compute_cov3D_python:
        raise RuntimeError("gaussian_renderer.render: pc.filter_3D filters the scales inside the kernels; it does not go with "
                           "pipe.compute_cov3D_python")
    fused = bool(getattr(pipe, "fused_activations", False)) and not variable_sh_bands
    raw_params = _raw_params(pc, pipe, override_color) if fused else None
    screenspace_points = torch.zeros_like(pc.get_xyz, dtype=pc.get_xyz.dtype, requires_grad=True, device=pc.get_xyz.device)
    screenspace_points_abs = None
    if absgrad:
        screenspace_points_abs = torch.zeros_like(pc.get_xyz, dtype=pc.get_xyz.dtype, requires_grad=True, device=pc.get_xyz.device)

    tanfovx = math.tan(viewpoint_camera.FoVx * 0.5)
    tanfovy = math.tan(viewpoint_camera.FoVy * 0.5)
    raster_settings = GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height), image_width=int(viewpoint_camera.image_width),
        tanfovx=tanfovx, tanfovy=tanfovy, bg=bg_color, scale_modifier=scaling_modifier,
        viewmatrix=viewpoint_camera.world_view_transform, projmatrix=viewpoint_camera.full_proj_transform,
        sh_degree=pc.active_sh_degree, campos=viewpoint_camera.camera_center, prefiltered=False, debug=pipe.debug,
        antialiasing=getattr(pipe, "antialiasing", False))
    rasterizer = GaussianRasterizer(raster_settings=raster_settings)

    means3D = pc.get_xyz
    means2D = screenspace_points
    opacity = pc._opacity
    degrees = pc._degrees
    prune_mask = getattr(pc, "prune_mask", None)
    quant = getattr(pc, "quant", None)

    scales = rotations = cov3D_precomp = None
    shs = colors_precomp = None
    if raw_params is not None:
        colors_precomp = override_color
    elif quant is None:
        if pipe.compute_cov3D_python:
            cov3D_precomp = pc.get_covariance(scaling_modifier)
        else:
            scales = pc.get_scaling
            rotations = pc.get_rotation
        if override_color is None:
            if pipe.convert_SHs_python:
                shs_view = pc.get_features.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
                dir_pp = (pc.get_xyz - viewpoint_camera.camera_center.repeat(pc.get_features.shape[0], 1))
                dir_pp_normalized = dir_pp / dir_pp.norm(dim=1, keepdim=True)
                sh2rgb = eval_sh(pc.active_sh_degree, shs_view, dir_pp_normalized)
                colors_precomp = torch.clamp_min(sh2rgb + 0.5, 0.0)
            else:
                shs = pc.get_features
                if variable_sh_bands:
                    shs = torch.cat([tensor.flatten() for tensor in shs])
        else:
            colors_precomp = override_color
    else:
        # quantised model: attributes are codebook ids, de-quantised inside the kernels.  override_color (depth / debug renders of
        # the reference's callers) replaces the SH colours there too; the PyTorch-side SH / covariance paths have nothing to work on.
        if pipe.convert_SHs_python or pipe.compute_cov3D_python:
            raise RuntimeError("gaussian_renderer.render: pipe.convert_SHs_python / compute_cov3D_python need fp32 attributes; "
                               "de-quantise the model first (QuantScene.dequantise()) or leave both options off")
        if override_color is not None:
            colors_precomp = override_color

    fps = 0
    if measure_fps:
        start_timer = torch.cuda.Event(enable_timing=True)
        end_timer = torch.cuda.Event(enable_timing=True)
        start_timer.record()
    if variable_sh_bands and quant is None:
        per_band_count = torch.tensor(pc.per_band_count, dtype=torch.int)
        cumsum_count = torch.cumsum(per_band_count, dim=0).to(dtype=torch.int)
        coeffs_num = torch.tensor([i * i for i in range(1, len(pc.per_band_count) + 1)], dtype=torch.int)
        empty = torch.Tensor([])
        out = rasterize_gaussians_variableSH_bands(
            raster_settings.bg, means3D, empty, opacity, scales, rotations, raster_settings.scale_modifier, empty,
            raster_settings.viewmatrix, raster_settings.projmatrix, raster_settings.tanfovx, raster_settings.tanfovy,
            raster_settings.image_height, raster_settings.image_width, shs, per_band_count, cumsum_count, coeffs_num,
            degrees, raster_settings.campos, raster_settings.prefiltered, raster_settings.debug, prune_mask=prune_mask,
            return_maps=return_maps, antialiasing=raster_settings.antialiasing, **({} if features is None else dict(features=features)),
            **({} if filter_3D is None else dict(filter_3D=filter_3D)))
        rendered_image, radii = out[1], out[2]
        maps = out[6:8] if return_maps else ()
        feature_image = out[6 + 2 * return_maps] if features is not None else None
        contrib = None
        if contributions:
            contrib = _C.contributions(out[3], out[4], out[5], out[0], raster_settings.image_width, raster_settings.image_height,
                                       means3D.shape[0], pixel_weights=pixel_weights)
    else:
        out = rasterizer(
            means3D=means3D, means2D=means2D, shs=shs, degrees=degrees, colors_precomp=colors_precomp, opacities=opacity,
            scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp, lambda_sh_sparsity=lambda_sh_sparsity,
            prune_mask=prune_mask, quant=quant, return_maps=return_maps, raw_params=raw_params, features=features,
            **({} if screenspace_points_abs is None else dict(means2D_abs=screenspace_points_abs)),
            **({} if filter_3D is None else dict(filter_3D=filter_3D)),
            **({} if not contributions else dict(contributions=True, pixel_weights=pixel_weights)))
        rendered_image, radii = out[0], out[1]
        maps = out[2:4] if return_maps else ()
        feature_image = out[2 + 2 * return_maps] if features is not None else None
        contrib = out[-1] if contributions else None
    if measure_fps:
        end_timer.record()
        torch.cuda.synchronize()
        fps = 1 / (start_timer.elapsed_time(end_timer))

    # Those Gaussians that were frustum culled or had a radius of 0 were not visible.
    # They will be excluded from value updates used in the splitting criteria.
    pkg = {"render": rendered_image,
           "viewspace_points": screenspace_points,
           "visibility_filter": radii > 0,
           "radii": radii,
           "FPS": fps}
    if return_maps:
        pkg["invdepth"], pkg["alpha"] = maps
    if features is not None:
        pkg["features"] = feature_image
    if absgrad:
        pkg["viewspace_points_abs"] = screenspace_points_abs
    if contributions:
        pkg["contributions"] = contrib
    return pkg
