"""Drop-in for the reference's pybind module `diff_gaussian_rasterization._C` (ext.cpp:17-20), re-hosted on the
C ABI of include/gs_b200.h through ctypes.  Same function names, positional signatures, return tuples and error
behaviour as rasterize_points.h:18-93; tensors in, torch.Tensors out.

Build-defined extensions (keyword-only, SURVEY §8(b)): `prune_mask` (u8/bool [P], 1 = pruned), `quant`
(a gs_b200.synth.QuantScene-like object with u8 id planes + [20,256] centres) and `debug_out` (dict that
receives the forward intermediates in the reference's GeometryState layouts).  `return_maps` (forward) also renders the
inverse-depth and alpha maps in the same pass; `dL_dinvdepth` / `dL_dalpha` (backward) take their gradients.
`camera_grads` (backward) also returns the gradients w.r.t. viewmatrix, projmatrix and campos.  `antialiasing` (forward and
backward, the same value for both) scales each Gaussian's opacity so that the 0.3 px^2 dilation no longer inflates sub-pixel splats.
`raw` (forward and backward) takes the model's leaf parameters (features_dc, features_rest, scaling, rotation) in place of sh,
scales and rotations, and applies exp / F.normalize / the SH concatenation inside the kernels.  `deterministic` (backward) sums
the per-Gaussian gradients in a fixed order: the same bytes on every run.  `calculate_colours_variance` and `kmeans_cuda` take the
same keyword (None: torch's deterministic-algorithms flag) for their statistics and centre sums (the forward request's
`deterministic`, gsb_kmeans's `deterministic`).  `features` (forward, also of the variable-SH entry point) composites a [P, F] fp32
tensor of per-Gaussian features over the pairs of the colour image, with background 0, and appends the [F, H, W] image to the
outputs; the backward's `features` and `dL_dfeatures_out` add that image's gradient and append dL_dfeatures [P, F].
`absgrad_out` (backward) takes a [P, 3] fp32 tensor that receives the absolute screen-space gradient.
`filter_3D` (forward, also of the variable-SH entry point, and backward) takes Mip-Splatting's 3D smoothing filter, [P] or [P, 1]
fp32 on the device (gs_b200.mip.compute_3D_filter): the scales become sqrt(s^2 + f^2) and the opacity sigmoid(logit) * c3 inside the
kernels (DESIGN.md §5o).  Its backward also needs the opacity logits, `opacity` (not with `quant`, whose ids are read).

Each keyword is one field of the library's request (GsbForwardRequest / GsbBackwardRequest): the forward and the backward make one
library call, gsb_forward / gsb_backward, whatever their keywords.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple

import torch

from gs_b200 import lib as _lib
from gs_b200.lib import (GsbBackwardRequest, GsbCamera, GsbDebug, GsbFeatures, GsbForwardRequest, GsbGrads, GsbQuant, GsbRawGrads,
                         GsbRawParams, GsbScene, BlobAllocator, f32, on_device, ptr)

RAW_REST_COEFFS = (0, 3, 8, 15)     # _features_rest widths of max SH degree 0..3


def _carve_f32(device, shapes):
    """The gradient outputs as views of ONE allocation (each starting on a 256-byte boundary).  Eight separate mid-size
    tensors per backward (1-100 MB, different sizes) fragment the caching allocator's split blocks and provoke a cudaMalloc
    inside the training loop every now and then (measured: 1-90 ms); one request of a constant size is always reused."""
    sizes = [int(math.prod(sh)) for sh in shapes]
    offs, total = [], 0
    for n in sizes:
        offs.append(total)
        total += (n + 63) // 64 * 64
    flat = torch.empty(max(total, 1), dtype=torch.float32, device=device)
    return [flat[o:o + n].view(sh) for o, n, sh in zip(offs, sizes, shapes)]


def _device_of(means3D: torch.Tensor) -> torch.device:
    if not means3D.is_cuda:
        raise RuntimeError("gs_b200: means3D must live on a CUDA device (no CPU path exists)")
    d = means3D.device
    return d if d.index is not None else torch.device("cuda", torch.cuda.current_device())


def _camera(device, bg, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, H, W, prefiltered, keep):
    bg, viewmatrix, projmatrix, campos = (f32(bg, device), f32(viewmatrix, device), f32(projmatrix, device),
                                           f32(campos, device))
    keep += [bg, viewmatrix, projmatrix, campos]
    return GsbCamera(int(W), int(H), float(tan_fovx), float(tan_fovy), ptr(viewmatrix), ptr(projmatrix), ptr(campos),
                     ptr(bg), int(bool(prefiltered)))


def _quant_struct(quant, device, keep):
    def u8(t):
        t = t.to(device=device, dtype=torch.uint8).contiguous()
        keep.append(t)
        return t.data_ptr()
    centers = f32(quant.centers, device)
    keep.append(centers)
    q = GsbQuant(u8(quant.ids_dc), u8(quant.ids_rest), u8(quant.ids_opacity), u8(quant.ids_scaling), u8(quant.ids_rot),
                 centers.data_ptr())
    keep.append(q)
    return C.pointer(q)


def check_features(features, P, cuda=True):
    """The checks of a `features` argument, made before anything runs: a [P, F] float32 tensor with 1 <= F <= FEATURES_MAX, on a CUDA
    device unless `cuda` is False (then the caller checks the device later).  -> F."""
    if not isinstance(features, torch.Tensor):
        raise RuntimeError(f"features must be a [P, F] tensor, got {type(features).__name__}")
    if features.dim() != 2 or int(features.shape[0]) != P:
        raise RuntimeError(f"features must have shape [P, F] with P = {P} Gaussians, got {tuple(features.shape)}")
    F = int(features.shape[1])
    if not 1 <= F <= _lib.FEATURES_MAX:
        raise RuntimeError(f"features has F = {F} channels; 1..{_lib.FEATURES_MAX} are supported")
    if features.dtype != torch.float32:
        raise RuntimeError(f"features must be float32, got {features.dtype}")
    if cuda and not features.is_cuda:
        raise RuntimeError("features must live on a CUDA device (no CPU path exists)")
    return F


def check_absgrad_out(absgrad_out, P, accumulate_into=None, features=None, dL_dfeatures_out=None):
    """The checks of the backward's `absgrad_out`, made before anything runs (the device is checked against means3D's later)."""
    if accumulate_into is not None:
        raise RuntimeError("absgrad: the absolute screen-space gradient has no accumulate_into form (view-batch accumulation)")
    if features is not None or dL_dfeatures_out is not None:
        raise RuntimeError("absgrad: the feature backward is a separate pass, so the absolute screen-space gradient has no feature form")
    if not isinstance(absgrad_out, torch.Tensor):
        raise RuntimeError(f"absgrad_out must be a [P, 3] tensor, got {type(absgrad_out).__name__}")
    if tuple(absgrad_out.shape) != (P, 3):
        raise RuntimeError(f"absgrad_out must have shape [P, 3] with P = {P} Gaussians, got {tuple(absgrad_out.shape)}")
    if absgrad_out.dtype != torch.float32:
        raise RuntimeError(f"absgrad_out must be float32, got {absgrad_out.dtype}")
    if not absgrad_out.is_contiguous():
        raise RuntimeError("absgrad_out must be contiguous (it is written in place)")
    if not absgrad_out.is_cuda:
        raise RuntimeError("absgrad_out must live on a CUDA device (no CPU path exists)")


def check_filter_3d(filter_3D, P):
    """The checks of a `filter_3D` argument, made before anything runs: a [P] or [P, 1] float32 tensor on a CUDA device."""
    if not isinstance(filter_3D, torch.Tensor):
        raise RuntimeError(f"filter_3D must be a [P] or [P, 1] tensor, got {type(filter_3D).__name__}")
    if tuple(filter_3D.shape) not in ((P,), (P, 1)):
        raise RuntimeError(f"filter_3D must have shape [P] or [P, 1] with P = {P} Gaussians, got {tuple(filter_3D.shape)}")
    if filter_3D.dtype != torch.float32:
        raise RuntimeError(f"filter_3D must be float32, got {filter_3D.dtype}")
    if not filter_3D.is_cuda:
        raise RuntimeError("filter_3D must live on a CUDA device (no CPU path exists)")


def _present(t):
    return t is not None and not (isinstance(t, torch.Tensor) and t.numel() == 0)


def _raw_struct(raw, device, P, want_sh, sh, scales, rotations, cov3D_precomp, quant):
    """raw = (features_dc [P,1,3], features_rest [P,C,3], scaling [P,3], rotation [P,4]): the model's leaf tensors, passed by
    pointer as they are (no cast), so each must already be a contiguous fp32 tensor on the device; only a rotation that does not
    start on a 16-byte boundary is copied (lib.aligned16: the kernels read its rows as one float4).  Everything is checked before
    anything is launched.  -> (GsbRawParams, C, the rotation tensor handed over, to keep alive for the call)."""
    if quant is not None:
        raise RuntimeError("raw parameters: a quantised model has no raw fp32 parameters (its kernels activate the codebooks already)")
    if any(_present(t) for t in (sh, scales, rotations, cov3D_precomp)):
        raise RuntimeError("raw parameters replace sh, scales and rotations; give those (and cov3D_precomp) empty")
    if not isinstance(raw, (tuple, list)) or len(raw) != 4:
        raise RuntimeError("raw parameters: expected (features_dc, features_rest, scaling, rotation)")
    dc, rest, scaling, rotation = raw
    if isinstance(rest, (list, tuple)) or isinstance(dc, (list, tuple)):
        raise RuntimeError("raw parameters: the packed variable-SH layout (a list of per-degree tensors) is not supported")

    checked = []

    def check(name, t, shape):
        if not isinstance(t, torch.Tensor):
            raise RuntimeError(f"raw parameters: {name} must be a tensor, got {type(t).__name__}")
        if t.dtype != torch.float32:
            raise RuntimeError(f"raw parameters: {name} must be float32, got {t.dtype}")
        if not t.is_contiguous():
            raise RuntimeError(f"raw parameters: {name} must be contiguous (it is read in place)")
        if tuple(t.shape) != tuple(shape):
            raise RuntimeError(f"raw parameters: {name} must have shape {tuple(shape)}, got {tuple(t.shape)}")
        checked.append((name, t))

    check("scaling", scaling, (P, 3))
    check("rotation", rotation, (P, 4))
    C_rest = 0
    if want_sh:
        check("features_dc", dc, (P, 1, 3))
        if not isinstance(rest, torch.Tensor) or rest.dim() != 3 or rest.shape[2] != 3:
            raise RuntimeError("raw parameters: features_rest must be a [P, C, 3] tensor")
        C_rest = int(rest.shape[1])
        if C_rest not in RAW_REST_COEFFS:
            raise RuntimeError(f"raw parameters: features_rest has C = {C_rest} coefficients; only {RAW_REST_COEFFS} exist")
        if int(rest.shape[0]) != P:
            raise RuntimeError(f"raw parameters: features_dc has {P} rows but features_rest {int(rest.shape[0])}")
        check("features_rest", rest, (P, C_rest, 3))
    elif _present(dc) or _present(rest):
        raise RuntimeError("raw parameters: SH features given together with colors_precomp")
    for name, t in checked:
        if not t.is_cuda or t.device != device:
            raise RuntimeError(f"raw parameters: {name} must live on {device}, got {t.device}")
    rotation = _lib.aligned16(rotation)
    return GsbRawParams(ptr(dc) if want_sh else None, ptr(rest) if want_sh else None, C_rest, ptr(scaling), ptr(rotation)), C_rest, rotation


def _scene(device, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, sh, degrees, keep,
           packed_counts=None, prune_mask=None, quant=None, filter_3D=None):
    means3D = f32(means3D, device)
    P = int(means3D.shape[0]) if means3D is not None else 0
    colors, opacity, scales, rotations = f32(colors, device), f32(opacity, device), f32(scales, device), f32(rotations, device)
    cov3D_precomp, sh = f32(cov3D_precomp, device), f32(sh, device)
    if degrees is not None and degrees.numel() > 0:
        degrees = degrees.to(device=device, dtype=torch.int32).contiguous()
    else:
        degrees = None
    if prune_mask is not None:
        prune_mask = prune_mask.to(device=device, dtype=torch.uint8).contiguous()
    if filter_3D is not None:
        if filter_3D.device != device:
            raise RuntimeError(f"filter_3D must live on {device}, got {filter_3D.device}")
        filter_3D = filter_3D.detach().reshape(-1).contiguous()
    keep += [means3D, colors, opacity, scales, rotations, cov3D_precomp, sh, degrees, prune_mask, filter_3D]
    M = 0
    if quant is not None:
        M = 16
    elif sh is not None and packed_counts is None:
        M = int(sh.shape[1])                                       # rasterize_points.cu:187-191
    s = GsbScene()
    s.P, s.M = P, M
    s.means3D, s.opacities, s.scales, s.rotations = ptr(means3D), ptr(opacity), ptr(scales), ptr(rotations)
    s.cov3D_precomp, s.shs, s.colors_precomp, s.degrees = ptr(cov3D_precomp), ptr(sh), ptr(colors), ptr(degrees)
    s.scale_modifier = float(scale_modifier)
    s.sh_packed = 0
    if packed_counts is not None:
        s.sh_packed = 1
        for d in range(4):
            s.band_count[d] = int(packed_counts[d]) if d < len(packed_counts) else 0
    s.prune_mask = ptr(prune_mask)
    s.filter_3D = ptr(filter_3D)
    s.quant = _quant_struct(quant, device, keep) if quant is not None else None
    return s, P, M


def _forward(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
             tan_fovx, tan_fovy, image_height, image_width, sh, degrees, campos, prefiltered, debug, packed_counts=None,
             prune_mask=None, quant=None, debug_out=None, statistics=None, return_maps=False, antialiasing=False, raw=None,
             statistics_workspace=None, features=None, filter_3D=None):
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")          # rasterize_points.cu:158-161
    if filter_3D is not None:
        check_filter_3d(filter_3D, int(means3D.shape[0]))
    F = check_features(features, int(means3D.shape[0])) if features is not None else 0
    device = _device_of(means3D)
    if features is not None and features.device != device:
        raise RuntimeError(f"features must live on {device}, got {features.device}")
    raw_s = None
    if raw is not None:
        if packed_counts is not None or statistics is not None:
            raise RuntimeError("raw parameters: the packed variable-SH and statistics forwards have no raw form")
        raw_s, _, raw_rot = _raw_struct(raw, device, int(means3D.shape[0]), not _present(colors), sh, scales, rotations, cov3D_precomp,
                                        quant)
    L = _lib.lib()
    keep = []
    H, W = int(image_height), int(image_width)
    with on_device(device):
        scene, P, M = _scene(device, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, sh, degrees,
                             keep, packed_counts, prune_mask, quant, filter_3D)
        cam = _camera(device, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, H, W, prefiltered, keep)
        out_color = torch.empty((3, H, W), dtype=torch.float32, device=device)
        maps = None
        if return_maps:
            maps = (torch.empty((1, H, W), dtype=torch.float32, device=device), torch.empty((1, H, W), dtype=torch.float32, device=device))
        radii = torch.empty((P,), dtype=torch.int32, device=device)
        blobs = BlobAllocator.for_device(device)
        cbs = blobs.cb
        dbg_ptr = None
        if debug_out is not None:
            d = dict(depths=torch.zeros(P, device=device), means2D=torch.zeros(P, 2, device=device),
                     cov3D=torch.zeros(P, 6, device=device), conic_opacity=torch.zeros(P, 4, device=device),
                     rgb=torch.zeros(P, 3, device=device), tiles_touched=torch.zeros(P, dtype=torch.int32, device=device),
                     clamped=torch.zeros(P, 3, dtype=torch.uint8, device=device))
            debug_out.update(d)
            dbg = GsbDebug(*[ptr(d[k]) for k in ("depths", "means2D", "cov3D", "conic_opacity", "rgb", "tiles_touched", "clamped")])
            dbg_ptr = C.pointer(dbg)
        R = C.c_int64(0)
        req = GsbForwardRequest(scene=C.pointer(scene), cam=C.pointer(cam), geom_alloc=cbs["geom"], binning_alloc=cbs["binning"],
                                image_alloc=cbs["image"], out_color=out_color.data_ptr(), radii=ptr(radii), num_rendered=C.pointer(R),
                                debug=dbg_ptr, antialiasing=int(bool(antialiasing)), stream=_lib.current_stream(device))
        if maps is not None:
            req.out_invdepth, req.out_alpha = maps[0].data_ptr(), maps[1].data_ptr()
        if raw_s is not None:
            req.raw = C.pointer(raw_s)
        if statistics is not None:                               # (touched_pixels int32 [P,1], transmittance_sum f32 [P,1]) to fill
            req.touched_pixels, req.transmittance_sum = ptr(statistics[0]), ptr(statistics[1])
            if statistics_workspace is not None:
                req.deterministic, req.workspace = 1, statistics_workspace.data_ptr()
        feat_img = ()
        if features is not None:
            # the feature channels, composited from the blobs this forward leaves behind
            feats = f32(features, device)
            feat_img = (torch.empty((F, H, W), dtype=torch.float32, device=device),)
            fs = GsbFeatures(F, ptr(feats), feat_img[0].data_ptr(), None, None)
            req.features = C.pointer(fs)
        st = L.gsb_forward(C.byref(req))
        geomB, binB, imgB = blobs.take("geom"), blobs.take("binning"), blobs.take("image")
        _lib.check(st)
        if debug:
            torch.cuda.synchronize(device)                      # reference CHECK_CUDA(debug) semantics, auxiliary.h:161-168
    if maps is not None:
        return (int(R.value), out_color, radii, geomB, binB, imgB, maps[0], maps[1]) + feat_img
    return (int(R.value), out_color, radii, geomB, binB, imgB) + feat_img


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                        projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degrees, campos, prefiltered, debug,
                        *, prune_mask=None, quant=None, debug_out=None, return_maps=False, antialiasing=False, raw=None, features=None,
                        filter_3D=None):
    """rasterize_points.h:43-63 RasterizeGaussiansCUDA -> (R, color, radii, geomBuffer, binningBuffer, imgBuffer).
    `return_maps`: -> (R, color, radii, geomBuffer, binningBuffer, imgBuffer, invdepth [1,H,W], alpha [1,H,W]) with
    invdepth = sum (1/depth) * alpha * T over the pairs that composite the colour and alpha = 1 - final_T.
    `antialiasing`: opacity-compensated 2D filter; its buffers need the backward's `antialiasing=True`.
    `raw`: (features_dc [P,1,3], features_rest [P,C,3], scaling [P,3], rotation [P,4]), the model's leaf parameters, with sh, scales
    and rotations empty; the kernels read them in place and activate them.  With colors, features_dc and
    features_rest are None.  The same output bits as the activated call on cat(dc, rest), exp(scaling), F.normalize(rotation).
    `features`: [P, F] fp32 on the device, 1 <= F <= 256; the tuple ends with the [F, H, W] feature image, each channel composited
    like a colour channel with background 0.  Every other output is the call's without it.
    `filter_3D`: [P] or [P, 1] fp32 on the device, Mip-Splatting's 3D filter applied to the scales and the opacity in the kernels;
    an all-zero filter gives the bytes of the call without it.  Not with cov3D_precomp."""
    return _forward(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                    projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degrees, campos, prefiltered, debug,
                    None, prune_mask, quant, debug_out, return_maps=return_maps, antialiasing=antialiasing, raw=raw, features=features,
                    filter_3D=filter_3D)


def rasterize_gaussians_variableSH_bands(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                                         viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh,
                                         perBandPrimitiveCount, cumSumPrimitiveCount, coeffsNum, degrees, campos, prefiltered,
                                         debug, *, prune_mask=None, debug_out=None, return_maps=False, antialiasing=False, features=None,
                                         filter_3D=None):
    """rasterize_points.h:18-41 RasterizeGaussiansVariableSHBandsCUDA (inference, packed per-degree SH groups).
    cumSumPrimitiveCount / coeffsNum are implied by perBandPrimitiveCount ([1,4,9,16] per gaussian_renderer:90-92).
    `return_maps`, `antialiasing`, `features` and `filter_3D` as in rasterize_gaussians (forward only, like the rest of this path)."""
    counts = [int(v) for v in perBandPrimitiveCount.detach().cpu().tolist()]
    return _forward(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                    projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degrees, campos, prefiltered, debug,
                    counts, prune_mask, None, debug_out, return_maps=return_maps, antialiasing=antialiasing, features=features,
                    filter_3D=filter_3D)


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                                 projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degrees, campos, geomBuffer, R,
                                 binningBuffer, imageBuffer, lambda_sh_sparsity, debug, *, prune_mask=None, quant=None,
                                 accumulate_into=None, want_conic=False, view_means2D=None, dL_dinvdepth=None, dL_dalpha=None,
                                 camera_grads=False, antialiasing=False, raw=None, deterministic=False, features=None,
                                 dL_dfeatures_out=None, absgrad_out=None, filter_3D=None, opacity=None):
    """rasterize_points.h:65-88 RasterizeGaussiansBackwardCUDA ->
    (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations).
    `accumulate_into`: the same 8-tuple from a previous call; gradients are added in place (view-batch accumulation);
    `view_means2D` ([P,3], accumulate mode): receives THIS view's dL_dmeans2D on its own (per-view densification statistics);
    `dL_dinvdepth` / `dL_dalpha` ([1,H,W] each, None = zero): gradients of the maps of `return_maps`;
    `camera_grads`: the tuple (after dL_dconic when `want_conic`) ends with (dL_dviewmatrix [4,4], dL_dprojmatrix [4,4],
    dL_dcampos [3]) in the layouts of the inputs; they are this view's gradients, also with `accumulate_into`;
    `antialiasing`: the backward of a forward with `antialiasing=True`; it must match the forward's flag.
    `raw`: the backward of a forward with the same `raw`.  The 8-tuple then becomes the 9-tuple
    (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, None, dL_dfeatures_dc, dL_dfeatures_rest, dL_dscaling, dL_drotation):
    the SH gradient split at coefficient 1, scaling / rotation chained through exp / F.normalize; dL_dcolors only with colors
    (else None), the SH gradients None with colors, and no dL_dcov3D.  `accumulate_into` takes that 9-tuple.
    `deterministic`: sum the per-Gaussian gradients in a fixed order instead of with float atomics:
    the same inputs give the same bytes on every run, in every mode above; the values agree with the default path to rounding.
    `features` / `dL_dfeatures_out`: the [P, F] features of the forward's `features` and the gradient of its [F, H, W] image; the
    feature image's share of the gradients is added to every output above and the tuple ends with dL_dfeatures [P, F].
    Neither `accumulate_into` nor `deterministic` has a feature form: both are refused.
    `absgrad_out`: a contiguous fp32 [P, 3] tensor on the device, overwritten with (sum_p |g_x|, sum_p |g_y|, 0), the per-pixel terms
    of dL_dmeans2D added as absolute values (AbsGS); every other output is the call's without it (bit for bit
    with `deterministic`).  It has no `accumulate_into` and no feature form: both are refused before anything runs.
    `filter_3D`: the forward's filter; `opacity` is then the forward's opacity logits (not with `quant`).  The filter gets no
    gradient; the scale and opacity gradients are chained through it."""
    if filter_3D is not None:
        check_filter_3d(filter_3D, int(means3D.shape[0]))
        if quant is None and not isinstance(opacity, torch.Tensor):
            raise RuntimeError("filter_3D: the backward needs the forward's opacity logits (opacity=...)")
    if absgrad_out is not None:
        check_absgrad_out(absgrad_out, int(means3D.shape[0]), accumulate_into, features, dL_dfeatures_out)
    feat_F = 0
    if features is not None:
        if accumulate_into is not None:
            raise RuntimeError("features: the feature backward has no accumulate_into form (view-batch accumulation)")
        if deterministic:
            raise RuntimeError("features: the feature backward has no deterministic form; render the features without a gradient "
                               "(torch.no_grad() or features.detach() and no loss on the image) or turn the deterministic mode off")
        feat_F = check_features(features, int(means3D.shape[0]))
    device = _device_of(means3D)
    if absgrad_out is not None and absgrad_out.device != device:
        raise RuntimeError(f"absgrad_out must live on {device}, got {absgrad_out.device}")
    if raw is not None:
        want_sh = not _present(colors)
        raw_s, C_rest, raw_rot = _raw_struct(raw, device, int(means3D.shape[0]), want_sh, sh, scales, rotations, cov3D_precomp, quant)
    L = _lib.lib()
    keep = []
    H, W = int(dL_dout_color.size(1)), int(dL_dout_color.size(2))
    with on_device(device):
        with_opacity = filter_3D is not None and quant is None
        scene, P, M = _scene(device, means3D, colors, opacity if with_opacity else None, scales, rotations, scale_modifier,
                             cov3D_precomp, sh, degrees, keep, None, prune_mask, quant, filter_3D)
        if quant is None and not with_opacity:
            scene.opacities = means3D.data_ptr() if P > 0 else None      # not read by the backward; keeps check_scene satisfied
        cam = _camera(device, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, H, W, False, keep)
        dL = f32(dL_dout_color, device)
        dmaps = [f32(m, device) for m in (dL_dinvdepth, dL_dalpha)]
        for m in dmaps:
            if m is not None and m.numel() != H * W:
                raise RuntimeError(f"dL_dinvdepth / dL_dalpha must have H*W = {H * W} elements, got {m.numel()}")
        keep += dmaps
        if raw is None:
            shapes = [(P, 3), (P, 3), (P, 1), (P, 3), (P, 6), (P, M, 3), (P, 3), (P, 4)]
        else:
            # slots: means2D, colors, opacity, means3D, (cov3D: none), features_dc, features_rest, scaling, rotation
            shapes = [(P, 3), (P, 3) if not want_sh else None, (P, 1), (P, 3), None, (P, 1, 3) if want_sh else None,
                      (P, C_rest, 3) if want_sh else None, (P, 3), (P, 4)]
        # camera gradients and their workspace ride in the same single allocation as the per-Gaussian outputs
        cam_shapes = [(4, 4), (4, 4), (3,), ((int(L.gsb_camera_grad_workspace_bytes(P)) + 3) // 4,)] if camera_grads else []
        if accumulate_into is not None:
            outs = list(accumulate_into)
            if raw is not None and len(outs) != 9:
                raise RuntimeError("accumulate_into: the raw backward's 9-tuple is expected")
            cam_out = _carve_f32(device, cam_shapes) if camera_grads else []
        else:
            live = [s for s in shapes if s is not None]
            carved = _carve_f32(device, live + cam_shapes)
            it = iter(carved)
            outs = [next(it) if s is not None else None for s in shapes]
            cam_out = carved[len(live):]
        # accumulate mode ADDS into every output, this fresh one included: it must start from zero
        conic = None
        if want_conic:
            conic = (torch.zeros if accumulate_into is not None else torch.empty)((P, 4), dtype=torch.float32, device=device)
        if view_means2D is not None and (accumulate_into is None or tuple(view_means2D.shape) != (P, 3) or
                                         view_means2D.dtype != torch.float32 or not view_means2D.is_contiguous()):
            raise RuntimeError("view_means2D needs accumulate_into and a contiguous fp32 [P,3] tensor")
        # raw mode: GsbRawGrads takes the SH, scaling and rotation slots, and GsbGrads leaves its own NULL
        g = GsbGrads(*[ptr(t) for t in (outs[:8] if raw is None else outs[:4] + [None] * 4)], ptr(conic),
                     1 if accumulate_into is not None else 0, ptr(view_means2D))
        radii = radii.to(device=device, dtype=torch.int32).contiguous()
        req = GsbBackwardRequest(scene=C.pointer(scene), cam=C.pointer(cam), num_rendered=int(R), radii=ptr(radii),
                                 geom_blob=ptr(geomBuffer), binning_blob=ptr(binningBuffer), image_blob=ptr(imageBuffer),
                                 dL_dout_color=ptr(dL), grads=C.pointer(g), dL_dinvdepth=ptr(dmaps[0]), dL_dalpha=ptr(dmaps[1]),
                                 lambda_sh_sparsity=float(lambda_sh_sparsity), antialiasing=int(bool(antialiasing)),
                                 dL_dmeans2D_abs=ptr(absgrad_out), stream=_lib.current_stream(device))
        if camera_grads:
            req.dL_dviewmatrix, req.dL_dprojmatrix, req.dL_dcampos, req.camera_workspace = [t.data_ptr() for t in cam_out]
        dfeat = ()
        if features is not None:
            dLf = f32(dL_dfeatures_out, device)
            if dLf is None or dLf.numel() != feat_F * H * W:
                raise RuntimeError(f"dL_dfeatures_out must have F*H*W = {feat_F * H * W} elements")
            feats = f32(features, device)
            keep += [dLf, feats]
            dfeat = (torch.empty((P, feat_F), dtype=torch.float32, device=device),)
            fs = GsbFeatures(feat_F, ptr(feats), None, dLf.data_ptr(), ptr(dfeat[0]))
            req.features = C.pointer(fs)
        if raw is not None:
            rg = GsbRawGrads(*[ptr(t) for t in outs[5:9]])
            req.raw, req.raw_grads = C.pointer(raw_s), C.pointer(rg)
        if deterministic:
            # per-instance partial slots, from the caching allocator on the current stream (freed in stream order after the call)
            ws_bytes = L.gsb_deterministic_workspace_bytes(P, int(R), int(absgrad_out is not None))
            det_ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device=device)
            req.deterministic, req.det_workspace = 1, ptr(det_ws)
        st = L.gsb_backward(C.byref(req))
        _lib.check(st)
        if debug:
            torch.cuda.synchronize(device)
    res = tuple(outs) + ((conic,) if want_conic else ())
    return (res + tuple(cam_out[:3]) if camera_grads else res) + dfeat


def calculate_colours_variance(cam_positions, means3D, opacity, scales, rotations, cam_viewmatrices, cam_projmatrices, tan_fovxs,
                               tan_fovys, image_height, image_width, sh, degrees, max_sh_deg, *, deterministic=None):
    """reduced_3dgs.h:28-43 Reduced3DGS::calculateColourVariance (reduced_3dgs.cu:41-203) ->
    (average colour distance to each lower SH truncation [P, max_sh_deg], weighted colour variance [P,1,3], weighted mean colour [P,1,3]).
    Per camera: one forward with the visibility statistics on + one fused statistics kernel
    (gsb_sh_statistics_update) in place of the reference's ~30 ATen ops; the camera parameters are read back once, not per camera.
    `deterministic`: sum the transmittances in 64-bit fixed point (the forward request's `deterministic`), the same bytes on every
    run; None follows torch.are_deterministic_algorithms_enabled() at the call, an explicit bool wins."""
    det = torch.are_deterministic_algorithms_enabled() if deterministic is None else bool(deterministic)
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")          # reduced_3dgs.cu:57-60
    device = _device_of(means3D)
    if int(max_sh_deg) != 3:
        raise RuntimeError("calculate_colours_variance: the reference's colour table has 4 slots per Gaussian "
                           "(reduced_3dgs/sh_culling.cu:21), i.e. it is only meaningful for max_sh_deg == 3")
    L = _lib.lib()
    P = int(means3D.size(0))
    n_cams = int(cam_positions.size(0))
    M = int(sh.size(1)) if (P != 0 and sh.size(0) != 0) else 0
    f = lambda t: f32(t, device)
    zeros = lambda *shape: torch.zeros(shape, dtype=torch.float32, device=device)
    wsum, wsumsq, dist, mean, var = zeros(P, 1), zeros(P, 1), zeros(P, 3), zeros(P, 1, 3), zeros(P, 1, 3)
    if P == 0 or n_cams == 0:
        return dist / wsum, var / wsum.view(-1, 1, 1), mean
    means3D, sh, cam_positions = f(means3D), f(sh), f(cam_positions)
    views, projs = f(cam_viewmatrices), f(cam_projmatrices)
    deg = degrees.to(device=device, dtype=torch.int32).contiguous()
    Hs, Ws = [int(v) for v in image_height.cpu().tolist()], [int(v) for v in image_width.cpu().tolist()]
    txs, tys = [float(v) for v in tan_fovxs.cpu().tolist()], [float(v) for v in tan_fovys.cpu().tolist()]
    bg = zeros(3)                                             # reduced_3dgs.cu:112 background is irrelevant here
    empty = torch.empty(0)
    touched = torch.empty((P, 1), dtype=torch.int32, device=device)
    tsum = torch.empty((P, 1), dtype=torch.float32, device=device)
    stream = _lib.current_stream(device)
    det_kw = {}
    if det:
        # one fixed-point workspace for all cameras (each forward clears it)
        det_kw["statistics_workspace"] = torch.empty(int(L.gsb_statistics_workspace_bytes(P)), dtype=torch.uint8, device=device)
    for i in range(n_cams):
        _, _, radii, _, _, _ = _forward(bg, means3D, empty, opacity, scales, rotations, 1.0, empty, views[i], projs[i], txs[i], tys[i],
                                        Hs[i], Ws[i], sh, deg, cam_positions[i], False, False, statistics=(touched, tsum), **det_kw)
        with on_device(device):
            _lib.check(L.gsb_sh_statistics_update(P, M, ptr(deg), ptr(means3D), cam_positions[i].data_ptr(), ptr(sh), ptr(radii), ptr(touched),
                                                  ptr(tsum), ptr(wsum), ptr(wsumsq), ptr(dist), ptr(mean), ptr(var), stream))
    return dist / wsum, var / wsum.view(-1, 1, 1), mean


def find_minimum_projected_pixel_size(w2ndc_transforms, w2ndc_transforms_inverse, means3D, image_height, image_width):
    """reduced_3dgs.h:61-66 Reduced3DGS::calculatePixelSize (reduced_3dgs.cu:246-268) -> float [P,1]."""
    device = _device_of(means3D)
    L = _lib.lib()
    P, n = int(means3D.size(0)), int(w2ndc_transforms.size(0))
    out = torch.empty((P, 1), dtype=torch.float32, device=device)
    if P == 0:
        return out
    i32 = lambda t: t.to(device=device, dtype=torch.int32).contiguous()
    m, mi, xyz, hs, ws = f32(w2ndc_transforms, device), f32(w2ndc_transforms_inverse, device), f32(means3D, device), i32(image_height), i32(image_width)
    with on_device(device):
        _lib.check(L.gsb_min_projected_pixel_size(P, ptr(xyz), n, ptr(m), ptr(mi), ptr(hs), ptr(ws), ptr(out), _lib.current_stream(device)))
    return out


def sphere_ellipsoid_intersection(means3D, scales, rotations, neighbours_indices, sphere_radius, knn):
    """reduced_3dgs.h:45-51 Reduced3DGS::intersectionTest (reduced_3dgs.cu:205-243) -> (redundancy_values int32 [P,1], intersection_mask bool [P,knn])."""
    device = _device_of(means3D)
    L = _lib.lib()
    P, knn = int(means3D.size(0)), int(knn)
    red = torch.empty((P, 1), dtype=torch.int32, device=device)
    mask = torch.empty((P, knn), dtype=torch.bool, device=device)
    if P == 0:
        return red, mask
    nb = neighbours_indices.to(device=device, dtype=torch.int32).contiguous()
    xyz, sc, rot, rad = f32(means3D, device), f32(scales, device), f32(rotations, device), f32(sphere_radius, device)
    with on_device(device):
        _lib.check(L.gsb_sphere_ellipsoid_intersection(P, ptr(xyz), ptr(sc), ptr(rot), ptr(nb), ptr(rad), knn, ptr(red), ptr(mask),
                                                       _lib.current_stream(device)))
    return red, mask


def allocate_minimum_redundancy_value(redundancy_values, neighbours_indices, intersection_mask, knn):
    """reduced_3dgs.h:53-59 Reduced3DGS::assignFinalRedundancyValue (reduced_3dgs.cu:270-287) -> 1-tuple (int32 [P,1],)."""
    device = _device_of(redundancy_values)
    L = _lib.lib()
    P, knn = int(redundancy_values.size(0)), int(knn)
    out = torch.empty((P, 1), dtype=torch.int32, device=device)
    if P == 0:
        return (out,)
    red = redundancy_values.to(device=device, dtype=torch.int32).contiguous()
    nb = neighbours_indices.to(device=device, dtype=torch.int32).contiguous()
    mask = intersection_mask.to(device=device, dtype=torch.bool).contiguous()
    with on_device(device):
        _lib.check(L.gsb_min_redundancy_value(P, ptr(red), ptr(nb), ptr(mask), knn, ptr(out), _lib.current_stream(device)))
    return (out,)


def kmeans_cuda(values, centers, tol, max_iterations, *, deterministic=None):
    """reduced_3dgs.h:21-26 Reduced3DGS::kmeans (reduced_3dgs.cu:289-338) -> (ids int32 [n,1], centers float32 [k]).
    `values` is the [n,1] column of one attribute, `centers` the [k] initial centres (gaussian_model.py:36-41).
    `deterministic`: add each cluster's values in an order fixed by the input (gsb_kmeans's `deterministic`), the same centres and ids
    on every run; None follows torch.are_deterministic_algorithms_enabled() at the call, an explicit bool wins."""
    det = torch.are_deterministic_algorithms_enabled() if deterministic is None else bool(deterministic)
    device = _device_of(values)
    L = _lib.lib()
    v = f32(values, device)
    c = f32(centers, device)
    n, k = int(values.size(0)), int(centers.size(0))
    ids = torch.zeros((n, 1), dtype=torch.int32, device=device)
    out = torch.empty((k,), dtype=torch.float32, device=device)
    with on_device(device):
        ws = torch.empty(int(L.gsb_kmeans_workspace_bytes(n, k, int(det))), dtype=torch.uint8, device=device)
        _lib.check(L.gsb_kmeans(ptr(v.reshape(-1)) if n else None, n, ptr(c.reshape(-1)), k, float(tol), int(max_iterations), int(det),
                                ptr(ids), out.data_ptr(), ws.data_ptr(), _lib.current_stream(device)))
    return ids, out


def mark_visible(means3D, viewmatrix, projmatrix):
    """rasterize_points.h:90-93 markVisible -> bool[P]."""
    device = _device_of(means3D)
    P = int(means3D.size(0))
    present = torch.zeros((P,), dtype=torch.bool, device=device)
    if P:
        m, v, p = f32(means3D, device), f32(viewmatrix, device), f32(projmatrix, device)
        with on_device(device):
            _lib.check(_lib.lib().gsb_mark_visible(P, ptr(m), ptr(v), ptr(p), present.data_ptr(), _lib.current_stream(device)))
    return present


def export_state(geomBuffer, binningBuffer, imageBuffer, R, W, H, P=0):
    """Decode the private blobs into reference-layout arrays (tests / tooling)."""
    device = imageBuffer.device
    L = _lib.lib()
    out = {}
    with on_device(device):
        keys = torch.zeros(max(R, 0), dtype=torch.int64, device=device)
        pl = torch.zeros(max(R, 0), dtype=torch.int32, device=device)
        if R > 0:
            _lib.check(L.gsb_export_binning(ptr(geomBuffer), int(P), ptr(binningBuffer), int(R), ptr(imageBuffer), W, H,
                                            ptr(keys), ptr(pl), _lib.current_stream(device)))
        T = ((W + 15) // 16) * ((H + 15) // 16)
        final_T = torch.zeros(H, W, device=device)
        n_contrib = torch.zeros(H, W, dtype=torch.int32, device=device)
        ranges = torch.zeros(T, 2, dtype=torch.int32, device=device)
        _lib.check(L.gsb_export_image(ptr(imageBuffer), W, H, ptr(final_T), ptr(n_contrib), ptr(ranges), _lib.current_stream(device)))
    out.update(keys=keys, point_list=pl, final_T=final_T, n_contrib=n_contrib, ranges=ranges)
    return out


class Contributions(NamedTuple):
    """One view's contribution statistics (gsb_contributions, DESIGN.md §5p): per Gaussian the sum of its blending weights
    w = alpha * T (times the clamped pixel weight), their maximum and the number of pixels it composites; per pixel the id of the
    Gaussian with the largest w (-1 where none)."""
    weight_sum: torch.Tensor     # [P] float32
    weight_max: torch.Tensor     # [P] float32
    pixels: torch.Tensor         # [P] int32
    top_id: torch.Tensor         # [H, W] int32


def check_pixel_weights(pixel_weights, H, W, device=None):
    """The checks of a `pixel_weights` map, made before anything runs: a contiguous float32 [H, W] or [1, H, W] tensor on `device`
    (on a CUDA device when `device` is None)."""
    if not isinstance(pixel_weights, torch.Tensor):
        raise RuntimeError(f"pixel_weights must be an [H, W] tensor, got {type(pixel_weights).__name__}")
    if tuple(pixel_weights.shape) not in ((H, W), (1, H, W)):
        raise RuntimeError(f"pixel_weights must have shape [H, W] or [1, H, W] with H, W = {H}, {W}, got {tuple(pixel_weights.shape)}")
    if pixel_weights.dtype != torch.float32:
        raise RuntimeError(f"pixel_weights must be float32, got {pixel_weights.dtype}")
    if not pixel_weights.is_contiguous():
        raise RuntimeError("pixel_weights must be contiguous (it is read in place)")
    if device is None and not pixel_weights.is_cuda:
        raise RuntimeError("pixel_weights must live on a CUDA device (no CPU path exists)")
    if device is not None and pixel_weights.device != device:
        raise RuntimeError(f"pixel_weights must live on {device}, got {pixel_weights.device}")


def contributions(geomBuffer, binningBuffer, imageBuffer, R, W, H, P, pixel_weights=None):
    """The contribution statistics of the forward that left these blobs (its R, image size and P), -> Contributions(weight_sum [P],
    weight_max [P], pixels [P], top_id [H, W]), views of one allocation.  `pixel_weights`: an [H, W] (or [1, H, W]) fp32 map on the
    blobs' device, clamped to [0, 1] on read (NaN reads as 0), that weights the sum.  The same bytes on every run; the blobs are only
    read.  No gradient."""
    device = imageBuffer.device
    if not imageBuffer.is_cuda:
        raise RuntimeError("contributions: the forward's buffers must live on a CUDA device (no CPU path exists)")
    W, H, P, R = int(W), int(H), int(P), int(R)
    if pixel_weights is not None:
        check_pixel_weights(pixel_weights, H, W, device)
    L = _lib.lib()
    with on_device(device):
        ws_words = (int(L.gsb_contributions_workspace_bytes(P)) + 3) // 4
        # int32 words: weight_sum, weight_max, pixels, top_id, then the 8-byte fixed-point workspace, each on a 256-byte boundary
        sizes = [P, P, P, H * W, ws_words]
        offs, total = [], 0
        for n in sizes:
            offs.append(total)
            total += (n + 63) // 64 * 64
        flat = torch.empty(total, dtype=torch.int32, device=device)
        ws, pw_sum, pw_max, pix, top = (flat[offs[4]:offs[4] + ws_words], flat[:P].view(torch.float32),
                                        flat[offs[1]:offs[1] + P].view(torch.float32), flat[offs[2]:offs[2] + P],
                                        flat[offs[3]:offs[3] + H * W].view(H, W))
        _lib.check(L.gsb_contributions(ptr(geomBuffer), P, ptr(binningBuffer), R, ptr(imageBuffer), W, H, ptr(pixel_weights), ptr(pw_sum),
                                       ptr(pw_max), ptr(pix), ptr(top), ptr(ws), _lib.current_stream(device)))
    return Contributions(pw_sum, pw_max, pix, top)


def debug_dequant(quant):
    """Fused de-quantisation on its own (test helper): -> (scales [P,3], rotations [P,4]) as the kernels compute them."""
    device = quant.means3D.device
    P = int(quant.means3D.shape[0])
    keep = []
    q = _quant_struct(quant, device, keep)
    scales = torch.empty(P, 3, device=device)
    rots = torch.empty(P, 4, device=device)
    with on_device(device):
        _lib.check(_lib.lib().gsb_debug_dequant(q, P, scales.data_ptr(), rots.data_ptr(), _lib.current_stream(device)))
    return scales, rots
