"""Native densification: the reference's GaussianModel.densify_and_prune / prune / prune_points / add_densification_stats
(scene/gaussian_model.py:553-695) on the model and its optimizer state, row for row (DESIGN.md §5g), and its resolution-aware
redundancy pruning, Scene.calculate_redundancy_metric + GaussianModel.mercy_points (DESIGN.md §5k).

    from gs_b200 import densify
    GaussianModel.densify_and_prune = densify.densify_and_prune      # INTEGRATION.md section D
    GaussianModel.prune = densify.prune
    GaussianModel.prune_points = densify.prune_points
    GaussianModel.add_densification_stats = densify.add_densification_stats
    GaussianModel.mercy_points = densify.mercy_points
    Scene.calculate_redundancy_metric = densify.calculate_redundancy_metric

The signatures are the reference's methods with `self` -> `model`.  The results are the reference's: the same rows in the same
order ([kept originals][kept clones][kept first children][kept second children]), the same values, the same optimizer state
dicts (their `step` tensors included) moved to the new nn.Parameters, the same statistics and dictionary entries, and the same
CUDA generator state (torch.normal is called once, with the reference's [2 S, 3] shape, also for S = 0).  The split children's
xyz goes through rotation @ sample, whose torch.bmm rounding depends on cuBLAS's kernel choice; those values agree to rounding.

densify_and_prune, prune and prune_points each read the host once (the counts that size the outputs), where the reference
synchronises about ten times; add_densification_stats never does.  torch.cuda.empty_cache() is not called.

Model contract (duck-typed on the reference's attribute names): the optimizer is torch.optim.Adam or GaussianAdam with exactly
the six groups "xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", one fp32 contiguous CUDA param each (f_rest a dense
[P, C, 3] tensor); `_degrees` int32 [P, 1]; `xyz_gradient_accum`, `denom` fp32 [P, 1]; `max_radii2D` fp32 [P];
`percent_dense`.  Anything else is refused before the model or the optimizer changes.

AbsGS (DESIGN.md §5m): add_densification_stats(..., viewspace_abs=pkg["viewspace_points_abs"]) also accumulates the norm of the
absolute screen-space gradient into `xyz_gradient_accum_abs` [P, 1] (created as zeros on the first call), and
densify_and_prune(..., max_grad_abs=...) splits on accum_abs / denom >= max_grad_abs instead of on the signed statistic.  Every prune
carries `xyz_gradient_accum_abs`, and densify_and_prune resets it, exactly as `xyz_gradient_accum`, when the model has one.

Mip-Splatting (DESIGN.md §5o): a model with `filter_3D` ([P, 1] or [P] fp32, gs_b200.mip.compute_3D_filter) has it carried row for
row by every pass here and in gs_b200.mcmc, a clone, split child or added row taking its source's value, so render() never sees a
stale row count; recompute it after densifying, as Mip-Splatting does.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from . import lib as gsl

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
        "rotation": "_rotation"}
ROW_SHAPE = {"xyz": (3,), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
SPLIT_N = 2


def split_scale_factor(n=SPLIT_N):
    """torch's CUDA division of an fp32 tensor by the Python number 0.8 * N multiplies by the fp32 reciprocal of its fp32 cast
    (tools/probe_torch_densify.py)."""
    return float(np.float32(1) / np.float32(0.8 * n))


def _check_viewspace_grad(g, P, what):
    if g is None:
        raise RuntimeError(f"densify: {what} has no gradient")
    if (not g.is_cuda or g.dtype != torch.float32 or g.dim() != 2 or g.shape[0] != P or g.shape[1] < 2 or g.stride(1) != 1
            or (P > 1 and g.stride(0) < 2)):
        raise RuntimeError(f"densify: the view-space gradient ({what}) must be an fp32 CUDA [P, >= 2] tensor with unit column stride")


def add_densification_stats(model, viewspace_point_tensor, update_filter, radii=None, viewspace_abs=None):
    """xyz_gradient_accum += |grad[:, :2]|; denom += update_filter; with radii, also train.py:134's
    max_radii2D[update_filter] = max(max_radii2D[update_filter], radii[update_filter]).  With viewspace_abs (render(absgrad=True)'s
    pkg["viewspace_points_abs"]), also xyz_gradient_accum_abs += |viewspace_abs.grad[:, :2]| (zeros [P, 1] created on the first call).
    One launch, no host synchronisation."""
    g = viewspace_point_tensor.grad
    accum, denom = model.xyz_gradient_accum, model.denom
    P = accum.shape[0] if accum.dim() > 0 else -1
    _check_viewspace_grad(g, P, "viewspace_point_tensor")
    dev = g.device
    ga = None
    if viewspace_abs is not None:
        ga = viewspace_abs.grad
        _check_viewspace_grad(ga, P, "viewspace_abs")
        if ga.device != dev:
            raise RuntimeError(f"densify: the gradient of viewspace_abs must live on {dev}")
        if getattr(model, "xyz_gradient_accum_abs", None) is not None:
            _check_f32(model.xyz_gradient_accum_abs, (P, 1), dev, "xyz_gradient_accum_abs")
    _check_f32(accum, (P, 1), dev, "xyz_gradient_accum")
    _check_f32(denom, (P, 1), dev, "denom")
    if (update_filter.dtype != torch.bool or update_filter.shape != (P,) or update_filter.device != dev
            or not update_filter.is_contiguous()):
        raise RuntimeError(f"densify: update_filter must be a contiguous bool tensor [{P}] on {dev}")
    mr = None
    if radii is not None:
        if radii.dtype != torch.int32 or radii.shape != (P,) or radii.device != dev or not radii.is_contiguous():
            raise RuntimeError(f"densify: radii must be a contiguous int32 tensor [{P}] on {dev}")
        mr = model.max_radii2D
        _check_f32(mr, (P,), dev, "max_radii2D")
    if ga is not None and getattr(model, "xyz_gradient_accum_abs", None) is None:
        model.xyz_gradient_accum_abs = torch.zeros((P, 1), device=dev)
    if P == 0:
        return
    with gsl.on_device(dev):
        gsl.check(gsl.lib().gsb_densify_stats(P, g.data_ptr(), g.stride(0), None if ga is None else ga.data_ptr(),
                                               0 if ga is None else ga.stride(0), update_filter.data_ptr(),
                                               None if radii is None else radii.data_ptr(), accum.data_ptr(),
                                               None if ga is None else model.xyz_gradient_accum_abs.data_ptr(), denom.data_ptr(),
                                               None if mr is None else mr.data_ptr(), gsl.current_stream(dev)))


def densify_and_prune(model, max_grad, min_opacity, extent, max_screen_size, densification_statistics_dict, store_grads=False,
                      max_grad_abs=None):
    """densify_and_clone + densify_and_split + prune of the reference, in one plan and one emit.  max_grad_abs (AbsGS): clone on
    accum / denom >= max_grad as before, split on xyz_gradient_accum_abs / denom >= max_grad_abs (NaN -> 0); None is the reference's
    rule."""
    groups, P, dev = _validate(model, store_grads, grads_everywhere=store_grads)
    if max_grad_abs is not None and getattr(model, "xyz_gradient_accum_abs", None) is None:
        raise RuntimeError("densify: max_grad_abs needs model.xyz_gradient_accum_abs (add_densification_stats(..., viewspace_abs=...))")
    counts, ws, dcounts = _plan(model, groups, P, dev, gsl.DENSIFY_CLONE_SPLIT, max_grad=max_grad, percent_dense=model.percent_dense,
                       min_opacity=min_opacity, extent=extent, max_screen_size=max_screen_size, max_grad_abs=max_grad_abs)
    n_kept, C, n_clones_kept, S, n_children, P_out = counts[:6]
    # the reference's draw (gaussian_model.py:633-635): std = exp(scaling) of the split parents, repeated N times
    off = gsl.lib().gsb_densify_split_std_offset(P)
    stds = ws[off:off + 12 * S].view(torch.float32).view(S, 3).repeat(SPLIT_N, 1)
    means = torch.zeros((stds.size(0), 3), device=dev)
    samples = torch.normal(mean=means, std=stds)
    _emit(model, groups, P, dev, ws, counts, store_grads, gather_stats=False, samples=samples)
    model.xyz_gradient_accum = torch.zeros((P_out, 1), device=dev)
    if getattr(model, "xyz_gradient_accum_abs", None) is not None:
        model.xyz_gradient_accum_abs = torch.zeros((P_out, 1), device=dev)
    # densification_postfix creates density_gradient_accum after the split's concatenation; the prunes that follow do not index it
    model.density_gradient_accum = torch.zeros((P + C + SPLIT_N * S, 1), device=dev)
    model.denom = torch.zeros((P_out, 1), device=dev)
    model.max_radii2D = torch.zeros((P_out), device=dev)
    densification_statistics_dict["n_points_pruned"] = _pruned(dcounts)
    densification_statistics_dict["n_points_cloned"] = C
    densification_statistics_dict["n_points_split"] = S


def prune(model, min_opacity, extent, max_screen_size, densification_statistics_dict, store_grads=False):
    """The reference's prune(): drop sigmoid(opacity) < min_opacity and, if max_screen_size, the rows too large on screen or in
    the world."""
    groups, P, dev = _validate(model, store_grads)
    counts, ws, dcounts = _plan(model, groups, P, dev, gsl.DENSIFY_PRUNE, min_opacity=min_opacity, extent=extent,
                       max_screen_size=max_screen_size)
    densification_statistics_dict["n_points_pruned"] = _pruned(dcounts)
    _emit(model, groups, P, dev, ws, counts, store_grads, gather_stats=True)


def prune_points(model, mask, store_grads=False):
    """The reference's prune_points(mask): drop the rows where mask (bool [P], e.g. from mercy_points) is True."""
    groups, P, dev = _validate(model, store_grads)
    if not torch.is_tensor(mask) or mask.dtype != torch.bool or mask.shape != (P,) or mask.device != dev:
        raise RuntimeError(f"densify: the prune mask must be a bool tensor [{P}] on {dev}")
    counts, ws, _ = _plan(model, groups, P, dev, gsl.DENSIFY_PRUNE_MASK, mask=mask.contiguous())
    _emit(model, groups, P, dev, ws, counts, store_grads, gather_stats=True)


MERCY_TYPES = (("redundancy_opacity", gsl.MERCY_REDUNDANCY_OPACITY), ("redundancy_random", gsl.MERCY_REDUNDANCY_RANDOM),
               ("opacity", gsl.MERCY_OPACITY), ("redundancy_opacity_opacity", gsl.MERCY_REDUNDANCY_OPACITY_OPACITY))
MERCY_QUANTILE = {gsl.MERCY_OPACITY: 0.045, gsl.MERCY_REDUNDANCY_OPACITY_OPACITY: 0.03}


def calculate_redundancy_metric(scene, pixel_scale=1.0, num_neighbours=30):
    """The reference's Scene.calculate_redundancy_metric -> (min_redundancy int32 [P, 1], cube_size fp32 [P, 1]): the pixel
    size, the kNN, the intersection test and the minimum in one native call with no host synchronisation and no [P, K] mask
    or [P, K + 1] copies.  Missing neighbours (P <= num_neighbours) are not counted.  1 <= num_neighbours <= 64."""
    cams = scene.getTrainCameras()
    g = scene.gaussians
    xyz = g._xyz
    if not torch.is_tensor(xyz) or not xyz.is_cuda or xyz.dtype != torch.float32 or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise RuntimeError("densify: the model's _xyz must be an fp32 CUDA tensor [P, 3]")
    dev, P = xyz.device, xyz.shape[0]
    K = int(num_neighbours)
    f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
    xyz, scales, rots = f32(xyz), f32(g.get_scaling), f32(g.get_rotation)
    if tuple(scales.shape) != (P, 3) or tuple(rots.shape) != (P, 4):
        raise RuntimeError(f"densify: get_scaling / get_rotation must be [{P}, 3] / [{P}, 4]")
    n = len(cams)
    if n:
        w2ndc = f32(torch.stack([c.full_proj_transform for c in cams], dim=0))
        inv = f32(torch.stack([c.inverse_full_proj_transform for c in cams], dim=0))
        if tuple(w2ndc.shape) != (n, 4, 4) or tuple(inv.shape) != (n, 4, 4):
            raise RuntimeError("densify: the cameras' full_proj_transform / inverse_full_proj_transform must be 4 x 4")
    else:
        w2ndc = inv = None
    heights = torch.tensor([c.image_height for c in cams], device=dev, dtype=torch.int32)
    widths = torch.tensor([c.image_width for c in cams], device=dev, dtype=torch.int32)
    L = gsl.lib()
    red = torch.empty((P, 1), dtype=torch.int32, device=dev)
    cube = torch.empty((P, 1), dtype=torch.float32, device=dev)
    ws = torch.empty(L.gsb_redundancy_workspace_bytes(P, K) if 1 <= K <= 64 else 0, dtype=torch.uint8, device=dev)  # else refused
    ptr = lambda t: None if t is None or t.numel() == 0 else t.data_ptr()  # noqa: E731
    with gsl.on_device(dev):
        gsl.check(L.gsb_redundancy_score(P, ptr(xyz), ptr(scales), ptr(rots), n, ptr(w2ndc), ptr(inv), ptr(heights),
                                         ptr(widths), float(pixel_scale), K, ptr(red), ptr(cube), ptr(ws), gsl.current_stream(dev)))
    return red, cube


def mercy_points(model, densification_statistics_dict, lambda_mercy=2, mercy_minimum=2, mercy_type='redundancy_opacity'):
    """The reference's mercy_points: threshold the redundancy counts in model._splatted_num_accum (int32 [P, 1, 1], [P, 1] or
    [P]) at max(mean + lambda_mercy * std, mercy_minimum), choose the rows to prune by mercy_type and prune them with
    prune_points' plan and emit.  The statistics dictionary gets the reference's types and shapes.  One host read-back (the
    prune's counts); 'redundancy_random' has a second one, the number of uniforms to draw."""
    groups, P, dev = _validate(model, False)
    c = getattr(model, "_splatted_num_accum", None)
    if (not torch.is_tensor(c) or c.dtype != torch.int32 or c.device != dev or not c.is_contiguous()
            or tuple(c.shape) not in ((P, 1, 1), (P, 1), (P,))):
        raise RuntimeError(f"densify: _splatted_num_accum must be a contiguous int32 tensor [{P}, 1, 1], [{P}, 1] or [{P}] on {dev}")
    code = next((v for k, v in MERCY_TYPES if mercy_type == k), gsl.MERCY_REDUNDANCY)
    q = MERCY_QUANTILE.get(code, 0.0)
    logits = next(p for name, _, p, _ in groups if name == "opacity")
    L = gsl.lib()
    ws = torch.empty(L.gsb_mercy_workspace_bytes(P), dtype=torch.uint8, device=dev)
    mask = torch.empty(P, dtype=torch.uint8, device=dev)
    thr = torch.empty(2, dtype=torch.float32, device=dev)
    cnt = torch.empty(2, dtype=torch.int64, device=dev)

    def plan(draws=None, n_draws=-1):
        with gsl.on_device(dev):
            gsl.check(L.gsb_mercy_plan(P, c.data_ptr(), logits.data_ptr(), code, lambda_mercy, mercy_minimum, q,
                                       None if draws is None else draws.data_ptr(), n_draws, ws.data_ptr(), mask.data_ptr(),
                                       thr.data_ptr(), cnt.data_ptr(), gsl.current_stream(dev)))
    plan()
    if code == gsl.MERCY_REDUNDANCY_RANDOM:
        # the reference's torch.rand(mask[mask].shape): one draw per redundant row, also when there is none
        draws = torch.rand((int(cnt[0]),), device=dev)
        plan(draws if draws.numel() else torch.zeros(1, device=dev), draws.numel())
    counts, pws, _ = _plan(model, groups, P, dev, gsl.DENSIFY_PRUNE_MASK, mask=mask)
    _emit(model, groups, P, dev, pws, counts, False, gather_stats=True)
    densification_statistics_dict["n_points_mercied"] = cnt[1].clone()
    # the reference's mean of squeeze(): [1], or 0-dim for a single row
    densification_statistics_dict["redundancy_threshold"] = thr[0].clone() if P == 1 else thr[0:1].clone()
    densification_statistics_dict["opacity_threshold"] = (thr[1].clone() if code == gsl.MERCY_OPACITY else thr[1:2].clone()
                                                          if code == gsl.MERCY_REDUNDANCY_OPACITY_OPACITY else 0)


# ------------------------------------------------------------------------------------------------ internals
def _check_f32(t, shape, dev, name):
    if not torch.is_tensor(t) or t.dtype != torch.float32 or tuple(t.shape) != tuple(shape) or t.device != dev or not t.is_contiguous():
        raise RuntimeError(f"densify: {name} must be a contiguous fp32 tensor {list(shape)} on {dev}")


def _validate(model, store_grads, grads_everywhere=False):
    """[(name, group, param, state or None)] in group order, P, device; raises before anything changes."""
    if getattr(model, "_codebook_dict", None) is not None:
        raise RuntimeError("densify: a quantised model (codebooks) cannot be densified")
    if isinstance(getattr(model, "_features_rest", None), (list, tuple)):
        raise RuntimeError("densify: variable-SH-band models (a list-valued _features_rest) are not supported")
    opt = getattr(model, "optimizer", None)
    if not isinstance(opt, torch.optim.Adam):
        raise RuntimeError("densify: the model's optimizer must be torch.optim.Adam or GaussianAdam")
    names = [g.get("name") for g in opt.param_groups]
    if sorted(names) != sorted(GROUPS) or any(len(g["params"]) != 1 for g in opt.param_groups):
        raise RuntimeError(f"densify: the optimizer needs exactly the groups {GROUPS}, one param each; it has {names}")
    p0 = next(g["params"][0] for g in opt.param_groups if g["name"] == "xyz")
    P, dev = p0.shape[0] if p0.dim() > 0 else -1, p0.device
    if not p0.is_cuda:
        raise RuntimeError("densify: the model's params must be CUDA tensors (there is no CPU path)")
    groups = []
    for g in opt.param_groups:
        name, p = g["name"], g["params"][0]
        want = (P,) + ROW_SHAPE[name] if name in ROW_SHAPE else None
        if p.dtype != torch.float32 or not p.is_contiguous() or p.device != dev or p.dim() < 2 or p.shape[0] != P \
                or (want is not None and tuple(p.shape) != want) or (name == "f_rest" and (p.dim() != 3 or p.shape[2] != 3)):
            raise RuntimeError(f"densify: param '{name}' must be a contiguous fp32 tensor of {P} rows on {dev} "
                               f"({'x'.join(map(str, want)) if want else '[P, C, 3]'}), got {tuple(p.shape)} {p.dtype} on {p.device}")
        state = opt.state.get(p, None)
        if state is not None:
            for k in ("exp_avg", "exp_avg_sq"):
                s = state.get(k)
                if not torch.is_tensor(s) or s.shape != p.shape or s.dtype != torch.float32 or s.device != dev or not s.is_contiguous():
                    raise RuntimeError(f"densify: state['{k}'] of '{name}' must be a contiguous fp32 tensor of the param's shape")
        if store_grads and (state is not None or grads_everywhere):
            gr = p.grad
            if gr is None or gr.shape != p.shape or gr.dtype != torch.float32 or gr.device != dev or not gr.is_contiguous():
                raise RuntimeError(f"densify: store_grads needs a contiguous fp32 gradient of '{name}' (the reference carries it)")
        groups.append((name, g, p, state))
    deg = getattr(model, "_degrees", None)
    if not torch.is_tensor(deg) or deg.dtype != torch.int32 or tuple(deg.shape) != (P, 1) or deg.device != dev or not deg.is_contiguous():
        raise RuntimeError(f"densify: _degrees must be a contiguous int32 tensor [{P}, 1] on {dev}")
    _check_f32(getattr(model, "xyz_gradient_accum", None), (P, 1), dev, "xyz_gradient_accum")
    _check_f32(getattr(model, "denom", None), (P, 1), dev, "denom")
    _check_f32(getattr(model, "max_radii2D", None), (P,), dev, "max_radii2D")
    if getattr(model, "xyz_gradient_accum_abs", None) is not None:
        _check_f32(model.xyz_gradient_accum_abs, (P, 1), dev, "xyz_gradient_accum_abs")
    f3d = getattr(model, "filter_3D", None)
    if f3d is not None:
        _check_f32(f3d, (P, 1) if torch.is_tensor(f3d) and f3d.dim() == 2 else (P,), dev, "filter_3D")
    return groups, P, dev


def _plan(model, groups, P, dev, mode, max_grad=0.0, percent_dense=0.0, min_opacity=0.0, extent=0.0, max_screen_size=None, mask=None,
          max_grad_abs=None):
    """Runs the plan and reads its counts back (the one host synchronisation).  The thresholds are the reference's Python
    doubles (percent_dense*extent, 0.1*extent), cast to fp32 by ctypes as torch casts a Python number it compares with."""
    param = {name: p for name, _, p, _ in groups}
    ws = torch.empty(gsl.lib().gsb_densify_workspace_bytes(P), dtype=torch.uint8, device=dev)
    counts = torch.empty(gsl.DENSIFY_COUNTS, dtype=torch.int64, device=dev)
    screen = bool(max_screen_size)
    with gsl.on_device(dev):
        gsl.check(gsl.lib().gsb_densify_plan(
            P, mode, model.xyz_gradient_accum.data_ptr(),
            None if max_grad_abs is None else model.xyz_gradient_accum_abs.data_ptr(), model.denom.data_ptr(),
            param["scaling"].data_ptr(), param["opacity"].data_ptr(), model.max_radii2D.data_ptr(),
            None if mask is None else mask.data_ptr(), max_grad, 0.0 if max_grad_abs is None else max_grad_abs, percent_dense * extent,
            min_opacity, 1 if screen else 0, max_screen_size if screen else 0.0, 0.1 * extent, split_scale_factor(), ws.data_ptr(),
            counts.data_ptr(), gsl.current_stream(dev)))
    return [int(v) for v in counts.tolist()], ws, counts


def _pruned(counts):
    """n_points_pruned: a 0-dim int64 device tensor, as the reference's prune_mask.sum() is; copied on the device."""
    return counts[6].clone()


def _emit(model, groups, P, dev, ws, counts, store_grads, gather_stats, samples=None):
    n_kept, _, n_clones_kept, S, n_children, P_out = counts[:6]
    entries, install = _resized(model, groups, P_out, dev, {"xyz": gsl.DENSIFY_XYZ, "scaling": gsl.DENSIFY_SCALING},
                                gsl.DENSIFY_COPY if gather_stats else None, store_grads)
    rot = next(p for name, _, p, _ in groups if name == "rotation")
    table = (gsl.GsbDensifyTensor * len(entries))(*entries)
    with gsl.on_device(dev):
        gsl.check(gsl.lib().gsb_densify_emit(table, len(entries), P, ws.data_ptr(), n_kept, n_clones_kept, S, n_children,
                                              rot.data_ptr(), None if samples is None or samples.numel() == 0 else samples.data_ptr(),
                                              split_scale_factor(), gsl.current_stream(dev)))
    install()


def _entry(src, dst, kind, moments_src=None, moments_dst=None, grad_src=None, grad_dst=None):
    """One GsbDensifyTensor row of the densify / MCMC emit tables; moments are (exp_avg, exp_avg_sq) pairs."""
    e = gsl.GsbDensifyTensor()
    e.src, e.dst = src.data_ptr(), dst.data_ptr()
    e.row_width = src.shape[1:].numel()
    e.kind = kind
    if moments_src is not None:
        e.exp_avg_src, e.exp_avg_dst = moments_src[0].data_ptr(), moments_dst[0].data_ptr()
        e.exp_avg_sq_src, e.exp_avg_sq_dst = moments_src[1].data_ptr(), moments_dst[1].data_ptr()
    if grad_src is not None:
        e.grad_src, e.grad_dst = grad_src.data_ptr(), grad_dst.data_ptr()
    return e


STATS = ("xyz_gradient_accum", "denom", "max_radii2D", "xyz_gradient_accum_abs")


def _resized(model, groups, P_out, dev, kinds, stat_kind, store_grads=False):
    """The [P_out] rows of a resized model and their emit table entries: each group's param (kind from `kinds`, else COPY), its
    moments if it has state and then with store_grads its .grad; _degrees and, when the model has one, filter_3D (Mip-Splatting's
    3D filter, DESIGN.md §5o) as COPY, so a child or an added row takes its source's value; unless stat_kind is None, the STATS the
    model has.
    -> (entries, install).  install(), after the emit, sets the statistics and does the reference's optimizer surgery
    (_prune_optimizer / cat_tensors_to_optimizer): the state dict object moves to the new Parameter with the new moments; a group
    without state only gets its param; .grad travels only with state and store_grads."""
    entries, new = [], []
    for name, g, p, state in groups:
        dst = torch.empty((P_out,) + tuple(p.shape[1:]), dtype=torch.float32, device=dev)
        mv = gr = None
        if state is not None:
            mv = (torch.empty_like(dst), torch.empty_like(dst))
            if store_grads:
                gr = torch.empty_like(dst)
        moments = None if state is None else (state["exp_avg"], state["exp_avg_sq"])
        entries.append(_entry(p, dst, kinds.get(name, gsl.DENSIFY_COPY), moments, mv, None if gr is None else p.grad, gr))
        new.append((name, g, p, state, dst, mv, gr))
    stats = [("_degrees", gsl.DENSIFY_COPY)]
    if getattr(model, "filter_3D", None) is not None:
        stats.append(("filter_3D", gsl.DENSIFY_COPY))
    if stat_kind is not None:
        stats += [(k, stat_kind) for k in STATS if getattr(model, k, None) is not None]
    out_stats = {}
    for attr, kind in stats:
        src = getattr(model, attr)
        out_stats[attr] = torch.empty((P_out,) + tuple(src.shape[1:]), dtype=src.dtype, device=dev)
        entries.append(_entry(src, out_stats[attr], kind))

    def install():
        opt = model.optimizer
        for name, g, p, state, dst, mv, gr in new:
            param = nn.Parameter(dst.requires_grad_(True))
            if state is not None:
                state["exp_avg"], state["exp_avg_sq"] = mv
                del opt.state[p]
                if gr is not None:
                    param.grad = gr
                opt.state[param] = state
            g["params"][0] = param
            setattr(model, ATTR[name], param)
        for attr, t in out_stats.items():
            setattr(model, attr, t)
    return entries, install
