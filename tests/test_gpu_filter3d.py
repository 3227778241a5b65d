"""GPU: Mip-Splatting's 3D smoothing filter (GsbScene.filter_3D, gsb_filter_3d, gs_b200.mip; DESIGN.md §5o).
  1. compute_3D_filter against the float64 and fp32 torch restatements (tests/filter3d_restatement.py) on points on the 0.2 depth
     plane and at the +-15 % screen margins, unseen points, cameras of different focals and sizes and more cameras than one
     shared-memory chunk; every disagreement beyond 2 ulp is a point within a few ulp of a visibility boundary; same bytes twice;
  2. a zero filter is the call without one, bit for bit (dense, raw, quantised, anti-aliased, maps);
  3. with a filter, cov3D / means2D / conic / radii / depths are those of a render on torch's sqrt(s^2 + f^2), and the opacity is
     the fp32 product sigmoid * c3 (times the AA factor);
  4. gradients: per Gaussian against the fp64 oracle with backward_edges.compare's bar on backward-edge scenes with a filter
     (filter3d_restatement.edge_rows: zero and moderate filters, compositing rows with c3 in [5e-3, 0.05] and flat ones with an axis
     of 1e-6, and axes of exactly 0), with and without AA; the new chain per Gaussian against float64 contracted with the kernel's
     own screen-space gradients on the dense, raw and quantised paths; the camera and deterministic paths against the dense one; end
     to end against the float64 restatement of the anti-aliased pipeline (render64.py);
  5. a short training run that recomputes the filter, densifies with it and renders features and absgrad with it.
Observed maxima are printed (pytest -s)."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import filter3d_restatement as F3
import ours as O
import restate64 as R64
from render64 import render64
from diff_gaussian_rasterization import _C
from gs_b200 import mip, synth

pytestmark = pytest.mark.gpu

DEV = "cuda"
F64 = torch.float64


def _ulps(a, b):
    """|a - b| in units in the last place of fp32 (both non-negative)."""
    return (a.contiguous().view(torch.int32).long() - b.contiguous().view(torch.int32).long()).abs()


# ---- 1. the filter computation ------------------------------------------------------------------------------------------------

def _cams(n, seed):
    g = torch.Generator().manual_seed(seed)
    cams = [F3.camera(torch.eye(4), 64, 48, 1.0, 0.8)]          # camera 0: view space == world space
    for i in range(1, n):
        a = 2 * math.pi * i / n
        R = torch.tensor([[math.cos(a), 0, -math.sin(a)], [0, 1, 0], [math.sin(a), 0, math.cos(a)]])
        view = torch.eye(4)
        view[:3, :3] = R.T
        view[3, 2] = 3.0 + 2.0 * float(torch.rand(1, generator=g))
        cams.append(F3.camera(view, 40 + 24 * (i % 5), 30 + 16 * (i % 3), 0.6 + 0.15 * (i % 4), 0.5 + 0.1 * (i % 3)))
    return cams


def _points(cams, seed, P=20_000):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.randn(P, 3, generator=g) * 2.0
    c = cams[0]
    fx, fy = F3.focals(c)
    k = 500
    # on camera 0's 0.2 depth plane (z is exactly 0.2 in fp32, as in the kernel: view space is world space)
    xyz[:k, 2] = 0.2
    xyz[:k, :2] = (torch.rand(k, 2, generator=g) - 0.5) * 0.05
    # at camera 0's screen margins: u = -0.15 W and 1.15 W, v = -0.15 H and 1.15 H
    z = 1.0 + torch.rand(4 * k, generator=g)
    xyz[k:5 * k, 2] = z
    for j, (lo_u, val) in enumerate(((True, -0.15 * c.image_width), (True, 1.15 * c.image_width),
                                     (False, -0.15 * c.image_height), (False, 1.15 * c.image_height))):
        rows = slice(k + j * k, k + (j + 1) * k)
        if lo_u:
            xyz[rows, 0] = ((val - c.image_width / 2.0) / fx * z[j * k:(j + 1) * k]).float()
            xyz[rows, 1] = 0.0
        else:
            xyz[rows, 1] = ((val - c.image_height / 2.0) / fy * z[j * k:(j + 1) * k]).float()
            xyz[rows, 0] = 0.0
    xyz[5 * k:6 * k] = torch.tensor([0.0, 300.0, 0.0])             # far above every camera: seen by none
    return xyz


@pytest.mark.parametrize("n_cams", [7, 1500])
def test_filter_against_the_restatements(n_cams):
    cams = _cams(n_cams, 11 + n_cams)
    xyz = _points(cams, 12 + n_cams)
    model = SimpleNamespace(get_xyz=xyz.to(DEV))
    f = mip.compute_3D_filter(model, cams).clone()
    f2 = mip.compute_3D_filter(model, cams).clone()
    assert f.shape == (xyz.shape[0], 1) and f.dtype == torch.float32 and model.filter_3D.data_ptr() != 0
    assert torch.equal(f.view(torch.int32), f2.view(torch.int32))                       # the same bytes on every run
    f = f.view(-1).cpu()
    ref32 = F3.filter_torch_fp32(xyz.to(DEV), cams).cpu()
    ref64, seen, _ = F3.filter_fp64(xyz, cams)
    assert 0 < int(seen.sum()) < xyz.shape[0] and bool((f > 0).all())
    near = F3.boundary_ulps(xyz, cams) <= 8
    d = _ulps(f, ref32)
    bad = d > 2
    print(f"\n[filter_3D] {n_cams} cameras: {int(seen.sum())} of {xyz.shape[0]} seen, {int(near.sum())} within 8 ulp of a boundary, "
          f"max ulp vs fp32 loop {int(d[~near].max())} away from boundaries ({int(bad.sum())} rows beyond 2 ulp), max rel vs fp64 "
          f"{float(((f.double() - ref64).abs() / ref64)[~near].max()):.2e}")
    # every disagreement beyond 2 ulp is a point within a few ulp of a boundary (whose max over the seen rows may move the unseen)
    unseen = ~seen
    assert bool(near[bad & seen].all()), "a decision differs away from any boundary"
    assert float(((f.double() - ref64).abs() / ref64)[~near & seen].max()) < 4e-6      # fp32 depths, a few ulp of them
    assert bool((f[unseen & ~near] == f[seen].max()).all())                             # unseen rows: the largest seen distance


def test_filter_edge_cases():
    xyz = torch.randn(1000, 3)
    m = SimpleNamespace(get_xyz=xyz.to(DEV))
    assert torch.equal(mip.compute_3D_filter(m, []).cpu(), torch.zeros(1000, 1))            # no camera: zeros
    behind = F3.camera(torch.diag(torch.tensor([1.0, 1.0, -1.0, 1.0])), 64, 48, 1.0, 0.8)
    xyz[:, 2] = xyz[:, 2].abs() + 1.0
    m = SimpleNamespace(get_xyz=xyz.to(DEV))
    assert torch.equal(mip.compute_3D_filter(m, [behind]).cpu(), torch.zeros(1000, 1))      # nothing seen: zeros
    m = SimpleNamespace(get_xyz=torch.zeros(0, 3, device=DEV))
    assert mip.compute_3D_filter(m, _cams(3, 1)).shape == (0, 1)


# ---- 2./3. the forward --------------------------------------------------------------------------------------------------------

W, H = 96, 64
BG = torch.tensor([0.2, 0.4, 0.6])


def _scene(seed, P=3000, ls=0.02):
    return synth.make_scene(P, seed, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(ls), M=16)


def _filter(P, seed, zero_frac=0.3, scale=0.02):
    g = torch.Generator().manual_seed(seed)
    f = torch.rand(P, generator=g) * scale
    f[torch.rand(P, generator=g) < zero_frac] = 0.0
    return f


def _raw(scene):
    return (scene.sh[:, :1].contiguous().to(DEV), scene.sh[:, 1:].contiguous().to(DEV), torch.log(scene.scales).to(DEV),
            scene.rotations.to(DEV).contiguous())


def _fwd(path, scene, cam, f=None, quant=None, maps=True, dbg=None):
    """-> (args, outputs) of _C.rasterize_gaussians on `path` (dense, raw, quant, aa)."""
    args = list(O.forward_args(scene, cam, BG))
    kw = dict(return_maps=maps, debug_out=dbg, antialiasing=path == "aa")
    if path == "raw":
        kw["raw"] = _raw(scene)
        args[4] = args[5] = args[14] = O.EMPTY
    if path == "quant":
        kw["quant"] = quant.to(DEV)
    if f is not None:
        kw["filter_3D"] = f.to(DEV)
    return args, _C.rasterize_gaussians(*args, **kw)


PATHS = ["dense", "raw", "quant", "aa"]


def _config(path, seed):
    scene = _scene(seed)
    quant = synth.quantise_scene(scene) if path == "quant" else None
    if quant is not None:
        scene = quant.dequantise()
    if path == "raw":
        scene.scales = torch.exp(torch.log(scene.scales))
    return scene, quant, O.yaw_cam(W, H, 4.0, dev=DEV)


@pytest.mark.parametrize("path", PATHS)
def test_zero_filter_is_the_call_without_one(path):
    scene, quant, cam = _config(path, 301)
    d0, d1 = {}, {}
    _, a = _fwd(path, scene, cam, None, quant, dbg=d0)
    _, b = _fwd(path, scene, cam, torch.zeros(scene.P, 1), quant, dbg=d1)
    assert a[0] == b[0] > 0
    for i in (1, 2, 6, 7):
        assert O.same(a[i], b[i]), i
    for k in d0:
        assert O.same(d0[k], d1[k]), k
    s0, s1 = O.state(a, cam, scene.P), O.state(b, cam, scene.P)
    for k in s0:
        assert torch.equal(s0[k], s1[k]), k


def _activated(path, scene, quant):
    """The activated scales and rotations the kernels use (the fused de-quantisation's own values for quant)."""
    if path == "quant":
        s, r = _C.debug_dequant(quant.to(DEV))
        return s, r
    return scene.scales.to(DEV), scene.rotations.to(DEV)


@pytest.mark.parametrize("path", PATHS)
def test_filtered_geometry_is_a_render_on_the_filtered_scales(path):
    scene, quant, cam = _config(path, 302)
    f = _filter(scene.P, 303).to(DEV)
    s, r = _activated(path, scene, quant)
    if path == "raw":
        s, r = torch.exp(_raw(scene)[2]), torch.nn.functional.normalize(_raw(scene)[3])
    sp, c3 = F3.filtered(s, f)
    d1, d0 = {}, {}
    _, fo = _fwd(path, scene, cam, f, quant, dbg=d1)
    # the same scene, unfiltered, on torch's sqrt(s^2 + f^2) (dense path, kernel-exact rotations and SH)
    ref = synth.Scene(scene.means3D, scene.opacity, sp.cpu(), r.cpu(), scene.sh, scene.degrees)
    _, no = _fwd("aa" if path == "aa" else "dense", ref, cam, None, None, dbg=d0)
    assert torch.equal(fo[2], no[2])
    for k in ("cov3D", "means2D", "depths"):
        assert O.same(d1[k], d0[k]), k
    assert O.same(d1["conic_opacity"][:, :3], d0["conic_opacity"][:, :3])
    vis = fo[2] > 0
    # the opacity: the fp32 product of the kernel's own sigmoid (a plain render's) and c3
    dp = {}
    _fwd("dense", ref, cam, None, None, dbg=dp)
    want = dp["conic_opacity"][:, 3] * c3
    got = d1["conic_opacity"][:, 3]
    if path != "aa":
        assert O.same(got[vis], want[vis])
    else:
        # times the AA factor s, restated in float64 from the kernel's cov3D (as test_gpu_antialias.py does)
        a_, b_, c_ = R64.screen_cov(scene.means3D.to(DEV, F64), cam.world_view_transform.to(DEV, F64), d1["cov3D"].to(F64), W, H,
                                    math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5))[2:]
        aa = torch.sqrt(torch.clamp((a_ * c_ - b_ * b_) / ((a_ + 0.3) * (c_ + 0.3) - b_ * b_), min=2.5e-5))
        rel = ((got.to(F64) - want.to(F64) * aa).abs() / (want.to(F64) * aa))[vis]
        print(f"\n[filter_3D aa] opacity vs sigmoid * c3 * s(fp64): max rel {float(rel.max()):.2e}")
        assert float(rel.max()) < 1e-3
    assert int(vis.sum()) > 500 and float(c3[vis].min()) < 0.9


# ---- 4. gradients -------------------------------------------------------------------------------------------------------------

def _grad_scene(seed, P=2000):
    """The rows of filter3d_restatement.edge_rows: zero filters, moderate ones, f >> s with c3 in [5e-3, 0.05] at a high sigmoid,
    flat splats with an axis of 1e-6 that still composite, and a few with an axis of exactly 0.  -> (scene, f, kind)."""
    scene = _scene(seed, P, ls=0.01)
    f, kind = F3.edge_rows(scene, seed + 1)
    return scene, f, kind


def _bwd(path, args, out, dL, f, quant=None, raw=None, **kw):
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, Hh, Ww, sh, degrees, campos, _, _) = args
    extra = dict(antialiasing=path == "aa", **kw)
    if raw is not None:
        extra["raw"] = raw
    if quant is not None:
        extra["quant"] = quant.to(DEV)
    if f is not None:
        extra.update(filter_3D=f.to(DEV), opacity=opacity)
    R, color, radii, geom, binning, img = out[:6]
    return _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, view, proj, tx, ty, dL.to(DEV), sh,
                                           degrees, campos, geom, R, binning, img, 0.0, False, **extra)


def _run(path, scene, cam, f, quant=None, dL=None, **kw):
    args, out = _fwd(path, scene, cam, f, quant, maps=False)
    return args, out, _bwd(path, args, out, dL, f, quant, _raw(scene) if path == "raw" else None, **kw)


def _chain_reference(path, scene, cam, f, dL, quant=None):
    """The filtered scale and logit gradients restated in float64 from an UNfiltered render on (s', logit(sigmoid * c3)): its
    scale gradient g (w.r.t. s') and G = dL/dlogit' / (sigma' (1 - sigma')) = dL/do^ a are the kernel's own screen-space chain."""
    s, r = _activated(path, scene, quant)
    if path == "raw":
        s, r = torch.exp(_raw(scene)[2]), torch.nn.functional.normalize(_raw(scene)[3])
    sp, c3 = F3.filtered(s, f.to(DEV))
    sig = torch.sigmoid(scene.opacity.to(DEV, F64).view(-1))
    p = sig * c3.to(F64)
    ok = p > 1e-30
    logit_p = torch.log(p / (1 - p)).float()
    ref_scene = synth.Scene(scene.means3D, torch.where(ok, logit_p, torch.zeros_like(logit_p)).view(-1, 1).cpu(), sp.cpu(), r.cpu(),
                            scene.sh, scene.degrees)
    _, out, g = _run("aa" if path == "aa" else "dense", ref_scene, cam, None, None, dL)
    g_m2 = g[0]
    sig_p = torch.sigmoid(ref_scene.opacity.to(DEV, F64).view(-1))
    G = g[2].to(F64).view(-1) / (sig_p * (1 - sig_p))
    s64, f64 = s.to(F64), f.to(DEV, F64)
    sp64, c364 = F3.filtered64(s64, f64)
    rr = (s64 * s64) / (sp64 * sp64)
    dc3 = torch.stack([torch.sqrt(rr[:, (k + 1) % 3] * rr[:, (k + 2) % 3]) * (1 - rr[:, k]) / sp64[:, k] for k in range(3)], 1)
    nz = (f64 != 0)[:, None]
    ds = torch.where(nz, g[6].to(F64) * s64 / sp64 + (G * sig)[:, None] * dc3, g[6].to(F64))
    dlogit = torch.where(nz[:, 0], G * c364 * sig * (1 - sig), g[2].to(F64).view(-1))
    return ds, dlogit, ok & (out[2] > 0), s, g_m2


def _row_ratio(got, ref, rows, r_rel=1e-4, a_abs=1e-6):
    """Largest e / max(r_rel |ref|_row, a_abs max|ref|) over the Gaussians `rows`, e = |got - ref| per element."""
    got, ref = got.to(F64).reshape(got.shape[0], -1), ref.to(F64).reshape(ref.shape[0], -1)
    e = (got - ref).abs()
    bar = torch.clamp((r_rel * ref.abs().amax(1, keepdim=True)), min=a_abs * float(ref[rows].abs().max()))
    return float((e / bar)[rows].max())


def _rel(a, b, rows):
    a, b = a[rows].to(F64), b[rows].to(F64)
    return float((a - b).abs().max()) / (float(b.abs().max()) + 1e-30)


@pytest.mark.parametrize("path", PATHS)
def test_gradient_chain_against_float64(path):
    scene, f, kind = _grad_scene(401 + PATHS.index(path))
    quant = None
    if path == "quant":
        quant = synth.quantise_scene(scene)
        scene = quant.dequantise()
    cam = O.yaw_cam(W, H, 2.0, dev=DEV)
    dL = torch.randn(3, H, W, generator=torch.Generator().manual_seed(7))
    args, out, g = _run(path, scene, cam, f, quant, dL)
    ds, dlogit, rows, s, g_m2 = _chain_reference(path, scene, cam, f, dL, quant)
    if path == "raw":
        ds = ds * s                                       # raw: dL/d_scaling = dL/ds * s
    got_s = g[7] if path == "raw" else g[6]
    got_o = g[2].view(-1)
    for t in g:
        if t is not None:
            assert bool(torch.isfinite(t).all())
    # rows whose filtered opacity is exactly 0 (an exactly flat axis): nothing to compare against, the logit gradient is 0
    dead = (out[2] > 0) & ~rows
    # the unfiltered reference renders sigmoid(fl32(logit(sigmoid * c3))), a few ulp from the kernel's fl32(sigmoid * c3): a pair at
    # the 1/255 alpha threshold may go the other way.  Such a row's screen-space gradient, which the new chain does not touch,
    # differs too; the rows whose dL/dmeans2D agrees to 1e-4 took the same decisions and are compared
    agree = ((g[0] - g_m2).abs().amax(1) <= 1e-4 * g_m2.abs().amax(1) + 1e-12) & rows
    # per Gaussian: e <= max(1e-4 |ref|_row, 1e-6 max|ref|) (backward_edges.compare's R_REL / A_ABS without the E32 term)
    es, eo = _row_ratio(got_s, ds, agree), _row_ratio(got_o, dlogit, agree)
    kinds = torch.from_numpy(kind).to(DEV)
    live = agree & (dlogit != 0)                                          # rows whose pairs composite
    counts = {k: int((live & (kinds == i)).sum()) for i, k in enumerate(F3.EDGE_KINDS)}
    print(f"\n[filter_3D grad] {path}: max e / bar dL/ds {es:.3f}, dL/dlogit {eo:.3f} over {int(agree.sum())} of {int(rows.sum())} "
          f"rows with the same decisions, compositing rows per kind {counts}; {int(dead.sum())} rows of zero opacity")
    assert int(agree.sum()) > 0.5 * int(rows.sum()) and int(agree.sum()) > 300
    if path != "quant":                                   # the codebooks move the scales off the kinds' targets
        assert counts["strong"] >= 20 and counts["flat"] >= 20, counts
    assert es <= 1.0 and eo <= 1.0
    if path != "raw" and bool(dead.any()):
        assert float(got_o[dead].abs().max()) == 0.0


def test_raw_quant_camera_and_deterministic_paths_agree():
    scene, f, _ = _grad_scene(411)
    cam = O.yaw_cam(W, H, 2.0, dev=DEV)
    dL = torch.randn(3, H, W, generator=torch.Generator().manual_seed(8))
    _, _, gd = _run("dense", scene, cam, f, None, dL)
    _, _, gr = _run("raw", scene, cam, f, None, dL)
    s = torch.exp(_raw(scene)[2])
    vis = gd[6].abs().sum(1) > 0
    assert _rel(gr[7], gd[6] * s, vis) < 1e-5 and _rel(gr[2], gd[2], vis) < 1e-5
    _, _, gc = _run("dense", scene, cam, f, None, dL, camera_grads=True)
    for i in range(8):
        assert _rel(gc[i], gd[i], slice(None)) < 1e-5, i
    assert all(bool(torch.isfinite(t).all()) for t in gc[8:11])
    _, _, g1 = _run("dense", scene, cam, f, None, dL, deterministic=True)
    _, _, g2 = _run("dense", scene, cam, f, None, dL, deterministic=True)
    for a, b in zip(g1, g2):
        assert O.same(a, b)
    for i in range(8):
        assert _rel(g1[i], gd[i], slice(None)) < 1e-4, i
    # quantised: quant.grads-style outputs against the dense path on the de-quantised scene
    quant = synth.quantise_scene(scene)
    dq = quant.dequantise()
    sdq, rdq = _C.debug_dequant(quant.to(DEV))
    dense = synth.Scene(dq.means3D, dq.opacity, sdq.cpu(), rdq.cpu(), dq.sh, dq.degrees)
    _, _, gq = _run("quant", dq, cam, f, quant, dL)
    _, _, gdq = _run("dense", dense, cam, f, None, dL)
    for i in (2, 6):
        assert _rel(gq[i], gdq[i], slice(None)) < 1e-5, i


def test_antialiased_filter_against_the_float64_pipeline():
    Wt = Ht = 32
    scene = synth.make_scene(48, 421, mixed_degrees=True, box=(1.3, 1.3, 0.8), log_scale_mean=math.log(0.05), M=16, near_frac=0.0)
    f = torch.rand(48, generator=torch.Generator().manual_seed(422)) * 0.04
    f[::5] = 0.0
    cam = O.yaw_cam(Wt, Ht, 3.0)
    bg = torch.tensor([0.3, 0.2, 0.1], device=DEV)
    gen = torch.Generator().manual_seed(423)
    args = O.forward_args(scene, cam, bg)
    out = _C.rasterize_gaussians(*args, antialiasing=True, return_maps=True, filter_3D=f.to(DEV))
    Gc = torch.randn(3, Ht, Wt, generator=gen)
    g = _C.rasterize_gaussians_backward(*args[:1], args[1], out[2], args[2], args[4], args[5], 1.0, args[7], args[8], args[9], args[10],
                                        args[11], Gc.to(DEV), args[14], args[15], args[16], out[3], out[0], out[4], out[5], 0.0, False,
                                        antialiasing=True, filter_3D=f.to(DEV), opacity=args[3])
    st = O.state(out, cam, scene.P)
    vis = out[2] > 0
    tiles = [st["point_list"][int(r0):int(r1)].long() for r0, r1 in st["ranges"].tolist()]
    leaf = lambda v: v.to(DEV, F64).detach().clone().requires_grad_(True)  # noqa: E731
    s, logit = leaf(scene.scales), leaf(scene.opacity)
    sp, c3 = F3.filtered64(s, f.to(DEV, F64))
    p = torch.sigmoid(logit.view(-1)) * c3
    x = dict(means=leaf(scene.means3D), logit=torch.log(p / (1 - p)), view=leaf(cam.world_view_transform),
             proj=leaf(cam.full_proj_transform), campos=leaf(cam.camera_center), scales=sp, rots=leaf(scene.rotations),
             sh=leaf(scene.sh), deg=scene.degrees.to(DEV))
    col, invd, alpha, nc, mid, (margin_a, margin_t) = render64(x, cam, bg, vis, tiles)
    assert torch.equal(nc, st["n_contrib"].long()), "compositing decisions differ from the kernel's"
    e_img = float((out[1].to(F64) - col.detach()).abs().max())
    (col * Gc.to(DEV, F64)).sum().backward()
    errs = dict(dL_dscales=_rel(g[6], s.grad, vis), dL_dopacity=_rel(g[2].view(-1), logit.grad.view(-1), vis),
                dL_dmeans3D=_rel(g[3], x["means"].grad, vis))
    print(f"\n[filter_3D aa fp64] image {e_img:.2e}; gradients {errs}")
    assert e_img <= 1e-5
    for k, e in errs.items():
        assert e <= 2e-4, (k, e)


# ---- 5. training --------------------------------------------------------------------------------------------------------------

def test_training_with_the_filter():
    from test_gpu_fused_activations import Model, _adam, _render
    from gs_b200 import densify
    from utils.loss_utils import l1_ssim_loss
    torch.manual_seed(3)
    Wt, Ht = 128, 96
    target = synth.make_scene(8_000, 431, sh_degree=3, box=(1.9 * Wt / Ht, 1.9, 1.0), log_scale_mean=math.log(0.03))
    cams = [O.yaw_cam(Wt, Ht, yaw) for yaw in (-8.0, 0.0, 8.0)]
    with torch.no_grad():
        gts = [_render(Model(target, 15, norm_range=(0.0, 0.0)), c, False)["render"].clone() for c in cams]
    g = torch.Generator().manual_seed(432)
    start = synth.Scene(target.means3D + 0.01 * torch.randn(target.means3D.shape, generator=g), target.opacity - 1.0,
                        target.scales * 1.3, target.rotations, target.sh + 0.1 * torch.randn(target.sh.shape, generator=g),
                        target.degrees)
    m = Model(start, 15)
    m.optimizer = _adam(m)
    m.percent_dense = 0.01
    P = m._xyz.shape[0]
    m.xyz_gradient_accum, m.denom, m.max_radii2D = torch.zeros(P, 1, device=DEV), torch.zeros(P, 1, device=DEV), torch.zeros(P, device=DEV)
    cam_objs = [F3.camera(c.world_view_transform, c.image_width, c.image_height, c.FoVx, c.FoVy) for c in cams]
    mip.compute_3D_filter(m, cam_objs)
    losses, sizes = [], [P]
    for it in range(40):
        k = it % len(cams)
        m.optimizer.zero_grad(set_to_none=True)
        pkg = _render(m, cams[k], it % 2 == 0)
        loss = l1_ssim_loss(pkg["render"], gts[k], 0.2)
        loss.backward()
        densify.add_densification_stats(m, pkg["viewspace_points"], pkg["visibility_filter"], pkg["radii"])
        m.optimizer.step()
        losses.append(float(loss.detach()))
        assert math.isfinite(losses[-1])
        if it == 19:
            densify.densify_and_prune(m, 1e-7, 0.005, 2.0, None, {})
            assert m.filter_3D.shape == (m._xyz.shape[0], 1)
            sizes.append(m._xyz.shape[0])
        if it % 5 == 4:
            mip.compute_3D_filter(m, cam_objs)
    print(f"\n40 steps with the 3D filter: loss {sum(losses[:3]) / 3:.4f} -> {sum(losses[-3:]) / 3:.4f}, P {sizes}")
    assert sum(losses[-3:]) < sum(losses[:3]) and sizes[1] != sizes[0]
    feats = torch.rand(m._xyz.shape[0], 2, device=DEV)
    pkg = _render(m, cams[0], False, features=feats)
    assert bool(torch.isfinite(pkg["features"]).all())
    pkg = _render(m, cams[1], True, absgrad=True)
    pkg["render"].sum().backward()
    assert bool(torch.isfinite(pkg["viewspace_points_abs"].grad).all())


# ---- 4b. per element against the fp64 oracle on the backward-edge scenes ------------------------------------------------------

def _filtered_oracle(case, f, aa, o_hat, dL=None, fwd=None):
    """The oracle's fp64 and fp32 backwards of the filtered scene, with the filter's chain applied in float64 per Gaussian.
    The oracle runs on the filtered scales s' (torch's fp32 sqrt(s^2 + f^2), the kernel's own) with the forward state's opacity
    replaced by the kernel's o^ (`o_hat`, which the test holds to fl32(sigmoid * c3), times s with AA; the AA chain differentiates
    at sigmoid * c3), and its render re-run on it.  Its dL/dlogit is then dL/do^ * o^ (1 - o^) (AA: dL/do^ s sg (1 - sg), sg = sigmoid * c3), from which A = dL/do^ a is
    recovered; dL/ds = g s / s' + A sigmoid dc3/ds and dL/dlogit = A c3 sigmoid (1 - sigmoid) on the rows with f != 0.
    -> (state, o64, o32, sigmoid, c3 fp32)."""
    import gs_oracle
    s = case.scene
    sp, c3 = F3.filtered(s.scales, f)
    kw = case.cam_kw()
    if fwd is None:
        fwd = gs_oracle.forward(s.means3D, s.opacity, sp, s.rotations, s.sh, s.degrees, bg=case.bg, antialiasing=aa, **kw)
        sig = (fwd["aa_sigmoid"] if aa else fwd["conic_opacity"][:, 3]).astype(np.float32).copy()
        c3n = c3.numpy()
        sc = (sig * c3n).astype(np.float32)
        fwd["sigma"] = sig
        fwd["o_hat_oracle"] = (sc * fwd["aa_s"]).astype(np.float32) if aa else sc
        fwd["conic_opacity"][:, 3] = o_hat
        if aa:
            fwd["aa_sigmoid"] = sc
        fwd.update(gs_oracle.render_forward(fwd, fwd, case.bg, case.W, case.H))
    sig = fwd["sigma"].astype(np.float64)
    bk = dict(bg=case.bg, lambda_sh_sparsity=case.lam, antialiasing=aa, **kw)
    dL = case.dL if dL is None else dL
    outs = [gs_oracle.backward(fwd, dL, s.means3D, sp, s.rotations, s.sh, s.degrees, f64=d, **bk) for d in (True, False)]
    s64 = s.scales.numpy().astype(np.float64)
    f64 = f.numpy().astype(np.float64)
    sp64 = np.sqrt(s64 * s64 + (f64 * f64)[:, None])
    c364 = np.prod(s64 / np.where(sp64 > 0, sp64, 1.0), 1)
    rr = (s64 * s64) / np.where(sp64 > 0, sp64 * sp64, 1.0)
    dc3 = np.stack([np.sqrt(rr[:, (k + 1) % 3] * rr[:, (k + 2) % 3]) * (1 - rr[:, k]) / np.where(sp64[:, k] > 0, sp64[:, k], 1.0)
                    for k in range(3)], 1)
    nz = f64 != 0
    o_hat = fwd["aa_sigmoid"] if aa else fwd["conic_opacity"][:, 3]
    o_hat = o_hat.astype(np.float64)
    for g in outs:
        dlo = np.asarray(g["dL_dopacity"], np.float64).reshape(-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            A = np.where(o_hat * (1 - o_hat) > 0, dlo / (o_hat * (1 - o_hat)), 0.0)
        gs = np.asarray(g["dL_dscales"], np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            ds = np.where(nz[:, None], gs * s64 / np.where(sp64 > 0, sp64, 1.0) + (A * sig)[:, None] * dc3, gs)
        g["dL_dscales"] = ds
        g["dL_dopacity"] = np.where(nz, A * c364 * sig * (1 - sig), dlo).reshape(-1, 1)
    return fwd, outs[0], outs[1]


FILTER_EDGE_CASES = [("staircase", False), ("odd_20x36", False), ("large", False), ("saturation", False), ("dense_4k", False),
                     ("aa_subpixel", True), ("odd_20x36", True), ("dense_4k", True)]


@pytest.mark.parametrize("name,aa", FILTER_EDGE_CASES)
def test_filtered_backward_per_element_against_fp64_oracle(name, aa):
    import backward_edges as BE
    case = BE.build(name, aa=aa)
    f, kind = F3.edge_rows(case.scene, 431 + FILTER_EDGE_CASES.index((name, aa)))
    args = O.forward_args(case.scene, case.cam, case.bg)
    dbg = {}
    out = _C.rasterize_gaussians(*args, antialiasing=aa, filter_3D=f.to(DEV), debug_out=dbg)
    got_o = dbg["conic_opacity"][:, 3].cpu().numpy()
    o, o64, o32 = _filtered_oracle(case, f, aa, got_o)
    excl = BE.excluded(case, o)
    st = O.state(out, case.cam, case.scene.P)
    assert out[0] == int(o["num_rendered"])
    for k in ("radii", "keys", "point_list", "ranges"):
        mine = out[2] if k == "radii" else st[k]
        assert np.array_equal(np.asarray(o[k]).reshape(-1).astype(np.int64), mine.cpu().numpy().reshape(-1).astype(np.int64)), k
    vis = o["radii"] > 0
    # o^ against fl32(sigmoid * c3) (times s) from the oracle's own sigmoid (and s), which may differ from the kernel's by an ulp
    u = np.abs(got_o.view(np.int32).astype(np.int64) - o["o_hat_oracle"].view(np.int32).astype(np.int64))[vis]
    print("\n[%s%s, filter_3D] o^: max %d ulp from fl32(sigmoid * c3)%s of the oracle, %d of %d bit-identical"
          % (name, ", aa" if aa else "", int(u.max()), " * s" if aa else "", int((u == 0).sum()), int(vis.sum())))
    assert int(u.max()) <= 16
    nb = ~o["borderline"]
    assert np.array_equal(o["n_contrib"][nb], st["n_contrib"].cpu().numpy()[nb]), "n_contrib"

    def run(dL):
        g = _C.rasterize_gaussians_backward(args[0], args[1], out[2], args[2], args[4], args[5], 1.0, args[7], args[8], args[9],
                                            args[10], args[11], dL.to(DEV), args[14], args[15], args[16], out[3], out[0], out[4],
                                            out[5], case.lam, False, antialiasing=aa, want_conic=True, filter_3D=f.to(DEV),
                                            opacity=args[3])
        return {n: t.cpu().numpy() for n, t in zip(BE.ARRAYS, g)}
    bar = BE.BAR_CASE.get(name, (BE.R_REL, BE.A_ABS))
    cmp = (lambda *a, **k: BE.compare_aa(*a, **k)) if aa else (lambda label, case_, *a, **k: BE.compare(label, *a, **k)[1])
    got = run(case.dL)
    label = "%s%s, filter_3D" % (name, ", aa" if aa else "")
    failures = cmp(label, case, o, o64, o32, got, ~excl, glob=(excl, BE.EXCLUDED_BAR), bar=bar)
    assert not failures, "\n" + BE.describe(failures, o, o64, got, case.W, case.H)
    if excl.any():
        dL = case.dL.clone()
        dL[:, torch.from_numpy(o["borderline"])] = 0.0
        _, m64, m32 = _filtered_oracle(case, f, aa, got_o, dL=dL, fwd=o)
        mgot = run(dL)
        failures = cmp(label + ", borderline dL = 0", case, o, m64, m32, mgot, np.ones_like(excl), bar=bar)
        assert not failures, "\n" + BE.describe(failures, o, m64, mgot, case.W, case.H)
    # which rows were held to the per-element bar: every kind composites (strong: c3 in [5e-3, 0.05]; flat: an axis of 1e-6)
    chk = vis & ~excl & (np.abs(o64["dL_dopacity"]).reshape(-1) > 0)
    counts = {k: int((chk & (kind == i)).sum()) for i, k in enumerate(F3.EDGE_KINDS)}
    flat0 = vis & (kind == 4)
    print("[%s] per element, compositing rows per kind: %s; exactly flat rows visible: %d (all gradients 0)" % (label, counts, int(flat0.sum())))
    for n in BE.ARRAYS:
        if n != "dL_dsh":                                 # the SH sparsity term reaches every visible row
            assert not np.asarray(got[n]).reshape(case.scene.P, -1)[flat0].any(), n
    assert counts["strong"] > 0 and counts["flat"] > 0 and counts["moderate"] > 0 and counts["zero"] > 0, counts
