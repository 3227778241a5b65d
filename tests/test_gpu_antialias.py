"""GPU: anti-aliased rendering (`antialiasing=True`, the requests' `antialiasing` field, DESIGN.md §5e).
  1. nothing else moves: radii, tiles, depths, means2D, conic, cov3D, rgb, clamped, R, sorted keys and point_list are bit-identical
     with and without anti-aliasing, and without it conic_opacity[:,3] is the plain sigmoid;
  2. the effective opacity is sigmoid * s, s = sqrt(max(2.5e-5, det0 / det1)), against float64;
  3. a float64 torch restatement of the whole pipeline (AA preprocess, front-to-back compositing with the reference's skip,
     saturate and stop rules, the maps) gives the colour, the maps and every gradient, camera included;
  4. resolution invariance, the point of the feature: one small Gaussian keeps its total alpha across a 4x zoom only with AA;
  5. equivalences: quantised == de-quantised, pruned == compacted, accumulate == sum of calls, quant.grads accumulates;
  6. a second device.
Translation / rotation invariance with the camera, the same bytes on every run and stream and P = 0 / R = 0 are checked with and
without anti-aliasing in test_gpu_camera.py, and Adam steps through render() with pipe.antialiasing in test_gpu_training.py.
Observed maxima are printed (pytest -s)."""
import math
from functools import partial
from types import SimpleNamespace

import pytest
import torch

import ours as O
import restate64 as R64
from render64 import render64
from diff_gaussian_rasterization import _C
from gs_b200 import synth
from gs_b200.model import GaussianModelView

pytestmark = pytest.mark.gpu

DEV = "cuda"
F64 = torch.float64
H_DIL = 0.3


def _config(name):
    """-> (scene, cam on DEV, prune_mask or None, quant or None)."""
    scene, cam, prune, quant = O.scene_config("aa", name)
    return scene, cam.to(DEV), prune, quant


# every call here is anti-aliased unless it passes aa=False
_forward = partial(O.forward, aa=True)
_backward = partial(O.backward, aa=True)


def _rel(a, b):
    """max |a - b| / max |b|."""
    a, b = a.to(F64), b.to(F64)
    return float((a - b).abs().max()) / (float(b.abs().max()) + 1e-30)


# ---- 1./2. nothing else moves; the effective opacity --------------------------------------------------------------------------

def _cov2D64(means, cov3D, cam):
    """Undilated screen covariance (a, b, c) in float64 from the kernel's own cov3D, following computeCov2D."""
    return R64.screen_cov(means.to(DEV, F64), cam.world_view_transform.to(DEV, F64), cov3D.to(DEV, F64), cam.image_width,
                          cam.image_height, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5))[2:]


@pytest.mark.parametrize("name", ["c1", "quant", "pruned"])
def test_antialiasing_moves_nothing_but_the_opacity(name):
    scene, cam, prune, quant = _config(name)
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    d0, d1 = {}, {}
    _, plain = _forward(scene, cam, bg, prune, quant, aa=False, dbg=d0)
    _, aa = _forward(scene, cam, bg, prune, quant, aa=True, dbg=d1)
    assert plain[0] == aa[0] and plain[0] > 0 and O.same(plain[2], aa[2])
    for k in ("depths", "means2D", "cov3D", "rgb", "tiles_touched", "clamped"):
        assert O.same(d0[k], d1[k]), k
    assert O.same(d0["conic_opacity"][:, :3], d1["conic_opacity"][:, :3])
    st0, st1 = O.state(plain, cam, scene.P), O.state(aa, cam, scene.P)
    for k in ("keys", "point_list", "ranges"):
        assert torch.equal(st0[k], st1[k]), k
    vis = plain[2] > 0
    logit = (quant.dequantise().opacity if quant is not None else scene.opacity).to(DEV).view(-1)
    sig = torch.sigmoid(logit.to(F64))
    # without AA: the plain sigmoid (the kernel's expf sequence is within 2 ulp of it)
    assert float((d0["conic_opacity"][vis, 3].to(F64) - sig[vis]).abs().max()) <= 3e-7
    # with AA: sigmoid * s in float64, from the undilated cov2D of the kernel's cov3D
    a, b, c = _cov2D64(scene.means3D, d1["cov3D"], cam)
    det0, det1 = a * c - b * b, (a + H_DIL) * (c + H_DIL) - b * b
    s = torch.sqrt(torch.clamp_min(det0 / det1, 2.5e-5))
    err = float((d1["conic_opacity"][vis, 3].to(F64) - (sig * s)[vis]).abs().max())
    print(f"\n[antialias] {name}: max |o^ - sigmoid * s| = {err:.3e} (bar 1e-5); s in [{float(s[vis].min()):.4f}, {float(s[vis].max()):.4f}]")
    assert err <= 1e-5
    assert float(s[vis].min()) < 0.5                                           # the scene has sub-pixel splats
    # lower opacities let more light through on the whole (not at every pixel: near saturation the early stop comes later)
    assert not torch.equal(plain[1], aa[1]) and float(st1["final_T"].mean()) > float(st0["final_T"].mean())


# ---- 3. float64 restatement of the pipeline (render64.py) ----------------------------------------------------------------------

def _tiny_scene(seed, P=48):
    return synth.make_scene(P, seed, mixed_degrees=True, box=(1.3, 1.3, 0.8), log_scale_mean=math.log(0.05), M=16, near_frac=0.0)


@pytest.mark.parametrize("case", ["sh", "colors_precomp", "cov3D_precomp", "maps_only"])
def test_antialiasing_against_a_float64_restatement(case):
    W = H = 32
    scene = _tiny_scene({"sh": 211, "colors_precomp": 212, "cov3D_precomp": 213, "maps_only": 214}[case])
    cam = O.yaw_cam(W, H, 3.0)
    bg = torch.tensor([0.3, 0.2, 0.1], device=DEV)
    gen = torch.Generator().manual_seed(215)
    extra = {}
    if case == "colors_precomp":
        extra["colors_precomp"] = torch.rand(scene.P, 3, generator=gen)
    if case == "cov3D_precomp":
        extra["cov3D_precomp"] = R64.cov3D_from(scene.scales.to(F64), scene.rotations.to(F64)).float()
    dbg = {}
    args, out = _forward(scene, cam, bg, extra=extra, maps=True, dbg=dbg)
    Gc = torch.zeros(3, H, W) if case == "maps_only" else torch.randn(3, H, W, generator=gen)
    Gd, Ga = torch.randn(1, H, W, generator=gen), torch.randn(1, H, W, generator=gen)
    g = _backward(args, out, Gc, dL_dinvdepth=Gd.to(DEV), dL_dalpha=Ga.to(DEV), camera_grads=True)
    st = O.state(out, cam, scene.P)
    vis = out[2] > 0
    assert int(vis.sum()) >= 30
    tiles = [st["point_list"][int(r0):int(r1)].long() for r0, r1 in st["ranges"].tolist()]
    leaf = lambda v: v.to(DEV, F64).detach().clone().requires_grad_(True)
    x = dict(means=leaf(scene.means3D), logit=leaf(scene.opacity), view=leaf(cam.world_view_transform),
             proj=leaf(cam.full_proj_transform), campos=leaf(cam.camera_center))
    if "cov3D_precomp" in extra:
        x["cov3D"] = leaf(extra["cov3D_precomp"])
    else:
        x["scales"], x["rots"] = leaf(scene.scales), leaf(scene.rotations)
    if "colors_precomp" in extra:
        x["colors"] = leaf(extra["colors_precomp"])
    else:
        x["sh"], x["deg"] = leaf(scene.sh), scene.degrees.to(DEV)
    col, invd, alpha, nc, mid, (margin_a, margin_t) = render64(x, cam, bg, vis, tiles)
    # the restatement took the kernel's decisions: the same last contributor everywhere, and no pair near a threshold
    assert torch.equal(nc, st["n_contrib"].long()), "compositing decisions differ from the kernel's"
    assert margin_a > 1e-7 and margin_t > 1e-9, (margin_a, margin_t)
    e_img = max(float((out[1].to(F64) - col.detach()).abs().max()), float((out[6].to(F64) - invd.detach()).abs().max()),
                float((out[7].to(F64) - alpha.detach()).abs().max()))
    loss = (col * Gc.to(DEV, F64)).sum() + (invd * Gd.to(DEV, F64)).sum() + (alpha * Ga.to(DEV, F64)).sum()
    loss.backward()
    ref = dict(dL_dmeans2D=mid["ndc"].grad, dL_dopacity=x["logit"].grad, dL_dmeans3D=x["means"].grad,
               view=x["view"].grad, proj=x["proj"].grad, campos=x["campos"].grad)
    got = dict(dL_dmeans2D=g[0][:, :2], dL_dopacity=g[2], dL_dmeans3D=g[3], view=g[8], proj=g[9], campos=g[10])
    if "colors" in x:
        ref["dL_dcolors"], got["dL_dcolors"] = x["colors"].grad, g[1]
    else:
        ref["dL_dcolors"], got["dL_dcolors"] = mid["rgb"].grad, g[1]
        ref["dL_dsh"], got["dL_dsh"] = x["sh"].grad, g[5]
    if "cov3D" in x:
        ref["dL_dcov3D"], got["dL_dcov3D"] = x["cov3D"].grad, g[4]
    else:
        ref["dL_dscales"], got["dL_dscales"] = x["scales"].grad, g[6]
        ref["dL_drotations"], got["dL_drotations"] = x["rots"].grad, g[7]
    # an input the loss does not depend on (campos without SH colours, the colours under a loss on the maps alone) must get zeros
    zero = [k for k in ref if ref[k] is None or float(ref[k].abs().max()) == 0]
    for k in zero:
        assert float(got[k].abs().max()) == 0.0, k
    errs = {k: _rel(got[k].reshape(ref[k].shape), ref[k]) for k in ref if k not in zero}
    worst = max(errs.items(), key=lambda kv: kv[1])
    print(f"\n[antialias fp64] {case}: image/maps max |diff| = {e_img:.3e} (bar 1e-5); worst gradient {worst[0]} {worst[1]:.3e} "
          f"(bar 2e-4); margins alpha {margin_a:.2e} T {margin_t:.2e}; exactly zero: {zero}")
    assert e_img <= 1e-5
    assert len(errs) >= 6
    for k, e in errs.items():
        assert e <= 2e-4, (k, e)


# ---- 4. resolution invariance -------------------------------------------------------------------------------------------------

def test_total_alpha_of_a_small_gaussian_is_resolution_invariant_only_with_aa():
    Wh = 256
    cam_hi, cam_lo = synth.make_camera(Wh, Wh).to(DEV), synth.make_camera(Wh // 4, Wh // 4).to(DEV)
    focal = Wh / (2.0 * math.tan(cam_hi.FoVx * 0.5))
    sigma = 2.0 * 4.0 / focal                                                  # 2 px at W, 0.5 px at W / 4 (depth 4)
    scene = synth.Scene(torch.tensor([[0.0013, -0.0021, 0.0]]), torch.tensor([[math.log(0.9 / 0.1)]]), torch.full((1, 3), sigma),
                        torch.tensor([[1.0, 0.0, 0.0, 0.0]]), torch.zeros(1, 1, 3), torch.zeros(1, 1, dtype=torch.int32))
    bg = torch.zeros(3, device=DEV)
    total = {}
    for aa in (False, True):
        for label, cam in (("hi", cam_hi), ("lo", cam_lo)):
            dbg = {}
            _, out = _forward(scene, cam, bg, aa=aa, maps=True, dbg=dbg)
            a = out[7][0].to(F64)
            # per pixel: min(0.99, o^ exp(power)), cut below 1/255, from the kernel's own conic / means2D / o^ in float64
            co, mu = dbg["conic_opacity"][0].to(F64), dbg["means2D"][0].to(F64)
            ys, xs = torch.meshgrid(torch.arange(cam.image_height, device=DEV, dtype=F64),
                                    torch.arange(cam.image_width, device=DEV, dtype=F64), indexing="ij")
            dx, dy = mu[0] - xs, mu[1] - ys
            raw = co[3] * torch.exp(-0.5 * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy)
            exp = torch.where(raw >= 1.0 / 255.0, torch.clamp_max(raw, 0.99), torch.zeros_like(raw))
            near_cut = (raw - 1.0 / 255.0).abs() < 1e-5
            assert float((a - exp).abs()[~near_cut].max()) <= 2e-6, (aa, label)
            total[(aa, label)] = float(a.sum())
    r_aa = 16.0 * total[(True, "lo")] / total[(True, "hi")]
    r_plain = 16.0 * total[(False, "lo")] / total[(False, "hi")]
    print(f"\n[antialias] 16 sum(alpha_lo) / sum(alpha_hi): with AA {r_aa:.4f}, without {r_plain:.4f}")
    assert abs(r_aa - 1.0) <= 0.03
    assert r_plain > 1.5


# ---- 5. equivalences ----------------------------------------------------------------------------------------------------------
# Backward comparisons use an 8x4 image: one warp block, where the render backward's accumulator receives one addition per
# Gaussian, so two calls agree bit for bit and only the kernels' own arithmetic can differ (see test_gpu_camera.py).

def _small(name):
    scene, _, prune, quant = _config(name)
    return scene, O.yaw_cam(8, 4, 2.0), prune, quant


def _grads_close(a, b, bar=1e-6):
    return all(_rel(x, y) <= bar if float(y.abs().max()) > 0 else float(x.abs().max()) == 0 for x, y in zip(a, b))


def test_quantised_aa_equals_dequantised_aa():
    scene, cam, _, quant = _small("quant")
    dense = quant.to(DEV).dequantise()                       # on the GPU, as the reference flow does (load_ply)
    bg = torch.tensor([0.1, 0.3, 0.2], device=DEV)
    G = torch.randn(3, 4, 8, generator=torch.Generator().manual_seed(221))
    Gd = torch.randn(1, 4, 8, generator=torch.Generator().manual_seed(222)).to(DEV)
    aq, oq = _forward(scene, cam, bg, quant=quant, maps=True)
    ad, od = _forward(dense, cam, bg, maps=True)
    assert int((oq[2] > 0).sum()) > 1000
    for i in (0, 1, 2, 6, 7):
        assert oq[i] == od[i] if i == 0 else O.same(oq[i], od[i]), i
    gq = _backward(aq, oq, G, quant=quant, dL_dinvdepth=Gd)
    gd = _backward(ad, od, G, dL_dinvdepth=Gd)
    assert _grads_close(gq, gd)


def test_pruned_aa_equals_compacted_aa():
    scene, cam, prune, _ = _small("pruned")
    keep = prune == 0
    bg = torch.tensor([0.1, 0.3, 0.2], device=DEV)
    G = torch.randn(3, 4, 8, generator=torch.Generator().manual_seed(223))
    ap, op = _forward(scene, cam, bg, prune=prune, maps=True)
    ac, oc = _forward(scene.compact(keep), cam, bg, maps=True)
    assert op[0] == oc[0] and op[0] > 0
    for i in (1, 6, 7):
        assert O.same(op[i], oc[i]), i
    gp = _backward(ap, op, G, prune=prune)
    gc = _backward(ac, oc, G)
    kd = keep.to(DEV)
    assert _grads_close([t[kd] for t in gp], gc)
    assert all(float(t[~kd].abs().max()) == 0 for t in gp if t.numel())


def test_aa_accumulate_equals_the_sum_of_two_calls_and_quant_grads_accumulate():
    scene, cam, _, _ = _small("mixed")
    cam2 = O.yaw_cam(8, 4, 3.5)
    bg = torch.tensor([0.1, 0.3, 0.2], device=DEV)
    G = torch.randn(3, 4, 8, generator=torch.Generator().manual_seed(224))
    a1, o1 = _forward(scene, cam, bg)
    a2, o2 = _forward(scene, cam2, bg)
    g1, g2 = _backward(a1, o1, G), _backward(a2, o2, G)
    acc = tuple(t.clone() for t in g1)
    _backward(a2, o2, G, accumulate_into=acc)
    assert _grads_close(acc, [x + y for x, y in zip(g1, g2)])
    # quant.grads accumulate over backward calls through render() with pipe.antialiasing
    from gaussian_renderer import render
    qscene, qcam, _, quant = _small("quant")
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False, antialiasing=True)
    pc = GaussianModelView(qscene, DEV, quant=quant)
    Gq = G.to(DEV)
    (render(qcam, pc, pipe, bg)["render"] * Gq).sum().backward()
    first = {k: v.clone() for k, v in pc.quant.grads.items()}
    (render(qcam, pc, pipe, bg)["render"] * Gq).sum().backward()
    for k, v in pc.quant.grads.items():
        assert float(first[k].abs().max()) > 0 and _rel(v, 2 * first[k]) <= 1e-6, k
    # and they are the AA gradients: they equal the raw entry point's
    aq, oq = _forward(qscene, qcam, bg, quant=quant)
    gq = _backward(aq, oq, G, quant=quant)
    assert _rel(first["opacity"], gq[2]) <= 1e-6 and _rel(first["scales"], gq[6]) <= 1e-6


# ---- 6. a second device --------------------------------------------------------------------------------------------------------

@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_aa_on_a_second_device():
    scene, _, _, _ = _small("mixed")
    bg = torch.tensor([0.1, 0.3, 0.2])
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        cam = O.yaw_cam(8, 4, 2.0, dev=dev)
        args = O.forward_args(scene, cam, bg, dev=dev)
        out = _C.rasterize_gaussians(*args, antialiasing=True)
        (bgd, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = args
        g = _C.rasterize_gaussians_backward(bgd, means3D, out[2], colors, scales, rotations, mod, cov, view, proj, tx, ty,
                                            torch.ones(3, H, W, device=dev), sh, degrees, campos, out[3], out[0], out[4], out[5], 0.0,
                                            False, antialiasing=True)
        outs.append((out[1].cpu(), [t.cpu() for t in g]))
    assert O.same(outs[0][0], outs[1][0])
    assert all(O.same(a, b) for a, b in zip(outs[0][1], outs[1][1]))
