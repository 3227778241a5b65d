"""GPU: the deterministic backward (`deterministic=True`, gsb_backward's `deterministic`, DESIGN.md §5i).
  1. one-warp identity: on an 8x4 image the default path adds one partial per Gaussian, so both paths give the same values (a zero's
     sign aside) in every output: dense, quantised, pruned, maps, AA, camera gradients, raw; on 3x2 tiles with multi-tile rects the
     two agree per element (the slot arithmetic and the gather); a num_rendered that does not match the blobs gives NaN;
  2. accuracy: the 16 scenes of backward_edges against the fp64 oracle with the bars of test_gpu_backward_edges;
  3. reproducibility at 1920x1080 (P = 1 M degree 3, dense, with maps, camera, AA and raw; the C3 quantised scene): five runs give the
     same bytes, also on a side stream, after unrelated allocations, on a second GPU and for a two-view accumulate_into sum;
  4. agreement with the default path at the same sizes: within 1e-4 of each array's largest magnitude or four times the largest
     gap between any two of six default runs, measured from their mean;
  5. edges: P = 0, R = 0, everything pruned, Gaussians over more than 32 tiles, rects clipped at the border, odd image sizes;
  6. end to end: under torch.use_deterministic_algorithms(True), two 60-iteration training runs end bit-identical."""
import math

import numpy as np
import pytest
import torch

import backward_edges as BE
import ours as O
from diff_gaussian_rasterization import _C
from gs_b200 import densify, synth
from test_gpu_fused_activations import NAMES, Model, _adam, _render

pytestmark = pytest.mark.gpu

DEV = "cuda"
BG = torch.tensor([0.2, 0.4, 0.6])


def _vals_equal(a, b):
    """The same values (torch.equal compares with ==, so +0 and -0 match) and shape; None matches None."""
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and torch.equal(a, b)


def _bytes_equal(a, b):
    if a is None or b is None:
        return a is None and b is None
    return O.same(a, b)


def _outs(g):
    return [t.clone() if t is not None else None for t in g]


# ---- scenes ---------------------------------------------------------------------------------------------------------------------

def _small(kind, W=8, H=4):
    box, ls = (1.9 * 320 / 200, 1.9, 1.0), math.log(0.03)
    scene = synth.make_scene(20_000, {"dense": 11, "quant": 12, "pruned": 13}.get(kind, 11), mixed_degrees=True, box=box, log_scale_mean=ls)
    prune = synth.prune_mask(scene.P, 14) if kind == "pruned" else None
    quant = synth.quantise_scene(scene) if kind == "quant" else None
    return scene, O.yaw_cam(W, H, 2.0, dev="cpu"), prune, quant


def _pair(scene, cam, prune=None, quant=None, maps=False, aa=False, dL=None, **extra):
    """(default, deterministic) gradient tuples of one forward."""
    W, H = cam.image_width, cam.image_height
    args, out = O.forward(scene, cam, BG, prune, quant, maps=maps, aa=aa)
    dL = synth.grad_image(W, H, 3).to(DEV) if dL is None else dL
    if maps:
        extra.update(dL_dinvdepth=synth.grad_image(W, H, 4)[:1].to(DEV).contiguous(), dL_dalpha=synth.grad_image(W, H, 5)[:1].to(DEV).contiguous())
    a = _outs(O.backward(args, out, dL, prune, quant, aa=aa, want_conic=True, **extra))
    b = _outs(O.backward(args, out, dL, prune, quant, aa=aa, want_conic=True, deterministic=True, **extra))
    torch.cuda.synchronize()
    return out, a, b


# ---- 1. one-warp identity -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["dense", "quant", "pruned", "maps", "aa", "camera", "aa_maps_camera"])
def test_one_warp_identity(case):
    kind = case if case in ("quant", "pruned") else "dense"
    scene, cam, prune, quant = _small(kind)
    maps, aa, camg = "maps" in case, "aa" in case, "camera" in case
    out, a, b = _pair(scene, cam, prune, quant, maps=maps, aa=aa, camera_grads=camg)
    assert int((out[2] > 0).sum()) > 50
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert _vals_equal(x, y), (case, k)


def _raw_forward(m, cam, aa=False, maps=True):
    e = torch.empty(0)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    args = (BG.to(DEV), m._xyz.detach(), e, m._opacity.detach(), e, e, 1.0, e, cam.world_view_transform, cam.full_proj_transform, tx, ty,
            cam.image_height, cam.image_width, e, m._degrees, cam.camera_center, False, False)
    raw = (m._features_dc.detach(), m._features_rest.detach(), m._scaling.detach(), m._rotation.detach())
    with torch.no_grad():
        return _C.rasterize_gaussians(*args, return_maps=maps, antialiasing=aa, raw=raw), raw


def _raw_backward(m, cam, out, raw, dL, aa=False, **kw):
    e = torch.empty(0)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    R, color, radii, geom, binning, img = out[:6]
    return _C.rasterize_gaussians_backward(BG.to(DEV), m._xyz.detach(), radii, e, e, e, 1.0, e, cam.world_view_transform,
                                           cam.full_proj_transform, tx, ty, dL, e, m._degrees, cam.camera_center, geom, R, binning, img,
                                           0.0, False, raw=raw, antialiasing=aa, **kw)


def _raw_kw(W, H):
    return dict(dL_dinvdepth=synth.grad_image(W, H, 4)[:1].to(DEV).contiguous(), dL_dalpha=synth.grad_image(W, H, 5)[:1].to(DEV).contiguous(),
                camera_grads=True)


@pytest.mark.parametrize("aa", [False, True])
def test_one_warp_identity_raw(aa):
    W, H = 8, 4
    m = Model(synth.make_scene(20_000, 15, mixed_degrees=True, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.03)), 15)
    cam = O.yaw_cam(W, H, 1.0)
    out, raw = _raw_forward(m, cam, aa)
    dL = synth.grad_image(W, H, 3).to(DEV)
    a = _outs(_raw_backward(m, cam, out, raw, dL, aa, **_raw_kw(W, H)))
    b = _outs(_raw_backward(m, cam, out, raw, dL, aa, deterministic=True, **_raw_kw(W, H)))
    assert int((out[2] > 0).sum()) > 50
    for k, (x, y) in enumerate(zip(a, b)):
        assert _vals_equal(x, y), k


def _row_close(a, b, rel_row=1e-4, rel_arr=1e-5):
    """Per element: |a - b| <= rel_row * max|b| over the Gaussian's row + rel_arr * max|b| over the array."""
    a2, b2 = a.reshape(a.shape[0], -1).double(), b.reshape(b.shape[0], -1).double()
    row = b2.abs().amax(1, keepdim=True)
    return bool(((a2 - b2).abs() <= rel_row * row + rel_arr * float(b2.abs().max())).all())


@pytest.mark.parametrize("maps", [False, True])
def test_multi_tile_slots_per_element(maps):
    """3x2 tiles, Gaussians spanning up to all six: every slot of a Gaussian's rect is used, so a wrong (ty - miny) * w + (tx - minx)
    or a gather over the wrong slots moves whole partials between rows; the default path differs from the fixed order only by
    rounding, so both agree per element far inside what such a bug would produce."""
    W, H = 48, 32
    scene = synth.make_scene(600, 41, mixed_degrees=True, box=(2.5, 1.7, 1.0), log_scale_mean=math.log(0.3))
    cam = O.yaw_cam(W, H, 1.0, dev="cpu")
    out, a, b = _pair(scene, cam, maps=maps, camera_grads=maps)
    radii = out[2]
    assert int((radii > 0).sum()) > 200 and int((radii > 8).sum()) > 50        # 17+ px across: 2 x 2 tiles and more
    for k, (x, y) in enumerate(zip(b, a)):
        if x is None or x.numel() == 0 or x.dim() < 2 or x.shape[0] != scene.P:
            continue
        assert _row_close(x, y), k


def test_num_rendered_mismatch_gives_nan():
    """The documented consistency check: a num_rendered other than the blobs' instance count (here R - 1 and R + 1) makes every
    accumulated gradient NaN instead of a plausible-looking wrong one; nothing is written outside the slots of num_rendered."""
    W, H = 64, 48
    scene = synth.make_scene(2_000, 43, mixed_degrees=True, box=(2.5, 1.9, 1.0), log_scale_mean=math.log(0.03))
    cam = O.yaw_cam(W, H, 0.0, dev="cpu")
    args, out = O.forward(scene, cam, BG)
    R = out[0]
    assert R > 100
    dL = synth.grad_image(W, H, 3).to(DEV)
    vis = out[2] > 0
    good = O.backward(args, out, dL, deterministic=True)
    assert all(bool(torch.isfinite(t).all()) for t in good)
    for r in (R - 1, R + 1):
        bad = O.backward(args, (r,) + tuple(out[1:]), dL, deterministic=True)
        torch.cuda.synchronize()
        # dL_dopacity and the x, y columns of dL_dmeans2D (its z column is always written as 0)
        assert bool(torch.isnan(bad[2][vis]).all()) and bool(torch.isnan(bad[0][vis][:, :2]).all()), r


# ---- 2. accuracy against the fp64 oracle ----------------------------------------------------------------------------------------

def _run_backward_det(args, out, dL, lam=0.0):
    """ours.run_backward with deterministic=True."""
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = args
    R, color, radii, geom, binning, img = out
    grads = _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, view, proj, tx, ty, dL.to(means3D.device),
                                            sh, degrees, campos, geom, R, binning, img, lam, False, want_conic=True, deterministic=True)
    torch.cuda.synchronize()
    return {n: g.cpu().numpy() for n, g in zip(O.GRAD_NAMES + ["dL_dconic"], grads)}


@pytest.mark.parametrize("name", BE.CASES)
def test_backward_per_element_against_fp64_oracle(name):
    case = BE.build(name)
    o, o64, o32 = BE.oracle(case)
    excl = BE.excluded(case, o)
    args, out, fwd = O.run_forward(case.scene, case.cam, case.bg)
    assert int(fwd["num_rendered"]) == int(o["num_rendered"])
    bar = BE.BAR_CASE.get(name, (BE.R_REL, BE.A_ABS))
    got = _run_backward_det(args, out, case.dL, case.lam)
    _, failures = BE.compare(name, o, o64, o32, got, ~excl, glob=(excl, BE.EXCLUDED_BAR), bar=bar)
    assert not failures, "\n" + BE.describe(failures, o, o64, got, case.W, case.H)
    if excl.any():
        dL = case.dL.clone()
        dL[:, torch.from_numpy(o["borderline"])] = 0.0
        _, m64, m32 = BE.oracle(case, dL=dL, fwd=o)
        mgot = _run_backward_det(args, out, dL, case.lam)
        _, failures = BE.compare(name + ", borderline dL = 0", o, m64, m32, mgot, np.ones_like(excl), bar=bar)
        assert not failures, "\n" + BE.describe(failures, o, m64, mgot, case.W, case.H)


# ---- 3. / 4. reproducibility and agreement at 1920x1080 -------------------------------------------------------------------------

W_FULL, H_FULL = 1920, 1080


@pytest.fixture(scope="module")
def dense_1m():
    scene = synth.make_scene(1_000_000, 21, sh_degree=3, box=(1.9 * W_FULL / H_FULL, 1.9, 1.0), log_scale_mean=math.log(0.01))
    return scene, O.yaw_cam(W_FULL, H_FULL, 3.0, dev="cpu")


@pytest.fixture(scope="module")
def c3():
    W, H = synth.config_image("C3")
    scene = synth.config_scene("C3")
    quant = synth.quantise_scene(scene, seed=0)
    return scene, synth.make_camera(W, H), quant


N_DEFAULT = 6


def _check_repro_and_agreement(run_default, run_det, tag):
    """Reproducibility (the contract): five deterministic runs give the same bytes in every output.
    Agreement: the deterministic result lies within max(1e-4 scale, 4 x floor) of the mean of N_DEFAULT default runs, where floor is
    the largest gap between any two of those runs (15 pairs) and scale the array's largest magnitude.  A floor from a single pair
    is not enough for the camera outputs: 3 or 16 sums over every Gaussian, often dominated by one element, whose one-sample gap
    can be arbitrarily small.  Nor does the default path's spread bound every array: its CTAs are scheduled in nearly the same
    order on every run, so its runs differ less from each other than from an unrelated fixed order (observed at C3: dL_drotations
    4.3e-3 from the default mean against 1.0e-3 between default runs, 5.5e-5 of the array's scale).  A wrong slot or order
    moves whole partials, orders of magnitude above either bound; per-element accuracy is checked against the fp64 oracle."""
    d = [_outs(run_det()) for _ in range(5)]
    torch.cuda.synchronize()
    for i, r in enumerate(d[1:], 1):
        for k, (x, y) in enumerate(zip(d[0], r)):
            assert _bytes_equal(x, y), f"reproducibility: [{tag}] deterministic run {i} differs from run 0 in output {k}"
    g = [_outs(run_default()) for _ in range(N_DEFAULT)]
    torch.cuda.synchronize()
    for k, x in enumerate(d[0]):
        if x is None or x.numel() == 0:
            continue
        runs = torch.stack([r[k].double() for r in g])
        floor = max(float((runs[i] - runs[j]).abs().max()) for i in range(N_DEFAULT) for j in range(i + 1, N_DEFAULT))
        mean = runs.mean(0)
        scale = float(mean.abs().max())
        err = float((x.double() - mean).abs().max())
        bound = max(1e-4 * scale, 4.0 * floor)
        print(f"[{tag}] output {k}: |det - mean default| {err:.3e}, scale {scale:.3e}, default max pair gap {floor:.3e}, "
              f"err / bound {err / bound if bound else 0.0:.3f}")
        assert err <= bound, f"agreement: [{tag}] output {k}: |det - mean default| {err:.3e} > bound {bound:.3e} (scale {scale:.3e}, floor {floor:.3e})"
    return d[0]


@pytest.mark.parametrize("mode", ["plain", "maps_camera", "aa"])
def test_dense_1m_reproducible_and_agrees(dense_1m, mode):
    scene, cam = dense_1m
    maps, aa = mode == "maps_camera", mode == "aa"
    args, out = O.forward(scene, cam, BG, maps=maps, aa=aa)
    dL = synth.grad_image(W_FULL, H_FULL, 3).to(DEV)
    extra = dict(camera_grads=True, dL_dinvdepth=synth.grad_image(W_FULL, H_FULL, 4)[:1].to(DEV).contiguous(),
                 dL_dalpha=synth.grad_image(W_FULL, H_FULL, 5)[:1].to(DEV).contiguous()) if maps else {}
    assert out[0] > 1_000_000
    ref = _check_repro_and_agreement(lambda: O.backward(args, out, dL, aa=aa, **extra),
                                     lambda: O.backward(args, out, dL, aa=aa, deterministic=True, **extra), "dense 1M " + mode)
    if mode != "plain":
        return
    # a side stream
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        side = _outs(O.backward(args, out, dL, deterministic=True))
    torch.cuda.current_stream().wait_stream(s)
    # unrelated allocations move the workspace
    hog = [torch.empty(n, dtype=torch.uint8, device=DEV) for n in (12345, 7 << 20, 333 << 20)]
    moved = _outs(O.backward(args, out, dL, deterministic=True))
    del hog
    torch.cuda.synchronize()
    for k, x in enumerate(ref):
        assert _bytes_equal(x, side[k]) and _bytes_equal(x, moved[k]), k
    # a second GPU
    if torch.cuda.device_count() > 1:
        d1 = torch.device("cuda", 1)
        a1 = O.forward_args(scene, cam, BG, dev=d1)
        o1 = _C.rasterize_gaussians(*a1)
        (bg, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = a1
        g1 = _C.rasterize_gaussians_backward(bg, means3D, o1[2], colors, scales, rotations, mod, cov, view, proj, tx, ty, dL.to(d1), sh,
                                             degrees, campos, o1[3], o1[0], o1[4], o1[5], 0.0, False, deterministic=True)
        torch.cuda.synchronize(d1)
        for k, x in enumerate(g1):
            assert _bytes_equal(ref[k], x.to(DEV)), k


def test_dense_1m_raw_reproducible_and_agrees(dense_1m):
    scene, c = dense_1m
    m = Model(scene, 15)
    cam = O.yaw_cam(W_FULL, H_FULL, 3.0)
    out, raw = _raw_forward(m, cam, aa=True)
    dL = synth.grad_image(W_FULL, H_FULL, 3).to(DEV)
    kw = _raw_kw(W_FULL, H_FULL)
    _check_repro_and_agreement(lambda: _raw_backward(m, cam, out, raw, dL, True, **kw),
                               lambda: _raw_backward(m, cam, out, raw, dL, True, deterministic=True, **kw), "dense 1M raw aa")


def test_dense_1m_accumulate_two_views(dense_1m):
    scene, _ = dense_1m
    cams = [O.yaw_cam(W_FULL, H_FULL, d, dev="cpu") for d in (-2.0, 2.0)]
    fw = [O.forward(scene, c, BG) for c in cams]
    dLs = [synth.grad_image(W_FULL, H_FULL, s).to(DEV) for s in (6, 7)]

    def run():
        acc = O.backward(*fw[0], dLs[0], deterministic=True)
        return _outs(O.backward(*fw[1], dLs[1], deterministic=True, accumulate_into=acc))
    a, b = run(), run()
    torch.cuda.synchronize()
    for k, (x, y) in enumerate(zip(a, b)):
        assert _bytes_equal(x, y), k


def test_c3_quantised_reproducible_and_agrees(c3):
    scene, cam, quant = c3
    args, out = O.forward(scene, cam, BG, quant=quant)
    W, H = cam.image_width, cam.image_height
    dL = synth.grad_image(W, H, 3).to(DEV)
    _check_repro_and_agreement(lambda: O.backward(args, out, dL, quant=quant),
                               lambda: O.backward(args, out, dL, quant=quant, deterministic=True), "C3")


# ---- 5. edges -------------------------------------------------------------------------------------------------------------------

def test_empty_culled_and_pruned():
    W, H = 64, 48
    scene = synth.make_scene(2_000, 31, mixed_degrees=True, box=(2.5, 1.9, 1.0), log_scale_mean=math.log(0.03))
    cam = O.yaw_cam(W, H, 0.0, dev="cpu")
    dL = synth.grad_image(W, H, 3).to(DEV)
    # P = 0
    empty = synth.Scene(*[getattr(scene, f)[:0] for f in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
    args, out = O.forward(empty, cam, BG)
    g = O.backward(args, out, dL, deterministic=True, camera_grads=True)
    assert all(t.numel() == 0 for t in g[:8]) and float(g[-3].abs().max()) == 0.0
    # everything behind the camera (R = 0), everything pruned
    behind = synth.Scene(scene.means3D - torch.tensor([0.0, 0.0, 100.0]), scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees)
    for sc, prune in ((behind, None), (scene, torch.ones(scene.P, dtype=torch.bool))):
        args, out = O.forward(sc, cam, BG, prune)
        assert out[0] == 0
        g = O.backward(args, out, dL, prune, deterministic=True, want_conic=True)
        torch.cuda.synchronize()
        for t in g:
            assert t.numel() == 0 or float(t.abs().max()) == 0.0


@pytest.mark.parametrize("W,H", [(333, 77), (129, 250), (17, 1)])
def test_big_clipped_and_odd_sizes(W, H):
    """Gaussians over more than 32 tiles (the scatter's warp path), rects clipped at every border, image sizes off the tile grid."""
    g = torch.Generator().manual_seed(W)
    P = 3_000
    scene = synth.make_scene(P, W + H, mixed_degrees=True, box=(2.4 * W / max(H, 8), 2.4, 1.0), log_scale_mean=math.log(0.03))
    # a tenth of the Gaussians are large (radii of tens of pixels up to beyond the image)
    big = torch.rand(P, generator=g) < 0.1
    scales = scene.scales.clone()
    scales[big] *= 12.0
    scene = synth.Scene(scene.means3D, scene.opacity, scales, scene.rotations, scene.sh, scene.degrees)
    cam = O.yaw_cam(W, H, 1.5, dev="cpu")
    out, a, b = _pair(scene, cam)
    radii = out[2]
    assert int((radii > 0).sum()) > 10
    if W * H > 1000:
        assert int((radii > 48).sum()) > 5                      # rects of more than 32 tiles
    c = _outs(O.backward(*O.forward(scene, cam, BG), synth.grad_image(W, H, 3).to(DEV), want_conic=True, deterministic=True))
    torch.cuda.synchronize()
    for k, (x, y, z) in enumerate(zip(a, b, c)):
        assert _bytes_equal(y, z), k
        scale = float(x.abs().max()) if x.numel() else 0.0
        assert float((x - y).abs().max()) <= 1e-4 * scale + 1e-30, k


# ---- 6. end to end --------------------------------------------------------------------------------------------------------------

def _train(fused_schedule, seed=5):
    from utils.loss_utils import l1_ssim_loss
    torch.manual_seed(seed)                                   # the split children's samples (torch.normal) come from torch's generator
    W, H = 256, 192
    target = synth.make_scene(6_000, 71, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04))
    cams = [O.yaw_cam(W, H, yaw) for yaw in (-10.0, 0.0, 10.0)]
    with torch.no_grad():
        gts = [_render(Model(target, 15, norm_range=(0.0, 0.0)), c, False)["render"].clone() for c in cams]
    g = torch.Generator().manual_seed(seed)
    start = synth.Scene(target.means3D + 0.01 * torch.randn(target.means3D.shape, generator=g),
                        target.opacity + 0.5 * torch.randn(target.opacity.shape, generator=g),
                        target.scales * torch.exp(0.2 * torch.randn(target.scales.shape, generator=g)),
                        torch.nn.functional.normalize(target.rotations + 0.1 * torch.randn(target.rotations.shape, generator=g)),
                        target.sh + 0.1 * torch.randn(target.sh.shape, generator=g), target.degrees)
    m = Model(start, 15)
    m.optimizer = _adam(m)
    P = m._xyz.shape[0]
    m.percent_dense = 0.01
    m.xyz_gradient_accum = torch.zeros(P, 1, device=DEV)
    m.denom = torch.zeros(P, 1, device=DEV)
    m.max_radii2D = torch.zeros(P, device=DEV)
    losses = []
    for it in range(60):
        k = it % len(cams)
        m.optimizer.zero_grad(set_to_none=True)
        pkg = _render(m, cams[k], fused_schedule(it))
        loss = l1_ssim_loss(pkg["render"], gts[k], 0.2)
        loss.backward()
        vis = pkg["visibility_filter"]
        densify.add_densification_stats(m, pkg["viewspace_points"], vis, pkg["radii"])
        m.optimizer.step(visibility=vis, degrees=m._degrees)
        losses.append(float(loss.detach()))
        if it == 30:
            densify.densify_and_prune(m, 2e-4, 0.005, 3.0, None, {})
    return m, losses


def test_training_is_bit_identical_under_torch_deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        sched = lambda it: it % 2 == 0                        # pipe.fused_activations on and off
        m1, l1 = _train(sched)
        m2, l2 = _train(sched)
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    print(f"60 deterministic steps: loss {sum(l1[:3]) / 3:.4f} -> {sum(l1[-3:]) / 3:.4f}")
    assert l1 == l2
    # the loss goes down (observed on an H100: mean over the three views 0.0930 -> 0.0922, densification at step 30 included)
    assert sum(l1[-3:]) < sum(l1[:3])
    for n in NAMES:
        p1, p2 = getattr(m1, n), getattr(m2, n)
        assert O.same(p1.detach(), p2.detach()), n
        s1, s2 = m1.optimizer.state[p1], m2.optimizer.state[p2]
        assert O.same(s1["exp_avg"], s2["exp_avg"]) and O.same(s1["exp_avg_sq"], s2["exp_avg_sq"]), n
    for n in ("xyz_gradient_accum", "denom", "max_radii2D"):
        assert O.same(getattr(m1, n), getattr(m2, n)), n
