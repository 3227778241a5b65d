"""GPU: the absolute screen-space gradient (AbsGS; DESIGN.md §5m) of render_backward_kernel<*, *, ABS = true> and its use in
densification.

1. Nothing else moves: under the deterministic mode every other output of a backward with absgrad is bitwise the call's without it
   (dense, quantised, pruned, maps, anti-aliased, camera, raw); on the default path within the run-to-run gap.
2. Against float64 per Gaussian on the backward-edge scenes: absgrad64.pair_sums restates the per-pair terms on the forward's own
   state (pinned to the oracle's dL_dmeans2D by test_absgrad_api.py); bar max(1e-4 |abs64|_row, 1e-6 max |abs64|).  The sums of
   absolute values have no cancellation of their own, so the bar of test_gpu_backward_edges.py holds unchanged, with the same
   looser bar for dense_faint (whose 30 000-entry lists recover T with MUFU.RCP: up to 4e-4 of a row's w there, which the
   absolute sums inherit) and the same Gaussians left to a global bar (BE.excluded: an ulp of the exponential may flip a pair).
3. Properties at 1080p with 1 M Gaussians, the collision case, abs(dL) == abs(-dL).
4. Determinism: five runs, a side stream, culled / pruned rows, P = 0 and R = 0.
5. Densification with the absolute statistic, against torch restatements.
6. Training with absgrad and max_grad_abs: the loss goes down, splits happen, and two runs are bit-identical.
"""
import math

import numpy as np
import pytest
import torch

import absgrad64
import backward_edges as BE
import ours as O
from diff_gaussian_rasterization import _C
from gs_b200 import densify, synth
from test_gpu_deterministic import BG, DEV, _outs, _raw_backward, _raw_forward, _raw_kw, _small
from test_gpu_fused_activations import NAMES, Model, _adam, _render

pytestmark = pytest.mark.gpu


def _abs_out(P):
    return torch.full((P, 3), float("nan"), device=DEV)


def _same_all(a, b, tag):
    assert len(a) == len(b), tag
    for k, (x, y) in enumerate(zip(a, b)):
        if x is None or y is None:
            assert x is None and y is None, (tag, k)
        else:
            assert O.same(x, y), (tag, k)


# ---- 1. nothing else moves ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["dense", "quant", "pruned", "maps", "aa", "camera", "aa_maps_camera"])
def test_nothing_else_moves(case):
    kind = case if case in ("quant", "pruned") else "dense"
    scene, cam, prune, quant = _small(kind, W=64, H=48)
    maps, aa, camg = "maps" in case, "aa" in case, "camera" in case
    W, H = cam.image_width, cam.image_height
    args, out = O.forward(scene, cam, BG, prune, quant, maps=maps, aa=aa)
    dL = synth.grad_image(W, H, 3).to(DEV)
    extra = dict(camera_grads=camg, want_conic=True)
    if maps:
        extra.update(dL_dinvdepth=synth.grad_image(W, H, 4)[:1].to(DEV).contiguous(), dL_dalpha=synth.grad_image(W, H, 5)[:1].to(DEV).contiguous())
    P = scene.P
    for det in (True, False):
        plain = _outs(O.backward(args, out, dL, prune, quant, aa=aa, deterministic=det, **extra))
        ab = _abs_out(P)
        with_abs = _outs(O.backward(args, out, dL, prune, quant, aa=aa, deterministic=det, absgrad_out=ab, **extra))
        torch.cuda.synchronize()
        assert bool(torch.isfinite(ab).all()) and float(ab[:, :2].max()) > 0 and bool((ab[:, 2] == 0).all())
        if det:
            _same_all(plain, with_abs, case)
        else:
            again = _outs(O.backward(args, out, dL, prune, quant, aa=aa, **extra))
            for k, (x, y, z) in enumerate(zip(plain, with_abs, again)):
                if x is None:
                    continue
                gap = float((x - z).abs().max())
                scale = float(x.abs().max())
                assert float((x - y).abs().max()) <= max(4 * gap, 1e-5 * scale) + 1e-30, (case, k)


def test_nothing_else_moves_raw():
    W, H = 64, 48
    m = Model(synth.make_scene(20_000, 15, mixed_degrees=True, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.03)), 15)
    cam = O.yaw_cam(W, H, 1.0)
    out, raw = _raw_forward(m, cam, True)
    dL = synth.grad_image(W, H, 3).to(DEV)
    a = _outs(_raw_backward(m, cam, out, raw, dL, True, deterministic=True, **_raw_kw(W, H)))
    ab = _abs_out(m._xyz.shape[0])
    b = _outs(_raw_backward(m, cam, out, raw, dL, True, deterministic=True, absgrad_out=ab, **_raw_kw(W, H)))
    _same_all(a, b, "raw")
    assert float(ab[:, :2].max()) > 0


# ---- 2. against float64 per Gaussian --------------------------------------------------------------------------------------------

BAR_CASE = {"dense_faint": (1e-3, 1e-5)}


@pytest.mark.parametrize("name", BE.CASES + BE.AA_CASES)
def test_against_float64_per_gaussian(name):
    case = BE.build(name)
    aa = case.meta["aa"]
    o, _, _ = BE.oracle(case, aa=aa)
    excl = BE.excluded(case, o)
    args, out, fwd = O.run_forward(case.scene, case.cam, case.bg, aa=aa)
    _, abs64 = absgrad64.pair_sums(fwd, case.bg.numpy(), case.dL.numpy(), case.W, case.H)
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = args
    R, color, radii, geom, binning, img = out
    P = case.scene.P
    for det in (False, True):
        ab = _abs_out(P)
        _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, view, proj, tx, ty, case.dL.to(DEV), sh,
                                        degrees, campos, geom, R, binning, img, case.lam, False, antialiasing=aa, deterministic=det,
                                        absgrad_out=ab)
        got = ab.cpu().double().numpy()
        assert (got[:, 2] == 0).all()
        got = got[:, :2]
        rel, a_abs = BAR_CASE.get(name, (1e-4, 1e-6))
        err = np.abs(got - abs64).max(axis=1)
        row = np.abs(abs64).max(axis=1)
        bar = np.maximum(rel * row, a_abs * np.abs(abs64).max())
        vis = fwd["radii"] > 0
        assert (got[~vis] == 0).all()
        chk = vis & ~excl
        worst = float((err[chk] / np.maximum(bar[chk], 1e-30)).max()) if chk.any() else 0.0
        print(f"[{name} det={det}] {int(chk.sum())} Gaussians per element, worst err / bar {worst:.3f}")
        assert (err[chk] <= bar[chk]).all(), (name, det, worst)
        if (excl & vis).any():
            assert err[excl & vis].max() <= BE.EXCLUDED_BAR * np.abs(abs64).max(), name


# ---- 3. properties ----------------------------------------------------------------------------------------------------------------

W_FULL, H_FULL = 1920, 1080


@pytest.fixture(scope="module")
def dense_1m():
    scene = synth.make_scene(1_000_000, 21, sh_degree=3, box=(1.9 * W_FULL / H_FULL, 1.9, 1.0), log_scale_mean=math.log(0.01))
    return scene, O.yaw_cam(W_FULL, H_FULL, 3.0, dev="cpu")


def _run_1m(scene, cam, dL, det, **kw):
    args, out = O.forward(scene, cam, BG, **kw.pop("fwd", {}))
    ab = _abs_out(scene.P)
    g = _outs(O.backward(args, out, dL, deterministic=det, absgrad_out=ab, **kw))
    return g, ab


def test_properties_1080p(dense_1m):
    scene, cam = dense_1m
    dL = synth.grad_image(W_FULL, H_FULL, 3).to(DEV)
    g, ab = _run_1m(scene, cam, dL, True)
    signed = g[0][:, :2]
    vis = ab[:, :2].abs().sum(1) > 0
    assert int(vis.sum()) > 100_000
    # abs >= |signed| per component, to rounding (both are fp32 sums of the same terms)
    slack = 1e-5 * ab[:, :2] + 1e-6 * float(ab.abs().max())
    assert bool((ab[:, :2] + slack >= signed.abs()).all())
    # the sign of dL/dpixel does not matter, bit for bit
    _, ab_neg = _run_1m(scene, cam, -dL, True)
    assert O.same(ab, ab_neg)


def test_single_pixel_gaussians_abs_equals_signed():
    """Sub-pixel Gaussians far apart, each reaching one pixel only: the sum has one term, so abs = |signed|."""
    W, H = 256, 192
    n = 400
    g = torch.Generator().manual_seed(3)
    cam = synth.make_camera(W, H)
    # 20 x 20 distinct pixels 8 apart; centres 0.2 / 0.15 px off the pixel and opacity 0.008: alpha 0.0072 at the own pixel, below
    # 1/255 at every other one (the nearest is 0.8 px away: 0.008 * exp(-0.66 / 0.6) = 0.0027)
    px = (torch.randperm(W // 8, generator=g)[:20].repeat(20) * 8 + 4).double() + 0.2
    py = (torch.randperm(H // 8, generator=g)[:20].repeat_interleave(20) * 8 + 4).double() - 0.15
    case = BE.pixel_scene(cam, px, py, torch.full((n,), 4.0, dtype=torch.float64), torch.full((n,), 0.05, dtype=torch.float64),
                          torch.full((n,), math.log(0.008 / 0.992)), torch.rand(n, 1, 3, generator=g), g)
    scene = case if isinstance(case, synth.Scene) else case[0]
    args, out = O.forward(scene, cam, BG)
    dL = synth.grad_image(W, H, 9).to(DEV)
    ab = _abs_out(scene.P)
    res = O.backward(args, out, dL, deterministic=True, absgrad_out=ab)
    signed = res[0][:, :2]
    hit = ab[:, :2].abs().sum(1) > 0
    assert int(hit.sum()) == n
    assert float((ab[hit, :2] - signed[hit].abs()).abs().max()) <= 1e-6 * float(ab.abs().max())


def test_collision_case():
    """An isotropic Gaussian centred on a pixel under a mirror-symmetric dL/dpixel: the signed x-gradient cancels, abs does not."""
    W, H = 64, 64
    cam = synth.make_camera(W, H)
    g = torch.Generator().manual_seed(1)
    px, py = torch.tensor([32.0], dtype=torch.float64), torch.tensor([32.0], dtype=torch.float64)
    case = BE.pixel_scene(cam, px, py, torch.tensor([4.0], dtype=torch.float64), torch.tensor([3.0], dtype=torch.float64),
                          torch.tensor([1.0]), torch.full((1, 1, 3), 0.5), g)
    scene = case if isinstance(case, synth.Scene) else case[0]
    args, out = O.forward(scene, cam, torch.zeros(3))
    x = torch.arange(W, dtype=torch.float32) - 32.0
    dL = (torch.sign(x).abs() * torch.ones(3, H, W)).to(DEV).contiguous()        # |x - 32| symmetric: the same on both sides
    ab = _abs_out(1)
    res = O.backward(args, out, dL, deterministic=True, absgrad_out=ab)
    sx, ax = float(res[0][0, 0]), float(ab[0, 0])
    assert ax > 0 and abs(sx) <= 1e-3 * ax, (sx, ax)


# ---- 4. determinism -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["plain", "raw_aa_maps"])
def test_five_runs_identical_1080p(dense_1m, mode):
    scene, cam = dense_1m
    dL = synth.grad_image(W_FULL, H_FULL, 3).to(DEV)
    if mode == "plain":
        args, out = O.forward(scene, cam, BG)
        run = lambda ab: O.backward(args, out, dL, deterministic=True, absgrad_out=ab)
    else:
        m = Model(scene, 15)
        camd = O.yaw_cam(W_FULL, H_FULL, 3.0)
        out, raw = _raw_forward(m, camd, True)
        run = lambda ab: _raw_backward(m, camd, out, raw, dL, True, deterministic=True, absgrad_out=ab, **_raw_kw(W_FULL, H_FULL))
    first = _abs_out(scene.P)
    g0 = _outs(run(first))
    for i in range(4):
        ab = _abs_out(scene.P)
        gi = _outs(run(ab))
        assert O.same(ab, first), i
        _same_all(g0, gi, mode)
    # a side stream gives the same bytes
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ab = _abs_out(scene.P)
        run(ab)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert O.same(ab, first)


def test_culled_pruned_and_empty():
    scene, cam, prune, _ = _small("pruned", W=64, H=48)
    args, out = O.forward(scene, cam, BG, prune)
    dL = synth.grad_image(64, 48, 3).to(DEV)
    for det in (False, True):
        ab = _abs_out(scene.P)
        O.backward(args, out, dL, prune, deterministic=det, absgrad_out=ab)
        invisible = out[2] == 0
        assert int(invisible.sum()) > 0 and bool((ab[invisible] == 0).all())
        assert bool((ab[prune.to(DEV).bool()] == 0).all())
    # R = 0: every Gaussian behind the camera
    far = synth.Scene(scene.means3D + torch.tensor([0.0, 0.0, -50.0]), scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees)
    args, out = O.forward(far, cam, BG)
    assert out[0] == 0
    for det in (False, True):
        ab = _abs_out(far.P)
        O.backward(args, out, dL, deterministic=det, absgrad_out=ab)
        assert bool((ab == 0).all())
    # P = 0
    empty = synth.Scene(scene.means3D[:0], scene.opacity[:0], scene.scales[:0], scene.rotations[:0], scene.sh[:0], scene.degrees[:0])
    args, out = O.forward(empty, cam, BG)
    for det in (False, True):
        ab = torch.empty(0, 3, device=DEV)
        O.backward(args, out, dL, deterministic=det, absgrad_out=ab)


# ---- 5. densification -----------------------------------------------------------------------------------------------------------

def _model_100k(seed=4):
    scene = synth.make_scene(100_000, seed, sh_degree=3, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.02))
    m = Model(scene, 15)
    P = scene.P
    g = torch.Generator(device="cpu").manual_seed(seed)
    m.percent_dense = 0.01
    m.xyz_gradient_accum = (torch.rand(P, 1, generator=g) * 4e-3).to(DEV)
    m.xyz_gradient_accum_abs = m.xyz_gradient_accum + (torch.rand(P, 1, generator=g) * 4e-3).to(DEV)
    m.denom = torch.randint(0, 8, (P, 1), generator=g).float().to(DEV)
    m.max_radii2D = torch.zeros(P, device=DEV)
    return m


def test_densify_stats_abs_matches_torch():
    P = 50_000
    g = torch.Generator(device=DEV).manual_seed(2)
    m = type("M", (), {})()
    m.xyz_gradient_accum = torch.zeros(P, 1, device=DEV)
    m.denom = torch.zeros(P, 1, device=DEV)
    m.max_radii2D = torch.zeros(P, device=DEV)
    acc, acc_abs, den = m.xyz_gradient_accum.clone(), torch.zeros(P, 1, device=DEV), m.denom.clone()
    vp = torch.zeros(P, 3, device=DEV, requires_grad=True)
    va = torch.zeros(P, 3, device=DEV, requires_grad=True)
    torch.cuda.set_sync_debug_mode("error")
    try:
        for it in range(10):
            vp.grad = torch.randn(P, 3, generator=g, device=DEV) * 1e-3
            va.grad = vp.grad.abs() + 1e-4
            vis = (vp.grad[:, 2] > 0).contiguous()
            radii = (vis.int() * 3).contiguous()
            densify.add_densification_stats(m, vp, vis, radii, viewspace_abs=va)
            acc += torch.norm(vp.grad[:, :2], dim=-1, keepdim=True)
            acc_abs += torch.norm(va.grad[:, :2], dim=-1, keepdim=True)
            den += vis.float().unsqueeze(1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert O.same(m.xyz_gradient_accum, acc) and O.same(m.xyz_gradient_accum_abs, acc_abs) and O.same(m.denom, den)


def _torch_plan_abs(m, max_grad, max_grad_abs, extent, min_opacity):
    """The AbsGS rule restated in torch (clone on grads, split on grads_abs; clones padded with zeros are never split) -> the
    (clone, split, kept-after-prune) masks of the original rows."""
    grads = (m.xyz_gradient_accum / m.denom).nan_to_num(0.0).squeeze(1)
    grads_abs = (m.xyz_gradient_accum_abs / m.denom).nan_to_num(0.0).squeeze(1)
    ms = torch.exp(m._scaling.detach()).max(dim=1).values
    clone = (grads >= max_grad) & (ms <= m.percent_dense * extent)
    split = (grads_abs >= max_grad_abs) & (ms > m.percent_dense * extent)
    return clone, split


@pytest.mark.parametrize("opt", ["adam", "gaussian_adam"])
def test_densify_and_prune_abs_rule(opt):
    from gs_b200.optim import GaussianAdam
    m = _model_100k()
    m.optimizer = _adam(m, torch.optim.Adam if opt == "adam" else GaussianAdam)
    clone, split = _torch_plan_abs(m, 2e-4, 6e-4, 3.0, 0.005)
    P = m._xyz.shape[0]
    old_xyz = m._xyz.detach().clone()
    d = {}
    densify.densify_and_prune(m, 2e-4, 0.005, 3.0, None, d, max_grad_abs=6e-4)
    assert d["n_points_cloned"] == int(clone.sum()) and d["n_points_split"] == int(split.sum())
    assert int(split.sum()) > 100 and int(clone.sum()) > 100
    # the rows: [kept originals][kept clones][kept first children][kept second children]
    n_out = P + int(clone.sum()) + int(split.sum()) - int(d["n_points_pruned"])
    assert m._xyz.shape[0] == n_out
    op = torch.sigmoid(m._opacity.detach()).squeeze(1)
    gone = torch.sigmoid(_model_100k()._opacity.detach()).squeeze(1) < 0.005
    kept_orig = ~split & ~gone
    assert O.same(m._xyz.detach()[:int(kept_orig.sum())], old_xyz[kept_orig])
    assert bool((op >= 0.005).all())
    assert tuple(m.xyz_gradient_accum_abs.shape) == (n_out, 1) and float(m.xyz_gradient_accum_abs.abs().sum()) == 0


def test_max_grad_abs_none_is_todays_call():
    from gs_b200.optim import GaussianAdam
    ma, mb = _model_100k(), _model_100k()
    del mb.xyz_gradient_accum_abs
    for m in (ma, mb):
        m.optimizer = _adam(m, GaussianAdam)
    torch.manual_seed(0)
    da = {}
    densify.densify_and_prune(ma, 2e-4, 0.005, 3.0, None, da)
    torch.manual_seed(0)
    db = {}
    densify.densify_and_prune(mb, 2e-4, 0.005, 3.0, None, db)
    assert da["n_points_cloned"] == db["n_points_cloned"] and da["n_points_split"] == db["n_points_split"]
    for n in NAMES:
        assert O.same(getattr(ma, n).detach(), getattr(mb, n).detach()), n
    assert float(ma.xyz_gradient_accum_abs.abs().sum()) == 0 and ma.xyz_gradient_accum_abs.shape == ma.xyz_gradient_accum.shape


def test_prunes_carry_the_abs_accumulator():
    from gs_b200.optim import GaussianAdam
    m = _model_100k()
    m.optimizer = _adam(m, GaussianAdam)
    P = m._xyz.shape[0]
    mask = torch.zeros(P, dtype=torch.bool, device=DEV)
    mask[::3] = True
    before, before_abs = m.xyz_gradient_accum.clone(), m.xyz_gradient_accum_abs.clone()
    densify.prune_points(m, mask)
    assert O.same(m.xyz_gradient_accum, before[~mask]) and O.same(m.xyz_gradient_accum_abs, before_abs[~mask])
    d = {}
    keep_before = m.xyz_gradient_accum_abs.clone()
    op = torch.sigmoid(m._opacity.detach()).squeeze(1)
    densify.prune(m, 0.3, 3.0, None, d)
    assert O.same(m.xyz_gradient_accum_abs, keep_before[~(op < 0.3)])


# ---- 6. training ------------------------------------------------------------------------------------------------------------------

def _train_abs(seed=5):
    from utils.loss_utils import l1_ssim_loss
    torch.manual_seed(seed)
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
    losses, stats = [], {}
    for it in range(60):
        k = it % len(cams)
        m.optimizer.zero_grad(set_to_none=True)
        pkg = _render(m, cams[k], it % 2 == 0, absgrad=True)
        loss = l1_ssim_loss(pkg["render"], gts[k], 0.2)
        loss.backward()
        vis = pkg["visibility_filter"]
        densify.add_densification_stats(m, pkg["viewspace_points"], vis, pkg["radii"], viewspace_abs=pkg["viewspace_points_abs"])
        m.optimizer.step(visibility=vis, degrees=m._degrees)
        losses.append(float(loss.detach()))
        if it == 30:
            densify.densify_and_prune(m, 2e-4, 0.005, 3.0, None, stats, max_grad_abs=4e-4)
    return m, losses, stats


def test_training_with_absgrad_is_bit_identical_and_splits():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        m1, l1, s1 = _train_abs()
        m2, l2, s2 = _train_abs()
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    print(f"60 deterministic absgrad steps: loss {sum(l1[:3]) / 3:.4f} -> {sum(l1[-3:]) / 3:.4f}, "
          f"cloned {s1['n_points_cloned']}, split {s1['n_points_split']}")
    assert l1 == l2
    assert sum(l1[-3:]) < sum(l1[:3])
    assert s1["n_points_split"] > 0 and s1["n_points_split"] == s2["n_points_split"] and s1["n_points_cloned"] == s2["n_points_cloned"]
    for n in NAMES:
        assert O.same(getattr(m1, n).detach(), getattr(m2, n).detach()), n
    for n in ("xyz_gradient_accum", "xyz_gradient_accum_abs", "denom", "max_radii2D", "_degrees"):
        assert O.same(getattr(m1, n), getattr(m2, n)), n
