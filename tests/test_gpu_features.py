"""GPU: per-Gaussian feature channels (`features=[P, F]`, the requests' `features` field) against the colour path,
which the parity tests pin to the reference, and against a float64 restatement of the compositing:
  - a feature channel equals the colour channel of a colors_precomp = features, bg = 0 render, bit for bit, on the dense, raw,
    quantised and anti-aliased paths, and the variable-SH inference path's feature image equals the dense path's;
  - channels are independent: an F = 67 render is the concatenation of its slices rendered on their own (chunk boundaries);
  - nothing else moves: colour, radii, n_contrib, final_T and the maps are bit-identical with features present, and a feature image
    without a gradient leaves the deterministic backward's gradients bit-identical;
  - the gradients of a loss on the features equal those of the equivalent colour render (dL_dfeatures == dL_dcolors_precomp), and a
    loss on colour and features together equals the sum of the two, within the maps tests' 1e-4 of each array's scale;
  - the feature image and dL_dfeatures against a float64 restatement on the backward-boundary scenes (tests/backward_edges.py);
  - P = 0 and R = 0 give zeros; Adam on 16 feature channels lowers an L2 loss; the full C3 scene with F = 32 stays finite and leaves
    the colour bit-identical."""
import math
from types import SimpleNamespace

import pytest
import torch

import backward_edges as BE
import ours as O
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _C
from gs_b200 import synth
from gs_b200.model import GaussianModelView

pytestmark = pytest.mark.gpu

DEV = "cuda"
EMPTY = torch.Tensor([])


def _features(P, F, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(P, F, generator=g).to(DEV)


def _colour_groups(feat):
    """The channels of `feat` as [P, 3] colour tensors (the last one padded with zeros)."""
    P, F = feat.shape
    pad = torch.zeros(P, (F + 2) // 3 * 3, device=feat.device)
    pad[:, :F] = feat
    return [pad[:, 3 * k:3 * k + 3].contiguous() for k in range(pad.shape[1] // 3)]


def _fwd(scene, cam, bg, prune=None, quant=None, colors=None, aa=False, maps=False, features=None, raw=False):
    """_C.rasterize_gaussians; `raw` renders from (features_dc, features_rest, log-scales, rotations) of the scene."""
    args = O.forward_args(scene, cam, bg, None if colors is None else {"colors_precomp": colors})
    kw = dict(return_maps=maps, antialiasing=aa, **O.device_kw(prune, quant))
    if features is not None:
        kw["features"] = features
    if raw:
        args = _raw_args(args)
        kw["raw"] = _raw_tuple(scene, colors is not None)
    return args, _C.rasterize_gaussians(*args, **kw)


def _raw_tuple(scene, with_colors):
    sh = scene.sh.to(DEV)
    scaling, rotation = torch.log(scene.scales.to(DEV)).contiguous(), scene.rotations.to(DEV).contiguous()
    if with_colors:
        return (None, None, scaling, rotation)
    return (sh[:, :1].contiguous(), sh[:, 1:].contiguous(), scaling, rotation)


def _raw_args(args):
    a = list(args)
    a[4] = a[5] = a[14] = EMPTY
    return tuple(a)


def _bwd(args, out, dL, scene=None, prune=None, quant=None, aa=False, raw=False, colors=False, **kw):
    (bg, means3D, col, opacity, scales, rotations, mod, cov, view, proj, tx, ty, H, W, sh, degrees, campos, _, _) = args
    R, color, radii, geom, binning, img = out[:6]
    if raw:
        kw["raw"] = _raw_tuple(scene, colors)
    return _C.rasterize_gaussians_backward(bg, means3D, radii, col, scales, rotations, mod, cov, view, proj, tx, ty, dL.to(DEV), sh,
                                           degrees, campos, geom, R, binning, img, 0.0, False, antialiasing=aa, **O.device_kw(prune, quant),
                                           **kw)


def _config(name):
    """-> (scene, cam on the device, prune, quant, aa, raw)."""
    if name == "dense":
        s, c, p, q = O.scene_config("maps", "c1")
        return s, c.to(DEV), p, q, False, False
    if name == "quant":
        s, c, p, q = O.scene_config("maps", "quant")
        return s, c.to(DEV), p, q, False, False
    if name == "aa":
        s, c, p, q = O.scene_config("aa", "pruned")
        return s, c.to(DEV), p, q, True, False
    s, c, p, q = O.scene_config("aa", "mixed")                   # raw: M = 16 -> 15 rest coefficients
    assert s.sh.shape[1] == 16
    return s, c.to(DEV), p, q, False, True


PATHS = ["dense", "quant", "aa", "raw"]


@pytest.mark.parametrize("path", PATHS)
def test_feature_channels_equal_the_colour_channels_bitwise(path):
    scene, cam, prune, quant, aa, raw = _config(path)
    feat = _features(scene.P, 7, 11)
    _, out = _fwd(scene, cam, torch.tensor([0.3, 0.2, 0.1], device=DEV), prune, quant, aa=aa, features=feat, raw=raw)
    img = out[-1]
    assert img.shape == (7, cam.image_height, cam.image_width) and len(out) == 7
    zero3 = torch.zeros(3, device=DEV)
    for k, col in enumerate(_colour_groups(feat)):
        _, ref = _fwd(scene, cam, zero3, prune, quant, colors=col, aa=aa, raw=raw)
        assert ref[0] == out[0] and torch.equal(ref[2], out[2])
        n = min(3, 7 - 3 * k)
        assert O.same(img[3 * k:3 * k + n], ref[1][:n]), k
    assert float(img.abs().max()) > 0


def test_variable_sh_feature_image_equals_the_dense_one():
    W, H = 320, 200
    scene = synth.make_scene(20_000, 85, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03), M=16)
    cam = synth.make_camera(W, H).to(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    flat, pbc, cum, cn = scene.packed_sh()
    a = O.forward_args(scene, cam, bg)
    feat = _features(scene.P, 5, 12)
    packed = _C.rasterize_gaussians_variableSH_bands(a[0], a[1], EMPTY, a[3], a[4], a[5], 1.0, EMPTY, a[8], a[9], a[10], a[11], H, W,
                                                     flat.to(DEV), pbc, cum, cn, a[15], a[16], False, False, features=feat)
    _, dense = _fwd(scene, cam, bg, features=feat)
    assert len(packed) == 7 and O.same(packed[-1], dense[-1]) and float(dense[-1].abs().max()) > 0


def test_channels_are_independent():
    scene, cam, prune, quant, _, _ = _config("dense")
    bg = torch.zeros(3, device=DEV)
    feat = _features(scene.P, 67, 13)
    _, full = _fwd(scene, cam, bg, features=feat)
    parts = []
    for lo, hi in ((0, 1), (1, 4), (4, 67)):
        _, o = _fwd(scene, cam, bg, features=feat[:, lo:hi].contiguous())
        parts.append(o[-1])
    assert O.same(full[-1], torch.cat(parts, 0))
    for lo, hi in ((8, 16), (15, 17), (63, 67)):
        _, o = _fwd(scene, cam, bg, features=feat[:, lo:hi].contiguous())
        assert O.same(full[-1][lo:hi], o[-1]), (lo, hi)


@pytest.mark.parametrize("path", PATHS)
def test_features_change_nothing_else(path):
    scene, cam, prune, quant, aa, raw = _config(path)
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    _, plain = _fwd(scene, cam, bg, prune, quant, aa=aa, maps=True, raw=raw)
    _, withf = _fwd(scene, cam, bg, prune, quant, aa=aa, maps=True, raw=raw, features=_features(scene.P, 19, 14))
    assert len(withf) == len(plain) + 1 and withf[0] == plain[0]
    for i in (1, 2, 6, 7):
        assert O.same(withf[i], plain[i]), i
    s0, s1 = O.state(plain, cam, scene.P), O.state(withf, cam, scene.P)
    for k in ("final_T", "n_contrib", "point_list", "ranges"):
        assert torch.equal(s0[k], s1[k]), k


def _settings(cam, bg, deterministic):
    return GaussianRasterizationSettings(image_height=cam.image_height, image_width=cam.image_width, tanfovx=math.tan(cam.FoVx * 0.5),
                                         tanfovy=math.tan(cam.FoVy * 0.5), bg=bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform,
                                         projmatrix=cam.full_proj_transform, sh_degree=3, campos=cam.camera_center, prefiltered=False,
                                         debug=False, deterministic=deterministic)


def test_a_feature_image_without_gradient_leaves_the_deterministic_backward_unchanged():
    W, H = 256, 160
    scene = synth.make_scene(8000, 15, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04))
    cam = O.yaw_cam(W, H, 5.0)
    bg = torch.tensor([0.1, 0.0, 0.3], device=DEV)
    g = torch.Generator().manual_seed(16)
    Gc, Gd = torch.randn(3, H, W, generator=g).to(DEV), torch.randn(1, H, W, generator=g).to(DEV)
    feat = _features(scene.P, 9, 17)
    runs = []
    for f in (None, feat):
        m = O.Model(scene, DEV)
        means2D = torch.zeros_like(m._xyz, requires_grad=True)
        out = GaussianRasterizer(_settings(cam, bg, True))(m.get_xyz, means2D, m._opacity, shs=m.get_features, degrees=m._degrees,
                                                          scales=m.get_scaling, rotations=m.get_rotation, return_maps=True, features=f)
        ((out[0] * Gc).sum() + (out[2] * Gd).sum()).backward()
        runs.append((out, [p.grad for p in m.params()] + [means2D.grad]))
    (o0, g0), (o1, g1) = runs
    assert len(o1) == len(o0) + 1
    for a, b in zip(o0, o1):
        assert O.same(a, b)
    for a, b in zip(g0, g1):
        assert O.same(a, b)


def _assert_close(got, exp, tol=1e-4, name=""):
    got, exp = got.detach().cpu().double(), exp.detach().cpu().double()
    scale = float(exp.abs().max())
    err = float((got - exp).abs().max())
    assert err <= tol * scale + 1e-30, (name, err, scale)


def _compare_grads(got, exp, skip, tol=1e-4):
    assert len(got) == len(exp)
    n = 0
    for i, (a, b) in enumerate(zip(got, exp)):
        if i in skip or a is None or b is None or a.numel() == 0:
            continue
        _assert_close(a, b, tol, i)
        n += 1
    return n


@pytest.mark.parametrize("path", PATHS)
def test_feature_gradients_equal_the_colour_gradients(path):
    scene, cam, prune, quant, aa, raw = _config(path)
    H, W = cam.image_height, cam.image_width
    feat = _features(scene.P, 3, 18)
    g = torch.Generator().manual_seed(19)
    Gf = torch.randn(3, H, W, generator=g).to(DEV)
    bg = torch.tensor([0.5, 0.5, 0.5], device=DEV)
    zero3 = torch.zeros(3, device=DEV)
    cfg = dict(prune=prune, quant=quant, aa=aa, raw=raw)
    args, out = _fwd(scene, cam, bg, features=feat, **{k: v for k, v in cfg.items()})
    got = _bwd(args, out, torch.zeros(3, H, W), scene, features=feat, dL_dfeatures_out=Gf, camera_grads=True, **cfg)
    argsc, outc = _fwd(scene, cam, zero3, colors=feat, **cfg)
    exp = _bwd(argsc, outc, Gf, scene, colors=True, camera_grads=True, **cfg)
    dfeat, got = got[-1], got[:-1]
    assert dfeat.shape == (scene.P, 3)
    _assert_close(dfeat, exp[1], name="dL_dfeatures")
    # colours and SH: the feature run has SH and no colour loss, the colour run has colours; everything else must agree
    sh_slots = (1, 5, 6) if raw else (1, 5)
    assert _compare_grads(got, exp, sh_slots) >= 5
    assert float(got[2].abs().max()) > 0 and float(dfeat.abs().max()) > 0
    # culled and pruned Gaussians: zero feature rows
    off = out[2] == 0
    if bool(off.any()):
        assert float(dfeat[off].abs().max()) == 0.0


@pytest.mark.parametrize("path", ["dense", "quant"])
def test_colour_and_feature_losses_add(path):
    scene, cam, prune, quant, aa, raw = _config(path)
    H, W = cam.image_height, cam.image_width
    feat = _features(scene.P, 5, 20)
    g = torch.Generator().manual_seed(21)
    Gc, Gf = torch.randn(3, H, W, generator=g).to(DEV), torch.randn(5, H, W, generator=g).to(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    args, out = _fwd(scene, cam, bg, prune, quant, features=feat)
    both = _bwd(args, out, Gc, prune=prune, quant=quant, features=feat, dL_dfeatures_out=Gf)
    colour = _bwd(args, out, Gc, prune=prune, quant=quant)
    fonly = _bwd(args, out, torch.zeros(3, H, W), prune=prune, quant=quant, features=feat, dL_dfeatures_out=Gf)
    exp = tuple(a + b for a, b in zip(colour, fonly[:-1]))
    assert _compare_grads(both[:-1], exp, (), tol=2e-4) >= 5
    _assert_close(both[-1], fonly[-1], name="dL_dfeatures")


# ---- float64 restatement ----------------------------------------------------------------------------------------------------------

def _restate64(o, st, feat, G, W, H):
    """The feature image and dL_dfeatures in float64 over the kernel's own lists and n_contrib: alpha = min(0.99, o exp(power)) of the
    forward's means2D / conic / opacity, pairs with power > 0 or alpha < 1/255 skipped, T the running product.  -> (image [F,H,W],
    dL_dfeatures [P,F], borderline pixel mask [H,W]: some pair's alpha or power lies within float rounding of a threshold)."""
    F64 = torch.float64
    m2, co = o["means2D"].to(F64), o["conic_opacity"].to(F64)
    f, G = feat.to(F64), G.to(F64)
    P, F = f.shape
    img = torch.zeros(F, H, W, dtype=F64, device=DEV)
    dfeat = torch.zeros(P, F, dtype=F64, device=DEV)
    border = torch.zeros(H, W, dtype=torch.bool, device=DEV)
    ranges, pl, nc = st["ranges"].long(), st["point_list"].long(), st["n_contrib"].long()
    tx = (W + 15) // 16
    for t in range(ranges.shape[0]):
        a, b = int(ranges[t, 0]), int(ranges[t, 1])
        if b <= a:
            continue
        ids = pl[a:b]
        x0, y0 = (t % tx) * 16, (t // tx) * 16
        ys, xs = torch.meshgrid(torch.arange(y0, min(y0 + 16, H), device=DEV), torch.arange(x0, min(x0 + 16, W), device=DEV), indexing="ij")
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        dx = m2[ids, 0][None, :] - xs[:, None].to(F64)
        dy = m2[ids, 1][None, :] - ys[:, None].to(F64)
        A, B, Cc, op = co[ids, 0][None], co[ids, 1][None], co[ids, 2][None], co[ids, 3][None]
        power = -0.5 * (A * dx * dx + Cc * dy * dy) - B * dx * dy
        raw_alpha = op * torch.exp(power)
        alpha = raw_alpha.clamp(max=0.99)
        pos = torch.arange(b - a, device=DEV)[None, :]
        inlist = pos < nc[ys, xs][:, None]
        keep = inlist & (power <= 0) & (alpha >= 1.0 / 255.0)
        border[ys, xs] |= (inlist & (((raw_alpha * 255.0 - 1.0).abs() < 1e-4) | (power.abs() < 1e-6))).any(1)
        al = torch.where(keep, alpha, torch.zeros_like(alpha))
        T = torch.cumprod(torch.cat([torch.ones_like(al[:, :1]), 1.0 - al[:, :-1]], 1), 1)
        w = al * T                                                    # [pixels, list]
        img[:, ys, xs] = (w @ f[ids]).T
        dfeat.index_add_(0, ids, w.T @ G[:, ys, xs].T)
    return img, dfeat, border


@pytest.mark.parametrize("F", [1, 5, 16, 67])
@pytest.mark.parametrize("name", ["staircase", "odd_3x7", "odd_17x15", "odd_33x1", "saturation"])
def test_against_float64_restatement(name, F):
    case = BE.build(name)
    scene, cam = case.scene, case.cam.to(DEV)
    W, H = cam.image_width, cam.image_height
    feat = _features(scene.P, F, 22)
    dbg = {}
    args = O.forward_args(scene, cam, case.bg.to(DEV) if isinstance(case.bg, torch.Tensor) else torch.tensor(case.bg, device=DEV))
    out = _C.rasterize_gaussians(*args, debug_out=dbg, features=feat)
    st = O.state(out, cam, scene.P)
    g = torch.Generator().manual_seed(23)
    G = torch.randn(F, H, W, generator=g).to(DEV)
    ref_img, _, border = _restate64(dbg, st, feat, G, W, H)
    ok = ~border
    got = out[-1].double()
    scale = float(ref_img.abs().max())
    assert scale > 0
    err = (got - ref_img).abs()[:, ok]
    assert float(err.max()) <= 1e-5 * scale, (float(err.max()), scale)
    # dL_dfeatures with the borderline pixels' gradient set to zero
    Gm = G * ok[None].to(G.dtype)
    _, ref_d, _ = _restate64(dbg, st, feat, Gm, W, H)
    _, ref_abs, _ = _restate64(dbg, st, feat, Gm.abs(), W, H)             # sum of |alpha T g|: the size of each sum's terms
    d = _bwd(args, out, torch.zeros(3, H, W), features=feat, dL_dfeatures_out=Gm)[-1].double()
    dscale = float(ref_d.abs().max())
    assert dscale > 0
    bar = 1e-4 * ref_abs + 1e-6 * dscale
    assert bool(((d - ref_d).abs() <= bar).all()), float(((d - ref_d).abs() / bar).max())
    off = out[2] == 0
    if bool(off.any()):
        assert float(d[off].abs().max()) == 0.0


def test_empty_and_culled_scenes_give_zeros():
    W, H = 64, 48
    cam = synth.make_camera(W, H).to(DEV)
    bg = torch.tensor([0.3, 0.3, 0.3], device=DEV)
    for scene in O.empty_and_culled_scenes():
        feat = _features(scene.P, 6, 24)
        args, out = _fwd(scene, cam, bg, features=feat)
        assert out[0] == 0 and out[-1].shape == (6, H, W) and float(out[-1].abs().max()) == 0.0
        gr = _bwd(args, out, torch.ones(3, H, W), features=feat, dL_dfeatures_out=torch.ones(6, H, W, device=DEV))
        assert gr[-1].shape == (scene.P, 6)
        for t in gr:
            if t is not None and t.numel():
                assert float(t.abs().max()) == 0.0


def test_adam_fits_a_16_channel_feature_map():
    from gaussian_renderer import render
    W, H = 192, 128
    scene = synth.make_scene(6_000, 25, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04), M=16)
    cam = O.yaw_cam(W, H, 0.0)
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    bg = torch.zeros(3, device=DEV)
    pc = GaussianModelView(scene, DEV)
    with torch.no_grad():
        target = render(cam, pc, pipe, bg, features=_features(scene.P, 16, 26))["features"].clone()
    feat = torch.zeros(scene.P, 16, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([feat], lr=0.05)
    losses = []
    for _ in range(30):
        opt.zero_grad(set_to_none=True)
        pkg = render(cam, pc, pipe, bg, features=feat)
        loss = ((pkg["features"] - target) ** 2).mean()
        loss.backward()
        assert feat.grad is not None and torch.isfinite(feat.grad).all()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < 0.3 * losses[0], losses


def test_full_size_c3_with_32_channels():
    import bench
    dev = torch.device(DEV, 0)
    _, W, H, scene, quant, _ = bench.build_workload(SimpleNamespace(config="C3", points=0), dev, 0, 1)
    cam = bench.bench_cameras(W, H, 1)[0].to(DEV)
    bg = torch.zeros(3, device=DEV)
    feat = _features(scene.P, 32, 27)
    args, plain = _fwd(scene, cam, bg, quant=quant)
    _, withf = _fwd(scene, cam, bg, quant=quant, features=feat)
    assert withf[0] == plain[0] > 0 and O.same(withf[1], plain[1]) and O.same(withf[2], plain[2])
    img = withf[-1]
    assert img.shape == (32, H, W) and bool(torch.isfinite(img).all()) and float(img.abs().max()) > 0
    G = torch.randn(32, H, W, device=DEV)
    gr = _bwd(args, withf, torch.zeros(3, H, W), quant=quant, features=feat, dL_dfeatures_out=G)
    for t in gr:
        if t is not None and t.numel():
            assert bool(torch.isfinite(t).all())
    assert float(gr[-1].abs().max()) > 0
