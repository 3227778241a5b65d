"""GPU: rendering from the model's raw parameters (`pipe.fused_activations`, DESIGN.md §5h) against today's path through the
model's get_scaling / get_rotation / get_features properties (autograd through torch.exp, F.normalize and torch.cat).
  1. forward: colour, radii, R, the maps and every debug export bit-identical, C = 0/3/8/15, mixed degrees, AA on and off, prune
     mask, quaternion norms from 1e-3 to 1e3; a C1-sized scene and P = 100 k at 1920x1080;
  2. gradients on an 8x4 image (one warp: the render backward has one addition order): the SH, opacity and screen-space gradients
     are bit-identical; those of xyz, scaling, rotation and the camera come from the separately compiled raw kernel, whose
     multiply-adds may fuse differently, and agree within 1e-5 of each array's largest magnitude.  On 16x16 and larger images the
     render backward's atomic additions have no fixed order (two runs of either path differ): there the gap between the paths is
     bounded by 1e-5 or by a few times the run-to-run gap of the activated path (observed values printed with pytest -s);
  3. the graph reaches the six parameters through the rasterizer's node and AccumulateGrad only; the .grad tensors are contiguous;
  4. combinations: a loss on invdepth only, override_color, lambda_sh_sparsity, `_C` accumulate over two views, P = 0 and R = 0,
     run-to-run forward bytes and a side stream;
  5. training: 25 GaussianAdam steps on 8x4 agree to rounding, 90 steps reduce the loss, a render after densify_and_prune uses the new params;
  6. memory: the peak over forward + backward drops by more than the 192 B per Gaussian of the [P,16,3] copy at P = 1 M (its
     gradient's clone is made after the copy is freed, so the two never add up at the peak)."""
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import ours as O
from diff_gaussian_rasterization import _C
from gs_b200 import densify, synth
from gs_b200.optim import GaussianAdam

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
DEG_OF_C = {0: 0, 3: 1, 8: 2, 15: 3}
NAMES = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")


class Model:
    """The reference GaussianModel's leaf attributes, activations and properties (scene/gaussian_model.py:32-47, 140-163)."""

    def __init__(self, scene, Cn=15, seed=0, norm_range=(-3.0, 3.0)):
        g = torch.Generator().manual_seed(seed)
        P = scene.P
        deg = DEG_OF_C[Cn]
        self._xyz = scene.means3D.to(DEV).clone().requires_grad_()
        self._features_dc = scene.sh[:, :1].to(DEV).contiguous().requires_grad_()
        self._features_rest = scene.sh[:, 1:1 + Cn].to(DEV).contiguous().requires_grad_()
        self._opacity = scene.opacity.to(DEV).clone().requires_grad_()
        self._scaling = torch.log(scene.scales).to(DEV).requires_grad_()
        norms = torch.pow(10.0, torch.empty(P, 1).uniform_(*norm_range, generator=g))
        self._rotation = (scene.rotations * norms).to(DEV).contiguous().requires_grad_()
        self._degrees = scene.degrees.clamp(max=deg).to(DEV).contiguous()
        self.scaling_activation = torch.exp
        self.rotation_activation = F.normalize
        self.active_sh_degree = self.max_sh_degree = deg
        self.per_band_count = [int((self._degrees == d).sum()) for d in range(4)]

    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: s.scaling_activation(s._scaling))
    get_rotation = property(lambda s: s.rotation_activation(s._rotation))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))

    def leaves(self):
        return [getattr(self, n) for n in NAMES]

    def clone(self):
        c = object.__new__(Model)
        c.__dict__.update(self.__dict__)
        for n in NAMES:
            setattr(c, n, getattr(self, n).detach().clone().requires_grad_())
        return c


def _pipe(fused, aa=False):
    return SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False, fused_activations=fused, antialiasing=aa)


def _scene(P, W, H, seed, mixed=True, ls=math.log(0.02)):
    return synth.make_scene(P, seed, mixed_degrees=mixed, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=ls)


def _render(m, cam, fused, aa=False, **kw):
    from gaussian_renderer import render
    return render(cam, m, _pipe(fused, aa), torch.tensor([0.2, 0.4, 0.6], device=DEV), **kw)


def _both(model, cam, aa=False, loss=None, **kw):
    """(activated, fused) renders of two copies of `model`, each followed by loss(pkg).backward() when loss is given."""
    out = []
    for fused in (False, True):
        m = model.clone()
        c = SimpleNamespace(**{k: (v.detach().clone().requires_grad_() if torch.is_tensor(v) and v.requires_grad else v)
                               for k, v in vars(cam).items()})
        pkg = _render(m, c, fused, aa, **kw)
        if loss is not None:
            loss(pkg).backward()
        out.append((m, c, pkg))
    return out


# ---- 1. forward -----------------------------------------------------------------------------------------------------------------

def _c_forward(m, cam, fused, aa, prune=None, dbg=None):
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    e = torch.empty(0)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    common = (cam.world_view_transform, cam.full_proj_transform, tx, ty, cam.image_height, cam.image_width)
    with torch.no_grad():
        if fused:
            args = (bg, m._xyz, e, m._opacity, e, e, 1.0, e) + common + (e, m._degrees, cam.camera_center, False, False)
            raw = (m._features_dc, m._features_rest, m._scaling, m._rotation)
            return _C.rasterize_gaussians(*args, prune_mask=prune, return_maps=True, antialiasing=aa, debug_out=dbg, raw=raw)
        args = (bg, m._xyz, e, m._opacity, m.get_scaling, m.get_rotation, 1.0, e) + common + \
            (m.get_features, m._degrees, cam.camera_center, False, False)
        return _C.rasterize_gaussians(*args, prune_mask=prune, return_maps=True, antialiasing=aa, debug_out=dbg)


def _check_forward(m, cam, aa, prune=None):
    d0, d1 = {}, {}
    o0 = _c_forward(m, cam, False, aa, prune, d0)
    o1 = _c_forward(m, cam, True, aa, prune, d1)
    torch.cuda.synchronize()
    assert o0[0] == o1[0] and o0[0] > 0
    for k in (1, 2, 6, 7):
        assert O.same(o0[k], o1[k]), k
    for k in d0:
        assert O.same(d0[k], d1[k]), k


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("Cn", [0, 3, 8, 15])
def test_forward_bit_identical(Cn, aa):
    W, H = 320, 200
    m = Model(_scene(20_000, W, H, 300 + Cn), Cn, seed=Cn)
    prune = synth.prune_mask(m._xyz.shape[0], 7).to(DEV) if Cn in (3, 15) else None
    _check_forward(m, O.yaw_cam(W, H, -4.0), aa, prune)


@pytest.mark.parametrize("size", ["c1", "100k_1080p"])
def test_forward_bit_identical_sizes(size):
    if size == "c1":
        W, H = synth.config_image("C1")
        scene = synth.config_scene("C1")
        Cn = 0
    else:
        W, H = 1920, 1080
        scene = _scene(100_000, W, H, 31, ls=math.log(0.01))
        Cn = 15
    m = Model(scene, Cn, seed=5)
    for aa in (False, True):
        _check_forward(m, O.yaw_cam(W, H, 3.0), aa)


def test_forward_tiny_and_zero_quaternions():
    W, H = 160, 120
    m = Model(_scene(5_000, W, H, 41), 15, seed=2)
    with torch.no_grad():
        m._rotation[:50] *= 1e-14                # below the 1e-12 clamp of F.normalize
        m._rotation[50:60] = 0
    _check_forward(m, O.yaw_cam(W, H), False)


# ---- 2. gradients ---------------------------------------------------------------------------------------------------------------

def _loss_all(weights):
    def f(pkg):
        return (pkg["render"] * weights[0]).sum() + (pkg["invdepth"] * weights[1]).sum() + (pkg["alpha"] * weights[2]).sum()
    return f


def _weights(W, H, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(3, H, W, generator=g).to(DEV), torch.randn(1, H, W, generator=g).to(DEV),
            torch.randn(1, H, W, generator=g).to(DEV)]


def _grads(m, c):
    return [p.grad for p in m.leaves()] + [c.world_view_transform.grad, c.full_proj_transform.grad, c.camera_center.grad]


EXACT = ("_features_dc", "_features_rest", "_opacity", "means2D")


def _rel(a, b):
    return float((a.double() - b.double()).abs().max()) / (float(a.double().abs().max()) + 1e-30) if a.numel() else 0.0


def _compare(names, ga, gb, tol=1e-5, tag="", exact=EXACT, floor=None):
    """Bit-identical for `exact`, else within max(tol, floor[name]) of the array's largest magnitude; prints the gaps."""
    for name, a, b in zip(names, ga, gb):
        if a is None and b is None:
            continue
        assert a is not None and b is not None and a.shape == b.shape, name
        if floor is not None:
            tol_n = max(tol, floor[name])
        else:
            tol_n = tol
        if name in exact:
            assert O.same(a, b), name
        else:
            err = _rel(a, b)
            print(f"{tag} {name:16s} max |fused - activated| / max |activated| = {err:.3e}, "
                  f"{int((O.bits(a) != O.bits(b)).sum())} of {a.numel()} differ" + (f" (run-to-run {floor[name]:.3e})" if floor else ""))
            assert err <= tol_n, (name, err)


def _floor(model, cam, aa, loss, names, **kw):
    """Run-to-run gap of the activated path per gradient (the render backward's atomic order is not fixed on larger images)."""
    (ma, ca, pa), (mb, cb, pb) = [_both(model, cam, aa, loss, **kw)[0] for _ in range(2)]
    ga, gb = _grads(ma, ca) + [pa["viewspace_points"].grad], _grads(mb, cb) + [pb["viewspace_points"].grad]
    return {n: (_rel(a, b) if a is not None and b is not None else 0.0) for n, a, b in zip(names, ga, gb)}


ALL = NAMES + ("view", "proj", "campos", "means2D")


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("size", [(8, 4), (16, 16)])
@pytest.mark.parametrize("Cn", [3, 15])
def test_single_tile_gradients(Cn, size, aa):
    W, H = size
    m = Model(_scene(3_000, W, H, 50 + Cn, ls=math.log(0.05)), Cn, seed=Cn)
    cam, loss = O.yaw_cam(W, H, 2.0, grad=True), _loss_all(_weights(W, H, 9))
    (m0, c0, p0), (m1, c1, p1) = _both(m, cam, aa, loss, return_maps=True)
    assert int((p0["radii"] > 0).sum()) > 100
    one_warp = W * H <= 32
    floor = None if one_warp else {n: 4 * v for n, v in _floor(m, cam, aa, loss, ALL, return_maps=True).items()}
    _compare(ALL, _grads(m0, c0) + [p0["viewspace_points"].grad], _grads(m1, c1) + [p1["viewspace_points"].grad],
             tag=f"tile C={Cn} {W}x{H} aa={aa}", exact=EXACT if one_warp else (), floor=floor)


def test_fullsize_gradients():
    W, H = 1920, 1080
    m = Model(_scene(100_000, W, H, 61, ls=math.log(0.01)), 15, seed=4)
    cam, loss = O.yaw_cam(W, H, 2.0, grad=True), _loss_all(_weights(W, H, 3))
    (m0, c0, p0), (m1, c1, p1) = _both(m, cam, False, loss, return_maps=True)
    floor = {n: 4 * v for n, v in _floor(m, cam, False, loss, ALL, return_maps=True).items()}
    _compare(ALL, _grads(m0, c0) + [p0["viewspace_points"].grad], _grads(m1, c1) + [p1["viewspace_points"].grad], tag="1080p",
             exact=(), floor=floor)


# ---- 3. graph -------------------------------------------------------------------------------------------------------------------

def test_graph_holds_no_activation_nodes():
    W, H = 64, 48
    m = Model(_scene(2_000, W, H, 71), 15)
    pkg = _render(m, O.yaw_cam(W, H), True)
    seen, stack, names, leaves = set(), [pkg["render"].grad_fn], [], set()
    while stack:
        fn = stack.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        names.append(type(fn).__name__)
        if type(fn).__name__ == "AccumulateGrad":
            leaves.add(id(fn.variable))
        stack.extend(f for f, _ in fn.next_functions)
    assert not [n for n in names if any(k in n for k in ("Cat", "Exp", "Div", "Norm", "Clamp", "Expand"))], names
    assert all(id(p) in leaves for p in m.leaves())
    pkg["render"].sum().backward()
    assert all(p.grad is not None and p.grad.is_contiguous() and p.grad.shape == p.shape for p in m.leaves())


# ---- 4. combinations ------------------------------------------------------------------------------------------------------------

def test_invdepth_only_loss():
    W, H = 8, 4
    m = Model(_scene(3_000, W, H, 81, ls=math.log(0.05)), 15)
    w = _weights(W, H, 4)[1]
    (m0, _, _), (m1, _, _) = _both(m, O.yaw_cam(W, H), False, lambda p: (p["invdepth"] * w).sum(), return_maps=True)
    _compare(NAMES, [p.grad for p in m0.leaves()], [p.grad for p in m1.leaves()], tag="invdepth-only")
    assert float(m1._features_rest.grad.abs().max()) == 0.0 and float(m1._scaling.grad.abs().max()) > 0


def test_override_color():
    W, H = 8, 4
    m = Model(_scene(3_000, W, H, 82, ls=math.log(0.05)), 15)
    colors = torch.rand(m._xyz.shape[0], 3, device=DEV)
    w = _weights(W, H, 5)[0]
    outs = []
    for fused in (False, True):
        mm = m.clone()
        col = colors.clone().requires_grad_()
        pkg = _render(mm, O.yaw_cam(W, H), fused, override_color=col)
        (pkg["render"] * w).sum().backward()
        outs.append((mm, col, pkg))
    (m0, col0, p0), (m1, col1, p1) = outs
    assert O.same(p0["render"], p1["render"]) and O.same(col0.grad, col1.grad)
    assert int((p0["radii"] > 0).sum()) > 100
    assert m1._features_dc.grad is None and m1._features_rest.grad is None
    _compare(("_xyz", "_opacity", "_scaling", "_rotation"), [getattr(m0, n).grad for n in ("_xyz", "_opacity", "_scaling", "_rotation")],
             [getattr(m1, n).grad for n in ("_xyz", "_opacity", "_scaling", "_rotation")], tag="override_color")


def test_lambda_sh_sparsity():
    W, H = 8, 4
    m = Model(_scene(3_000, W, H, 83, ls=math.log(0.05)), 15)
    w = _weights(W, H, 6)[0]
    (m0, _, _), (m1, _, p1) = _both(m, O.yaw_cam(W, H), False, lambda p: (p["render"] * w).sum(), lambda_sh_sparsity=0.5)
    # the sign term's addition may fuse with the colour term differently in the raw kernel: the rest gradients agree to rounding
    _compare(NAMES, [p.grad for p in m0.leaves()], [p.grad for p in m1.leaves()], tag="lambda_sh_sparsity",
             exact=("_features_dc", "_opacity"))
    # the sign term lives in the active bands only: every rest coefficient beyond a Gaussian's degree has a zero gradient
    g = m1._features_rest.grad
    ncoef = (m1._degrees.view(-1) + 1) ** 2 - 1
    inactive = torch.arange(15, device=DEV).view(1, 15) >= ncoef.view(-1, 1)
    assert float(g[inactive].abs().max()) == 0.0
    vis = p1["radii"] > 0
    assert float(g[vis & (ncoef > 0)].abs().max()) > 0


def _c_raw_backward(m, cam, out, dL, acc=None):
    e = torch.empty(0)
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    R, color, radii, geom, binning, img = out[:6]
    raw = (m._features_dc.detach(), m._features_rest.detach(), m._scaling.detach(), m._rotation.detach())
    return _C.rasterize_gaussians_backward(torch.tensor([0.2, 0.4, 0.6], device=DEV), m._xyz.detach(), radii, e, e, e, 1.0, e,
                                           cam.world_view_transform, cam.full_proj_transform, tx, ty, dL, e, m._degrees,
                                           cam.camera_center, geom, R, binning, img, 0.0, False, raw=raw, accumulate_into=acc)


def test_c_accumulate_is_the_sum_of_two_views():
    W, H = 8, 4                                        # one warp: every backward has one addition order
    m = Model(_scene(3_000, W, H, 84, ls=math.log(0.05)), 8)
    cams = [O.yaw_cam(W, H, -1.0), O.yaw_cam(W, H, 1.0)]
    outs = [_c_forward(m, c, True, False) for c in cams]
    dLs = [synth.grad_image(W, H, s).to(DEV) for s in (1, 2)]
    g1 = [t.clone() if t is not None else None for t in _c_raw_backward(m, cams[0], outs[0], dLs[0])]
    g2 = _c_raw_backward(m, cams[1], outs[1], dLs[1])
    acc = _c_raw_backward(m, cams[0], outs[0], dLs[0])
    acc = _c_raw_backward(m, cams[1], outs[1], dLs[1], acc=acc)
    torch.cuda.synchronize()
    assert len(acc) == 9 and acc[1] is None and acc[4] is None
    assert int((outs[0][2] > 0).sum()) > 100 and int((outs[1][2] > 0).sum()) > 100
    # equal values (accumulate mode skips adding a zero, so a -0 may stay where torch's sum gives +0)
    for k in (0, 2, 3, 5, 6, 7, 8):
        assert torch.equal(acc[k], g1[k] + g2[k]), k


def test_empty_scene_and_no_instance():
    W, H = 32, 32
    for P in (0, 500):                                 # P = 0; every Gaussian behind the camera (R = 0)
        m = Model(_scene(max(P, 1), W, H, 85), 15)
        if P == 0:
            for n in NAMES:
                setattr(m, n, getattr(m, n).detach()[:0].clone().requires_grad_())
            m._degrees = m._degrees[:0]
        else:
            with torch.no_grad():
                m._xyz[:, 2] -= 100.0
        m1 = m.clone()
        p1 = _render(m1, O.yaw_cam(W, H), True)
        p1["render"].sum().backward()
        assert int(p1["radii"].sum()) == 0
        if P:
            assert O.same(p1["render"], _render(m.clone(), O.yaw_cam(W, H), False)["render"])
        for p in m1.leaves():
            assert p.grad is not None and p.grad.shape == p.shape and (p.numel() == 0 or float(p.grad.abs().max()) == 0.0)


def test_run_to_run_and_side_stream():
    W, H = 160, 120
    m = Model(_scene(10_000, W, H, 86), 15)
    w = _weights(W, H, 7)[0]

    def run():
        mm = m.clone()
        pkg = _render(mm, O.yaw_cam(W, H), True)
        (pkg["render"] * w).sum().backward()
        return [pkg["render"]] + [p.grad for p in mm.leaves()]

    a, b = run(), run()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c = run()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    # the forward is the same bytes on every run and stream; the gradients to the render backward's atomic order
    assert O.same(a[0], b[0]) and O.same(a[0], c[0])
    for x, y, z in zip(a[1:], b[1:], c[1:]):
        assert _rel(y, x) <= 1e-4 and _rel(z, x) <= 1e-4


# ---- 5. training ----------------------------------------------------------------------------------------------------------------

def _adam(m, cls=GaussianAdam):
    lrs = dict(_xyz=2e-4, _features_dc=2.5e-3, _features_rest=1.25e-4, _opacity=5e-2, _scaling=5e-3, _rotation=1e-3)
    names = dict(_xyz="xyz", _features_dc="f_dc", _features_rest="f_rest", _opacity="opacity", _scaling="scaling", _rotation="rotation")
    return cls([{"params": [getattr(m, n)], "lr": lrs[n], "name": names[n]} for n in NAMES], lr=0.0, eps=1e-15)


def test_25_adam_steps_agree():
    W, H = 8, 4
    m = Model(_scene(3_000, W, H, 91, ls=math.log(0.05)), 15)
    gt = torch.rand(3, H, W, device=DEV)
    cam = O.yaw_cam(W, H, 1.0)
    models = [m.clone(), m.clone()]
    opts = [_adam(mm) for mm in models]
    for _ in range(25):
        for fused, mm, opt in zip((False, True), models, opts):
            opt.zero_grad(set_to_none=True)
            pkg = _render(mm, cam, fused)
            (pkg["render"] - gt).abs().mean().backward()
            opt.step()
    # the rounding-level gaps of the xyz / scaling / rotation gradients move those params by a fraction of one step's size
    for n in NAMES:
        p0, p1 = getattr(models[0], n), getattr(models[1], n)
        s0, s1 = opts[0].state[p0], opts[1].state[p1]
        errs = [_rel(p0.detach(), p1.detach()), _rel(s0["exp_avg"], s1["exp_avg"]), _rel(s0["exp_avg_sq"], s1["exp_avg_sq"])]
        print(f"25 steps {n:16s} param / exp_avg / exp_avg_sq rel gap {errs[0]:.2e} {errs[1]:.2e} {errs[2]:.2e}")
        if n in ("_features_dc", "_features_rest", "_opacity") and max(errs) == 0.0:
            continue
        assert errs[0] <= 1e-5 and errs[1] <= 1e-3 and errs[2] <= 1e-3, (n, errs)


def test_90_steps_reduce_the_loss():
    from utils.loss_utils import l1_ssim_loss
    W, H = 256, 192
    target = synth.make_scene(6_000, 71, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04))
    cams = [O.yaw_cam(W, H, yaw) for yaw in (-10.0, 0.0, 10.0)]
    with torch.no_grad():
        gts = [_render(Model(target, 15, norm_range=(0.0, 0.0)), c, False)["render"].clone() for c in cams]
    g = torch.Generator().manual_seed(5)
    start = synth.Scene(target.means3D + 0.01 * torch.randn(target.means3D.shape, generator=g),
                        target.opacity + 0.5 * torch.randn(target.opacity.shape, generator=g),
                        target.scales * torch.exp(0.2 * torch.randn(target.scales.shape, generator=g)),
                        F.normalize(target.rotations + 0.1 * torch.randn(target.rotations.shape, generator=g)),
                        target.sh + 0.1 * torch.randn(target.sh.shape, generator=g), target.degrees)
    m = Model(start, 15)
    opt = _adam(m)
    losses = []
    for it in range(90):
        k = it % len(cams)
        opt.zero_grad(set_to_none=True)
        pkg = _render(m, cams[k], True)
        loss = l1_ssim_loss(pkg["render"], gts[k], 0.2)
        loss.backward()
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.leaves())
        opt.step()
        losses.append(float(loss.detach()))
    first, last = sum(losses[:3]) / 3, sum(losses[-3:]) / 3
    print(f"90 fused steps: loss {first:.4f} -> {last:.4f}")
    assert last < 0.8 * first, (first, last)


def test_render_after_densify_uses_the_new_parameters():
    W, H = 160, 120
    m = Model(_scene(10_000, W, H, 92, ls=math.log(0.05)), 15)
    m.optimizer = _adam(m)
    P = m._xyz.shape[0]
    m.percent_dense = 0.01
    m.xyz_gradient_accum = torch.zeros(P, 1, device=DEV)
    m.denom = torch.zeros(P, 1, device=DEV)
    m.max_radii2D = torch.zeros(P, device=DEV)
    cam = O.yaw_cam(W, H)
    pkg = _render(m, cam, True)
    (pkg["render"] * _weights(W, H, 8)[0]).sum().backward()
    m.optimizer.step()
    densify.add_densification_stats(m, pkg["viewspace_points"], pkg["visibility_filter"])
    densify.densify_and_prune(m, 1e-7, 0.005, 3.0, None, {})
    assert m._xyz.shape[0] != P
    m.active_sh_degree = m.max_sh_degree
    _check_forward(m, cam, False)
    pkg = _render(m, cam, True)
    pkg["render"].sum().backward()
    assert all(p.grad is not None and p.grad.shape == p.shape for p in m.leaves())


# ---- 6. memory ------------------------------------------------------------------------------------------------------------------

def test_peak_memory_drops():
    W, H = 1920, 1080
    P = 1_000_000
    m = Model(_scene(P, W, H, 93, ls=math.log(0.004)), 15)
    cam = O.yaw_cam(W, H)
    w = _weights(W, H, 9)[0]
    peaks = []
    for fused in (False, True, False, True):
        mm = m.clone()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        pkg = _render(mm, cam, fused)
        (pkg["render"] * w).sum().backward()
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del pkg, mm
    drop = min(peaks[0], peaks[2]) - max(peaks[1], peaks[3])
    print(f"P = 1M: peak over forward + backward {peaks[0] / 2**20:.1f} MiB activated, {peaks[1] / 2**20:.1f} MiB fused, "
          f"drop {drop / P:.0f} B per Gaussian")
    assert drop >= 192 * P
