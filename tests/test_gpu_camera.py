"""GPU: gradients w.r.t. the camera (viewmatrix, projmatrix, campos; gsb_backward_camera / camera_grads=True).
  1. nothing else moves: with the camera gradients on, the per-Gaussian outputs taken from the accumulator are bit-identical and
     the computed ones agree to fp32 rounding; with and without anti-aliasing the camera outputs (and with it every output) are
     the same bytes on every run and on any stream; P = 0 and R = 0 give zeros, with the camera gradients, the maps or both;
  2./3. chain check: the kernel's own screen-space gradients (dL_dmeans2D, dL_dconic, dL_dcolors) chained through the float64
     restatement of the preprocess (restate64.py) w.r.t. view, proj and campos as three independent tensors give the kernel's
     camera gradients; the same chain applied to the fp64 oracle's screen-space gradients agrees at the oracle gradient bar;
  4. invariance, with and without anti-aliasing: translating or rotating the whole world together with the camera leaves the
     image unchanged, so the directional derivative formed from dL_dmeans3D / dL_drotations and the camera gradients vanishes;
  5. maps: the camera gradients of the invdepth and alpha maps equal those of the colour renders that emulate the maps;
  6. end to end: Adam on a 6-vector pose through render() recovers a perturbed camera.
Observed ratios are printed (pytest -s) so that the bars below can be read against what the kernels actually do."""
import math
from functools import partial
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import ours as O
import restate64 as R64
from camera_chain import chain as _chain, check as _check
from gs_b200 import synth
from gs_b200.model import GaussianModelView

pytestmark = pytest.mark.gpu

DEV = "cuda"
F64 = torch.float64

_config = partial(O.scene_config, "camera")


# Outputs the preprocess backward copies or scales from the accumulator are bit-identical with the camera gradients on.  The ones
# it computes through the covariance / SH chains come from a separately compiled kernel (CAM = true), whose multiply-adds the
# compiler may fuse differently: they agree to fp32 rounding.
_BITWISE = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dconic")


def _close(a, b):
    return a.shape == b.shape and float((a - b).abs().max()) <= 1e-6 * float(a.abs().max()) + 1e-30


# ---- 1. nothing else moves ---------------------------------------------------------------------------------------------------
# The render backward adds each Gaussian's per-warp sums (one warp = an 8x4 pixel block) into its accumulator with float
# reductions, in whatever order the warps finish: two backward calls over a larger image agree only to rounding, with or without
# the camera gradients.  An 8x4 image is one warp block, so there every accumulator receives one addition and two calls must
# agree bit for bit; with the default 50 degree field of view every Gaussian in the frustum still lands in it.

def _small(name):
    scene, _, prune, quant = _config({"maps": "mixed", "accumulate": "mixed"}.get(name, name))
    return scene, O.yaw_cam(8, 4, 2.0, dev="cpu"), prune, quant


def _small_case(name):
    """One 8x4 case: -> (scene, cam, prune, quant, bg, dL, backward keywords, forward args, forward outputs)."""
    scene, cam, prune, quant = _small(name)
    cam = cam.to(DEV)
    H, W = cam.image_height, cam.image_width
    g = torch.Generator().manual_seed(170)
    dL = torch.randn(3, H, W, generator=g).to(DEV)
    extra = dict(want_conic=True)
    if name == "maps":
        extra.update(dL_dinvdepth=torch.randn(1, H, W, generator=g).to(DEV), dL_dalpha=torch.randn(1, H, W, generator=g).to(DEV))
    bg = torch.tensor([0.1, 0.3, 0.2], device=DEV)
    args, out = O.forward(scene, cam, bg, prune, quant, maps=(name == "maps"))
    return scene, cam, prune, quant, bg, dL, extra, args, out


@pytest.mark.parametrize("name", ["c1", "quant", "pruned", "maps", "accumulate"])
def test_camera_grads_change_nothing_else(name):
    scene, cam, prune, quant, bg, dL, extra, args, out = _small_case(name)
    H, W = cam.image_height, cam.image_width
    assert int((out[2] > 0).sum()) > 1000
    if name == "accumulate":
        # two views into one set of buffers; the second call also exports its own dL_dmeans2D
        args0, out0 = O.forward(scene, O.yaw_cam(W, H, 3.0), bg, prune, quant)
        base = O.backward(args0, out0, dL, prune, quant)
        acc_a, acc_b = tuple(t.clone() for t in base), tuple(t.clone() for t in base)
        v_a, v_b = torch.empty(scene.P, 3, device=DEV), torch.empty(scene.P, 3, device=DEV)
        plain = O.backward(args, out, dL, prune, quant, accumulate_into=acc_a, view_means2D=v_a, **extra)
        cam1 = O.backward(args, out, dL, prune, quant, accumulate_into=acc_b, view_means2D=v_b, camera_grads=True, **extra)
        assert O.same(v_a, v_b)
        for n, a, b in zip(O.GRAD_NAMES, acc_a, acc_b):
            assert O.same(a, b) if n in _BITWISE else _close(a, b), n
    else:
        plain = O.backward(args, out, dL, prune, quant, **extra)
        cam1 = O.backward(args, out, dL, prune, quant, camera_grads=True, **extra)
    assert len(plain) == 9 and len(cam1) == 12
    for n, a, b in zip(O.GRAD_NAMES + ["dL_dconic"], plain, cam1[:9]):
        assert O.same(a, b) if n in _BITWISE else _close(a, b), n
    dview, dproj, dcampos = cam1[9:]
    assert dview.shape == (4, 4) and dproj.shape == (4, 4) and dcampos.shape == (3,)
    assert torch.isfinite(dview).all() and torch.isfinite(dproj).all() and torch.isfinite(dcampos).all()
    # entries the preprocess never reads are exactly zero, the others are not
    assert float(dview[:, 3].abs().max()) == 0.0 and float(dproj[:, 2].abs().max()) == 0.0
    assert float(dview[:, :3].abs().min()) > 0 and float(dproj[:, [0, 1, 3]].abs().min()) > 0
    if name == "accumulate":
        # the camera outputs are this view's: equal to an overwrite-mode call of the same view
        ref = O.backward(args, out, dL, prune, quant, camera_grads=True, **extra)
        assert all(O.same(a, b) for a, b in zip(ref[9:], cam1[9:]))


def _on_a_side_stream(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        res = fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    return res


@pytest.mark.parametrize("name", ["c1", "quant", "pruned", "maps", "aa"])
def test_the_same_bytes_on_every_run_and_stream(name):
    """The camera outputs of the 8x4 cases above on a second run and on a non-default stream; with anti-aliasing, the colour,
    radii and maps of two 320x200 forwards, and every 8x4 backward output with the forward repeated on the other stream."""
    if name != "aa":
        scene, cam, prune, quant, bg, dL, extra, args, out = _small_case(name)
        run = partial(O.backward, args, out, dL, prune, quant, camera_grads=True, **extra)
        first, again, other = run(), run(), _on_a_side_stream(run)
        for a, b, c in zip(first[9:], again[9:], other[9:]):
            assert O.same(a, b) and O.same(a, c)
        return
    scene, _, _, _ = O.scene_config("aa", "mixed")
    bg = torch.tensor([0.1, 0.3, 0.2], device=DEV)
    big = O.yaw_cam(320, 200, 1.0)
    _, f1 = O.forward(scene, big, bg, maps=True, aa=True)
    _, f2 = O.forward(scene, big, bg, maps=True, aa=True)
    assert all(O.same(f1[i], f2[i]) for i in (1, 2, 6, 7))
    cam = O.yaw_cam(8, 4, 2.0)
    G = torch.randn(3, 4, 8, generator=torch.Generator().manual_seed(228)).to(DEV)
    args, out = O.forward(scene, cam, bg, maps=True, aa=True)
    kw = dict(dL_dalpha=torch.ones(1, 4, 8, device=DEV), camera_grads=True, aa=True)
    first = O.backward(args, out, G, **kw)
    again = O.backward(args, out, G, **kw)

    def on_side():
        a3, o3 = O.forward(scene, cam, bg, maps=True, aa=True)
        return o3, O.backward(a3, o3, G, **kw)
    o3, other = _on_a_side_stream(on_side)
    assert O.same(o3[1], out[1]) and O.same(o3[7], out[7])
    for a, b, c in zip(first, again, other):
        assert O.same(a, b) and O.same(a, c)


def test_quant_grads_unchanged_by_a_learnable_camera():
    from gaussian_renderer import render
    scene, cam, _, quant = _small("quant")                                   # one warp block: see above
    cam = cam.to(DEV)
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    G = synth.grad_image(cam.image_width, cam.image_height, 171).to(DEV)
    res = []
    for learn in (False, True):
        pc = GaussianModelView(scene, DEV, quant=quant)
        c = SimpleNamespace(**vars(cam))
        if learn:
            c.world_view_transform = cam.world_view_transform.clone().requires_grad_(True)
            c.full_proj_transform = cam.full_proj_transform.clone().requires_grad_(True)
            c.camera_center = cam.camera_center.clone().requires_grad_(True)
        pkg = render(c, pc, pipe, bg)
        (pkg["render"] * G).sum().backward()
        res.append((pc, pkg, c))
    (pa, ka, _), (pb, kb, cb) = res
    assert O.same(pa.quant.grads["opacity"], pb.quant.grads["opacity"])
    for k in ("sh", "scales", "rotations"):
        assert _close(pa.quant.grads[k], pb.quant.grads[k]), k
    assert _close(pa._xyz.grad, pb._xyz.grad) and O.same(ka["viewspace_points"].grad, kb["viewspace_points"].grad)
    for t in (cb.world_view_transform, cb.full_proj_transform, cb.camera_center):
        assert t.grad is not None and t.grad.shape == t.shape and float(t.grad.abs().max()) > 0


@pytest.mark.parametrize("option", ["camera", "camera_accumulate", "maps", "aa"])
def test_empty_and_fully_culled_scenes_give_zeros(option):
    """P = 0 and R = 0: zero maps and zero gradients, with the camera gradients (overwriting or accumulating), with the maps'
    backward, and anti-aliased with the maps, dL_dalpha and the camera gradients."""
    W, H = 100, 60
    cam = synth.make_camera(W, H).to(DEV)
    bg = torch.tensor([0.25, 0.5, 0.75], device=DEV)
    aa, maps, camera_grads = option == "aa", option in ("maps", "aa"), option != "maps"
    ones = torch.ones(1, H, W, device=DEV)
    for scene in O.empty_and_culled_scenes():
        args, out = O.forward(scene, cam, bg, maps=maps, aa=aa)
        assert out[0] == 0 and int((out[2] > 0).sum()) == 0
        if maps:
            assert out[6].shape == (1, H, W) and out[7].shape == (1, H, W)
            assert float(out[6].abs().max()) == 0.0 and float(out[7].abs().max()) == 0.0
        extra = dict(camera_grads=camera_grads, aa=aa)
        if option == "camera_accumulate":
            extra["accumulate_into"] = tuple(t.clone() for t in O.backward(args, out, torch.ones(3, H, W), None, None))
        if maps:
            extra.update(dL_dalpha=ones, **({} if aa else dict(dL_dinvdepth=ones)))
        g = O.backward(args, out, torch.ones(3, H, W), **extra)
        # poison-free check: every output, the camera's included, is written (not left as whatever the allocation held)
        assert all(float(t.abs().max()) == 0.0 for t in g if t.numel()), (option, scene.P)
        if camera_grads:
            assert [tuple(t.shape) for t in g[8:]] == [(4, 4), (4, 4), (3,)]


# ---- 2./3. chain check in float64 --------------------------------------------------------------------------------------------

def _kernel_and_chain(name):
    scene, cam, prune, quant = _config(name)
    cam = cam.to(DEV)
    H, W = cam.image_height, cam.image_width
    bg = torch.tensor([0.2, 0.1, 0.3], device=DEV)
    dL = synth.grad_image(W, H, 172).to(DEV)
    dbg = {}
    args, out = O.forward(scene, cam, bg, prune, quant, dbg=dbg)
    g = O.backward(args, out, dL, prune, quant, want_conic=True, camera_grads=True)
    vis = out[2] > 0
    sh = scene.sh if scene.sh.shape[1] > 0 else None
    per = _chain(cam.world_view_transform, cam.full_proj_transform, cam.camera_center, W, H, math.tan(cam.FoVx * 0.5),
                 math.tan(cam.FoVy * 0.5), scene.means3D, dbg["cov3D"], sh, scene.degrees, dbg["clamped"], vis, g[0], g[8], g[1])
    return scene, cam, dbg, out, g, per


@pytest.mark.parametrize("name", ["c1", "sh3", "mixed", "pruned"])
def test_camera_grads_are_the_chain_of_the_screen_space_gradients(name):
    _, _, _, out, g, per = _kernel_and_chain(name)
    assert int((out[2] > 0).sum()) > 1000
    _check(g[9:], per, 1e-5, name)


def test_camera_grads_against_the_fp64_oracle():
    import gs_oracle
    scene, cam = synth.config_scene("C1"), synth.make_camera(*synth.config_image("C1"))
    H, W = cam.image_height, cam.image_width
    bg = torch.tensor([0.2, 0.1, 0.3])
    dL = synth.grad_image(W, H, 173)
    kw = dict(viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, campos=cam.camera_center, W=W, H=H,
              tan_fovx=math.tan(cam.FoVx * 0.5), tan_fovy=math.tan(cam.FoVy * 0.5))
    o = gs_oracle.forward(scene.means3D, scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees, bg=bg, **kw)
    ob = gs_oracle.backward(o, dL, scene.means3D, scene.scales, scene.rotations, scene.sh, scene.degrees, bg=bg, f64=True, **kw)
    dbg = {}
    args, out = O.forward(scene, cam.to(DEV), bg.to(DEV), None, None, dbg=dbg)
    assert np.array_equal(out[2].cpu().numpy(), o["radii"])
    g = O.backward(args, out, dL, None, None, camera_grads=True)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    per = _chain(cam.world_view_transform, cam.full_proj_transform, cam.camera_center, W, H, kw["tan_fovx"], kw["tan_fovy"],
                 scene.means3D, t(o["cov3D"]), scene.sh, scene.degrees, t(o["clamped"]), out[2] > 0, t(ob["dL_dmeans2D"]),
                 t(ob["dL_dconic"]), t(ob["dL_dcolors"]))
    _check(g[8:], per, 2e-4, "C1 vs fp64 oracle")


# ---- 4. invariance identities ------------------------------------------------------------------------------------------------

# Each case keeps its option's scene table and grad-image seeds; the printed label tells the options apart.
_LABEL = {False: "camera invariance", True: "antialias camera"}


@pytest.mark.parametrize("aa, name, seed", [pytest.param(False, n, 174, id=n) for n in ("c1", "mixed", "quant")] +
                         [pytest.param(True, n, 225, id="aa-" + n) for n in ("c1", "quant")])
def test_translating_the_world_and_the_camera_together_changes_nothing(aa, name, seed):
    scene, cam, prune, quant = O.scene_config("aa" if aa else "camera", name)
    cam = cam.to(DEV)
    H, W = cam.image_height, cam.image_width
    args, out = O.forward(scene, cam, torch.tensor([0.3, 0.2, 0.1], device=DEV), prune, quant, aa=aa)
    g = O.backward(args, out, synth.grad_image(W, H, seed).to(DEV), prune, quant, aa=aa, camera_grads=True)
    gm = g[3].to(F64)
    gv, gp, gc = g[8].to(F64), g[9].to(F64), g[10].to(F64)
    V, Pf = cam.world_view_transform.to(DEV, F64), cam.full_proj_transform.to(DEV, F64)
    # means += tau, campos += tau, view[3,:] -= tau . view[:3,:], full_proj[3,:] -= tau . full_proj[:3,:] keep every t and ndc
    worst = 0.0
    for k in range(3):
        terms = [gm[:, k], gc[k:k + 1], -gv[3, :] * V[k, :], -gp[3, :] * Pf[k, :]]
        s = sum(float(x.sum()) for x in terms)
        scale = sum(float(x.abs().sum()) for x in terms)
        worst = max(worst, abs(s) / scale)
        assert abs(s) <= 1e-5 * scale, (name, k, s, scale)
    print(f"\n[{_LABEL[aa]}] translation {name}: max |sum| / sum|terms| = {worst:.3e}")


@pytest.mark.parametrize("aa, colour_seed, grad_seed", [pytest.param(False, 175, 176, id="camera"), pytest.param(True, 226, 227, id="aa")])
def test_rotating_the_world_and_the_camera_together_changes_nothing(aa, colour_seed, grad_seed):
    scene, cam, _, _ = O.scene_config("aa" if aa else "camera", "mixed")
    cam = cam.to(DEV)
    H, W = cam.image_height, cam.image_width
    col = torch.rand(scene.P, 3, generator=torch.Generator().manual_seed(colour_seed))
    args, out = O.forward(scene, cam, torch.tensor([0.3, 0.2, 0.1], device=DEV), None, None, colors=col, aa=aa)
    g = O.backward(args, out, synth.grad_image(W, H, grad_seed).to(DEV), None, None, aa=aa, camera_grads=True)
    gm, gq = g[3].to(F64), g[7].to(F64)
    gv, gp = g[8].to(F64), g[9].to(F64)
    m, q = scene.means3D.to(DEV, F64), scene.rotations.to(DEV, F64)
    V, Pf = cam.world_view_transform.to(DEV, F64), cam.full_proj_transform.to(DEV, F64)
    # column-vector world rotation R = exp([w]x): means -> R m, quaternions -> q_R (x) q (Sigma -> R Sigma R^T), the first three
    # rows of both transposed matrices -> R rows (t and ndc unchanged); the derivative at w = 0 along e_k:
    worst = 0.0
    for k in range(3):
        e = torch.zeros(3, dtype=F64, device=DEV)
        e[k] = 1.0
        S = R64.skew(e)
        dm = m @ S.T                                                         # e_k x m
        dq = R64.qmul(torch.cat([torch.zeros(1, dtype=F64, device=DEV), 0.5 * e]).expand_as(q), q)
        terms = [(gm * dm).sum(1), (gq * dq).sum(1), (gv[:3, :] * (S @ V[:3, :])).reshape(-1), (gp[:3, :] * (S @ Pf[:3, :])).reshape(-1)]
        s = sum(float(x.sum()) for x in terms)
        scale = sum(float(x.abs().sum()) for x in terms)
        worst = max(worst, abs(s) / scale)
        assert abs(s) <= 1e-5 * scale, (aa, k, s, scale)
    print(f"\n[{_LABEL[aa]}] rotation: max |sum| / sum|terms| = {worst:.3e}")


# ---- 5. maps ------------------------------------------------------------------------------------------------------------------

def test_camera_grads_of_the_maps_equal_those_of_the_colour_emulation():
    scene, cam, _, _ = _config("mixed")
    cam = cam.to(DEV)
    H, W = cam.image_height, cam.image_width
    g = torch.Generator().manual_seed(177)
    Gd, Ga = torch.randn(1, H, W, generator=g).to(DEV), torch.randn(1, H, W, generator=g).to(DEV)
    zero3 = torch.zeros(3, H, W, device=DEV)
    dbg = {}
    args, out = O.forward(scene, cam, torch.tensor([0.3, 0.1, 0.2], device=DEV), None, None, maps=True, dbg=dbg)
    vis = out[2] > 0
    z = dbg["depths"]
    got_d = O.backward(args, out, zero3, None, None, dL_dinvdepth=Gd, camera_grads=True)
    got_a = O.backward(args, out, zero3, None, None, dL_dalpha=Ga, camera_grads=True)
    # invdepth: colour (1/z, 0, 0) without background, plus the direct term d(1/z_i)/dview[4r+2] = -m_r / z_i^2
    col = torch.zeros(scene.P, 3)
    col[:, 0] = torch.where(vis.cpu(), 1.0 / torch.where(vis, z, torch.ones_like(z)).cpu(), torch.zeros(scene.P))
    ab, ob = O.forward(scene, cam, torch.zeros(3, device=DEV), None, None, colors=col)
    dLb = torch.zeros(3, H, W, device=DEV)
    dLb[0] = Gd[0]
    gb = O.backward(ab, ob, dLb, None, None, camera_grads=True)
    m = scene.means3D.to(DEV, F64)[vis]
    w = (-gb[1][:, 0].to(F64)[vis] / (z.to(F64)[vis] ** 2))
    direct = torch.zeros(4, 4, dtype=F64, device=DEV)
    direct[:3, 2] = (w[:, None] * m).sum(0)
    direct[3, 2] = w.sum()
    exp_d = (gb[8].to(F64) + direct, gb[9].to(F64), gb[10].to(F64))
    # alpha: colour 0 with background (-1, 0, 0)
    ac, oc = O.forward(scene, cam, torch.tensor([-1.0, 0.0, 0.0], device=DEV), None, None, colors=torch.zeros(scene.P, 3))
    dLc = torch.zeros(3, H, W, device=DEV)
    dLc[0] = Ga[0]
    gc = O.backward(ac, oc, dLc, None, None, camera_grads=True)
    exp_a = (gc[8].to(F64), gc[9].to(F64), gc[10].to(F64))
    scale_d = (w.abs()[:, None] * torch.cat([m.abs(), torch.ones_like(w)[:, None]], 1)).sum()
    for label, got, exp in (("invdepth", got_d[8:], exp_d), ("alpha", got_a[8:], exp_a)):
        for n, a, e in zip(("view", "proj", "campos"), got, exp):
            tol = 1e-4 * (float(e.abs().max()) + (float(scale_d) if label == "invdepth" and n == "view" else 0.0)) + 1e-30
            assert float((a.to(F64) - e).abs().max()) <= tol, (label, n, a.tolist(), e.tolist())
    assert float(got_d[8][:3, 2].abs().max()) > 0 and float(got_a[8][:3, :3].abs().max()) > 0
    assert float(got_d[10].abs().max()) == 0.0 and float(got_a[10].abs().max()) == 0.0   # the maps do not depend on the view direction


# ---- 6. end to end: pose refinement through render() -------------------------------------------------------------------------

def _pose_camera(xi, W, H, proj_T, fovx, fovy):
    """Camera from a 6-vector (axis-angle, translation) applied to the default camera (R = I, T = (0, 0, 4)), built in torch the
    way scene/cameras.py builds it: world_view_transform = [R | T]^T, full = view @ proj, campos = inverse(view)[3, :3]."""
    w, dt = xi[:3], xi[3:]
    K = torch.zeros(3, 3, dtype=xi.dtype, device=xi.device)
    K[0, 1], K[0, 2], K[1, 0], K[1, 2], K[2, 0], K[2, 1] = -w[2], w[1], w[2], -w[0], -w[1], w[0]
    Rwc = torch.linalg.matrix_exp(K)                                         # world -> camera rotation
    T = torch.tensor([0.0, 0.0, 4.0], dtype=xi.dtype, device=xi.device) + dt
    top = torch.cat([Rwc, T[:, None]], 1)
    Mwc = torch.cat([top, torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=xi.dtype, device=xi.device)], 0)
    view = Mwc.transpose(0, 1)
    full = view @ proj_T
    campos = torch.inverse(view)[3, :3]
    return SimpleNamespace(FoVx=fovx, FoVy=fovy, image_height=H, image_width=W, world_view_transform=view,
                           full_proj_transform=full, camera_center=campos)


def test_pose_refinement_through_render_recovers_the_camera():
    from gaussian_renderer import render
    W, H = 256, 192
    scene = synth.make_scene(8_000, 178, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.05), M=16)
    base = synth.make_camera(W, H)
    proj_T = synth._projection(base.znear, base.zfar, base.FoVx, base.FoVy).transpose(0, 1).to(DEV)
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    bg = torch.zeros(3, device=DEV)
    pc = GaussianModelView(scene, DEV, requires_grad=False)
    with torch.no_grad():
        cam0 = _pose_camera(torch.zeros(6, device=DEV), W, H, proj_T, base.FoVx, base.FoVy)
        assert torch.allclose(cam0.world_view_transform.cpu(), base.world_view_transform, atol=1e-6)
        gt = render(cam0, pc, pipe, bg)["render"].clone()
    # about 1 degree and 3 cm off
    xi0 = torch.tensor([0.01, -0.012, 0.008, 0.02, -0.015, 0.02], device=DEV)
    xi = xi0.clone().requires_grad_(True)
    opt = torch.optim.Adam([xi], lr=2e-3)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.985)
    losses = []
    for _ in range(200):
        opt.zero_grad(set_to_none=True)
        img = render(_pose_camera(xi, W, H, proj_T, base.FoVx, base.FoVy), pc, pipe, bg)["render"]
        loss = (img - gt).abs().mean()
        loss.backward()
        assert xi.grad is not None and torch.isfinite(xi.grad).all() and float(xi.grad.abs().max()) > 0
        opt.step()
        sched.step()
        losses.append(float(loss.detach()))
    err0, err1 = float(xi0.norm()), float(xi.detach().norm())
    first, last = sum(losses[:3]) / 3, sum(losses[-3:]) / 3
    print(f"\n[camera pose] pose error {err0:.4f} -> {err1:.5f}, L1 {first:.5f} -> {last:.6f}")
    assert err1 < err0 / 5 and last < first / 5, (err0, err1, first, last)
