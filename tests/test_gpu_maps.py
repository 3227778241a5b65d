"""GPU: the inverse-depth and alpha maps of `return_maps` (the requests' map fields) against the colour path, which the
parity tests pin to the reference bit for bit.  Every check is a linear identity:
  - the maps change nothing else (colour, radii, R, final_T, n_contrib, point_list are bit-identical with the maps on);
  - alpha == 1 - final_T, and invdepth == channel 0 of a render with colour (1/depth, 0, 0) and no background, bitwise;
  - the maps' gradients == the sum of three existing backwards (colour; the 1/depth colour render, chained through
    d(1/z)/dmeans3D in torch; a zero-colour render with background (-1, 0, 0)), within 1e-4 of each array's magnitude;
  - a few Adam steps on the means with an L1 loss on invdepth alone reduce that loss (sign and scale of the direct depth term).
The maps of P = 0 and R = 0 scenes and their backward are checked with the other options' in test_gpu_camera.py."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import backward_edges as BE
import ours as O
from diff_gaussian_rasterization import _C
from gs_b200 import synth
from gs_b200.model import GaussianModelView

pytestmark = pytest.mark.gpu

DEV = "cuda"
EMPTY = torch.Tensor([])


def _config(name):
    """-> (scene, cam, prune_mask or None, quant or None) on the CPU."""
    if name == "staircase" or name.startswith("odd_"):
        case = BE.build(name)                       # the per-element backward's boundary scenes (tests/backward_edges.py)
        return case.scene, case.cam, None, None
    return O.scene_config("maps", name)


def _invdepth_colours(radii, depths):
    """(1/depth, 0, 0) per Gaussian (IEEE division on the host), 0 for culled ones."""
    d = depths.cpu().numpy()
    inv = np.zeros_like(d)
    vis = radii.cpu().numpy() > 0
    inv[vis] = np.float32(1.0) / d[vis]
    col = torch.zeros(d.shape[0], 3)
    col[:, 0] = torch.from_numpy(inv)
    return col


@pytest.mark.parametrize("name", ["c1", "hd", "quant", "pruned"])
def test_maps_change_nothing_else_and_match_the_colour_path(name):
    scene, cam, prune, quant = _config(name)
    cam = cam.to(DEV)
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    _, plain = O.forward(scene, cam, bg, prune, quant)
    dbg = {}
    _, mapped = O.forward(scene, cam, bg, prune, quant, maps=True, dbg=dbg)
    assert len(plain) == 6 and len(mapped) == 8
    st0, st1 = O.state(plain, cam, scene.P), O.state(mapped, cam, scene.P)
    assert mapped[0] == plain[0] and plain[0] > 0
    assert torch.equal(mapped[1], plain[1]) and torch.equal(mapped[2], plain[2])
    for k in ("final_T", "n_contrib", "point_list", "ranges"):
        assert torch.equal(st0[k], st1[k]), k
    invdepth, alpha = mapped[6], mapped[7]
    H, W = cam.image_height, cam.image_width
    assert invdepth.shape == (1, H, W) and alpha.shape == (1, H, W) and invdepth.dtype == alpha.dtype == torch.float32
    # alpha == 1 - final_T, bitwise
    assert torch.equal(alpha[0], 1.0 - st1["final_T"])
    # invdepth == channel 0 of the colour render with colour (1/depth, 0, 0) and no background, bitwise
    col = _invdepth_colours(mapped[2], dbg["depths"])
    _, ref = O.forward(scene, cam, torch.zeros(3, device=DEV), prune, quant, colors=col)
    assert torch.equal(ref[2], mapped[2])
    assert torch.equal(invdepth[0], ref[1][0])
    assert float(invdepth.max()) > 0 and float(alpha.max()) > 0.5
    # the maps are a deterministic function of the inputs
    _, again = O.forward(scene, cam, bg, prune, quant, maps=True)
    assert torch.equal(again[6].view(torch.int32), invdepth.view(torch.int32))
    assert torch.equal(again[7].view(torch.int32), alpha.view(torch.int32))


def test_maps_of_the_variable_sh_entry_point():
    W, H = 320, 200
    scene = synth.make_scene(20_000, 85, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03), M=16)
    cam = synth.make_camera(W, H).to(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    flat, pbc, cum, cn = scene.packed_sh()
    a = O.forward_args(scene, cam, bg)

    def packed(maps):
        return _C.rasterize_gaussians_variableSH_bands(a[0], a[1], EMPTY, a[3], a[4], a[5], 1.0, EMPTY, a[8], a[9], a[10], a[11], H, W,
                                                       flat.to(DEV), pbc, cum, cn, a[15], a[16], False, False, return_maps=maps)
    plain, mapped = packed(False), packed(True)
    assert len(plain) == 6 and len(mapped) == 8
    assert mapped[0] == plain[0] and torch.equal(mapped[1], plain[1]) and torch.equal(mapped[2], plain[2])
    st0, st1 = O.state(plain, cam, scene.P), O.state(mapped, cam, scene.P)
    for k in ("final_T", "n_contrib", "point_list"):
        assert torch.equal(st0[k], st1[k]), k
    assert torch.equal(mapped[7][0], 1.0 - st1["final_T"])
    # the geometry is the dense path's: so are the maps
    _, dense = O.forward(scene, cam, bg, None, None, maps=True)
    assert torch.equal(mapped[6], dense[6]) and torch.equal(mapped[7], dense[7])


def _expected_grads(scene, cam, prune, quant, Gc, Gd, Ga):
    """Sum of three existing backwards (see the module docstring) -> (maps backward, expected, radii)."""
    bg = torch.tensor([0.3, 0.1, 0.2], device=DEV)
    dbg = {}
    args, out = O.forward(scene, cam, bg, prune, quant, maps=True, dbg=dbg)
    got = O.backward(args, out, Gc, prune, quant, dL_dinvdepth=Gd, dL_dalpha=Ga)
    # (a) the colour backward
    ga = O.backward(args, out, Gc, prune, quant)
    # (b) colour (1/depth, 0, 0), no background, dL/dpixel (Gd, 0, 0); dL/dcolour[:,0] chained through d(1/z)/dmeans3D
    zero3 = torch.zeros(3, device=DEV)
    col = _invdepth_colours(out[2], dbg["depths"])
    argsb, outb = O.forward(scene, cam, zero3, prune, quant, colors=col)
    dLb = torch.zeros(3, cam.image_height, cam.image_width, device=DEV)
    dLb[0] = Gd[0]
    gb = O.backward(argsb, outb, dLb, prune, quant)
    # (c) colour 0, background (-1, 0, 0), dL/dpixel (Ga, 0, 0)
    argsc, outc = O.forward(scene, cam, torch.tensor([-1.0, 0.0, 0.0], device=DEV), prune, quant, colors=torch.zeros(scene.P, 3))
    dLc = torch.zeros_like(dLb)
    dLc[0] = Ga[0]
    gc = O.backward(argsc, outc, dLc, prune, quant)
    # dL_dcolors and dL_dsh are the colour path's alone (the override renders have no SH: their dL_dsh is empty)
    exp = [a if i in (1, 5) else a + b + c for i, (a, b, c) in enumerate(zip(ga, gb, gc))]
    z = dbg["depths"]
    V = cam.world_view_transform.to(DEV).reshape(-1)
    vis = out[2] > 0                                                         # culled Gaussians have no depth (debug_out leaves 0)
    dz = torch.where(vis, -gb[1][:, 0] / torch.where(vis, z * z, torch.ones_like(z)), torch.zeros_like(z))
    exp[3] = exp[3] + dz[:, None] * torch.stack([V[2], V[6], V[10]])[None, :]
    return got, exp, out[2]


def _assert_close(got, exp, radii):
    off = (radii == 0).cpu()
    for n, g, e in zip(O.GRAD_NAMES, got, exp):
        g, e = g.cpu().reshape(g.shape[0], -1), e.cpu().reshape(e.shape[0], -1)
        if g.numel() == 0:
            continue
        scale = float(e.abs().max())
        assert scale > 0 or n == "dL_dsh", n
        assert float((g - e).abs().max()) <= 1e-4 * scale + 1e-30, (n, float((g - e).abs().max()), scale)
        if bool(off.any()):
            assert float(g[off].abs().max()) == 0.0, n


@pytest.mark.parametrize("name", ["c1", "quant", "pruned", "staircase"] + ["odd_%dx%d" % s for s in BE.ODD_SIZES])
def test_map_gradients_equal_the_sum_of_colour_backwards(name):
    scene, cam, prune, quant = _config(name)
    cam = cam.to(DEV)
    H, W = cam.image_height, cam.image_width
    g = torch.Generator().manual_seed(90)
    Gc, Gd, Ga = [torch.randn(c, H, W, generator=g).to(DEV) for c in (3, 1, 1)]
    got, exp, radii = _expected_grads(scene, cam, prune, quant, Gc, Gd, Ga)
    _assert_close(got, exp, radii)
    assert float(got[3].abs().max()) > 0 and float(got[2].abs().max()) > 0


def test_map_gradients_through_autograd_and_accumulation():
    from gaussian_renderer import render
    W, H = 256, 160
    scene = synth.make_scene(8000, 91, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04))
    cams = [O.yaw_cam(W, H, 0.0), O.yaw_cam(W, H, 6.0)]
    bg = torch.tensor([0.0, 0.3, 0.0], device=DEV)
    g = torch.Generator().manual_seed(92)
    Gd, Ga = torch.randn(1, H, W, generator=g).to(DEV), torch.randn(1, H, W, generator=g).to(DEV)
    # a loss on the maps alone: the colour's incoming gradient is None
    pc = GaussianModelView(scene, DEV)
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    pkg = render(cams[0], pc, pipe, bg, return_maps=True)
    assert pkg["invdepth"].shape == (1, H, W) and pkg["alpha"].shape == (1, H, W)
    ((pkg["invdepth"] * Gd).sum() + (pkg["alpha"] * Ga).sum()).backward()
    args, out = O.forward(scene, cams[0], bg, None, None, maps=True)
    assert torch.equal(out[1], pkg["render"].detach()) and torch.equal(out[6], pkg["invdepth"].detach())
    ref = O.backward(args, out, torch.zeros(3, H, W), None, None, dL_dinvdepth=Gd, dL_dalpha=Ga)

    def close(t, r):
        r = r.reshape(t.shape)
        return float((t - r).abs().max()) <= 1e-4 * (float(r.abs().max()) + 1e-12)
    assert close(pc._xyz.grad, ref[3]) and close(pc._opacity.grad, ref[2]) and close(pc._scaling.grad, ref[6])
    assert close(pc._rotation.grad, ref[7]) and close(pkg["viewspace_points"].grad, ref[0])
    assert float(pc._features.grad.abs().max()) == 0.0                      # no colour loss: no SH gradient
    assert float(pkg["viewspace_points"].grad[:, :2].norm(dim=1).max()) > 0  # the densification statistic sees the maps
    # accumulate_into over two views == the sum of two separate calls
    Gc = torch.randn(3, H, W, generator=g).to(DEV)
    runs = [O.forward(scene, c, bg, None, None, maps=True) for c in cams]
    sep = [O.backward(a, o, Gc, None, None, dL_dinvdepth=Gd, dL_dalpha=Ga) for a, o in runs]
    acc = tuple(t.clone() for t in sep[0])
    O.backward(*runs[1], Gc, None, None, dL_dinvdepth=Gd, dL_dalpha=Ga, accumulate_into=acc)
    for a, s0, s1 in zip(acc, *sep):
        s = s0 + s1
        assert float((a - s).abs().max()) <= 2e-4 * (float(s.abs().max()) + 1e-12)


def test_quantised_map_gradients_reach_quant_grads():
    from gaussian_renderer import render
    scene, cam, _, quant = _config("quant")
    cam = cam.to(DEV)
    H, W = cam.image_height, cam.image_width
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    g = torch.Generator().manual_seed(93)
    Gd, Ga = torch.randn(1, H, W, generator=g).to(DEV), torch.randn(1, H, W, generator=g).to(DEV)
    pc = GaussianModelView(scene, DEV, quant=quant)
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    pkg = render(cam, pc, pipe, bg, return_maps=True)
    ((pkg["invdepth"] * Gd).sum() + (pkg["alpha"] * Ga).sum()).backward()
    args, out = O.forward(scene, cam, bg, None, quant, maps=True)
    ref = O.backward(args, out, torch.zeros(3, H, W), None, quant, dL_dinvdepth=Gd, dL_dalpha=Ga)
    for k, i in (("opacity", 2), ("scales", 6), ("rotations", 7)):
        r = ref[i]
        assert float((pc.quant.grads[k].reshape(r.shape) - r).abs().max()) <= 1e-4 * float(r.abs().max()), k
        assert float(r.abs().max()) > 0, k


def test_invdepth_loss_alone_pulls_the_means_back():
    """Adam on the means only, L1 on invdepth only, against the maps of the scene the means were perturbed from."""
    from gaussian_renderer import render
    W, H = 256, 192
    target = synth.make_scene(6_000, 94, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04), M=16)
    cams = [O.yaw_cam(W, H, yaw) for yaw in (-10.0, 0.0, 10.0)]
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    bg = torch.zeros(3, device=DEV)
    with torch.no_grad():
        tpc = GaussianModelView(target, DEV, requires_grad=False)
        gts = [render(c, tpc, pipe, bg, return_maps=True)["invdepth"].clone() for c in cams]
    g = torch.Generator().manual_seed(95)
    means = target.means3D.clone()
    means[:, 2] += 0.05 * torch.randn(target.P, generator=g)
    start = synth.Scene(means, target.opacity, target.scales, target.rotations, target.sh, target.degrees)
    pc = GaussianModelView(start, DEV)
    for p in pc.params()[1:]:
        p.requires_grad_(False)
    opt = torch.optim.Adam([pc._xyz], lr=2e-3)
    losses = []
    for it in range(60):
        k = it % len(cams)
        opt.zero_grad(set_to_none=True)
        pkg = render(cams[k], pc, pipe, bg, return_maps=True)
        loss = (pkg["invdepth"] - gts[k]).abs().mean()
        loss.backward()
        assert pc._xyz.grad is not None and torch.isfinite(pc._xyz.grad).all()
        opt.step()
        losses.append(float(loss.detach()))
    first, last = sum(losses[:3]) / 3, sum(losses[-3:]) / 3
    assert last < 0.8 * first, (first, last)
