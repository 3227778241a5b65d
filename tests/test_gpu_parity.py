"""GPU: our CUDA path (through the reference-facing `_C` API -> C ABI) against
  (a) the golden vectors produced by the reference itself (bit-exact integers AND floats),
  (b) the CPU oracle on seeded inputs (integers bit-exact; colour <= 1e-4 off borderline pixels; gradients rel 2e-4 vs fp64),
  (c) size-independent properties at the full BASELINE sizes (sortedness, range consistency, determinism).
Tolerances: integers / indices / depth bits: exact.  Colour: 1e-4 abs (north_star).  Gradients: 2e-4 of the gradient scale
(the reference's own atomic-order noise is ~1e-5..1e-4 of scale, see noise_* in the goldens)."""
import math
import os

import numpy as np
import pytest
import torch

import backward_edges
import cases
import gs_oracle
import make_golden
import refsummary
from gs_b200 import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _ours():
    import ours
    return ours


def cam_kw(cam, W, H):
    return dict(viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, campos=cam.camera_center, W=W, H=H,
                tan_fovx=math.tan(cam.FoVx * 0.5), tan_fovy=math.tan(cam.FoVy * 0.5))


def assert_forward_equal(a, b, exact_float=True, check_lists=True, precomp=False):
    """a: reference-like dict, b: ours."""
    assert int(a["num_rendered"]) == int(b["num_rendered"])
    for k in ("radii", "tiles_touched"):
        assert np.array_equal(np.asarray(a[k]).reshape(-1), np.asarray(b[k]).reshape(-1)), k
    vis = np.asarray(a["radii"]) > 0
    assert np.array_equal(a["depths"][vis].view(np.uint32), b["depths"][vis].view(np.uint32)), "depth bits (sort key)"
    if check_lists:
        for k in ("keys", "point_list", "ranges", "n_contrib"):
            assert np.array_equal(np.asarray(a[k]).reshape(-1), np.asarray(b[k]).reshape(-1)), k
    if exact_float:
        for k in (("means2D", "conic_opacity", "final_T", "color") if precomp else
                  ("means2D", "cov3D", "conic_opacity", "rgb", "clamped", "final_T", "color")):
            x, y = np.asarray(a[k]), np.asarray(b[k])
            if k in ("final_T", "color"):
                assert np.array_equal(x, y), k
            else:
                assert np.array_equal(x[vis], y[vis]), k


@pytest.mark.parametrize("name", [n for n in cases.CASES if os.path.isfile(os.path.join(GOLD, n + ".npz"))])
def test_against_reference_goldens(name):
    ours = _ours()
    ref = refsummary.load_parts(name)
    c, scene, cam, bg, dL, extra = cases.build_inputs(name)
    args, out, fwd = ours.run_forward(scene, cam, bg, extra)
    assert_forward_equal(ref, fwd, precomp=c["precomp"])
    if c["backward"]:
        bwd = ours.run_backward(args, out, dL, c["lam"])
        vis = ref["radii"] > 0
        for n in make_golden.GRAD_NAMES:
            a = ref[n].astype(np.float64)
            if a.size == 0:
                continue
            b = bwd[n].astype(np.float64).reshape(a.shape)
            assert np.abs(a - b).max() / (np.abs(a).max() + 1e-30) < 5e-5, n
            assert not np.any(b[~vis]), n + ": culled Gaussians must carry zero gradient"
    if c["packed"]:
        from diff_gaussian_rasterization import _C
        flat, pbc, cs, cn = scene.packed_sh()
        E, d = torch.Tensor([]), "cuda"
        o2 = _C.rasterize_gaussians_variableSH_bands(
            bg.to(d), scene.means3D.to(d), E, scene.opacity.to(d), scene.scales.to(d), scene.rotations.to(d), 1.0, E,
            cam.world_view_transform.to(d), cam.full_proj_transform.to(d), math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5),
            c["H"], c["W"], flat.to(d), pbc, cs, cn, scene.degrees.to(d), cam.camera_center.to(d), False, False)
        assert o2[0] == int(ref["packed_num_rendered"])
        assert np.array_equal(o2[2].cpu().numpy(), ref["packed_radii"])
        assert np.array_equal(o2[1].cpu().numpy(), ref["packed_color"])
    from diff_gaussian_rasterization import _C
    mv = _C.mark_visible(scene.means3D.cuda(), cam.world_view_transform.cuda(), cam.full_proj_transform.cuda())
    assert np.array_equal(mv.cpu().numpy(), ref["mark_visible"])


def test_against_oracle_midsize():
    """60k Gaussians, mixed degrees, 640x368 (23 tile rows), fwd+bwd with the sparsity term."""
    ours = _ours()
    W, H = 640, 368
    scene = synth.make_scene(60_000, 21, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.012))
    cam = synth.make_camera(W, H)
    bg = torch.tensor([0.2, 0.1, 0.7])
    dL = synth.grad_image(W, H, 22)
    args, out, fwd = ours.run_forward(scene, cam, bg)
    o = gs_oracle.forward(scene.means3D, scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees, bg=bg, **cam_kw(cam, W, H))
    assert_forward_equal(o, fwd, exact_float=False, check_lists=False)
    for k in ("keys", "point_list", "ranges"):
        assert np.array_equal(np.asarray(o[k]).reshape(-1), fwd[k].reshape(-1)), k
    nb = ~o["borderline"]
    assert np.array_equal(o["n_contrib"][nb], fwd["n_contrib"][nb])
    assert (~nb).mean() < 1e-3
    assert np.abs(o["color"] - fwd["color"])[:, nb].max() <= 1e-4
    vis = o["radii"] > 0
    for k in ("means2D", "cov3D", "rgb"):
        assert np.array_equal(o[k][vis], fwd[k][vis]), k
    assert np.array_equal(o["conic_opacity"][vis, :3], fwd["conic_opacity"][vis, :3])
    # backward vs the fp64 oracle
    bwd = ours.run_backward(args, out, dL, 0.05)
    o64 = gs_oracle.backward(o, dL, scene.means3D, scene.scales, scene.rotations, scene.sh, scene.degrees, bg=bg,
                             lambda_sh_sparsity=0.05, f64=True, **cam_kw(cam, W, H))
    for n in make_golden.GRAD_NAMES + ["dL_dconic"]:
        a, b = o64[n].reshape(bwd[n].shape), bwd[n].astype(np.float64)
        assert np.abs(a - b).max() / (np.abs(a).max() + 1e-30) < 2e-4, n
    # PSNR criterion (north_star): |PSNR(ours, gt) - PSNR(reference arithmetic, gt)| <= 0.01 dB
    import test_oracle_golden as tog
    img64 = gs_oracle.render_forward(o, o, bg, W, H, f64=True)["color64"]
    gt = tog.pseudo_ground_truth(img64)
    assert abs(gs_oracle.psnr(fwd["color"], gt) - gs_oracle.psnr(o["color"], gt)) <= 0.01


def test_edge_cases():
    from diff_gaussian_rasterization import _C
    ours = _ours()
    d = "cuda"
    W, H = 100, 60
    cam = synth.make_camera(W, H)
    bg = torch.tensor([0.25, 0.5, 0.75])
    E = torch.Tensor([])

    def call(s):
        return _C.rasterize_gaussians(bg.to(d), s.means3D.to(d), E, s.opacity.to(d), s.scales.to(d), s.rotations.to(d), 1.0, E,
                                      cam.world_view_transform.to(d), cam.full_proj_transform.to(d), math.tan(cam.FoVx * .5),
                                      math.tan(cam.FoVy * .5), H, W, s.sh.to(d), s.degrees.to(d), cam.camera_center.to(d), False, False)
    empty, culled = ours.empty_and_culled_scenes()
    # P == 0 -> zero image WITHOUT background (rasterize_points.cu:184-185)
    R, color, radii, *_ = call(empty)
    assert R == 0 and float(color.abs().max()) == 0.0 and radii.numel() == 0
    # everything culled -> R == 0, pure background, backward gives zeros
    out = call(culled)
    assert out[0] == 0 and torch.allclose(out[1], bg.to(d)[:, None, None].expand(3, H, W))
    g = _C.rasterize_gaussians_backward(bg.to(d), culled.means3D.to(d), out[2], E, culled.scales.to(d), culled.rotations.to(d), 1.0, E,
                                        cam.world_view_transform.to(d), cam.full_proj_transform.to(d), math.tan(cam.FoVx * .5),
                                        math.tan(cam.FoVy * .5), torch.ones(3, H, W).to(d), culled.sh.to(d), culled.degrees.to(d),
                                        cam.camera_center.to(d), out[3], 0, out[4], out[5], 0.0, False)
    assert all(float(t.abs().max()) == 0.0 for t in g)
    # one huge opaque Gaussian covering every tile + one tiny one; compare with the oracle
    means = torch.tensor([[0.0, 0.0, 0.0], [0.3, 0.2, -0.5]])
    sc = torch.tensor([[5.0, 5.0, 5.0], [0.01, 0.01, 0.01]])
    q = torch.tensor([[1.0, 0, 0, 0], [0.5, 0.5, 0.5, 0.5]])
    op = torch.tensor([[8.0], [2.0]])
    sh = torch.tensor([[[1.0, 0.5, -0.2]], [[-3.0, 2.0, 0.1]]])
    deg = torch.zeros(2, 1, dtype=torch.int32)
    scene = synth.Scene(means, op, sc, q, sh, deg)
    args, out, fwd = ours.run_forward(scene, cam, bg)
    o = gs_oracle.forward(means, op, sc, q, sh, deg, bg=bg, **cam_kw(cam, W, H))
    assert fwd["num_rendered"] == o["num_rendered"] == int(o["tiles_touched"].sum())
    assert int(o["tiles_touched"][0]) == ((W + 15) // 16) * ((H + 15) // 16)
    for k in ("radii", "keys", "point_list", "ranges", "n_contrib"):
        assert np.array_equal(np.asarray(o[k]).reshape(-1), fwd[k].reshape(-1)), k
    assert np.abs(o["color"] - fwd["color"]).max() <= 1e-4


@pytest.mark.parametrize("kind", ["ties", "dense_4k", "dense_12k", "dense_40k", "dense_ties"])
def test_sort_paths_ties_and_dense_tiles(kind):
    """Every branch of the per-tile sort: bit-identical depths (tie order = ascending Gaussian id, as the reference's stable
    sort leaves them), clustered depths (distribution-sort fallback), and tiles with > 2048 / > 8192 instances
    (persistent shared-memory class and the global-memory fallback).  Integers must equal the oracle exactly."""
    ours = _ours()
    scene, cam, bg = backward_edges.dense_scene(kind)      # shared with test_gpu_backward_edges, which runs their backward
    W, H = cam.image_width, cam.image_height
    args, out, fwd = ours.run_forward(scene, cam, bg)
    o = gs_oracle.forward(scene.means3D, scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees, bg=bg, **cam_kw(cam, W, H))
    assert fwd["num_rendered"] == o["num_rendered"]
    counts = (o["ranges"][:, 1] - o["ranges"][:, 0]).astype(np.int64)
    if kind == "dense_4k":
        assert counts.max() > 2048
    if kind == "dense_12k":
        assert counts.max() > 8192
    if kind == "dense_ties":
        assert ((counts > 2048) & (counts <= 8192)).any(), counts
    if kind in ("ties", "dense_ties"):
        k = o["keys"]
        assert (k[1:] == k[:-1]).sum() > 1000, "the case must contain many exact depth ties"
    for k in ("radii", "keys", "point_list", "ranges"):
        assert np.array_equal(np.asarray(o[k]).reshape(-1), fwd[k].reshape(-1)), k
    nb = ~o["borderline"]          # pixels where a MUFU.EX2-vs-exp2f ulp can legitimately flip a threshold of the CPU oracle
    assert np.array_equal(o["n_contrib"][nb], fwd["n_contrib"][nb]), "n_contrib"
    assert (~nb).mean() < 5e-3
    assert np.abs(o["color"] - fwd["color"])[:, nb].max() <= 1e-4


def test_prune_mask_equals_compacted_scene():
    """Fused mask == reference semantics (rows physically deleted, gaussian_model.py:553-563), indices remapped."""
    ours = _ours()
    W, H = 320, 200
    scene = synth.make_scene(20_000, 31, sh_degree=2, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03))
    cam = synth.make_camera(W, H)
    bg = torch.zeros(3)
    dL = synth.grad_image(W, H, 32)
    mask = synth.prune_mask(scene.P, 4)
    keep = ~mask.bool()
    a1, o1, f1 = ours.run_forward(scene, cam, bg, prune_mask=mask)
    a2, o2, f2 = ours.run_forward(scene.compact(keep), cam, bg)
    idx = np.nonzero(keep.numpy())[0]
    assert f1["num_rendered"] == f2["num_rendered"]
    assert not f1["radii"][mask.numpy().astype(bool)].any()
    assert np.array_equal(f1["radii"][idx], f2["radii"])
    assert np.array_equal(f1["keys"], f2["keys"]) and np.array_equal(f1["point_list"], idx[f2["point_list"]])
    assert np.array_equal(f1["color"], f2["color"]) and np.array_equal(f1["n_contrib"], f2["n_contrib"])
    g1 = ours.run_backward(a1, o1, dL, prune_mask=mask)
    g2 = ours.run_backward(a2, o2, dL)
    for n in make_golden.GRAD_NAMES:
        assert not np.any(g1[n][mask.numpy().astype(bool)]), n
        x, y = g1[n][idx].astype(np.float64), g2[n].astype(np.float64)
        assert np.abs(x - y).max() / (np.abs(y).max() + 1e-30) < 1e-4, n


def test_prune_mask_against_oracle():
    """Fused mask vs the CPU oracle's reference-equivalent computation (`gs_oracle.forward(prune_mask=)`: the reference run on the
    physically compacted scene, outputs scattered back to the original indices — SURVEY §8(b), gaussian_model.py:553-563)."""
    ours = _ours()
    W, H = 320, 200
    scene = synth.make_scene(20_000, 33, sh_degree=2, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03))
    cam = synth.make_camera(W, H)
    bg = torch.tensor([0.2, 0.1, 0.05])
    mask = synth.prune_mask(scene.P, 5)
    o = gs_oracle.forward(scene.means3D, scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees, bg=bg.numpy(),
                          prune_mask=mask.numpy(), **cam_kw(cam, W, H))
    _, _, fwd = ours.run_forward(scene, cam, bg, prune_mask=mask)
    assert int(o["num_rendered"]) == fwd["num_rendered"]
    for k in ("radii", "tiles_touched", "keys", "point_list", "ranges"):
        assert np.array_equal(np.asarray(o[k]).reshape(-1), fwd[k].reshape(-1)), k
    assert not fwd["radii"][mask.numpy().astype(bool)].any()
    vis = o["radii"] > 0
    assert np.array_equal(o["depths"][vis].view(np.uint32), fwd["depths"][vis].view(np.uint32))
    for k in ("means2D", "cov3D", "rgb"):
        assert np.array_equal(np.asarray(o[k])[vis], fwd[k][vis]), k
    assert np.array_equal(o["conic_opacity"][vis, :3], fwd["conic_opacity"][vis, :3])     # opacity: oracle exp2f vs MUFU.EX2, <= 2 ulp
    nb = ~o["borderline"]
    assert np.array_equal(o["n_contrib"][nb], fwd["n_contrib"][nb]) and (~nb).mean() < 5e-3
    assert np.abs(o["color"] - fwd["color"])[:, nb].max() <= 1e-4


def test_fused_dequant_equals_dequantised_fp32():
    """Codebook ids + centres in the kernel == centers[ids] -> exp / normalize in PyTorch -> fp32 path (SURVEY §8(b))."""
    ours = _ours()
    W, H = 480, 272
    scene = synth.make_scene(40_000, 41, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.02))
    q = synth.quantise_scene(scene)
    cam = synth.make_camera(W, H)
    bg = torch.tensor([0.1, 0.1, 0.1])
    dL = synth.grad_image(W, H, 42)
    deq = q.to("cuda").dequantise()            # the reference flow de-quantises on the GPU (load_ply)
    deq_cpu = synth.Scene(*[getattr(deq, f).cpu() for f in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
    a1, o1, f1 = ours.run_forward(deq_cpu, cam, bg, quant=q)
    a2, o2, f2 = ours.run_forward(deq_cpu, cam, bg)
    # scales: exp in-kernel vs torch.exp; rotations: in-kernel normalise vs F.normalize -> may differ by an ulp; report and bound
    assert f1["num_rendered"] == f2["num_rendered"], "instance count differs between fused and torch de-quantisation"
    assert np.array_equal(f1["radii"], f2["radii"])
    assert np.array_equal(f1["keys"], f2["keys"]) and np.array_equal(f1["point_list"], f2["point_list"])
    assert np.abs(f1["color"] - f2["color"]).max() <= 1e-4
    g1 = ours.run_backward(a1, o1, dL, quant=q)
    g2 = ours.run_backward(a2, o2, dL)
    for n in make_golden.GRAD_NAMES:
        x, y = g1[n].astype(np.float64), g2[n].astype(np.float64)
        assert np.abs(x - y).max() / (np.abs(y).max() + 1e-30) < 2e-4, n


def test_autograd_and_render_api():
    """gaussian_renderer.render + autograd == direct _C calls; accumulate_into adds; repeated forward is deterministic."""
    import ours as O
    from types import SimpleNamespace
    from gaussian_renderer import render
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench", os.path.join(root, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    W, H = 256, 160
    scene = synth.make_scene(8000, 51, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04))
    cam = synth.make_camera(W, H).to("cuda")
    bg = torch.tensor([0.0, 0.3, 0.0], device="cuda")
    dL = synth.grad_image(W, H, 52).cuda()
    pc = bench.ModelView(scene, "cuda")
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    pkg = render(cam, pc, pipe, bg, lambda_sh_sparsity=0.0)
    (pkg["render"] * dL).sum().backward()
    args, out, fwd = O.run_forward(scene, cam, bg)
    g = O.run_backward(args, out, dL)
    assert np.array_equal(pkg["render"].detach().cpu().numpy(), fwd["color"])
    assert np.array_equal(pkg["radii"].cpu().numpy(), fwd["radii"]) and bool((pkg["visibility_filter"] == (pkg["radii"] > 0)).all())

    def close(t, ref):
        ref = ref.reshape(t.shape)
        return np.abs(t.detach().cpu().numpy() - ref).max() <= 1e-4 * (np.abs(ref).max() + 1e-12)
    assert close(pc._xyz.grad, g["dL_dmeans3D"]) and close(pc._features.grad, g["dL_dsh"]) and close(pc._opacity.grad, g["dL_dopacity"])
    assert close(pc._scaling.grad, g["dL_dscales"]) and close(pc._rotation.grad, g["dL_drotations"])
    assert close(pkg["viewspace_points"].grad, g["dL_dmeans2D"])
    # python-side SH / covariance paths of the reference (pipe.convert_SHs_python / compute_cov3D_python) give the same picture
    pipe2 = SimpleNamespace(debug=False, convert_SHs_python=True, compute_cov3D_python=False)
    with torch.no_grad():
        img2 = render(cam, pc, pipe2, bg)["render"]
    assert float((img2 - pkg["render"]).abs().max()) < 1e-4
    # accumulate_into: second call adds
    from diff_gaussian_rasterization import _C
    (bgt, m3, col, opa, sc, rot, mod, cov, view, proj, tx, ty, Hh, Ww, sh, deg, campos, _, _) = args
    R, color, radii, gb, bb, ib = out
    one = _C.rasterize_gaussians_backward(bgt, m3, radii, col, sc, rot, mod, cov, view, proj, tx, ty, dL, sh, deg, campos, gb, R, bb, ib, 0.0, False)
    acc = tuple(t.clone() for t in one)
    _C.rasterize_gaussians_backward(bgt, m3, radii, col, sc, rot, mod, cov, view, proj, tx, ty, dL, sh, deg, campos, gb, R, bb, ib, 0.0, False,
                                    accumulate_into=acc)
    for a, b in zip(acc, one):
        assert float((a - 2 * b).abs().max()) <= 2e-4 * float(b.abs().max() + 1e-12)
    # determinism of the forward
    _, _, fwd2 = O.run_forward(scene, cam, bg)
    assert np.array_equal(fwd2["color"], fwd["color"]) and np.array_equal(fwd2["point_list"], fwd["point_list"])


def test_render_variable_sh_bands_against_golden():
    """gaussian_renderer.render(..., variable_sh_bands=True) (GR:84-86, 99-125) with the model's list-of-tensors get_features
    (gaussian_model.py:153-163) == the reference's rasterize_gaussians_variableSH_bands output (golden g3, packed_*)."""
    from types import SimpleNamespace
    from gaussian_renderer import render
    from gs_b200.model import GaussianModelView
    ref = refsummary.load_parts("g3")
    c, scene, cam, bg, dL, extra = cases.build_inputs("g3")
    pc = GaussianModelView(scene, "cuda", requires_grad=False, variable_sh_bands=True)
    feats = pc.get_features
    assert isinstance(feats, list) and [tuple(f.shape[1:]) for f in feats] == [(1, 3), (4, 3), (9, 3), (16, 3)]
    assert [f.shape[0] for f in feats] == pc.per_band_count
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    with torch.no_grad():
        pkg = render(cam.to("cuda"), pc, pipe, bg.cuda(), variable_sh_bands=True)
    assert np.array_equal(pkg["radii"].cpu().numpy(), ref["packed_radii"])
    assert np.array_equal(pkg["render"].cpu().numpy(), ref["packed_color"])
    # and the dense path on the same model gives the same picture
    pc2 = GaussianModelView(scene, "cuda", requires_grad=False)
    with torch.no_grad():
        img2 = render(cam.to("cuda"), pc2, pipe, bg.cuda())["render"]
    assert np.array_equal(img2.cpu().numpy(), ref["packed_color"])


def test_quantised_model_with_override_color():
    """A quantised model rendered with override_color (reference callers: depth / debug renders) uses the given colours, forward
    and backward, exactly like the fp32 path with colors_precomp; the python-side SH / covariance options are refused."""
    from types import SimpleNamespace
    from gaussian_renderer import render
    from gs_b200.model import GaussianModelView
    ours = _ours()
    W, H = 320, 200
    scene = synth.make_scene(20_000, 61, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03))
    q = synth.quantise_scene(scene)
    deq = q.to("cuda").dequantise()
    deq_cpu = synth.Scene(*[getattr(deq, f).cpu() for f in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
    cam = synth.make_camera(W, H).to("cuda")
    bg = torch.tensor([0.1, 0.2, 0.3], device="cuda")
    dL = synth.grad_image(W, H, 62).cuda()
    col = torch.rand(scene.P, 3, generator=torch.Generator().manual_seed(63)).cuda().requires_grad_(True)
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    pc = GaussianModelView(deq_cpu, "cuda", quant=q)
    pkg = render(cam, pc, pipe, bg, override_color=col)
    (pkg["render"] * dL).sum().backward()
    args, out, fwd = ours.run_forward(deq_cpu, cam, bg, extra={"colors_precomp": col.detach().cpu()})
    g = ours.run_backward(args, out, dL)
    assert np.abs(pkg["render"].detach().cpu().numpy() - fwd["color"]).max() <= 1e-6
    assert np.array_equal(pkg["radii"].cpu().numpy(), fwd["radii"])
    ref = g["dL_dcolors"]
    assert np.abs(col.grad.cpu().numpy() - ref).max() <= 1e-4 * (np.abs(ref).max() + 1e-12)
    assert float(pc.quant.grads["sh"].abs().max()) == 0.0, "SH coefficients were not used: their gradient is zero"
    # quant.grads has the semantics of .grad: a second backward accumulates, `= None` resets
    first = {k: v.clone() for k, v in pc.quant.grads.items()}
    (render(cam, pc, pipe, bg, override_color=col)["render"] * dL).sum().backward()
    for k, v in first.items():
        assert float((pc.quant.grads[k] - 2 * v).abs().max()) <= 2e-4 * (float(v.abs().max()) + 1e-12), k
    pc.quant.grads = None
    (render(cam, pc, pipe, bg, override_color=col)["render"] * dL).sum().backward()
    for k, v in first.items():
        assert float((pc.quant.grads[k] - v).abs().max()) <= 2e-4 * (float(v.abs().max()) + 1e-12), k
    with pytest.raises(RuntimeError):
        render(cam, pc, SimpleNamespace(debug=False, convert_SHs_python=True, compute_cov3D_python=False), bg)


def test_speculative_binning_across_workload_jumps():
    """The binning blob is carved for the capacity recent frames needed (+6 %) before this frame's instance count is known
    (gsb_api.cu gsb_forward).  A frame whose count outgrows that speculation must be re-launched transparently, and a much
    smaller one must not inherit a stale layout: small -> large -> small -> large, every frame compared with the oracle."""
    ours = _ours()
    W, H = 320, 200
    cam = synth.make_camera(W, H)
    bg = torch.tensor([0.1, 0.0, 0.2])
    small = synth.make_scene(3_000, 81, sh_degree=1, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.02))
    large = synth.make_scene(40_000, 82, sh_degree=1, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04))
    ref = {}
    for name, sc in (("small", small), ("large", large)):
        ref[name] = gs_oracle.forward(sc.means3D, sc.opacity, sc.scales, sc.rotations, sc.sh, sc.degrees, bg=bg.numpy(), **cam_kw(cam, W, H))
    assert ref["large"]["num_rendered"] > 4 * ref["small"]["num_rendered"]
    for name in ("small", "large", "small", "large", "large", "small"):
        sc = small if name == "small" else large
        _, _, fwd = ours.run_forward(sc, cam, bg)
        o = ref[name]
        assert fwd["num_rendered"] == o["num_rendered"]
        for k in ("radii", "keys", "point_list", "ranges"):
            assert np.array_equal(np.asarray(o[k]).reshape(-1), fwd[k].reshape(-1)), (name, k)
        nb = ~o["borderline"]
        assert np.array_equal(o["n_contrib"][nb], fwd["n_contrib"][nb]) and np.abs(o["color"] - fwd["color"])[:, nb].max() <= 1e-4


def test_accumulate_mode_keeps_the_per_view_screen_gradient():
    """View-batch accumulation (GsbGrads.accumulate): the eight buffers receive the SUM over views, while `view_means2D` holds THIS
    view's dL_dmeans2D alone — what the per-view densification statistic needs (gaussian_model.py:693-695)."""
    from diff_gaussian_rasterization import _C
    from gs_b200 import multi
    O = _ours()
    W, H = 320, 200
    scene = synth.make_scene(15_000, 85, sh_degree=3, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03))
    bg = torch.zeros(3)
    cams = synth.orbit_cameras(3, W, H)
    dLs = [synth.grad_image(W, H, 90 + i) for i in range(3)]
    acc = multi.GradAccumulator(scene.P, 16, "cuda")
    singles = []
    for cam, dL in zip(cams, dLs):
        args, out, _ = O.run_forward(scene, cam, bg)
        (bgt, m3, col, opa, sc, rot, mod, cov, view, proj, tx, ty, Hh, Ww, sh, deg, campos, _, _) = args
        R, color, radii, gb, bb, ib = out
        one = _C.rasterize_gaussians_backward(bgt, m3, radii, col, sc, rot, mod, cov, view, proj, tx, ty, dL.cuda(), sh, deg, campos, gb, R, bb, ib, 0.0, False)
        _C.rasterize_gaussians_backward(bgt, m3, radii, col, sc, rot, mod, cov, view, proj, tx, ty, dL.cuda(), sh, deg, campos, gb, R, bb, ib, 0.0, False,
                                        accumulate_into=acc.buffers(), view_means2D=acc.view_means2D)
        torch.cuda.synchronize()
        scale = float(one[0].abs().max()) + 1e-12
        assert float((acc.view_means2D - one[0]).abs().max()) <= 2e-4 * scale, "per-view screen-space gradient"
        acc.observe_view(radii)
        singles.append([t.clone() for t in one])
    for i, buf in enumerate(acc.buffers()):
        tot = sum(s[i] for s in singles)
        assert float((buf - tot.reshape(buf.shape)).abs().max()) <= 3e-4 * (float(tot.abs().max()) + 1e-12), multi.GRAD_NAMES[i]
    # the statistic is the sum of per-view norms, not the norm of the sum
    want = sum(torch.where((s[0][:, :2].norm(dim=-1) > 0), s[0][:, :2].norm(dim=-1), torch.zeros_like(s[0][:, 0])) for s in singles)
    assert float((acc.xyz_gradient_accum.view(-1) - want).abs().max()) <= 1e-3 * (float(want.max()) + 1e-12)

    # degree-banded model: the accumulated dL_dsh is zero outside every Gaussian's active coefficients — what GradAccumulator's
    # banded all-reduce payload (band_counts) relies on — and non-zero inside
    banded = synth.make_scene(15_000, 86, sh_degree=3, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03))
    counts = [int((banded.degrees.view(-1) == d).sum()) for d in range(4)]
    accb = multi.GradAccumulator(banded.P, 16, "cuda", band_counts=counts)
    for cam, dL in zip(cams, dLs):
        args, out, _ = O.run_forward(banded, cam, bg)
        (bgt, m3, col, opa, sc, rot, mod, cov, view, proj, tx, ty, Hh, Ww, sh, deg, campos, _, _) = args
        R, color, radii, gb, bb, ib = out
        _C.rasterize_gaussians_backward(bgt, m3, radii, col, sc, rot, mod, cov, view, proj, tx, ty, dL.cuda(), sh, deg, campos, gb, R, bb, ib, 0.0, False,
                                        accumulate_into=accb.buffers(), view_means2D=accb.view_means2D)
    assert accb.inactive_sh_is_zero() and float(accb.sh.abs().max()) > 0
    assert accb.payload_floats < banded.P * (62 + 2)


def test_full_size_properties():
    """BASELINE config C2 (500k, 1080p): size-independent properties of the integer pipeline + determinism."""
    ours = _ours()
    scene = synth.config_scene("C2")
    W, H = synth.config_image("C2")
    cam = synth.make_camera(W, H)
    bg = torch.zeros(3)
    args, out, fwd = ours.run_forward(scene, cam, bg)
    R = fwd["num_rendered"]
    assert R == int(fwd["tiles_touched"].astype(np.uint64).sum()) and R > scene.P
    keys = fwd["keys"]
    assert np.all(keys[1:] >= keys[:-1]), "keys sorted by (tile, depth bits)"
    same = keys[1:] == keys[:-1]
    assert np.all(fwd["point_list"][1:][same] > fwd["point_list"][:-1][same]), "stable sort: ties keep ascending Gaussian index"
    tiles = (keys >> np.uint64(32)).astype(np.int64)
    rng = fwd["ranges"].astype(np.int64)
    counts = np.bincount(tiles, minlength=rng.shape[0])
    assert np.array_equal(rng[:, 1] - rng[:, 0], counts), "ranges partition the sorted list by tile"
    assert np.array_equal(np.sort(fwd["point_list"]), np.repeat(np.arange(scene.P), fwd["tiles_touched"]).astype(np.uint32)), "checksum of instances"
    vis = fwd["radii"] > 0
    assert np.array_equal((keys & np.uint64(0xffffffff)).astype(np.uint32), fwd["depths"].view(np.uint32)[fwd["point_list"]]), "depth bits ride in the key"
    assert np.all(fwd["n_contrib"].reshape(-1) <= np.repeat(counts.reshape((H + 15) // 16, (W + 15) // 16), 16, 0).repeat(16, 1)[:H, :W].reshape(-1))
    assert np.all(fwd["final_T"] >= 0) and np.all(fwd["final_T"] <= 1)
    assert 0.7 < vis.mean() < 0.95
    _, _, fwd2 = ours.run_forward(scene, cam, bg)
    assert np.array_equal(fwd2["color"], fwd["color"]) and np.array_equal(fwd2["keys"], keys)


def test_quantised_ply_to_fused_render(tmp_path):
    """SURVEY §8(f) row 1: a reduced-3dgs quantised PLY loaded straight into the id planes renders, through the fused
    de-quantising path, exactly what the original quantised model renders (same ids, same centres -> same bits)."""
    from gs_b200 import ply
    ours = _ours()
    W, H = 320, 200
    scene = synth.make_scene(20_000, 43, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03))
    order = torch.argsort(scene.degrees.view(-1), stable=True)
    scene = synth.Scene(*[getattr(scene, f)[order].contiguous() for f in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
    q = synth.quantise_scene(scene)
    path = str(tmp_path / "point_cloud_quantised.ply")
    ply.save_reduced_ply(path, q)
    loaded = ply.load_reduced_ply(path, quantised=True, device="cuda")
    assert loaded.ids_rest.is_cuda and loaded.ids_rest.dtype == torch.uint8
    cam = synth.make_camera(W, H)
    bg = torch.tensor([0.0, 0.2, 0.4])
    deq = q.to("cuda").dequantise()
    deq_cpu = synth.Scene(*[getattr(deq, f).cpu() for f in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
    _, _, f1 = ours.run_forward(deq_cpu, cam, bg, quant=q)
    _, _, f2 = ours.run_forward(deq_cpu, cam, bg, quant=loaded)
    assert f1["num_rendered"] == f2["num_rendered"] and np.array_equal(f1["point_list"], f2["point_list"])
    assert np.array_equal(f1["color"], f2["color"]) and np.array_equal(f1["n_contrib"], f2["n_contrib"])


def test_render_from_quantised_ply_through_model_view(tmp_path):
    """render() on a GaussianModelView built from a quantised PLY == render() on the fp32 model the file was made from
    (same ids and centres; the fused path de-quantises in the kernel), and == the reference-equivalent fp32 expansion within 1e-4."""
    from types import SimpleNamespace
    from gs_b200 import ply
    from gs_b200.model import GaussianModelView
    from gaussian_renderer import render
    W, H = 320, 200
    scene = synth.make_scene(20_000, 44, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.03))
    order = torch.argsort(scene.degrees.view(-1), stable=True)
    scene = synth.Scene(*[getattr(scene, f)[order].contiguous() for f in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
    q = synth.quantise_scene(scene)
    path = str(tmp_path / "point_cloud_quantised.ply")
    ply.save_reduced_ply(path, q)
    view = GaussianModelView.from_ply(path, quantised=True, device="cuda")
    cam = synth.make_camera(W, H).to("cuda")
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    bg = torch.tensor([0.2, 0.1, 0.0], device="cuda")
    with torch.no_grad():
        img_q = render(cam, view, pipe, bg)["render"]
        img_f = render(cam, GaussianModelView(q.to("cuda").dequantise(), "cuda", requires_grad=False), pipe, bg)["render"]
    assert float((img_q - img_f).abs().max()) <= 1e-4
    assert float(img_q.abs().max()) > 0.05


def test_global_atomics_binning_path_beyond_shared_memory():
    """Images with more than 40 960 tiles do not fit the per-CTA shared-memory tile histogram (BinPlan.priv == 0): counting and
    scattering fall back to global atomics.  Same integer results and image as the oracle."""
    ours = _ours()
    W, H = 3840, 2880                                    # 240 x 180 = 43 200 tiles -> 172.8 KB of histogram > 160 KB
    scene = synth.make_scene(30_000, 91, sh_degree=1, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.01))
    cam = synth.make_camera(W, H)
    bg = torch.tensor([0.0, 0.0, 0.0])
    args, out, fwd = ours.run_forward(scene, cam, bg)
    o = gs_oracle.forward(scene.means3D, scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees, bg=bg,
                          viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, campos=cam.camera_center,
                          W=W, H=H, tan_fovx=math.tan(cam.FoVx * 0.5), tan_fovy=math.tan(cam.FoVy * 0.5))
    assert fwd["num_rendered"] == o["num_rendered"] > 0
    for k in ("radii", "tiles_touched", "keys", "point_list", "ranges"):
        assert np.array_equal(np.asarray(fwd[k]), np.asarray(o[k])), k
    nb = ~o["borderline"]
    assert np.array_equal(fwd["n_contrib"][nb], o["n_contrib"][nb])
    assert np.abs(fwd["color"] - o["color"])[:, nb].max() <= 1e-4
    dL = synth.grad_image(W, H, 92)
    g = ours.run_backward(args, out, dL)
    assert all(np.isfinite(v).all() for v in g.values())


def test_second_device_in_the_same_process():
    """The library keeps no process-wide per-device state: after cuda:0 has run every kernel, cuda:1 in the SAME process must get its
    own dynamic-shared-memory opt-ins (preprocess 52 KB with codebooks, render backward 55 KB, per-tile sort) and its own
    instance-count landing buffer, and produce identical results.  Needs 2 visible GPUs (skipped otherwise)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs in one process")
    ours = _ours()
    W, H = 640, 368
    scene0 = synth.make_scene(60_000, 71, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.012))
    q = synth.quantise_scene(scene0)
    deq = q.to("cuda:0").dequantise()
    scene = synth.Scene(*[getattr(deq, f).cpu() for f in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
    cam = synth.make_camera(W, H)
    bg = torch.tensor([0.3, 0.2, 0.1])
    dL = synth.grad_image(W, H, 72)
    res = []
    for dev in ("cuda:0", "cuda:1", "cuda:0"):
        with torch.cuda.device(dev):
            args, out, fwd = ours.run_forward(scene, cam, bg, quant=q, dev=dev)
            g = ours.run_backward(args, out, dL, quant=q)
            torch.cuda.synchronize(dev)
        res.append((fwd, g))
    for fwd, g in res[1:]:
        for k in ("radii", "keys", "point_list", "ranges", "n_contrib", "color"):
            assert np.array_equal(fwd[k], res[0][0][k]), k
        for n in make_golden.GRAD_NAMES:
            a, b = res[0][1][n].astype(np.float64), g[n].astype(np.float64)
            assert np.abs(a - b).max() <= 2e-4 * (np.abs(a).max() + 1e-30), n
