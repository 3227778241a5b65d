"""CPU: the rasterizer's options together, through GaussianRasterizer and render(), against the stand-in `_C` of stub_c (no GPU).
Every combination of input form, learnable camera tensors, return_maps, features, means2D_abs and the deterministic mode: the
keywords of each `_C` call, the outputs, and that each input's .grad is the stub's output for its own slot (None where it needs
none); the combinations without a form are refused with their message before anything is called."""
import itertools
from types import SimpleNamespace

import pytest
import torch

import stub_c
from stub_c import marked

P, F, H, W = 4, 5, 8, 8
FORMS = ("sh", "colors", "cov3D", "quant", "raw_sh", "raw_colors")
CAMERA_KEYS = (("viewmatrix", "world_view_transform", "dL_dviewmatrix"), ("projmatrix", "full_proj_transform", "dL_dprojmatrix"),
               ("campos", "camera_center", "dL_dcampos"))
CAMERAS = ((), (0,), (1,), (2,), (0, 2), (0, 1, 2))         # which camera tensors require grad
MATRIX = list(itertools.product(FORMS, CAMERAS, (False, True), (None, "const", "grad"), (False, True), (False, True)))


@pytest.fixture
def torch_deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _scene(form):
    """-> (model, colors, quant, rasterizer keywords, {input: the stub output its gradient must be})."""
    m = stub_c.Model(P, C=3)
    colors = torch.rand(P, 3, requires_grad=True)
    quant = SimpleNamespace() if form == "quant" else None
    kw, grads = {}, {}
    if form in ("sh", "cov3D"):
        kw.update(shs=m.get_features)
        grads[m.get_features] = "dL_dsh"
    if form in ("colors", "raw_colors"):
        kw.update(colors_precomp=colors)
        grads[colors] = "dL_dcolors"
    if form in ("sh", "colors"):
        kw.update(scales=m.get_scaling, rotations=m.get_rotation)
        grads.update({m.get_scaling: "dL_dscales", m.get_rotation: "dL_drotations"})
    if form == "cov3D":
        kw.update(cov3D_precomp=m.cov3D)
        grads[m.cov3D] = "dL_dcov3D"
    if form == "quant":
        kw.update(quant=quant)
    if form == "raw_sh":
        kw.update(raw_params=(m._features_dc, m._features_rest, m._scaling, m._rotation))
        grads.update({m._features_dc: "dL_dfeatures_dc", m._features_rest: "dL_dfeatures_rest"})
    if form == "raw_colors":
        kw.update(raw_params=(None, None, m._scaling, m._rotation))
    if form.startswith("raw"):
        grads.update({m._scaling: "dL_dscaling", m._rotation: "dL_drotation"})
    grads.update({m.get_xyz: "dL_dmeans3D", m._opacity: "dL_dopacity"})
    return m, colors, quant, kw, grads


def _refusal(features, absgrad, det, via_render):
    if absgrad and features is not None:
        return ("gaussian_renderer.render: absgrad has no feature form" if via_render else
                "means2D_abs: the absolute screen-space gradient has no feature form")
    if features == "grad" and det:
        return "features: the feature gradient has no deterministic form"
    return None


@pytest.mark.parametrize("via_render", [False, True])
@pytest.mark.parametrize("form, cam_grad, maps, features, absgrad, det", MATRIX)
def test_every_option_reaches_its_slot(monkeypatch, torch_deterministic, via_render, form, cam_grad, maps, features, absgrad, det):
    stub = stub_c.StubC().install(monkeypatch)
    m, colors, quant, kw, grads = _scene(form)
    cam = stub_c.camera(H, W, grad=[CAMERA_KEYS[i][1] for i in cam_grad])
    feats = None if features is None else torch.rand(P, F, requires_grad=features == "grad")
    means2D_abs = torch.zeros(P, 3, requires_grad=True) if absgrad else None

    def run():
        if via_render:
            torch.use_deterministic_algorithms(det)
            if form == "quant":
                m.quant = quant
            pipe = stub_c.pipe(compute_cov3D_python=form == "cov3D", fused_activations=form.startswith("raw"))
            pkg = __import__("gaussian_renderer").render(cam, m, pipe, torch.zeros(3), override_color=kw.get("colors_precomp"),
                                                         return_maps=maps, features=feats, absgrad=absgrad)
            out = (pkg["render"], pkg["radii"]) + ((pkg["invdepth"], pkg["alpha"]) if maps else ())
            out += (pkg["features"],) if features is not None else ()
            assert set(pkg) == ({"render", "viewspace_points", "visibility_filter", "radii", "FPS"} | ({"invdepth", "alpha"} if maps else set())
                                | ({"features"} if features is not None else set()) | ({"viewspace_points_abs"} if absgrad else set()))
            return out, pkg["viewspace_points"], pkg.get("viewspace_points_abs")
        import diff_gaussian_rasterization as dgr
        torch.use_deterministic_algorithms(False)
        settings = dgr.GaussianRasterizationSettings(H, W, 0.5, 0.5, torch.zeros(3), 1.0, cam.world_view_transform,
                                                     cam.full_proj_transform, 0, cam.camera_center, False, False, deterministic=det)
        means2D = torch.zeros(P, 3, requires_grad=True)
        out = dgr.GaussianRasterizer(settings)(m.get_xyz, means2D, m._opacity, degrees=m._degrees, return_maps=maps, features=feats,
                                               **kw, **({} if means2D_abs is None else dict(means2D_abs=means2D_abs)))
        return out, means2D, means2D_abs

    msg = _refusal(features, absgrad, det, via_render)
    if msg is not None:
        with pytest.raises(RuntimeError, match=msg):
            run()
        assert stub.calls == 0
        return
    out, means2D, means2D_abs = run()
    grads[means2D] = "dL_dmeans2D"

    # the forward: one call with the option keywords, and its outputs in order
    assert len(stub.forward_calls) == 1
    fkw = stub.forward_calls[0][1]
    raw = kw.get("raw_params")
    assert set(fkw) == ({"prune_mask", "return_maps", "antialiasing"} | ({"raw"} if raw else {"quant"})
                        | ({"features"} if features is not None else set()))
    assert fkw["prune_mask"] is None and fkw["return_maps"] is maps and fkw["antialiasing"] is False
    assert fkw["raw"] == raw if raw else fkw["quant"] is quant
    if features is not None:
        assert fkw["features"] is feats
    expect = [marked("color", (3, H, W)), torch.ones(P, dtype=torch.int32)]
    expect += [marked("invdepth", (1, H, W)), marked("alpha", (1, H, W))] if maps else []
    expect += [marked("feature_image", (F, H, W))] if features is not None else []
    assert len(out) == len(expect) and all(torch.equal(a, b) for a, b in zip(out, expect))

    # the backward: a loss on every output (but a feature image that may not have a gradient), distinct weights per output
    feature_loss = features is not None and not (det and features == "const")
    loss = out[0].sum() + ((2 * out[2].sum() + 3 * out[3].sum()) if maps else 0) + (4 * out[-1].sum() if feature_loss else 0)
    loss.backward()
    assert len(stub.backward_calls) == 1
    bkw = stub.backward_calls[0][1]
    assert set(bkw) == ({"prune_mask", "dL_dinvdepth", "dL_dalpha", "camera_grads", "antialiasing"} | ({"raw"} if raw else {"quant"})
                        | ({"deterministic"} if det else set()) | ({"features", "dL_dfeatures_out"} if feature_loss else set())
                        | ({"absgrad_out"} if absgrad else set()))
    assert bkw["prune_mask"] is None and bkw["antialiasing"] is False and bkw["camera_grads"] is bool(cam_grad)
    assert bkw["raw"] == raw if raw else bkw["quant"] is quant
    assert bkw.get("deterministic") is (True if det else None)
    if maps:
        assert torch.equal(bkw["dL_dinvdepth"], torch.full((1, H, W), 2.0)) and torch.equal(bkw["dL_dalpha"], torch.full((1, H, W), 3.0))
    else:
        assert bkw["dL_dinvdepth"] is None and bkw["dL_dalpha"] is None
    if feature_loss:
        assert bkw["features"] is feats and torch.equal(bkw["dL_dfeatures_out"], torch.full((F, H, W), 4.0))

    # every gradient in its own slot
    if features == "grad":
        grads[feats] = "dL_dfeatures"
    if absgrad:
        grads[means2D_abs] = "absgrad"
    for i, (_, attr, name) in enumerate(CAMERA_KEYS):
        t = getattr(cam, attr)
        assert torch.equal(t.grad, marked(name, t.shape)) if i in cam_grad else t.grad is None, name
    inputs = m.leaves() + [colors, means2D] + ([feats] if feats is not None else []) + ([means2D_abs] if absgrad else [])
    for t in inputs:
        name = grads.get(t)
        assert (t.grad is None) if name is None else torch.equal(t.grad, marked(name, t.shape)), (name, t.shape)
    if quant is not None:
        assert set(quant.grads) == {"sh", "opacity", "scales", "rotations"}
        for k, name in (("sh", "dL_dsh"), ("opacity", "dL_dopacity"), ("scales", "dL_dscales"), ("rotations", "dL_drotations")):
            assert torch.equal(quant.grads[k], marked(name, quant.grads[k].shape)), k
