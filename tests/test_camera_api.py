"""CPU: argument checks of the camera-gradient backward (gsb_backward's dL_dviewmatrix / dL_dprojmatrix / dL_dcampos) and
gsb_camera_grad_workspace_bytes, the Python layer's refusal of CPU tensors with
camera_grads, and the autograd plumbing of a learnable camera, checked against a stub of `_C` (no GPU, no kernel)."""
import ctypes as C

import pytest
import torch

import stub_c
from gs_b200 import lib


def _call(L, scene, cam, view=None, proj=None, campos=None, ws=None):
    req = lib.GsbBackwardRequest(scene=scene, cam=cam, grads=C.pointer(lib.GsbGrads()), dL_dviewmatrix=view, dL_dprojmatrix=proj,
                                 dL_dcampos=campos, camera_workspace=ws)
    return L.gsb_backward(C.byref(req))


def test_backward_camera_rejects_bad_arguments():
    L = lib.lib()
    cam = lib.GsbCamera()
    for scene in (None, C.pointer(lib.GsbScene(P=-1))):
        assert _call(L, scene, C.pointer(cam)) < 0 and len(L.gsb_last_error()) > 0
    # a camera output without a workspace is refused before anything else is looked at (here: an empty camera struct)
    buf = (C.c_float * 16)()
    for k in range(3):
        outs = [None, None, None]
        outs[k] = C.addressof(buf)
        scene = lib.GsbScene(P=10)
        assert _call(L, C.pointer(scene), C.pointer(cam), *outs) == -1
        assert b"workspace" in L.gsb_last_error()
    # without any camera output the workspace is not needed: the call goes on to the usual scene / camera checks
    assert _call(L, C.pointer(lib.GsbScene(P=10)), C.pointer(cam)) == -1
    assert b"workspace" not in L.gsb_last_error()


def test_camera_workspace_bytes():
    L = lib.lib()
    f = L.gsb_camera_grad_workspace_bytes
    # one row of 32 floats per CTA of the preprocess backward: ceil(P / 256), at most 4 per SM; never empty
    assert f(0) == 128 and f(1) == 128 and f(256) == 128 and f(257) == 256
    assert f(10 ** 6) == f(3 * 10 ** 6) == f(10 ** 8) and f(10 ** 6) % 128 == 0
    assert 128 * 256 < f(10 ** 6) <= 128 * 4 * 160
    assert all(f(p) <= f(p + 1000) for p in range(0, 300_000, 7919))


def test_camera_grads_refuse_cpu_tensors():
    from diff_gaussian_rasterization import _C
    P, H, W = 4, 16, 16
    z = torch.zeros(P, 3)
    with pytest.raises(RuntimeError):
        _C.rasterize_gaussians_backward(torch.zeros(3), z, torch.ones(P, dtype=torch.int32), torch.empty(0), z, torch.zeros(P, 4), 1.0,
                                        torch.empty(0), torch.eye(4), torch.eye(4), 1.0, 1.0, torch.zeros(3, H, W), torch.zeros(P, 1, 3),
                                        torch.zeros(P, 1, dtype=torch.int32), torch.zeros(3), torch.empty(0), 0, torch.empty(0),
                                        torch.empty(0), 0.0, False, camera_grads=True)


def _render(monkeypatch, view, proj, campos):
    import diff_gaussian_rasterization as dgr
    stub = stub_c.StubC().install(monkeypatch)
    P = 5
    settings = dgr.GaussianRasterizationSettings(image_height=8, image_width=8, tanfovx=0.5, tanfovy=0.5, bg=torch.zeros(3),
                                                 scale_modifier=1.0, viewmatrix=view, projmatrix=proj, sh_degree=0, campos=campos,
                                                 prefiltered=False, debug=False)
    means = torch.zeros(P, 3, requires_grad=True)
    color, radii = dgr.GaussianRasterizer(settings)(means, torch.zeros(P, 3, requires_grad=True), torch.zeros(P, 1),
                                                    shs=torch.zeros(P, 1, 3), degrees=torch.zeros(P, 1, dtype=torch.int32),
                                                    scales=torch.ones(P, 3), rotations=torch.ones(P, 4))
    color.sum().backward()
    assert means.grad is not None and float(means.grad[0, 0]) == stub_c.MARK["dL_dmeans3D"]
    return stub


def test_constant_camera_passes_camera_grads_false(monkeypatch):
    view, proj, campos = torch.eye(4), torch.eye(4), torch.zeros(3)
    stub = _render(monkeypatch, view, proj, campos)
    assert len(stub.backward_calls) == 1 and stub.backward_calls[0][1]["camera_grads"] is False
    assert view.grad is None and proj.grad is None and campos.grad is None


def test_learnable_camera_receives_its_gradients(monkeypatch):
    view = torch.eye(4, dtype=torch.float64, requires_grad=True)         # gradients come back in the input's dtype and shape
    proj = torch.eye(4)
    campos = torch.zeros(1, 3, requires_grad=True)
    stub = _render(monkeypatch, view, proj, campos)
    assert stub.backward_calls[0][1]["camera_grads"] is True
    assert view.grad.dtype == torch.float64 and torch.equal(view.grad, stub_c.marked("dL_dviewmatrix", (4, 4)).double())
    assert proj.grad is None                                                # not requested
    assert campos.grad.shape == (1, 3) and torch.equal(campos.grad, stub_c.marked("dL_dcampos", (3,)).view(1, 3))


def test_learnable_camera_under_no_grad_is_todays_call(monkeypatch):
    view = torch.eye(4, requires_grad=True)
    import diff_gaussian_rasterization as dgr
    seen = []
    orig = dgr._RasterizeGaussians.apply
    monkeypatch.setattr(dgr._RasterizeGaussians, "apply", lambda *a: seen.append(len(a)) or orig(*a))
    stub_c.StubC().install(monkeypatch)
    settings = dgr.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, view, torch.eye(4), 0, torch.zeros(3), False, False)
    with torch.no_grad():
        dgr.GaussianRasterizer(settings)(torch.zeros(2, 3), torch.zeros(2, 3), torch.zeros(2, 1), shs=torch.zeros(2, 1, 3),
                                         degrees=torch.zeros(2, 1, dtype=torch.int32), scales=torch.ones(2, 3),
                                         rotations=torch.ones(2, 4))
    assert seen == [14]
