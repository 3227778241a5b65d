"""CPU: anti-aliased requests (the `antialiasing` field of GsbForwardRequest / GsbBackwardRequest): argument checks before any CUDA
call, refusal of CPU tensors, and the plumbing of the `antialiasing` flag from GaussianRasterizationSettings and `pipe` to both
kernels, checked against a stub of `_C` (no GPU, no kernel)."""
import ctypes as C

import pytest
import torch

import stub_c
from gs_b200 import lib


def test_antialiased_symbols_are_exported():
    L = lib.lib()
    for sym in ("gsb_forward", "gsb_backward"):
        assert sym in lib.EXPORTED_SYMBOLS
        getattr(L, sym)
    assert lib.GsbForwardRequest.antialiasing.size == lib.GsbBackwardRequest.antialiasing.size == 4


def _fwd(L, scene, cam, invdepth=None, alpha=None):
    req = lib.GsbForwardRequest(scene=scene, cam=cam, num_rendered=C.pointer(C.c_int64(0)), out_invdepth=invdepth, out_alpha=alpha,
                                antialiasing=1)
    return L.gsb_forward(C.byref(req))


def _bwd(L, scene, cam, view=None, proj=None, campos=None, ws=None):
    req = lib.GsbBackwardRequest(scene=scene, cam=cam, grads=C.pointer(lib.GsbGrads()), dL_dviewmatrix=view, dL_dprojmatrix=proj,
                                 dL_dcampos=campos, camera_workspace=ws, antialiasing=1)
    return L.gsb_backward(C.byref(req))


def test_forward_antialiased_rejects_bad_arguments():
    L = lib.lib()
    cam = lib.GsbCamera()
    for scene in (None, C.pointer(lib.GsbScene(P=-1))):
        assert _fwd(L, scene, C.pointer(cam)) == -1 and b"P < 0" in L.gsb_last_error()
    # one map output without the other is refused before the scene / camera are looked at (here: an empty camera struct)
    buf = (C.c_float * 16)()
    for maps in ((C.addressof(buf), None), (None, C.addressof(buf))):
        assert _fwd(L, C.pointer(lib.GsbScene(P=10)), C.pointer(cam), *maps) == -1
        assert b"both map outputs" in L.gsb_last_error()
    # both or neither: the call goes on to the usual scene / camera checks
    for maps in ((None, None), (C.addressof(buf), C.addressof(buf))):
        assert _fwd(L, C.pointer(lib.GsbScene(P=10)), C.pointer(cam), *maps) == -1
        assert b"map outputs" not in L.gsb_last_error()


def test_backward_antialiased_rejects_bad_arguments():
    L = lib.lib()
    cam = lib.GsbCamera()
    for scene in (None, C.pointer(lib.GsbScene(P=-1))):
        assert _bwd(L, scene, C.pointer(cam)) == -1 and b"P < 0" in L.gsb_last_error()
    buf = (C.c_float * 16)()
    for k in range(3):
        outs = [None, None, None]
        outs[k] = C.addressof(buf)
        assert _bwd(L, C.pointer(lib.GsbScene(P=10)), C.pointer(cam), *outs) == -1
        assert b"workspace" in L.gsb_last_error()
    assert _bwd(L, C.pointer(lib.GsbScene(P=10)), C.pointer(cam)) == -1
    assert b"workspace" not in L.gsb_last_error()


def test_antialiasing_refuses_cpu_tensors():
    from diff_gaussian_rasterization import _C
    P, H, W = 4, 16, 16
    z = torch.zeros(P, 3)
    with pytest.raises(RuntimeError):
        _C.rasterize_gaussians(torch.zeros(3), z, torch.empty(0), torch.zeros(P, 1), z, torch.zeros(P, 4), 1.0, torch.empty(0),
                               torch.eye(4), torch.eye(4), 1.0, 1.0, H, W, torch.zeros(P, 1, 3), torch.zeros(P, 1, dtype=torch.int32),
                               torch.zeros(3), False, False, antialiasing=True)
    with pytest.raises(RuntimeError):
        _C.rasterize_gaussians_backward(torch.zeros(3), z, torch.ones(P, dtype=torch.int32), torch.empty(0), z, torch.zeros(P, 4), 1.0,
                                        torch.empty(0), torch.eye(4), torch.eye(4), 1.0, 1.0, torch.zeros(3, H, W), torch.zeros(P, 1, 3),
                                        torch.zeros(P, 1, dtype=torch.int32), torch.zeros(3), torch.empty(0), 0, torch.empty(0),
                                        torch.empty(0), 0.0, False, antialiasing=True)


def test_settings_default_to_no_antialiasing():
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    args = (8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)
    s = GaussianRasterizationSettings(*args)
    assert s.antialiasing is False and len(s) == 12 and s.debug is False
    # upstream 3DGS passes it as a trailing keyword; a 13th positional argument works too; _replace keeps or changes it
    assert GaussianRasterizationSettings(*args, antialiasing=True).antialiasing is True
    t = GaussianRasterizationSettings(*args, True)
    assert t.antialiasing is True and tuple(t) == tuple(s)
    assert t._replace(debug=True).antialiasing is True and t._replace(antialiasing=False).antialiasing is False
    assert s._replace(antialiasing=True).antialiasing is True and s._replace(image_height=4).image_height == 4


@pytest.mark.parametrize("aa", [False, True])
def test_settings_flag_reaches_forward_and_backward(monkeypatch, aa):
    import diff_gaussian_rasterization as dgr
    stub = stub_c.StubC().install(monkeypatch)
    P = 5
    settings = dgr.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3),
                                                 False, False, antialiasing=aa)
    means = torch.zeros(P, 3, requires_grad=True)
    opac = torch.zeros(P, 1, requires_grad=True)
    color, _ = dgr.GaussianRasterizer(settings)(means, torch.zeros(P, 3, requires_grad=True), opac, shs=torch.zeros(P, 1, 3),
                                                degrees=torch.zeros(P, 1, dtype=torch.int32), scales=torch.ones(P, 3),
                                                rotations=torch.ones(P, 4))
    (color * 1.0).sum().backward()
    assert [kw["antialiasing"] for _, kw in stub.forward_calls] == [aa]
    assert [kw["antialiasing"] for _, kw in stub.backward_calls] == [aa]
    assert float(opac.grad[0, 0]) == stub_c.MARK["dL_dopacity"] and float(means.grad[0, 0]) == stub_c.MARK["dL_dmeans3D"]


@pytest.mark.parametrize("pipe_aa", [None, False, True])
def test_render_takes_the_flag_from_pipe(monkeypatch, pipe_aa):
    import gaussian_renderer
    stub = stub_c.StubC().install(monkeypatch)
    pipe = stub_c.pipe()
    if pipe_aa is not None:
        pipe.antialiasing = pipe_aa
    want = bool(pipe_aa)                                    # a pipe without the attribute (reduced-3dgs's) renders without
    gaussian_renderer.render(stub_c.camera(), stub_c.Model(), pipe, torch.zeros(3))
    gaussian_renderer.render(stub_c.camera(), stub_c.Model(), pipe, torch.zeros(3), variable_sh_bands=True)
    assert [kw["antialiasing"] for _, kw in stub.forward_calls] == [want]
    assert [kw["antialiasing"] for _, kw in stub.variable_sh_calls] == [want]
