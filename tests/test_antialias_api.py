"""CPU: the anti-aliased entry points (gsb_forward_antialiased / gsb_backward_antialiased): exported, argument checks before any CUDA
call, refusal of CPU tensors, and the plumbing of the `antialiasing` flag from GaussianRasterizationSettings and `pipe` to both
kernels, checked against a stub of `_C` (no GPU, no kernel)."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

from gs_b200 import lib


def test_antialiased_symbols_are_exported():
    L = lib.lib()
    for sym in ("gsb_forward_antialiased", "gsb_backward_antialiased"):
        assert sym in lib.EXPORTED_SYMBOLS
        getattr(L, sym)


def _fwd(L, scene, cam, invdepth=None, alpha=None):
    R = C.c_int64(0)
    return L.gsb_forward_antialiased(scene, cam, lib.ALLOC_FN(0), None, lib.ALLOC_FN(0), None, lib.ALLOC_FN(0), None, None, None,
                                     C.byref(R), None, invdepth, alpha, None)


def _bwd(L, scene, cam, view=None, proj=None, campos=None, ws=None):
    g = lib.GsbGrads()
    return L.gsb_backward_antialiased(scene, cam, 0, None, None, None, None, None, C.byref(g), None, None, 0.0, view, proj, campos, ws,
                                      None)


def test_forward_antialiased_rejects_bad_arguments():
    L = lib.lib()
    cam = lib.GsbCamera()
    for scene in (None, C.byref(lib.GsbScene(P=-1))):
        assert _fwd(L, scene, C.byref(cam)) == -1 and b"P < 0" in L.gsb_last_error()
    # one map output without the other is refused before the scene / camera are looked at (here: an empty camera struct)
    buf = (C.c_float * 16)()
    for maps in ((C.addressof(buf), None), (None, C.addressof(buf))):
        assert _fwd(L, C.byref(lib.GsbScene(P=10)), C.byref(cam), *maps) == -1
        assert b"both map outputs" in L.gsb_last_error()
    # both or neither: the call goes on to the usual scene / camera checks
    for maps in ((None, None), (C.addressof(buf), C.addressof(buf))):
        assert _fwd(L, C.byref(lib.GsbScene(P=10)), C.byref(cam), *maps) == -1
        assert b"map outputs" not in L.gsb_last_error()


def test_backward_antialiased_rejects_bad_arguments():
    L = lib.lib()
    cam = lib.GsbCamera()
    for scene in (None, C.byref(lib.GsbScene(P=-1))):
        assert _bwd(L, scene, C.byref(cam)) == -1 and b"P < 0" in L.gsb_last_error()
    buf = (C.c_float * 16)()
    for k in range(3):
        outs = [None, None, None]
        outs[k] = C.addressof(buf)
        assert _bwd(L, C.byref(lib.GsbScene(P=10)), C.byref(cam), *outs) == -1
        assert b"workspace" in L.gsb_last_error()
    assert _bwd(L, C.byref(lib.GsbScene(P=10)), C.byref(cam)) == -1
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


class _StubC:
    """Stands in for the kernels: records the `antialiasing` keyword of each call and returns outputs of the right shapes."""

    def __init__(self):
        self.forward_aa, self.backward_aa, self.variable_sh_aa = [], [], []

    def rasterize_gaussians(self, *args, antialiasing=False, return_maps=False, **kw):
        self.forward_aa.append(antialiasing)
        means3D, H, W = args[1], args[12], args[13]
        P = means3D.shape[0]
        color = torch.ones(3, H, W)
        out = (1, color, torch.ones(P, dtype=torch.int32), torch.zeros(8, dtype=torch.uint8), torch.zeros(8, dtype=torch.uint8),
               torch.zeros(8, dtype=torch.uint8))
        return out + ((torch.zeros(1, H, W), torch.zeros(1, H, W)) if return_maps else ())

    def rasterize_gaussians_backward(self, *args, antialiasing=False, **kw):
        self.backward_aa.append(antialiasing)
        means3D, sh = args[1], args[13]
        P = means3D.shape[0]
        M = sh.shape[1] if sh.numel() else 0
        return tuple(torch.full(s, 0.5) for s in [(P, 3), (P, 3), (P, 1), (P, 3), (P, 6), (P, M, 3), (P, 3), (P, 4)])

    def rasterize_gaussians_variableSH_bands(self, *args, antialiasing=False, **kw):
        self.variable_sh_aa.append(antialiasing)
        H, W, P = args[12], args[13], args[1].shape[0]
        return (1, torch.ones(3, H, W), torch.ones(P, dtype=torch.int32), None, None, None)


@pytest.mark.parametrize("aa", [False, True])
def test_settings_flag_reaches_forward_and_backward(monkeypatch, aa):
    import diff_gaussian_rasterization as dgr
    stub = _StubC()
    monkeypatch.setattr(dgr._C, "rasterize_gaussians", stub.rasterize_gaussians)
    monkeypatch.setattr(dgr._C, "rasterize_gaussians_backward", stub.rasterize_gaussians_backward)
    P = 5
    settings = dgr.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3),
                                                 False, False, antialiasing=aa)
    means = torch.zeros(P, 3, requires_grad=True)
    opac = torch.zeros(P, 1, requires_grad=True)
    color, _ = dgr.GaussianRasterizer(settings)(means, torch.zeros(P, 3, requires_grad=True), opac, shs=torch.zeros(P, 1, 3),
                                                degrees=torch.zeros(P, 1, dtype=torch.int32), scales=torch.ones(P, 3),
                                                rotations=torch.ones(P, 4))
    (color * 1.0).sum().backward()
    assert stub.forward_aa == [aa] and stub.backward_aa == [aa]
    assert float(opac.grad[0, 0]) == 0.5 and float(means.grad[0, 0]) == 0.5


class _Model:
    def __init__(self, P=4):
        self.get_xyz = torch.zeros(P, 3)
        self._opacity = torch.zeros(P, 1)
        self._degrees = torch.zeros(P, 1, dtype=torch.int32)
        self.get_scaling = torch.ones(P, 3)
        self.get_rotation = torch.ones(P, 4)
        self.get_features = torch.zeros(P, 1, 3)
        self.active_sh_degree = self.max_sh_degree = 0
        self.per_band_count = [P, 0, 0, 0]


def _camera():
    return SimpleNamespace(FoVx=1.0, FoVy=1.0, image_height=8, image_width=8, world_view_transform=torch.eye(4),
                           full_proj_transform=torch.eye(4), camera_center=torch.zeros(3))


@pytest.mark.parametrize("pipe_aa", [None, False, True])
def test_render_takes_the_flag_from_pipe(monkeypatch, pipe_aa):
    import diff_gaussian_rasterization as dgr
    import gaussian_renderer
    stub = _StubC()
    monkeypatch.setattr(dgr._C, "rasterize_gaussians", stub.rasterize_gaussians)
    monkeypatch.setattr(gaussian_renderer, "rasterize_gaussians_variableSH_bands", stub.rasterize_gaussians_variableSH_bands)
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    if pipe_aa is not None:
        pipe.antialiasing = pipe_aa
    want = bool(pipe_aa)                                    # a pipe without the attribute (reduced-3dgs's) renders without
    gaussian_renderer.render(_camera(), _Model(), pipe, torch.zeros(3))
    gaussian_renderer.render(_camera(), _Model(), pipe, torch.zeros(3), variable_sh_bands=True)
    assert stub.forward_aa == [want] and stub.variable_sh_aa == [want]
