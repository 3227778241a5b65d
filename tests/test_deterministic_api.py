"""CPU: the deterministic backward (gsb_deterministic_workspace_bytes, gsb_backward's `deterministic` / `det_workspace`): exported,
workspace size, argument checks before any CUDA call, and the plumbing of GaussianRasterizationSettings' `deterministic` keyword
and torch's deterministic-algorithms flag to `_C.rasterize_gaussians_backward`, checked against a stub of `_C` (no GPU)."""
import ctypes as C

import pytest
import torch

import stub_c
from gs_b200 import lib


@pytest.fixture
def torch_deterministic():
    """Restores torch's deterministic-algorithms flag (and its warn-only mode) after the test."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def test_symbols_are_exported():
    L = lib.lib()
    for sym in ("gsb_deterministic_workspace_bytes", "gsb_backward"):
        assert sym in lib.EXPORTED_SYMBOLS
        getattr(L, sym)


def test_workspace_size():
    L = lib.lib()
    for P, R in ((0, 0), (1, 1), (1000, 5000), (10 ** 6, 7 * 10 ** 6), (3 * 10 ** 6, 4 * 10 ** 7)):
        assert L.gsb_deterministic_workspace_bytes(P, R, 0) >= P * 4 + R * 36
    assert L.gsb_deterministic_workspace_bytes(2000, 5000, 0) > L.gsb_deterministic_workspace_bytes(1000, 5000, 0)
    assert L.gsb_deterministic_workspace_bytes(1000, 6000, 0) > L.gsb_deterministic_workspace_bytes(1000, 5000, 0)


def _bwd(L, scene, R=0, ws=None, det_ws=None, cam_out=(None, None, None), raw=None, raw_grads=None, grads=None):
    g = grads if grads is not None else lib.GsbGrads()
    req = lib.GsbBackwardRequest(scene=scene, cam=C.pointer(lib.GsbCamera()), num_rendered=R, grads=C.pointer(g), camera_workspace=ws,
                                 raw=raw, raw_grads=raw_grads, deterministic=1, det_workspace=det_ws)
    req.dL_dviewmatrix, req.dL_dprojmatrix, req.dL_dcampos = cam_out
    return L.gsb_backward(C.byref(req))


def test_backward_deterministic_rejects_bad_arguments():
    L = lib.lib()
    for scene in (None, C.pointer(lib.GsbScene(P=-1))):
        assert _bwd(L, scene) == -1 and b"P < 0" in L.gsb_last_error()
    assert _bwd(L, C.pointer(lib.GsbScene(P=10)), R=-1) == -1 and b"num_rendered < 0" in L.gsb_last_error()
    assert _bwd(L, C.pointer(lib.GsbScene(P=10)), R=1 << 30) == -4 and b"2^30" in L.gsb_last_error()
    # a NULL workspace is refused only when there is something to sum (P > 0 and R > 0)
    assert _bwd(L, C.pointer(lib.GsbScene(P=10)), R=5) == -1 and b"det_workspace is NULL" in L.gsb_last_error()
    buf = (C.c_char * 256)()
    for scene, R, ws in ((lib.GsbScene(P=10), 0, None), (lib.GsbScene(P=0), 5, None), (lib.GsbScene(P=10), 5, C.addressof(buf))):
        assert _bwd(L, C.pointer(scene), R=R, det_ws=ws) == -1            # goes on to the camera / scene checks (an empty camera)
        assert b"det_workspace" not in L.gsb_last_error()
    fbuf = (C.c_float * 16)()
    for k in range(3):
        outs = [None, None, None]
        outs[k] = C.addressof(fbuf)
        assert _bwd(L, C.pointer(lib.GsbScene(P=10)), R=5, det_ws=C.addressof(buf), cam_out=outs) == -1
        assert b"workspace is NULL" in L.gsb_last_error()
    rg = lib.GsbRawGrads()
    assert _bwd(L, C.pointer(lib.GsbScene(P=10)), R=5, det_ws=C.addressof(buf), raw_grads=C.pointer(rg)) == -1
    assert b"raw_grads given without raw" in L.gsb_last_error()


def test_backward_deterministic_applies_the_raw_checks():
    L = lib.lib()
    buf = (C.c_char * 256)()
    ws = C.addressof(buf)
    scene = lib.GsbScene(P=10)
    # C outside {0, 3, 8, 15}
    assert _bwd(L, C.pointer(scene), R=5, det_ws=ws, raw=C.pointer(lib.GsbRawParams(C=4)), raw_grads=C.pointer(lib.GsbRawGrads())) == -1
    assert b"C = 4" in L.gsb_last_error()
    # a scene field the raw parameters replace
    fbuf = (C.c_float * 16)()
    s2 = lib.GsbScene(P=10)
    s2.scales = C.addressof(fbuf)
    assert _bwd(L, C.pointer(s2), R=5, det_ws=ws, raw=C.pointer(lib.GsbRawParams(C=3)), raw_grads=C.pointer(lib.GsbRawGrads())) == -1
    assert b"must be NULL" in L.gsb_last_error()
    # raw without raw_grads
    full = lib.GsbRawParams(C.addressof(fbuf), C.addressof(fbuf), 3, C.addressof(fbuf), C.addressof(fbuf))
    s3 = lib.GsbScene(P=10)
    s3.degrees = C.addressof(fbuf)
    assert _bwd(L, C.pointer(s3), R=5, det_ws=ws, raw=C.pointer(full)) == -1 and b"raw_grads are NULL" in L.gsb_last_error()
    # grads->dL_dsh given next to raw_grads
    g = lib.GsbGrads()
    g.dL_dsh = C.addressof(fbuf)
    assert _bwd(L, C.pointer(s3), R=5, det_ws=ws, raw=C.pointer(full), raw_grads=C.pointer(lib.GsbRawGrads()), grads=g) == -1
    assert b"raw_grads replaces them" in L.gsb_last_error()
    # dL_dfeatures_rest with C == 0
    rg = lib.GsbRawGrads()
    rg.dL_dfeatures_rest = C.addressof(fbuf)
    c0 = lib.GsbRawParams(C.addressof(fbuf), None, 0, C.addressof(fbuf), C.addressof(fbuf))
    assert _bwd(L, C.pointer(s3), R=5, det_ws=ws, raw=C.pointer(c0), raw_grads=C.pointer(rg)) == -1
    assert b"C == 0" in L.gsb_last_error()


def test_deterministic_refuses_cpu_tensors():
    from diff_gaussian_rasterization import _C
    P, H, W = 4, 16, 16
    z = torch.zeros(P, 3)
    with pytest.raises(RuntimeError):
        _C.rasterize_gaussians_backward(torch.zeros(3), z, torch.ones(P, dtype=torch.int32), torch.empty(0), z, torch.zeros(P, 4), 1.0,
                                        torch.empty(0), torch.eye(4), torch.eye(4), 1.0, 1.0, torch.zeros(3, H, W), torch.zeros(P, 1, 3),
                                        torch.zeros(P, 1, dtype=torch.int32), torch.zeros(3), torch.empty(0), 0, torch.empty(0),
                                        torch.empty(0), 0.0, False, deterministic=True)


ARGS = (8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)


def test_settings_keyword():
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    s = GaussianRasterizationSettings(*ARGS)
    assert s.deterministic is None and len(s) == 12
    assert len(s._fields) == 12 and "deterministic" not in s._fields
    t = GaussianRasterizationSettings(*ARGS, deterministic=True)
    assert t.deterministic is True and tuple(t) == tuple(s)
    # the 13-positional layout (trailing antialiasing) is unchanged; deterministic is keyword-only
    u = GaussianRasterizationSettings(*ARGS, True, deterministic=False)
    assert u.antialiasing is True and u.deterministic is False and len(u) == 12
    with pytest.raises(TypeError):
        GaussianRasterizationSettings(*ARGS, True, True)
    # _replace keeps the value, or changes it when asked
    assert t._replace(debug=True).deterministic is True and t._replace(debug=True).debug is True
    assert u._replace(image_height=4).deterministic is False and u._replace(image_height=4).antialiasing is True
    assert t._replace(deterministic=None).deterministic is None and s._replace(deterministic=True).deterministic is True


def _run(monkeypatch, settings, raw=False):
    import diff_gaussian_rasterization as dgr
    stub = stub_c.StubC().install(monkeypatch)
    P = 5
    means = torch.zeros(P, 3, requires_grad=True)
    opac = torch.zeros(P, 1, requires_grad=True)
    rz = dgr.GaussianRasterizer(settings)
    if raw:
        leaves = (torch.zeros(P, 1, 3, requires_grad=True), torch.zeros(P, 3, 3, requires_grad=True), torch.zeros(P, 3, requires_grad=True),
                  torch.ones(P, 4, requires_grad=True))
        color, _ = rz(means, torch.zeros(P, 3, requires_grad=True), opac, degrees=torch.zeros(P, 1, dtype=torch.int32), raw_params=leaves)
    else:
        color, _ = rz(means, torch.zeros(P, 3, requires_grad=True), opac, shs=torch.zeros(P, 1, 3),
                      degrees=torch.zeros(P, 1, dtype=torch.int32), scales=torch.ones(P, 3), rotations=torch.ones(P, 4))
    (color * 1.0).sum().backward()
    assert float(opac.grad[0, 0]) == stub_c.MARK["dL_dopacity"]
    assert len(stub.backward_calls) == 1
    return stub.backward_calls[0][1]


@pytest.mark.parametrize("raw", [False, True])
def test_settings_keyword_reaches_the_backward(monkeypatch, torch_deterministic, raw):
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    torch.use_deterministic_algorithms(False)
    assert _run(monkeypatch, GaussianRasterizationSettings(*ARGS, deterministic=True), raw).get("deterministic") is True


@pytest.mark.parametrize("raw", [False, True])
def test_torch_flag_reaches_the_backward(monkeypatch, torch_deterministic, raw):
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    torch.use_deterministic_algorithms(True)
    assert _run(monkeypatch, GaussianRasterizationSettings(*ARGS), raw).get("deterministic") is True
    # read when the backward runs: a _replace'd copy still follows the flag
    assert _run(monkeypatch, GaussianRasterizationSettings(*ARGS)._replace(debug=False), raw).get("deterministic") is True


def test_explicit_false_wins_over_the_torch_flag(monkeypatch, torch_deterministic):
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    torch.use_deterministic_algorithms(True)
    kw = _run(monkeypatch, GaussianRasterizationSettings(*ARGS, deterministic=False))
    assert "deterministic" not in kw


def test_default_leaves_the_call_unchanged(monkeypatch, torch_deterministic):
    """Flag off and no keyword: the backward is called with exactly the keywords it had before the option existed."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    torch.use_deterministic_algorithms(False)
    expected = {"prune_mask", "dL_dinvdepth", "dL_dalpha", "camera_grads", "antialiasing", "quant"}
    assert set(_run(monkeypatch, GaussianRasterizationSettings(*ARGS))) == expected
    assert set(_run(monkeypatch, GaussianRasterizationSettings(*ARGS), raw=True)) == expected - {"quant"} | {"raw"}
