"""CPU: the absolute screen-space gradient (DESIGN.md §5m).  The backward request with dL_dmeans2D_abs, its workspace size,
gsb_densify_stats and gsb_densify_plan with their absolute-gradient arguments reject each bad argument before any CUDA call; the Python layer refuses what has no
absgrad form before anything runs and, against stand-in kernels, carries `absgrad` through both autograd ops and render() while
leaving the calls without it exactly as they were; and the float64 restatement of the per-pair terms (absgrad64.py) sums, with
signs, to the fp64 oracle's dL_dmeans2D on the backward-edge scenes, which pins it to the pairs and terms the oracle uses."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import absgrad64
import backward_edges as BE
import stub_c
from gs_b200 import lib

NEW = ("gsb_backward", "gsb_deterministic_workspace_bytes", "gsb_densify_stats", "gsb_densify_plan")


def test_symbols_exported():
    L = lib.lib()
    for sym in NEW:
        assert sym in lib.EXPORTED_SYMBOLS
        getattr(L, sym)


def test_workspace_grows_and_adds_eight_bytes_per_instance():
    L = lib.lib()
    for P, R in ((0, 0), (1, 1), (1000, 5000), (100_000, 3_000_000)):
        base, ab = int(L.gsb_deterministic_workspace_bytes(P, R, 0)), int(L.gsb_deterministic_workspace_bytes(P, R, 1))
        assert ab >= base + 8 * R
    assert L.gsb_deterministic_workspace_bytes(1000, 10, 1) < L.gsb_deterministic_workspace_bytes(1000, 11_000, 1)
    assert L.gsb_deterministic_workspace_bytes(1000, 10, 1) < L.gsb_deterministic_workspace_bytes(100_000, 10, 1)


def _bwd(L, scene, R=5, grads=None, out=True, det_ws=None, raw=None, raw_grads=None, cam_out=None, workspace=None, features=None):
    g = grads if grads is not None else lib.GsbGrads()
    buf = (C.c_float * 16)()
    req = lib.GsbBackwardRequest(scene=scene, cam=C.pointer(lib.GsbCamera()), num_rendered=R, grads=C.pointer(g), dL_dviewmatrix=cam_out,
                                 camera_workspace=workspace, raw=raw, raw_grads=raw_grads, deterministic=int(det_ws is not None),
                                 det_workspace=det_ws, features=features, dL_dmeans2D_abs=C.addressof(buf) if out else None)
    return L.gsb_backward(C.byref(req))


def test_backward_absgrad_rejects_bad_arguments():
    L = lib.lib()
    scene = C.pointer(lib.GsbScene(P=10))
    fbuf = (C.c_float * 16)()
    for sc in (None, C.pointer(lib.GsbScene(P=-1))):
        assert _bwd(L, sc) == -1 and b"P < 0" in L.gsb_last_error()
    feats = lib.GsbFeatures(4, C.addressof(fbuf), None, C.addressof(fbuf), C.addressof(fbuf))
    assert _bwd(L, scene, features=C.pointer(feats)) == -1 and b"no feature form" in L.gsb_last_error()
    assert _bwd(L, scene, grads=lib.GsbGrads(accumulate=1)) == -1 and b"accumulate" in L.gsb_last_error()
    assert _bwd(L, scene, R=-1) == -1 and b"num_rendered < 0" in L.gsb_last_error()
    buf = (C.c_char * 256)()
    assert _bwd(L, scene, R=1 << 30, det_ws=C.addressof(buf)) == -4 and b"2^30" in L.gsb_last_error()
    assert _bwd(L, scene, cam_out=C.addressof(fbuf)) == -1 and b"workspace is NULL" in L.gsb_last_error()
    assert _bwd(L, scene, raw_grads=C.pointer(lib.GsbRawGrads())) == -1 and b"raw_grads given without raw" in L.gsb_last_error()
    assert _bwd(L, scene, raw=C.pointer(lib.GsbRawParams(C=4)), raw_grads=C.pointer(lib.GsbRawGrads())) == -1
    assert b"C = 4" in L.gsb_last_error()
    # valid absgrad arguments go on to the scene checks of the backward (an empty camera is refused there), and so does a request
    # without the output
    assert _bwd(L, scene) == -1 and b"image size" in L.gsb_last_error()
    assert _bwd(L, C.pointer(lib.GsbScene(P=0)), out=False) == -1 and b"image size" in L.gsb_last_error()
    assert _bwd(L, scene, out=False) == -1 and b"image size" in L.gsb_last_error()


def test_densify_abs_entry_points_reject_bad_arguments():
    L = lib.lib()
    b = (C.c_float * 64)()
    p = C.addressof(b)
    assert L.gsb_densify_stats(-1, p, 3, p, 3, p, None, p, p, p, None, None) == -1 and b"P < 0" in L.gsb_last_error()
    assert L.gsb_densify_stats(4, p, 3, p, 1, p, None, p, p, p, None, None) == -1 and b">= 2" in L.gsb_last_error()
    assert L.gsb_densify_stats(4, p, 3, p, 3, p, p, p, p, p, None, None) == -1 and b"without max_radii2D" in L.gsb_last_error()
    assert L.gsb_densify_stats(4, p, 3, None, 3, p, None, p, p, p, None, None) == -1 and b"NULL" in L.gsb_last_error()
    assert L.gsb_densify_stats(4, p, 3, p, 3, p, None, p, None, p, None, None) == -1 and b"NULL" in L.gsb_last_error()
    assert L.gsb_densify_stats(0, None, 3, None, 3, None, None, None, None, None, None, None) == 0
    # one of the pair without the other is refused at any P
    for ga, acc_abs in ((p, None), (None, p)):
        assert L.gsb_densify_stats(0, None, 3, ga, 3, None, None, None, acc_abs, None, None, None) == -1 and b"both" in L.gsb_last_error()
    cnt = (C.c_int64 * 8)()
    args = lambda P, acc_abs, ws=p, mode=lib.DENSIFY_CLONE_SPLIT: (P, mode, p, acc_abs, p, p, p, None, None, 0.1, 0.2, 0.01, 0.005, 0,
                                                                   0.0, 1.0, 0.625, ws, C.addressof(cnt), None)
    # the absolute accumulator selects the AbsGS split test, which only the clone / split mode has
    for mode in (lib.DENSIFY_PRUNE, lib.DENSIFY_PRUNE_MASK):
        assert L.gsb_densify_plan(*args(4, p, mode=mode)) == -1 and b"xyz_gradient_accum_abs" in L.gsb_last_error()
    assert L.gsb_densify_plan(*args(4, p, None)) == -1 and b"workspace" in L.gsb_last_error()
    assert L.gsb_densify_plan(*args(-1, p)) == -1 and b"outside" in L.gsb_last_error()


# ---- Python refusals ---------------------------------------------------------------------------------------------------------------

def _backward_call(**kw):
    from diff_gaussian_rasterization import _C
    P, H, W = 4, 16, 16
    z = torch.zeros(P, 3)
    return _C.rasterize_gaussians_backward(torch.zeros(3), z, torch.ones(P, dtype=torch.int32), torch.empty(0), z, torch.zeros(P, 4), 1.0,
                                           torch.empty(0), torch.eye(4), torch.eye(4), 1.0, 1.0, torch.zeros(3, H, W), torch.zeros(P, 1, 3),
                                           torch.zeros(P, 1, dtype=torch.int32), torch.zeros(3), torch.empty(0), 0, torch.empty(0),
                                           torch.empty(0), 0.0, False, **kw)


@pytest.mark.parametrize("kw, msg", [
    (dict(absgrad_out=torch.zeros(4, 3), accumulate_into=tuple(torch.zeros(1) for _ in range(8))), "accumulate_into"),
    (dict(absgrad_out=torch.zeros(4, 3), features=torch.zeros(4, 5), dL_dfeatures_out=torch.zeros(5, 16, 16)), "feature"),
    (dict(absgrad_out=torch.zeros(5, 3)), r"shape \[P, 3\]"),
    (dict(absgrad_out=torch.zeros(4, 2)), r"shape \[P, 3\]"),
    (dict(absgrad_out=torch.zeros(4, 3, dtype=torch.float64)), "float32"),
    (dict(absgrad_out=torch.zeros(3, 4).t()), "contiguous"),
    (dict(absgrad_out=torch.zeros(4, 3)), "CUDA device"),
    (dict(absgrad_out="no"), "tensor"),
])
def test_backward_refusals_leave_nothing_called(monkeypatch, kw, msg):
    from gs_b200 import lib as gl
    monkeypatch.setattr(gl, "lib", lambda: (_ for _ in ()).throw(AssertionError("the library was reached")))
    with pytest.raises(RuntimeError, match=msg):
        _backward_call(**kw)


def _render(monkeypatch, fused=False, **kw):
    from gaussian_renderer import render
    stub = stub_c.StubC().install(monkeypatch)
    pkg = render(stub_c.camera(), stub_c.Model(), stub_c.pipe(fused_activations=fused), torch.zeros(3), **kw)
    return stub, pkg


@pytest.mark.parametrize("fused", [False, True])
def test_render_absgrad_reaches_both_ops(monkeypatch, fused):
    stub, pkg = _render(monkeypatch, fused, absgrad=True)
    v = pkg["viewspace_points_abs"]
    assert v.is_leaf and v.requires_grad and tuple(v.shape) == (4, 3) and float(v.abs().sum()) == 0
    pkg["render"].sum().backward()
    assert "absgrad_out" in stub.backward_calls[0][1]
    assert torch.equal(v.grad, stub_c.marked("absgrad", (4, 3)))
    assert float(pkg["viewspace_points"].grad[0, 0]) == stub_c.MARK["dL_dmeans2D"]
    assert ("raw" in stub.backward_calls[0][1]) == fused


@pytest.mark.parametrize("fused", [False, True])
def test_render_without_absgrad_is_unchanged(monkeypatch, fused):
    stub, pkg = _render(monkeypatch, fused)
    assert "viewspace_points_abs" not in pkg
    pkg["render"].sum().backward()
    kw = stub.backward_calls[0][1]
    assert "absgrad_out" not in kw
    assert set(kw) == {"prune_mask", "dL_dinvdepth", "dL_dalpha", "camera_grads", "antialiasing"} | ({"raw"} if fused else {"quant"})
    assert "means2D_abs" not in stub.forward_calls[0][1] and "absgrad_out" not in stub.forward_calls[0][1]


def test_absgrad_accumulates_over_backward_calls(monkeypatch):
    stub, pkg = _render(monkeypatch, absgrad=True)
    pkg["render"].sum().backward(retain_graph=True)
    pkg["render"].sum().backward()
    assert torch.equal(pkg["viewspace_points_abs"].grad, 2 * stub_c.marked("absgrad", (4, 3)))


@pytest.mark.parametrize("kw, msg", [(dict(variable_sh_bands=True), "variable-SH"), (dict(features=torch.zeros(4, 2)), "feature")])
def test_render_refuses_absgrad_without_a_form(monkeypatch, kw, msg):
    from gaussian_renderer import render
    stub = stub_c.StubC().install(monkeypatch)
    with pytest.raises(RuntimeError, match=msg):
        render(stub_c.camera(), stub_c.Model(), stub_c.pipe(), torch.zeros(3), absgrad=True, **kw)
    assert not stub.calls


# ---- the float64 restatement against the oracle ---------------------------------------------------------------------------------

_cache = {}


def _run(name):
    if name not in _cache:
        case = BE.build(name)
        aa = case.meta["aa"]
        o, o64, _ = BE.oracle(case, aa=aa)
        excl = BE.excluded(case, o)
        signed, ab = absgrad64.pair_sums(o, case.bg.numpy(), case.dL.numpy(), case.W, case.H)
        _cache[name] = case, o, o64, excl, signed, ab
    return _cache[name]


@pytest.mark.parametrize("name", BE.CASES + BE.AA_CASES)
def test_restatement_signed_sums_are_the_oracles_means2D(name):
    case, o, o64, excl, signed, ab = _run(name)
    ref = np.asarray(o64["dL_dmeans2D"], np.float64).reshape(-1, 3)[:, :2]
    vis = np.asarray(o["radii"]) > 0
    chk = vis & ~excl
    assert chk.sum() > 0
    err = np.abs(signed - ref).max(axis=1)
    row = np.maximum(np.abs(ref).max(axis=1), ab.max(axis=1))
    # agreement to ~1e-6 of the row (the oracle recovers T by division along the list, this by a product): a pair too many or
    # too few, or a wrong term, moves a row by orders of magnitude more
    bar = np.maximum(1e-5 * row, 1e-8 * np.abs(ref).max())
    assert (err[chk] <= bar[chk]).all(), (name, float((err[chk] / np.maximum(row[chk], 1e-30)).max()))
    # the absolute sums bound the signed ones and are zero exactly where nothing was visited
    assert (ab + 1e-12 * ab.max() >= np.abs(signed)).all()
    assert (ab[~vis] == 0).all()
