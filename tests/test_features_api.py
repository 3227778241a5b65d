"""CPU: the feature-channel requests (the `features` field of GsbForwardRequest / GsbBackwardRequest) reject each bad argument before
any CUDA call, with gsb_last_error() set, and the Python layer refuses what the feature pass does not take (CPU tensors, a shape other than
[P, F], F out of range, accumulate_into, a feature gradient under the deterministic mode) before anything runs."""
import ctypes as C
import os
import re

import pytest
import torch

import stub_c
from gs_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbols_struct_and_limit():
    L = lib.lib()
    for sym in ("gsb_forward", "gsb_backward"):
        assert sym in lib.EXPORTED_SYMBOLS
        getattr(L, sym)
    assert C.sizeof(lib.GsbFeatures) == 8 + 4 * 8 and lib.GsbFeatures.features.offset == 8
    header = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
    assert int(re.search(r"#define GSB_FEATURES_MAX (\d+)", header).group(1)) == lib.FEATURES_MAX == 256


def _fwd(L, feats, P=10, W=16, H=16):
    buf = (C.c_float * 64)()
    b = C.addressof(buf)
    scene = lib.GsbScene(P=P, means3D=b, opacities=b, degrees=b)
    cam = lib.GsbCamera(width=W, height=H, viewmatrix=b, projmatrix=b, campos=b, background=b)
    req = lib.GsbForwardRequest(scene=C.pointer(scene), cam=C.pointer(cam), out_color=b, radii=b, num_rendered=C.pointer(C.c_int64(0)),
                                features=C.pointer(feats))
    return L.gsb_forward(C.byref(req))


def test_forward_features_rejects_bad_arguments():
    L = lib.lib()
    fbuf = (C.c_float * 16)()
    p = C.addressof(fbuf)
    cases = [
        (lib.GsbFeatures(0, p, p, None, None), {}, b"F = 0"),
        (lib.GsbFeatures(257, p, p, None, None), {}, b"F = 257"),
        (lib.GsbFeatures(-3, p, p, None, None), {}, b"F = -3"),
        (lib.GsbFeatures(4, None, p, None, None), {}, b"features->features is NULL"),
        (lib.GsbFeatures(4, p, None, None, None), {}, b"out is NULL"),
        (lib.GsbFeatures(4, p, p, None, None), dict(P=-1), b"P < 0"),
        (lib.GsbFeatures(4, p, p, None, None), dict(W=0), b"image size"),
        # with P == 0 the features themselves may be NULL: the request goes on to the scene's checks (a camera without tensors)
        (lib.GsbFeatures(4, None, p, None, None), dict(P=0, W=0), b"image size"),
    ]
    for feats, kw, msg in cases:
        assert _fwd(L, feats, **kw) == -1, msg
        assert msg in L.gsb_last_error(), (msg, L.gsb_last_error())


def _bwd(L, scene, feats, R=5, det_ws=None, raw=None, raw_grads=None):
    req = lib.GsbBackwardRequest(scene=scene, cam=C.pointer(lib.GsbCamera()), num_rendered=R, grads=C.pointer(lib.GsbGrads()), raw=raw,
                                 raw_grads=raw_grads, deterministic=int(det_ws is not None), det_workspace=det_ws,
                                 features=None if feats is None else C.pointer(feats))
    return L.gsb_backward(C.byref(req))


def test_backward_features_rejects_bad_arguments():
    L = lib.lib()
    fbuf = (C.c_float * 16)()
    p = C.addressof(fbuf)
    ok = lib.GsbFeatures(4, p, None, p, p)
    scene = C.pointer(lib.GsbScene(P=10))
    for sc in (None, C.pointer(lib.GsbScene(P=-1))):
        assert _bwd(L, sc, ok) == -1 and b"P < 0" in L.gsb_last_error()
    buf = (C.c_char * 256)()
    assert _bwd(L, scene, ok, det_ws=C.addressof(buf)) == -1 and b"no deterministic form" in L.gsb_last_error()
    for feats, msg in ((lib.GsbFeatures(0, p, None, p, p), b"F = 0"), (lib.GsbFeatures(300, p, None, p, p), b"F = 300"),
                       (lib.GsbFeatures(4, None, None, p, p), b"features->features is NULL"),
                       (lib.GsbFeatures(4, p, None, None, p), b"dL_dout / dL_dfeatures is NULL"),
                       (lib.GsbFeatures(4, p, None, p, None), b"dL_dout / dL_dfeatures is NULL")):
        assert _bwd(L, scene, feats) == -1, msg
        assert msg in L.gsb_last_error(), (msg, L.gsb_last_error())
    assert _bwd(L, scene, ok, R=-1) == -1 and b"num_rendered < 0" in L.gsb_last_error()
    assert _bwd(L, scene, ok, raw_grads=C.pointer(lib.GsbRawGrads())) == -1 and b"raw_grads given without raw" in L.gsb_last_error()
    assert _bwd(L, scene, ok, raw=C.pointer(lib.GsbRawParams(C=4)), raw_grads=C.pointer(lib.GsbRawGrads())) == -1
    assert b"C = 4" in L.gsb_last_error()
    # valid feature arguments go on to the scene checks of the backward (an empty camera is refused there)
    assert _bwd(L, scene, ok) == -1 and b"image size" in L.gsb_last_error()
    # without features it is the deterministic backward (with det_workspace) or the plain backward
    assert _bwd(L, scene, None, det_ws=None, R=1 << 30) == -1 and b"image size" in L.gsb_last_error()
    assert _bwd(L, scene, None, det_ws=C.addressof(buf), R=1 << 30) == -4 and b"2^30" in L.gsb_last_error()


def _render(features, deterministic=None):
    from gaussian_renderer import render
    return render(stub_c.camera(16, 16), stub_c.Model(), stub_c.pipe(), torch.zeros(3), features=features)


@pytest.fixture
def torch_deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.mark.parametrize("features, msg", [
    (torch.zeros(4, 8), "CUDA device"),
    (torch.zeros(5, 8), r"shape \[P, F\]"),
    (torch.zeros(4, 8, 1), r"shape \[P, F\]"),
    (torch.zeros(4), r"shape \[P, F\]"),
    (torch.zeros(4, 0), "F = 0"),
    (torch.zeros(4, 257), "F = 257"),
    (torch.zeros(4, 8, dtype=torch.float64), "float32"),
    ("not a tensor", "tensor"),
])
def test_render_refuses_bad_features(features, msg, torch_deterministic):
    torch.use_deterministic_algorithms(False)
    with pytest.raises(RuntimeError, match=msg):
        _render(features)


def test_render_refuses_a_deterministic_feature_gradient(torch_deterministic):
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match="deterministic"):
        _render(torch.zeros(4, 8, requires_grad=True))
    # without a gradient the features are only refused for living on the CPU
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match="CUDA device"):
        _render(torch.zeros(4, 8))


def test_settings_deterministic_refuses_a_feature_gradient(torch_deterministic):
    import diff_gaussian_rasterization as dgr
    torch.use_deterministic_algorithms(False)
    s = dgr.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False,
                                          deterministic=True)
    P = 4
    with pytest.raises(RuntimeError, match="deterministic"):
        dgr.GaussianRasterizer(s)(torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 1), shs=torch.zeros(P, 1, 3),
                                  degrees=torch.zeros(P, 1, dtype=torch.int32), scales=torch.ones(P, 3), rotations=torch.ones(P, 4),
                                  features=torch.zeros(P, 3, requires_grad=True))


def _backward_call(**kw):
    from diff_gaussian_rasterization import _C
    P, H, W = 4, 16, 16
    z = torch.zeros(P, 3)
    return _C.rasterize_gaussians_backward(torch.zeros(3), z, torch.ones(P, dtype=torch.int32), torch.empty(0), z, torch.zeros(P, 4), 1.0,
                                           torch.empty(0), torch.eye(4), torch.eye(4), 1.0, 1.0, torch.zeros(3, H, W), torch.zeros(P, 1, 3),
                                           torch.zeros(P, 1, dtype=torch.int32), torch.zeros(3), torch.empty(0), 0, torch.empty(0),
                                           torch.empty(0), 0.0, False, features=torch.zeros(P, 5), dL_dfeatures_out=torch.zeros(5, H, W),
                                           **kw)


def test_backward_refuses_accumulate_into_and_deterministic():
    with pytest.raises(RuntimeError, match="accumulate_into"):
        _backward_call(accumulate_into=tuple(torch.zeros(1) for _ in range(8)))
    with pytest.raises(RuntimeError, match="deterministic"):
        _backward_call(deterministic=True)
    with pytest.raises(RuntimeError, match="CUDA device"):
        _backward_call()
