"""CPU: the contribution statistics' C entry point refuses each bad argument before any CUDA call, the Python layer refuses what the
pass does not take before the library is called, and the request reaches `_C.contributions` on every render() path (against the
stand-in `_C` of stub_c) while a call without it carries exactly the arguments it carries without the feature."""
import ctypes as C
import os
import re

import pytest
import torch

import stub_c
from gs_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_INVAL, E_RANGE = -1, -4


def test_symbols_and_workspace():
    L = lib.lib()
    header = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
    for s in ("gsb_contributions", "gsb_contributions_workspace_bytes"):
        assert s in lib.EXPORTED_SYMBOLS and re.search(rf"GSB_API \w+ {s}\(", header), s
        getattr(L, s)
    sizes = [L.gsb_contributions_workspace_bytes(P) for P in (0, 1, 1000, 10 ** 6)]
    assert all(s >= 8 * P for s, P in zip(sizes, (0, 1, 1000, 10 ** 6))) and sizes == sorted(sizes) and sizes[-1] > sizes[-2]


def _call(P=10, R=5, W=16, H=16, blobs=True, outs=True, ws=256, top=True):
    L = lib.lib()
    b = 256 if blobs else None
    o = 256 if outs else None
    return L.gsb_contributions(b, P, b, R, b, W, H, None, o, o, o, 256 if top else None, ws, None), L.gsb_last_error()


@pytest.mark.parametrize("kw, code, msg", [
    (dict(P=-1), E_INVAL, b"negative size"),
    (dict(R=-1), E_INVAL, b"negative size"),
    (dict(W=0), E_INVAL, b"image size"),
    (dict(H=-3), E_INVAL, b"image size"),
    (dict(W=1 << 14, H=1 << 14), E_RANGE, b"2^28"),
    (dict(W=(1 << 28), H=1), E_RANGE, b"2^28"),
    (dict(outs=False), E_INVAL, b"output is NULL"),
    (dict(top=False, P=0, R=0, blobs=False, outs=False), E_INVAL, b"output is NULL"),
    (dict(blobs=False), E_INVAL, b"blob is NULL"),
    (dict(blobs=False, P=0), E_INVAL, b"blob is NULL"),
    (dict(ws=None), E_INVAL, b"workspace"),
    (dict(ws=260), E_INVAL, b"workspace"),
])
def test_refusals(kw, code, msg):
    st, err = _call(**kw)
    assert st == code and msg in err and err.startswith(b"contributions: "), (st, err)


def test_pixel_count_limit():
    # 2^28 - 1 pixels pass the range check: the call goes on to the next one (a NULL top_id here), nothing runs
    st, err = _call(W=(1 << 28) - 1, H=1, top=False)
    assert st == E_INVAL and b"output is NULL" in err
    st, err = _call(W=(1 << 27), H=2, top=False)
    assert st == E_RANGE


# ---- the Python layer ---------------------------------------------------------------------------------------------------------

@pytest.fixture
def no_library(monkeypatch):
    """The library must not be reached: any use of it fails the test."""
    def fail():
        raise AssertionError("the library was called")
    monkeypatch.setattr(lib, "lib", fail)


def test_C_refusals_leave_the_library_uncalled(no_library):
    from diff_gaussian_rasterization import _C
    blob = torch.zeros(8, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA device"):
        _C.contributions(blob, blob, blob, 1, 16, 8, 4)
    cuda0 = torch.device("cuda", 0)
    for bad, match in ((torch.zeros(8, 16, dtype=torch.float64), "float32"), (torch.zeros(16, 8).t(), "contiguous"),
                       (torch.zeros(8, 15), "shape"), (torch.zeros(2, 8, 16), "shape"), (torch.zeros(8, 16), "live on cuda:0"),
                       ("map", "tensor")):
        with pytest.raises(RuntimeError, match=match):
            _C.check_pixel_weights(bad, 8, 16, cuda0)
    with pytest.raises(RuntimeError, match="CUDA device"):
        _C.check_pixel_weights(torch.zeros(8, 16), 8, 16)
    _C.check_pixel_weights(torch.zeros(1, 8, 16), 8, 16, torch.device("cpu"))


class _Recorder:
    """Stands in for _C.contributions: records each call and returns a Contributions of marked tensors."""

    def __init__(self):
        self.calls = []

    def __call__(self, *args, **kw):
        from diff_gaussian_rasterization import _C
        self.calls.append((args, kw))
        P, H, W = args[6], args[5], args[4]
        self.result = _C.Contributions(torch.full((P,), 0.5), torch.full((P,), 0.25), torch.full((P,), 3, dtype=torch.int32),
                                       torch.full((H, W), 7, dtype=torch.int32))
        return self.result


def _install(monkeypatch):
    import diff_gaussian_rasterization as dgr
    stub = stub_c.StubC().install(monkeypatch)
    rec = _Recorder()
    monkeypatch.setattr(dgr._C, "contributions", rec)
    monkeypatch.setattr(dgr._C, "check_filter_3d", lambda f, P: None)
    return stub, rec


PATHS = ["dense", "quant", "pruned", "fused", "aa", "filter_3D", "maps", "features", "variable_sh"]


def _render(path, **kw):
    from types import SimpleNamespace
    from gaussian_renderer import render
    pc = stub_c.Model(4, C=3)
    pipe = stub_c.pipe(**({"fused_activations": True} if path == "fused" else {"antialiasing": True} if path == "aa" else {}))
    if path == "quant":
        pc.quant = SimpleNamespace()
    if path == "pruned":
        pc.prune_mask = torch.tensor([0, 1, 0, 0], dtype=torch.bool)
    if path == "filter_3D":
        pc.filter_3D = torch.rand(4, 1)
    extra = dict(return_maps=path == "maps", features=torch.rand(4, 2) if path == "features" else None,
                 variable_sh_bands=path == "variable_sh")
    return render(stub_c.camera(8, 16), pc, pipe, torch.zeros(3), **extra, **kw)


@pytest.mark.parametrize("path", PATHS)
def test_the_request_reaches_the_call_on_every_path(monkeypatch, path):
    runs = {}
    for name, kw in (("without", {}), ("off", dict(contributions=False)), ("plain", dict(contributions=True)),
                     ("map", dict(contributions=True, pixel_weights=torch.rand(8, 16)))):
        stub, rec = _install(monkeypatch)
        pkg = _render(path, **kw)
        if path != "variable_sh":
            pkg["render"].sum().backward()
        runs[name] = stub, rec, pkg, kw
    for name in ("without", "off"):
        stub, rec, pkg, _ = runs[name]
        assert not rec.calls and "contributions" not in pkg
    fwd = lambda s: s.variable_sh_calls if path == "variable_sh" else s.forward_calls
    base_stub = runs["without"][0]
    for name in ("off", "plain", "map"):
        stub, rec, pkg, kw = runs[name]
        # the rasterizer's own calls carry the arguments of a call without contributions
        (a0, k0), (a1, k1) = fwd(base_stub)[0], fwd(stub)[0]
        assert len(a0) == len(a1) and k0.keys() == k1.keys()
        if path != "variable_sh":
            assert base_stub.backward_calls[0][1].keys() == stub.backward_calls[0][1].keys()
        if name == "off":
            continue
        got = pkg["contributions"]
        assert len(rec.calls) == 1 and type(got) is type(rec.result) and all(torch.equal(a, b) for a, b in zip(got, rec.result))
        assert not any(t.requires_grad for t in got)
        args, ckw = rec.calls[0]
        out = stub._forward_outputs(a1, k1)
        assert args[3:] == (out[0], 16, 8, 4) and ckw["pixel_weights"] is kw.get("pixel_weights")


def test_the_op_takes_the_request_only_when_given(monkeypatch):
    import diff_gaussian_rasterization as dgr
    _install(monkeypatch)
    seen = []
    apply = dgr._RasterizeGaussians.apply
    monkeypatch.setattr(dgr._RasterizeGaussians, "apply", lambda *a: seen.append(len(a)) or apply(*a))
    _render("dense")
    _render("dense", contributions=True)
    _render("features")
    _render("features", contributions=True)
    assert seen == [14, dgr.N_INPUTS, dgr.N_INPUTS - 1, dgr.N_INPUTS]


def test_weights_without_the_flag_are_refused(monkeypatch):
    import diff_gaussian_rasterization as dgr
    stub, rec = _install(monkeypatch)
    with pytest.raises(RuntimeError, match="needs contributions=True"):
        _render("dense", pixel_weights=torch.rand(8, 16))
    s = dgr.GaussianRasterizationSettings(8, 16, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)
    P = 4
    call = lambda **kw: dgr.GaussianRasterizer(s)(torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 1), shs=torch.zeros(P, 1, 3),
                                                  degrees=torch.zeros(P, 1, dtype=torch.int32), scales=torch.ones(P, 3),
                                                  rotations=torch.ones(P, 4), **kw)
    with pytest.raises(RuntimeError, match="needs contributions=True"):
        call(pixel_weights=torch.rand(8, 16))
    for bad, match in ((torch.rand(8, 16, dtype=torch.float64), "float32"), (torch.rand(16, 8).t(), "contiguous"), (torch.rand(16, 8), "shape")):
        with pytest.raises(RuntimeError, match=match):
            call(contributions=True, pixel_weights=bad)
        with pytest.raises(RuntimeError, match=match):
            _render("fused", contributions=True, pixel_weights=bad)
    assert stub.calls == 0 and not rec.calls
    out = call(contributions=True)
    assert len(out) == 3 and isinstance(out[-1], dgr._C.Contributions) and len(rec.calls) == 1
