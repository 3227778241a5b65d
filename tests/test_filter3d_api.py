"""Mip-Splatting's 3D smoothing filter (DESIGN.md §5o) without a GPU: the ABI mirror and the request refusals in their documented
order, the plumbing from render() to `_C` (through tests/stub_c.py), the densify / MCMC row carry of filter_3D, and the float64
restatement of compute_3D_filter against Mip-Splatting's fp32 torch loop."""
import ctypes as C
import math
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import densify_golden as dg  # noqa: E402
import filter3d_restatement as F3  # noqa: E402
import stub_c  # noqa: E402
from gs_b200 import densify, mcmc  # noqa: E402
from gs_b200 import lib as gsl  # noqa: E402

HEADER = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
E = -1


# ------------------------------------------------------------------------------------------------ the ABI
def test_abi_mirror():
    L = gsl.lib()
    for s in ("gsb_filter_3d", "gsb_filter_3d_workspace_bytes"):
        assert s in gsl.EXPORTED_SYMBOLS and re.search(rf"GSB_API \w+ {s}\(", HEADER), s
        getattr(L, s)
    S = gsl.GsbScene
    assert S.filter_3D.offset == S.prune_mask.offset + 8 and S.quant.offset == S.filter_3D.offset + 8
    assert C.sizeof(S) == S.quant.offset + 8
    # the requests do not grow
    assert C.sizeof(gsl.GsbForwardRequest) == 22 * 8 and C.sizeof(gsl.GsbBackwardRequest) == 24 * 8
    assert L.gsb_filter_3d_workspace_bytes() >= 8


def test_filter_3d_refusals():
    L = gsl.lib()
    fake = C.c_void_p(256)

    def call(P=10, xyz=fake, n=3, views=fake, focals=fake, sizes=fake, out=fake, ws=fake):
        return L.gsb_filter_3d(P, xyz, n, views, focals, sizes, out, ws, None)
    assert call(P=-1) == E and b"filter_3d" in L.gsb_last_error()
    assert call(P=1 << 30) == E
    assert call(n=-1) == E
    for bad in (dict(xyz=None), dict(out=None), dict(ws=None), dict(views=None), dict(focals=None), dict(sizes=None)):
        assert call(**bad) == E, bad
    assert call(P=0, xyz=None, out=None) == 0                  # nothing to do, nothing launched


def _requests(P=5):
    """A forward / backward request whose every check passes up to the scene's tensors (fake device pointers: nothing runs)."""
    cb = gsl.ALLOC_FN(lambda user, n: 0)
    fake = 256
    scene = gsl.GsbScene(P=P, M=1, means3D=fake, opacities=fake, scales=fake, rotations=fake, shs=fake, degrees=fake, scale_modifier=1.0,
                         filter_3D=fake)
    m = (C.c_float * 16)()
    cam = gsl.GsbCamera(16, 16, 1.0, 1.0, fake, fake, fake, fake, 0)
    R = C.c_int64(0)
    keep = [cb, scene, cam, R, m]
    fwd = gsl.GsbForwardRequest(scene=C.pointer(scene), cam=C.pointer(cam), geom_alloc=cb, binning_alloc=cb, image_alloc=cb,
                                out_color=fake, radii=fake, num_rendered=C.pointer(R))
    bwd = gsl.GsbBackwardRequest(scene=C.pointer(scene), cam=C.pointer(cam))
    return scene, fwd, bwd, keep


def test_request_refusals_in_order():
    L = gsl.lib()
    scene, fwd, bwd, keep = _requests()
    # forward step 4: statistics with a filter (the SH-culling statistics keep the reference's definition)
    fwd.touched_pixels = fwd.transmittance_sum = 256
    assert L.gsb_forward(C.byref(fwd)) == E
    assert b"filter_3D" in L.gsb_last_error() and L.gsb_last_error().startswith(b"forward: statistics")
    # ... after the statistics' own earlier refusal (one output without the other)
    fwd.transmittance_sum = None
    assert L.gsb_forward(C.byref(fwd)) == E and b"statistics output" in L.gsb_last_error()
    fwd.touched_pixels = None
    # step 7: a filter with cov3D_precomp, after the exactly-one-of check
    scene.scales = scene.rotations = None
    scene.cov3D_precomp = 256
    assert L.gsb_forward(C.byref(fwd)) == E and b"filter_3D" in L.gsb_last_error() and b"cov3D_precomp" in L.gsb_last_error()
    scene.scales = scene.rotations = 256
    assert L.gsb_forward(C.byref(fwd)) == E and b"exactly one" in L.gsb_last_error()
    scene.scales = scene.rotations = None
    bwd.grads = None
    assert L.gsb_backward(C.byref(bwd)) == E
    assert L.gsb_last_error().startswith(b"backward: ") and b"filter_3D" in L.gsb_last_error()


# ------------------------------------------------------------------------------------------------ the plumbing
def _render(monkeypatch, pc, **kw):
    import gaussian_renderer
    from diff_gaussian_rasterization import _C
    stub = stub_c.StubC().install(monkeypatch)
    monkeypatch.setattr(_C, "check_filter_3d", lambda f, P: None)
    pipe = stub_c.pipe(**kw.pop("pipe", {}))
    out = gaussian_renderer.render(stub_c.camera(), pc, pipe, torch.zeros(3), **kw)
    return stub, out


@pytest.mark.parametrize("mode", ["activated", "fused", "aa", "variable_sh"])
def test_filter_reaches_C_only_when_the_model_has_one(monkeypatch, mode):
    pipe = dict(fused_activations=True) if mode == "fused" else dict(antialiasing=True) if mode == "aa" else {}
    kw = dict(variable_sh_bands=True) if mode == "variable_sh" else {}
    stubs = []
    pc = None
    for with_filter in (False, True):
        pc = stub_c.Model()
        if with_filter:
            pc.filter_3D = torch.rand(4, 1)
        stub, out = _render(monkeypatch, pc, pipe=pipe, **kw)
        if mode != "variable_sh":
            out["render"].sum().backward()
        stubs.append(stub)
    stub0, stub1 = stubs
    calls0 = stub0.variable_sh_calls if mode == "variable_sh" else stub0.forward_calls
    calls1 = stub1.variable_sh_calls if mode == "variable_sh" else stub1.forward_calls
    (a0, k0), (a1, k1) = calls0[0], calls1[0]
    assert "filter_3D" not in k0 and k1["filter_3D"] is pc.filter_3D
    assert {k: v for k, v in k1.items() if k != "filter_3D"}.keys() == k0.keys() and len(a0) == len(a1)
    if mode == "variable_sh":
        return
    (b0, kb0), (b1, kb1) = stub0.backward_calls[0], stub1.backward_calls[0]
    assert "filter_3D" not in kb0 and "opacity" not in kb0 and len(b0) == len(b1)
    assert kb1["filter_3D"] is pc.filter_3D and kb1["opacity"] is pc._opacity
    assert pc.filter_3D.grad is None


def test_render_refuses_filter_with_python_covariance(monkeypatch):
    pc = stub_c.Model()
    pc.filter_3D = torch.rand(4, 1)
    with pytest.raises(RuntimeError, match="compute_cov3D_python"):
        _render(monkeypatch, pc, pipe=dict(compute_cov3D_python=True))


def test_C_checks_the_filter_before_anything_runs():
    from diff_gaussian_rasterization import _C
    for bad, match in ((torch.zeros(4, 2), "shape"), (torch.zeros(5), "shape"), (torch.zeros(4, dtype=torch.float64), "float32"),
                       (torch.zeros(4), "CUDA"), ([0.0] * 4, "tensor")):
        with pytest.raises(RuntimeError, match=match):
            _C.check_filter_3d(bad, 4)


# ------------------------------------------------------------------------------------------------ the row carry
class _McmcStub:
    def __init__(self):
        self.calls = []

    def gsb_mcmc_workspace_bytes(self, P):
        return 64

    def gsb_mcmc_plan(self, *a):
        if a[7] is None:
            (C.c_int64 * 4).from_address(a[9])[:] = [7, 1 << 40, 0, 0]
        return 0

    def gsb_mcmc_emit(self, table, n_tensors, P, mode, n, ws, stream):
        self.calls.append([(table[i].src, table[i].dst, table[i].kind, table[i].row_width) for i in range(n_tensors)])
        return 0


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(gsl, "on_device", lambda dev: __import__("contextlib").nullcontext())
    monkeypatch.setattr(gsl, "current_stream", lambda dev: 0)

    def install(stub):
        monkeypatch.setattr(gsl, "lib", lambda: stub)
        return stub
    return install


@pytest.mark.parametrize("shape", [(300, 1), (300,)])
@pytest.mark.parametrize("stat_kind", [None, gsl.DENSIFY_COPY, gsl.MCMC_FRESH])
def test_resized_carries_the_filter_as_a_copy(stubbed, shape, stat_kind):
    m = dg.make_model(dg.load("dp_none"), "cpu")
    m.filter_3D = torch.rand(shape)
    groups, P, dev = densify._validate(m, False)
    entries, install = densify._resized(m, groups, 321, dev, {}, stat_kind)
    mine = [e for e in entries if e.src == m.filter_3D.data_ptr()]
    assert len(mine) == 1 and mine[0].kind == gsl.DENSIFY_COPY and mine[0].row_width == 1 and not mine[0].exp_avg_src
    install()
    assert tuple(m.filter_3D.shape) == (321,) + shape[1:] and m.filter_3D.data_ptr() == mine[0].dst


def test_models_without_a_filter_emit_the_same_table(stubbed):
    m = dg.make_model(dg.load("dp_none"), "cpu")
    groups, P, dev = densify._validate(m, False)
    n0 = len(densify._resized(m, groups, 321, dev, {}, gsl.DENSIFY_COPY)[0])
    m.filter_3D = torch.rand(P, 1)
    assert len(densify._resized(m, groups, 321, dev, {}, gsl.DENSIFY_COPY)[0]) == n0 + 1


def test_validate_refuses_a_stale_filter(stubbed):
    m = dg.make_model(dg.load("dp_none"), "cpu")
    m.filter_3D = torch.rand(299, 1)
    with pytest.raises(RuntimeError, match="filter_3D"):
        densify._validate(m, False)


def test_mcmc_carries_the_filter(stubbed, monkeypatch):
    stub = stubbed(_McmcStub())
    m = dg.make_model(dg.load("dp_none"), "cpu")
    m.filter_3D = torch.rand(300, 1)
    f = m.filter_3D
    mcmc.relocate_gs(m)
    (table,) = stub.calls
    assert (f.data_ptr(), f.data_ptr(), gsl.DENSIFY_COPY, 1) in table             # in place, the dead row takes its source's
    assert m.filter_3D is f
    n = mcmc.add_new_gs(m, 1000)
    table = stub.calls[-1]
    assert any(s == f.data_ptr() and k == gsl.DENSIFY_COPY for s, _, k, _ in table)
    assert tuple(m.filter_3D.shape) == (300 + n, 1)


# ------------------------------------------------------------------------------------------------ the restatement
def _cams(n, g, W=64, H=48):
    cams = []
    for i in range(n):
        a = 2 * math.pi * i / n
        R = torch.tensor([[math.cos(a), 0, -math.sin(a)], [0, 1, 0], [math.sin(a), 0, math.cos(a)]], dtype=F3.F64)
        view = torch.eye(4, dtype=F3.F64)
        view[:3, :3] = R.T            # rows as the transposed world_view_transform holds them
        view[3, 2] = 4.0 + float(torch.rand(1, generator=g))
        w, h = W + 8 * (i % 3), H + 4 * (i % 2)
        cams.append(F3.camera(view.float(), w, h, 0.9 + 0.1 * (i % 4), 0.7 + 0.05 * (i % 3)))
    return cams


def test_fp64_restatement_against_the_torch_loop():
    g = torch.Generator().manual_seed(5)
    xyz = torch.randn(4000, 3, generator=g) * 2.5
    xyz[:50] = torch.tensor([0.0, 0.0, 100.0])                      # behind or beyond every camera's screen: unseen rows
    cams = _cams(12, g)
    f64, seen, _ = F3.filter_fp64(xyz, cams)
    f32 = F3.filter_torch_fp32(xyz, cams)
    assert 0 < int(seen.sum()) < xyz.shape[0]
    near = F3.boundary_ulps(xyz, cams) < 64
    rel = ((f32.double() - f64).abs() / f64).numpy()
    assert rel[~near.numpy()].max() < 4e-7                          # the fp32 loop rounds a few times
    assert bool((f64[~seen] == f64[seen].max()).all())               # unseen rows take the largest seen distance
    assert torch.equal(F3.filter_torch_fp32(xyz, []), torch.zeros(xyz.shape[0]))


def test_filtered_scales_restatement():
    s = torch.tensor([[0.1, 0.2, 0.0], [1e-6, 0.5, 0.5], [0.3, 0.3, 0.3]])
    f = torch.tensor([0.05, 0.0, 0.3])
    sp, c3 = F3.filtered(s, f)
    assert torch.equal(sp[1], s[1]) and float(c3[1]) == 1.0                 # zero filter: unchanged
    assert float(c3[0]) == 0.0 and bool(torch.isfinite(sp).all())          # an exactly flat axis: c3 = 0
    sp64, c364 = F3.filtered64(s.double(), f.double())
    assert torch.allclose(sp64[[0, 2]].float(), sp[[0, 2]]) and abs(float(c364[2]) - 0.5 ** 1.5) < 1e-12
