"""CPU: rendering from the model's raw parameters (`pipe.fused_activations`, the `raw` / `raw_grads` fields of the
rasterizer requests, DESIGN.md §5h): the struct layouts, the GSB_EINVAL cases of the C calls (all raised before any CUDA call), every refusal of the
Python layers (raised before anything runs, parameters untouched), and, against a stub of `_C`, that render() hands the
parameters' own storage to the rasterizer, that the flag reaches the backward, and that the `.grad` tensors are the rasterizer's
own outputs with no Cat / Exp / Div node in the graph."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest
import torch

import stub_c
from gs_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_raw_symbols_are_exported():
    L = lib.lib()
    for sym in ("gsb_forward", "gsb_backward"):
        assert sym in lib.EXPORTED_SYMBOLS
        getattr(L, sym)
    assert lib.GsbForwardRequest.raw.size == lib.GsbBackwardRequest.raw.size == lib.GsbBackwardRequest.raw_grads.size == 8


def test_raw_struct_layouts_match_header():
    assert C.sizeof(lib.GsbRawParams) == 40
    assert [getattr(lib.GsbRawParams, f).offset for f in ("features_dc", "features_rest", "C", "scaling", "rotation")] == [0, 8, 16, 24, 32]
    assert C.sizeof(lib.GsbRawGrads) == 32
    assert [getattr(lib.GsbRawGrads, f).offset for f in ("dL_dfeatures_dc", "dL_dfeatures_rest", "dL_dscaling", "dL_drotation")] == \
        [0, 8, 16, 24]
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler to read the header's own offsets")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "gs_b200.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu %zu\\n",'
           'sizeof(GsbRawParams), offsetof(GsbRawParams, C), offsetof(GsbRawParams, scaling), offsetof(GsbRawParams, rotation),'
           'sizeof(GsbRawGrads), offsetof(GsbRawGrads, dL_dscaling), offsetof(GsbRawGrads, dL_drotation)); return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")], check=True)
        got = subprocess.run([os.path.join(d, "t")], check=True, capture_output=True, text=True).stdout.split()
    assert [int(v) for v in got] == [40, 16, 24, 32, 32, 16, 24]


# ---- GSB_EINVAL: nothing below is dereferenced, the checks come before any CUDA call ------------------------------------------

_BUF = (C.c_float * 64)()
_A = C.addressof(_BUF)


def _scene(P=10, **kw):
    s = lib.GsbScene(P=P)
    s.means3D = s.opacities = _A
    s.degrees = _A
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def _raw(Cn=15, dc=_A, rest=_A, scaling=_A, rotation=_A):
    return lib.GsbRawParams(dc, rest if Cn else None, Cn, scaling, rotation)


def _fwd(scene, raw, invdepth=None, alpha=None):
    req = lib.GsbForwardRequest(scene=C.pointer(scene) if scene is not None else None, cam=C.pointer(lib.GsbCamera()),
                                num_rendered=C.pointer(C.c_int64(0)), out_invdepth=invdepth, out_alpha=alpha, raw=C.pointer(raw))
    return lib.lib().gsb_forward(C.byref(req))


def _bwd(scene, raw, grads=None, raw_grads=None):
    g = grads if grads is not None else lib.GsbGrads()
    rg = raw_grads if raw_grads is not None else lib.GsbRawGrads(_A, _A, _A, _A)
    req = lib.GsbBackwardRequest(scene=C.pointer(scene), cam=C.pointer(lib.GsbCamera()), grads=C.pointer(g), raw=C.pointer(raw),
                                 raw_grads=C.pointer(rg))
    return lib.lib().gsb_backward(C.byref(req))


@pytest.mark.parametrize("case, msg", [
    ("C5", b"C = 5"),
    ("scales_set", b"must be NULL"),
    ("shs_set", b"must be NULL"),
    ("cov3D_set", b"must be NULL"),
    ("quant_set", b"must be NULL"),
    ("packed", b"must be NULL"),
    ("no_scaling", b"scaling / rotation missing"),
    ("no_rotation", b"scaling / rotation missing"),
    ("no_dc", b"features_dc"),
    ("no_rest", b"features_rest"),
    ("rest_with_C0", b"features_rest"),
    ("sh_and_colors", b"colors_precomp"),
])
def test_raw_entry_points_refuse(case, msg):
    scene, raw = _scene(), _raw()
    if case == "C5":
        raw = _raw(Cn=5)
    elif case == "scales_set":
        scene.scales = _A
    elif case == "shs_set":
        scene.shs = _A
    elif case == "cov3D_set":
        scene.cov3D_precomp = _A
    elif case == "quant_set":
        q = lib.GsbQuant()
        scene.quant = C.pointer(q)
    elif case == "packed":
        scene.sh_packed = 1
    elif case == "no_scaling":
        raw.scaling = None
    elif case == "no_rotation":
        raw.rotation = None
    elif case == "no_dc":
        raw.features_dc = None
    elif case == "no_rest":
        raw.features_rest = None
    elif case == "rest_with_C0":
        raw = _raw(Cn=0)
        raw.features_rest = _A
    elif case == "sh_and_colors":
        scene.colors_precomp = _A
    L = lib.lib()
    assert _fwd(scene, raw) == -1 and msg in L.gsb_last_error()
    assert _bwd(scene, raw) == -1 and msg in L.gsb_last_error()


def test_raw_entry_points_refuse_bad_outputs():
    L = lib.lib()
    assert _fwd(None, _raw()) == -1 and b"P < 0" in L.gsb_last_error()
    assert _fwd(_scene(), _raw(), invdepth=_A) == -1 and b"both map outputs" in L.gsb_last_error()
    for field in ("dL_dsh", "dL_dscales", "dL_drotations"):
        g = lib.GsbGrads()
        setattr(g, field, _A)
        assert _bwd(_scene(), _raw(), grads=g) == -1 and b"must be NULL" in L.gsb_last_error()
    scene = _scene(colors_precomp=_A)
    raw = _raw(dc=None, rest=None)
    assert _bwd(scene, raw, raw_grads=lib.GsbRawGrads(_A, None, _A, _A)) == -1 and b"colors_precomp" in L.gsb_last_error()
    assert _bwd(_scene(), _raw(Cn=0), raw_grads=lib.GsbRawGrads(_A, _A, _A, _A)) == -1 and b"C == 0" in L.gsb_last_error()
    # P == 0 needs no tensor at all: the checks pass and the call reaches the scene / camera checks (here: an empty camera)
    assert _fwd(_scene(P=0), _raw(dc=None, rest=None, scaling=None, rotation=None)) == -1
    assert b"raw" not in L.gsb_last_error()


# ---- Python-side refusals -----------------------------------------------------------------------------------------------------

def _leaves(P=6, Cn=15, device="cpu"):
    g = torch.Generator().manual_seed(3)
    return (torch.randn(P, 1, 3, generator=g).to(device), torch.randn(P, Cn, 3, generator=g).to(device),
            torch.randn(P, 3, generator=g).to(device), torch.randn(P, 4, generator=g).to(device))


@pytest.mark.parametrize("case, msg", [
    ("f64", "float32"), ("noncontig", "contiguous"), ("C5", "C = 5"), ("P_differ", "rows"), ("dc_shape", "shape"),
    ("rot_shape", "shape"), ("list_rest", "packed"), ("cpu", "must live on"),
])
def test_raw_struct_refusals(case, msg):
    from diff_gaussian_rasterization import _C
    dc, rest, sc, rot = _leaves()
    if case == "f64":
        sc = sc.double()
    elif case == "noncontig":
        rot = torch.randn(4, 6).t()
    elif case == "C5":
        rest = torch.zeros(6, 5, 3)
    elif case == "P_differ":
        rest = torch.zeros(7, 15, 3)
    elif case == "dc_shape":
        dc = torch.zeros(6, 3)
    elif case == "rot_shape":
        rot = torch.zeros(6, 3)
    elif case == "list_rest":
        rest = [torch.zeros(3, 3, 3), torch.zeros(3, 8, 3)]
    with pytest.raises(RuntimeError, match=msg):
        _C._raw_struct((dc, rest, sc, rot), torch.device("cpu"), 6, True, None, None, None, None, None)


def test_raw_keyword_refuses_activated_inputs_and_cpu():
    from diff_gaussian_rasterization import _C
    dc, rest, sc, rot = _leaves()
    z = torch.zeros(6, 3)
    with pytest.raises(RuntimeError, match="replace"):
        _C._raw_struct((dc, rest, sc, rot), torch.device("cpu"), 6, True, torch.zeros(6, 16, 3), None, None, None, None)
    with pytest.raises(RuntimeError, match="quantised"):
        _C._raw_struct((dc, rest, sc, rot), torch.device("cpu"), 6, True, None, None, None, None, object())
    with pytest.raises(RuntimeError):              # CPU means3D: refused before anything else
        _C.rasterize_gaussians(torch.zeros(3), z, torch.empty(0), torch.zeros(6, 1), torch.empty(0), torch.empty(0), 1.0, torch.empty(0),
                               torch.eye(4), torch.eye(4), 1.0, 1.0, 8, 8, torch.empty(0), torch.zeros(6, 1, dtype=torch.int32),
                               torch.zeros(3), False, False, raw=(dc, rest, sc, rot))


@pytest.mark.parametrize("case, msg", [
    ("quant", "quantised"), ("cov3D_python", "compute_cov3D_python"), ("shs_python", "convert_SHs_python"),
    ("scaling_act", "scaling_activation"), ("rotation_act", "rotation_activation"), ("no_act", "scaling_activation"),
    ("packed", "packed"),
])
def test_render_refusals_leave_the_model_untouched(monkeypatch, case, msg):
    import diff_gaussian_rasterization as dgr
    import gaussian_renderer
    calls = []
    monkeypatch.setattr(dgr._C, "rasterize_gaussians", lambda *a, **k: calls.append(1))
    pc, pipe = stub_c.Model(6, C=15), stub_c.pipe(fused_activations=True)
    if case == "quant":
        pc.quant = object()
    elif case == "cov3D_python":
        pipe.compute_cov3D_python = True
    elif case == "shs_python":
        pipe.convert_SHs_python = True
    elif case == "scaling_act":
        pc.scaling_activation = torch.nn.functional.softplus
    elif case == "rotation_act":
        pc.rotation_activation = lambda q: q
    elif case == "no_act":
        del pc.scaling_activation
    elif case == "packed":
        pc._features_rest = [torch.zeros(3, 3, 3), torch.zeros(3, 8, 3)]
    before = [t.detach().clone() for t in pc.leaves() if isinstance(t, torch.Tensor)]
    with pytest.raises(RuntimeError, match=msg):
        gaussian_renderer.render(stub_c.camera(), pc, pipe, torch.zeros(3))
    after = [t for t in pc.leaves() if isinstance(t, torch.Tensor)]
    assert not calls
    assert all(torch.equal(a.detach(), b) and a.grad is None for a, b in zip(after, before))


# ---- plumbing against a stub _C ------------------------------------------------------------------------------------------------

def _graph_names(root):
    seen, stack, names = set(), [root], []
    while stack:
        fn = stack.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        names.append(type(fn).__name__)
        stack.extend(f for f, _ in fn.next_functions)
    return names


@pytest.mark.parametrize("Cn", [0, 3, 8, 15])
def test_render_passes_the_parameters_own_storage_and_grads(monkeypatch, Cn):
    import gaussian_renderer
    stub = stub_c.StubC().install(monkeypatch)
    pc = stub_c.Model(6, C=Cn)
    pkg = gaussian_renderer.render(stub_c.camera(), pc, stub_c.pipe(fused_activations=True, antialiasing=True), torch.zeros(3))
    args, f = stub.forward_calls[0]
    assert f["antialiasing"] is True
    assert [t.data_ptr() for t in f["raw"]] == [pc._features_dc.data_ptr(), pc._features_rest.data_ptr(), pc._scaling.data_ptr(),
                                               pc._rotation.data_ptr()]
    assert all(not (isinstance(t, torch.Tensor) and t.numel()) for t in (args[14], args[4], args[5]))     # sh, scales, rotations
    names = _graph_names(pkg["render"].grad_fn)
    assert not [n for n in names if any(k in n for k in ("Cat", "Exp", "Div", "Norm", "Clamp", "Expand"))], names
    assert names.count("AccumulateGrad") == 7                 # xyz, screen-space points, dc, rest, opacity, scaling, rotation
    pkg["render"].sum().backward()
    b = stub.backward_calls[0][1]
    assert [t.data_ptr() for t in b["raw"]] == [t.data_ptr() for t in (pc._features_dc, pc._features_rest, pc._scaling, pc._rotation)]
    assert b["antialiasing"] is True
    # the rasterizer's own outputs became .grad: no clone
    got = [pc._features_dc.grad, pc._features_rest.grad, pc._scaling.grad, pc._rotation.grad]
    out_ptrs = stub.backward_output_ptrs[0]
    assert [g.data_ptr() for g in got[:1] + got[2:]] == [out_ptrs[5], out_ptrs[7], out_ptrs[8]]
    assert all(g.is_contiguous() for g in got) and tuple(got[1].shape) == (6, Cn, 3)


def test_render_override_color_reads_no_sh(monkeypatch):
    import gaussian_renderer
    stub = stub_c.StubC().install(monkeypatch)
    pc = stub_c.Model(6, C=15)
    colors = torch.rand(6, 3, requires_grad=True)
    pkg = gaussian_renderer.render(stub_c.camera(), pc, stub_c.pipe(fused_activations=True), torch.zeros(3), override_color=colors)
    args, f = stub.forward_calls[0]
    assert f["raw"][:2] == (None, None) and args[2] is colors
    pkg["render"].sum().backward()
    assert stub.backward_calls[0][1]["raw"][:2] == (None, None)
    assert pc._features_dc.grad is None and pc._features_rest.grad is None
    assert colors.grad is not None and pc._scaling.grad is not None


def test_flag_off_changes_nothing(monkeypatch):
    import gaussian_renderer
    stub = stub_c.StubC().install(monkeypatch)
    pc = stub_c.Model(6, C=15)
    for pipe in (stub_c.pipe(fused_activations=False), stub_c.pipe()):
        gaussian_renderer.render(stub_c.camera(), pc, pipe, torch.zeros(3))
    assert [f.get("raw") for _, f in stub.forward_calls] == [None, None]
    assert all(tuple(args[14].shape) == (6, 16, 3) and args[4].numel() == 18 for args, _ in stub.forward_calls)
