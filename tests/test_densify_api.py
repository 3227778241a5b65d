"""gs_b200.densify without a GPU: the C ABI's symbols, layout and argument errors, the refusals (each leaving the model and the
optimizer as they were), the host arithmetic against a stub of the library, and the torch restatement of the reference's
semantics against the reference's own goldens (so that the GPU tests may compare the kernels with it)."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import densify_golden as dg  # noqa: E402
import densify_restatement as rs  # noqa: E402
from gs_b200 import densify  # noqa: E402
from gs_b200 import lib as gsl  # noqa: E402

HEADER = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
NEW = ["gsb_densify_stats", "gsb_densify_workspace_bytes", "gsb_densify_split_std_offset", "gsb_densify_plan", "gsb_densify_emit"]


def test_symbols_exported():
    L = gsl.lib()
    for s in NEW:
        assert s in gsl.EXPORTED_SYMBOLS
        getattr(L, s)
        assert re.search(rf"GSB_API \w+ {s}\(", HEADER), s


def test_table_layout_matches_header():
    body = re.search(r"typedef struct GsbDensifyTensor \{(.*?)\} GsbDensifyTensor;", HEADER, re.S).group(1)
    names = re.findall(r"(\w+);", body)
    assert names == [f[0] for f in gsl.GsbDensifyTensor._fields_]
    assert C.sizeof(gsl.GsbDensifyTensor) == 8 * 8 + 2 * 4
    for name, value in (("GSB_DENSIFY_MAX_TENSORS", gsl.DENSIFY_MAX_TENSORS), ("GSB_DENSIFY_COUNTS", gsl.DENSIFY_COUNTS),
                        ("GSB_DENSIFY_CLONE_SPLIT", gsl.DENSIFY_CLONE_SPLIT), ("GSB_DENSIFY_PRUNE", gsl.DENSIFY_PRUNE),
                        ("GSB_DENSIFY_PRUNE_MASK", gsl.DENSIFY_PRUNE_MASK), ("GSB_DENSIFY_COPY", gsl.DENSIFY_COPY),
                        ("GSB_DENSIFY_XYZ", gsl.DENSIFY_XYZ), ("GSB_DENSIFY_SCALING", gsl.DENSIFY_SCALING)):
        assert int(re.search(rf"#define {name} (\d+)", HEADER).group(1)) == value, name


def test_workspace_grows_with_P():
    L = gsl.lib()
    assert L.gsb_densify_workspace_bytes(0) > 0
    assert L.gsb_densify_workspace_bytes(1 << 20) >= 28 * (1 << 20)
    assert L.gsb_densify_split_std_offset(1000) + 12 * 1000 <= L.gsb_densify_workspace_bytes(1000)


def test_einval():
    L = gsl.lib()
    fake = C.c_void_p(256)
    E = -1
    stats = lambda P, grad, stride, vis, radii, accum, denom, max_radii2D: L.gsb_densify_stats(  # noqa: E731
        P, grad, stride, None, 0, vis, radii, accum, None, denom, max_radii2D, None)                # without the AbsGS pair
    assert stats(-1, None, 3, None, None, None, None, None) == E
    assert stats(10, fake, 1, fake, None, fake, fake, None) == E                                # stride < 2
    assert stats(10, None, 3, fake, None, fake, fake, None) == E                                # NULL grad
    assert stats(10, fake, 3, fake, fake, fake, fake, None) == E                                # radii without max_radii2D
    assert stats(0, None, 3, None, None, None, None, None) == 0
    plan = lambda P, mode, ws=fake, counts=fake, mask=None: L.gsb_densify_plan(  # noqa: E731
        P, mode, fake, None, fake, fake, fake, fake, mask, 0.0, 0.0, 1.0, 0.005, 0, 0.0, 10.0, 0.625, ws, counts, None)
    assert plan(-1, 0) == E
    assert plan(1 << 30, 0) == E
    assert plan(10, 3) == E
    assert plan(10, 0, ws=None) == E
    assert plan(10, 0, counts=None) == E
    assert plan(10, 2) == E                                                                     # mask mode without a mask
    e = gsl.GsbDensifyTensor(src=256, dst=256, row_width=3, kind=0)
    emit = lambda tab, n, P=10, ws=fake, k=(5, 0, 0, 0): L.gsb_densify_emit(  # noqa: E731
        tab, n, P, ws, *k, fake, fake, 0.625, None)
    assert emit(None, 1) == E
    assert emit((gsl.GsbDensifyTensor * 1)(e), 17) == E
    assert emit((gsl.GsbDensifyTensor * 1)(e), 1, P=-1) == E
    assert emit((gsl.GsbDensifyTensor * 1)(e), 1, ws=None) == E
    assert emit((gsl.GsbDensifyTensor * 1)(e), 1, k=(-1, 0, 0, 0)) == E
    assert emit((gsl.GsbDensifyTensor * 1)(e), 1, k=(5, 0, 1, 2)) == E                        # more kept children than splits
    for bad in (dict(row_width=0), dict(kind=3), dict(kind=1, row_width=4), dict(exp_avg_src=256), dict(grad_dst=256),
                dict(src=258), dict(src=None)):
        f = gsl.GsbDensifyTensor(src=256, dst=256, row_width=3, kind=0)
        for k, v in bad.items():
            setattr(f, k, v)
        assert emit((gsl.GsbDensifyTensor * 1)(f), 1) == E, bad
    x = gsl.GsbDensifyTensor(src=256, dst=256, row_width=3, kind=1)
    assert L.gsb_densify_emit((gsl.GsbDensifyTensor * 1)(x), 1, 10, fake, 5, 0, 2, 1, None, fake, 0.625, None) == E   # no rotation
    assert emit((gsl.GsbDensifyTensor * 1)(e), 0) == 0


# ------------------------------------------------------------------------------------------------ refusals
def _model(name="dp_none"):
    return dg.make_model(dg.load(name), "cpu")


def _fingerprint(m):
    groups = [(g["name"], g["params"][0]) for g in m.optimizer.param_groups]
    state = {id(p): (id(m.optimizer.state[p]), {k: id(v) for k, v in m.optimizer.state[p].items()}) for _, p in groups if p in m.optimizer.state}
    return [(n, id(p)) for n, p in groups], state, {k: id(v) for k, v in vars(m).items()}


class _FakeCuda:
    """Makes _validate see CUDA tensors so that the refusal under test is the one that fires (no GPU here)."""

    def __init__(self, monkeypatch):
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def _refused(m, fn, match):
    before = _fingerprint(m)
    with pytest.raises(RuntimeError, match=match):
        fn(m)
    assert _fingerprint(m) == before


def test_refuses_cpu_tensors():
    _refused(_model(), lambda m: densify.densify_and_prune(m, 0.0002, 0.005, 100.0, None, {}), "CUDA")
    _refused(_model(), lambda m: densify.prune_points(m, torch.zeros(300, dtype=torch.bool)), "CUDA")


@pytest.mark.parametrize("case", ["dtype", "contiguous", "list_f_rest", "quantised", "extra_group", "optimizer", "degrees",
                                  "stats", "store_grads_missing"])
def test_refusals_leave_model_untouched(monkeypatch, case):
    _FakeCuda(monkeypatch)
    m = _model()
    match = "densify"
    if case == "dtype":
        m.optimizer.param_groups[3]["params"][0] = torch.nn.Parameter(m._opacity.detach().double())
    elif case == "contiguous":
        m.optimizer.param_groups[0]["params"][0] = torch.nn.Parameter(m._xyz.detach().t().contiguous().t())
    elif case == "list_f_rest":
        m._features_rest = [m._features_rest]
        match = "variable-SH"
    elif case == "quantised":
        m._codebook_dict = {"opacity": None}
        match = "quantised"
    elif case == "extra_group":
        m.optimizer.add_param_group({"params": [torch.nn.Parameter(torch.zeros(300, 2))], "name": "extra"})
        match = "groups"
    elif case == "optimizer":
        m.optimizer = torch.optim.SGD(m.optimizer.param_groups, lr=0.1)
        match = "Adam"
    elif case == "degrees":
        m._degrees = m._degrees.long()
        match = "_degrees"
    elif case == "stats":
        m.denom = m.denom[:-1]
        match = "denom"
    elif case == "store_grads_missing":
        _refused(m, lambda m: densify.densify_and_prune(m, 0.0002, 0.005, 100.0, None, {}, store_grads=True), "store_grads")
        return
    _refused(m, lambda m: densify.densify_and_prune(m, 0.0002, 0.005, 100.0, None, {}), match)


@pytest.mark.parametrize("mask", [torch.zeros(299, dtype=torch.bool), torch.zeros(300, dtype=torch.uint8), [False] * 300])
def test_refuses_bad_mask(monkeypatch, mask):
    _FakeCuda(monkeypatch)
    _refused(_model(), lambda m: densify.prune_points(m, mask), "mask")


# ------------------------------------------------------------------------------------------------ host logic against a stub library
class _Stub:
    """Records the plan's arguments, "computes" a plan that keeps every row, and copies rows on the CPU in emit."""

    def __init__(self, P):
        self.P, self.plan_args, self.table = P, None, None

    def gsb_densify_workspace_bytes(self, P):
        return 64

    def gsb_densify_split_std_offset(self, P):
        return 0

    def gsb_densify_plan(self, *a):
        self.plan_args = a
        counts = (C.c_int64 * 8).from_address(a[-2])
        counts[:] = [self.P, 0, 0, 0, 0, self.P, 0, 0]
        return 0

    def gsb_densify_emit(self, table, n, P, ws, n_kept, n_clones, S, n_children, rot, samples, factor, stream):
        self.table = [table[i] for i in range(n)]
        for e in self.table:
            for s, d in ((e.src, e.dst), (e.exp_avg_src, e.exp_avg_dst), (e.exp_avg_sq_src, e.exp_avg_sq_dst), (e.grad_src, e.grad_dst)):
                if s:
                    C.memmove(d, s, 4 * P * e.row_width)
        return 0


def test_host_thresholds_and_state_rekeying(monkeypatch):
    m = _model("dp_screen_sg")
    stub = _Stub(300)
    monkeypatch.setattr(gsl, "lib", lambda: stub)
    monkeypatch.setattr(gsl, "on_device", lambda dev: __import__("contextlib").nullcontext())
    monkeypatch.setattr(gsl, "current_stream", lambda dev: 0)
    monkeypatch.setattr(densify, "_validate", lambda model, sg, grads_everywhere=False: (
        [(g["name"], g, g["params"][0], model.optimizer.state.get(g["params"][0], None)) for g in model.optimizer.param_groups],
        300, torch.device("cpu")))
    steps = {g["name"]: m.optimizer.state[g["params"][0]]["step"] for g in m.optimizer.param_groups if g["params"][0] in m.optimizer.state}
    states = {g["name"]: m.optimizer.state[g["params"][0]] for g in m.optimizer.param_groups if g["params"][0] in m.optimizer.state}
    extent, pd = 3.7, m.percent_dense
    d = {}
    densify.densify_and_prune(m, 0.0002, 0.005, extent, 20, d, store_grads=True)
    a = stub.plan_args
    # the ctypes float fields hold the fp32 casts of the reference's double products
    f = lambda x: float(np.float32(x))  # noqa: E731
    assert a[1] == gsl.DENSIFY_CLONE_SPLIT
    argtypes = [C.c_int32, C.c_int32] + [C.c_void_p] * 7 + [C.c_float] * 4 + [C.c_int32] + [C.c_float] * 3
    vals = [t(v).value for t, v in zip(argtypes[9:], a[9:17])]
    assert vals == [f(0.0002), 0.0, f(pd * extent), f(0.005), 1, f(20), f(0.1 * extent), f(1.0 / f(0.8 * 2))]
    assert a[3] is None                                                   # no xyz_gradient_accum_abs: the reference's split test
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        if g["name"] in states:
            assert m.optimizer.state[p] is states[g["name"]]
            assert m.optimizer.state[p]["step"] is steps[g["name"]]
            assert p.grad is not None
        else:
            assert p not in m.optimizer.state and p.grad is None
        assert getattr(m, dg.GROUPS[g["name"]]) is p and isinstance(p, torch.nn.Parameter)
    assert len(m.optimizer.state) == len(states)
    assert d["n_points_cloned"] == 0 and d["n_points_split"] == 0 and d["n_points_pruned"].dim() == 0
    kinds = {e.kind for e in stub.table}
    assert kinds == {gsl.DENSIFY_COPY, gsl.DENSIFY_XYZ, gsl.DENSIFY_SCALING}


# ------------------------------------------------------------------------------------------------ the restatement vs the goldens
@pytest.mark.parametrize("name", dg.CASES)
def test_restatement_reproduces_reference_goldens(name):
    z = dg.load(name)
    m = dg.make_model(z, "cpu")
    a, d = dg.args(z), {}
    op, sg = str(z["op"]), bool(z["store_grads"])
    calls = []

    def recorded(mean, std):
        calls.append(tuple(mean.shape))
        return torch.from_numpy(z["samples"])

    if op == "densify_and_prune":
        rs.densify_and_prune(m, a["max_grad"], a["min_opacity"], a["extent"], a["max_screen_size"], d, sg, normal=recorded)
        assert calls == [tuple(z["samples"].shape)] and z["n_normal_calls"] == 1
    elif op == "prune":
        rs.prune(m, a["min_opacity"], a["extent"], a["max_screen_size"], d, sg)
    elif op == "prune_points":
        rs.prune_points(m, torch.from_numpy(z["mask"]), sg)
    else:
        vs = torch.zeros_like(torch.from_numpy(z["view_grad"]), requires_grad=True)
        vs.grad = torch.from_numpy(z["view_grad"])
        rs.add_densification_stats(m, vs, torch.from_numpy(z["visibility"]), torch.from_numpy(z["radii"]))
    dg.compare(dg.outputs(m), z)
    got = {k: (int(v) if not torch.is_tensor(v) else int(v.item())) for k, v in d.items()}
    assert got == {k[5:]: int(v) for k, v in z.items() if k.startswith("dict.")}
    for k, v in d.items():
        assert torch.is_tensor(v) == (k == "n_points_pruned")
