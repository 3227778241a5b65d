"""gs_b200.mcmc without a GPU: the C ABI's symbols and argument errors, the refusals (each leaving the params, moments and step
tensors as they were), the host side against a stub of the library, and the restatement (tests/mcmc_restatement.py) against first
principles: the integer sampler against a brute-force inverse CDF, the relocation values in 50-digit decimal, and the precision
the fp32 evaluation of D would lose."""
import ctypes as C
import math
import os
import re
import sys
from decimal import Decimal

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import densify_golden as dg  # noqa: E402
import mcmc_restatement as rs  # noqa: E402
from gs_b200 import lib as gsl  # noqa: E402
from gs_b200 import mcmc  # noqa: E402

HEADER = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
NEW = ["gsb_mcmc_noise", "gsb_mcmc_workspace_bytes", "gsb_mcmc_plan", "gsb_mcmc_emit"]
E = -1


def test_symbols_exported():
    L = gsl.lib()
    for s in NEW:
        assert s in gsl.EXPORTED_SYMBOLS
        getattr(L, s)
        assert re.search(rf"GSB_API \w+ {s}\(", HEADER), s
    for name, value in (("GSB_MCMC_RELOCATE", gsl.MCMC_RELOCATE), ("GSB_MCMC_ADD", gsl.MCMC_ADD), ("GSB_MCMC_COUNTS", gsl.MCMC_COUNTS),
                        ("GSB_MCMC_OPACITY", gsl.MCMC_OPACITY), ("GSB_MCMC_FRESH", gsl.MCMC_FRESH)):
        assert int(re.search(rf"#define {name} (\d+)", HEADER).group(1)) == value, name


def test_workspace_grows_with_P():
    L = gsl.lib()
    assert L.gsb_mcmc_workspace_bytes(0) > 0
    assert L.gsb_mcmc_workspace_bytes(1 << 20) >= 40 * (1 << 20)          # the value table comes first: 16 bytes per row
    assert L.gsb_mcmc_workspace_bytes(1000) < L.gsb_mcmc_workspace_bytes(2000)


def test_einval():
    L = gsl.lib()
    fake = C.c_void_p(256)
    noise = lambda P=10, a=5e5, b=1e-4, ptr=fake: L.gsb_mcmc_noise(P, ptr, fake, fake, fake, fake, a, b, None)  # noqa: E731
    assert noise(P=-1) == E
    assert noise(P=1 << 30) == E
    assert noise(a=float("nan")) == E and b"finite" in L.gsb_last_error()
    assert noise(b=float("inf")) == E
    assert noise(b=1e39) == E                                                     # finite in double, inf as fp32
    assert noise(ptr=None) == E
    assert noise(P=0, ptr=None) == 0                                              # nothing to launch

    def plan(P=10, mode=0, logits=fake, scaling=fake, mask=None, n=0, draws=None, ws=fake, counts=fake):
        return L.gsb_mcmc_plan(P, mode, logits, scaling, mask, 0.005, n, draws, ws, counts, None)
    assert plan(P=-1) == E
    assert plan(P=1 << 30) == E
    assert plan(mode=2) == E
    assert plan(mode=gsl.MCMC_ADD, mask=fake) == E
    assert plan(ws=None) == E
    assert plan(n=3) == E                                                          # n without draws
    assert plan(draws=fake, n=0) == E
    assert plan(draws=fake, n=11) == E                                             # more draws than rows
    assert plan(counts=None) == E
    assert plan(logits=None) == E
    assert plan(draws=fake, n=5, scaling=None) == E

    e = lambda **kw: gsl.GsbDensifyTensor(**{**dict(src=256, dst=256, row_width=3, kind=0), **kw})  # noqa: E731

    def emit(entries, n_tensors=None, P=10, mode=gsl.MCMC_RELOCATE, n=5, ws=fake):
        tab = (gsl.GsbDensifyTensor * len(entries))(*entries) if entries else None
        return L.gsb_mcmc_emit(tab, len(entries) if n_tensors is None else n_tensors, P, mode, n, ws, None)
    assert emit([], n_tensors=1) == E
    assert emit([e()], n_tensors=17) == E
    assert emit([e()], P=-1) == E
    assert emit([e()], mode=2) == E
    assert emit([e()], n=-1) == E
    assert emit([e()], n=11) == E
    assert emit([e()], ws=None) == E
    for bad in (dict(row_width=0), dict(kind=gsl.DENSIFY_XYZ), dict(kind=5), dict(kind=gsl.DENSIFY_SCALING, row_width=4),
                dict(kind=gsl.MCMC_OPACITY), dict(kind=gsl.MCMC_FRESH, row_width=1), dict(grad_src=256, grad_dst=256),
                dict(exp_avg_src=256), dict(src=None, dst=None), dict(dst=512), dict(src=258, dst=258)):
        assert emit([e(**bad)]) == E, bad
    fresh_with_moments = e(kind=gsl.MCMC_FRESH, row_width=1, dst=512, exp_avg_src=256, exp_avg_dst=768, exp_avg_sq_src=1024,
                           exp_avg_sq_dst=1280)
    assert emit([fresh_with_moments], mode=gsl.MCMC_ADD) == E
    moved = e(exp_avg_src=256, exp_avg_dst=512, exp_avg_sq_src=768, exp_avg_sq_dst=768)   # relocate works in place
    assert emit([moved]) == E
    assert emit([e()], n=0) == 0                                                   # no rows: nothing launched
    assert emit([]) == 0


# ------------------------------------------------------------------------------------------------ refusals
def _model():
    return dg.make_model(dg.load("dp_none"), "cpu")


def _snapshot(m):
    groups = [(g["name"], g["params"][0]) for g in m.optimizer.param_groups]
    ids = ([(n, id(p)) for n, p in groups], {k: id(v) for k, v in vars(m).items()})
    values = {n: p.detach().clone() for n, p in groups}
    for n, p in groups:
        st = m.optimizer.state.get(p)
        if st is not None:
            values.update({f"{n}.{k}": v.clone() for k, v in st.items()})
            ids[1][f"{n}.step"] = id(st["step"])
    values["_degrees"] = m._degrees.clone()
    return ids, values


def _refused(m, fn, match):
    ids, values = _snapshot(m)
    rng = torch.get_rng_state()
    with pytest.raises(RuntimeError, match=match):
        fn(m)
    ids2, values2 = _snapshot(m)
    assert ids2 == ids
    assert values.keys() == values2.keys() and all(torch.equal(values[k], values2[k]) for k in values)
    assert torch.equal(torch.get_rng_state(), rng)                              # nothing drawn


@pytest.fixture
def fake_cuda(monkeypatch):
    """Makes densify._validate see CUDA tensors, so that the refusal under test is the one that fires (no GPU here)."""
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def test_refuses_cpu_tensors():
    _refused(_model(), lambda m: mcmc.relocate_gs(m), "CUDA")
    _refused(_model(), lambda m: mcmc.add_new_gs(m, 1000), "CUDA")
    _refused(_model(), lambda m: mcmc.inject_noise(m, 1e-4), "CUDA")


@pytest.mark.parametrize("mask", [torch.zeros(299, dtype=torch.bool), torch.zeros(300, dtype=torch.uint8), [False] * 300,
                                  torch.zeros(300, 1, dtype=torch.bool)])
def test_refuses_bad_dead_mask(fake_cuda, mask):
    _refused(_model(), lambda m: mcmc.relocate_gs(m, mask), "dead_mask")


@pytest.mark.parametrize("cap_max", [-1, 1000.0, "1000", True, None])
def test_refuses_bad_cap_max(fake_cuda, cap_max):
    _refused(_model(), lambda m: mcmc.add_new_gs(m, cap_max), "cap_max")


@pytest.mark.parametrize("lrs", [(float("nan"), 1e-4), (5e5, float("inf")), (5e5, -float("inf")), (1e39, 1e-4)])
def test_refuses_non_finite_learning_rates(fake_cuda, lrs):
    _refused(_model(), lambda m: mcmc.inject_noise(m, lrs[1], noise_lr=lrs[0]), "finite")


@pytest.mark.parametrize("case", ["quantised", "list_f_rest", "optimizer", "extra_group", "degrees"])
@pytest.mark.parametrize("call", ["relocate_gs", "add_new_gs", "inject_noise"])
def test_model_contract_is_densify(fake_cuda, case, call):
    m = _model()
    match = {"quantised": "quantised", "list_f_rest": "variable-SH", "optimizer": "Adam", "extra_group": "groups", "degrees": "_degrees"}[case]
    if case == "quantised":
        m._codebook_dict = {"opacity": None}
    elif case == "list_f_rest":
        m._features_rest = [m._features_rest]
    elif case == "optimizer":
        m.optimizer = torch.optim.SGD(m.optimizer.param_groups, lr=0.1)
    elif case == "extra_group":
        m.optimizer.add_param_group({"params": [torch.nn.Parameter(torch.zeros(300, 2))], "name": "extra"})
    else:
        m._degrees = m._degrees.long()
    fn = {"relocate_gs": lambda m: mcmc.relocate_gs(m), "add_new_gs": lambda m: mcmc.add_new_gs(m, 1000),
          "inject_noise": lambda m: mcmc.inject_noise(m, 1e-4)}[call]
    _refused(m, fn, match)


# ------------------------------------------------------------------------------------------------ host logic against a stub library
class _Stub:
    """Records every call; the first plan reports `dead` dead rows and a total weight of `total`."""

    def __init__(self, dead, total=1 << 40):
        self.dead, self.total, self.calls = dead, total, []

    def gsb_mcmc_workspace_bytes(self, P):
        return 64

    def gsb_mcmc_noise(self, *a):
        self.calls.append(("noise", a))
        return 0

    def gsb_mcmc_plan(self, *a):
        self.calls.append(("plan", a))
        if a[7] is None:
            (C.c_int64 * 4).from_address(a[9])[:] = [self.dead, self.total, 0, 0]
        return 0

    def gsb_mcmc_emit(self, table, n_tensors, P, mode, n, ws, stream):
        self.calls.append(("emit", (mode, n, [(table[i].kind, table[i].row_width, table[i].src == table[i].dst)
                                              for i in range(n_tensors)])))
        return 0


@pytest.fixture
def stubbed(monkeypatch, fake_cuda):
    draws = []
    real_randint = torch.randint

    def randint(low, high, size, dtype=None, device=None):
        draws.append((low, high, tuple(size), dtype))
        return real_randint(0, 1 << 62, size, dtype=dtype)

    def install(stub):
        monkeypatch.setattr(gsl, "lib", lambda: stub)
        monkeypatch.setattr(gsl, "on_device", lambda dev: __import__("contextlib").nullcontext())
        monkeypatch.setattr(gsl, "current_stream", lambda dev: 0)
        monkeypatch.setattr(torch, "randint", randint)
        return stub
    install.draws = draws
    return install


def test_noise_arguments_are_fp32_casts(stubbed):
    stub = stubbed(_Stub(0))
    m = _model()
    for p in m.optimizer.param_groups:
        p["params"][0].grad = torch.ones_like(p["params"][0])
    mcmc.inject_noise(m, 1.6e-4 / 3, noise_lr=5e5 / 7)
    (kind, a), = stub.calls
    assert kind == "noise" and a[0] == 300
    argtypes = gsl.SIGNATURES["gsb_mcmc_noise"][1]
    assert [t(v).value for t, v in zip(argtypes[6:8], a[6:8])] == [float(np.float32(5e5 / 7)), float(np.float32(1.6e-4 / 3))]
    assert a[1] == m._xyz.data_ptr() and a[4] == m._opacity.data_ptr()
    assert all(g["params"][0].grad is not None for g in m.optimizer.param_groups)     # the noise leaves .grad alone


def test_relocate_draws_one_per_dead_row(stubbed):
    stub = stubbed(_Stub(37))
    m = _model()
    for g in m.optimizer.param_groups:
        g["params"][0].grad = torch.ones_like(g["params"][0])
    ids, _ = _snapshot(m)
    mcmc.relocate_gs(m)
    assert stubbed.draws == [(0, 2 ** 62, (37,), torch.int64)]
    (k0, a0), (k1, a1), (k2, (mode, n, table)) = stub.calls
    assert (k0, k1, k2) == ("plan", "plan", "emit")
    assert a0[1] == gsl.MCMC_RELOCATE and a0[4] is None and a0[6] == 0 and a1[6] == 37 and a1[7] is not None
    assert C.c_float(a0[5]).value == np.float32(0.005)
    assert mode == gsl.MCMC_RELOCATE and n == 37
    assert [k for k, _, _ in table] == [0, 0, 0, gsl.MCMC_OPACITY, gsl.DENSIFY_SCALING, 0, 0] and all(s for _, _, s in table)
    assert _snapshot(m)[0] == ids                                                       # in place: the same objects
    assert all(g["params"][0].grad is None for g in m.optimizer.param_groups)


@pytest.mark.parametrize("dead,total", [(0, 1 << 40), (12, 0)])
def test_relocate_without_dead_or_weight_changes_nothing(stubbed, dead, total):
    stub = stubbed(_Stub(dead, total))
    m = _model()
    mcmc.relocate_gs(m, torch.zeros(300, dtype=torch.bool))
    assert stubbed.draws == [] and [k for k, _ in stub.calls] == ["plan"]
    assert stub.calls[0][1][4] is not None                                            # the mask reached the plan


@pytest.mark.parametrize("P,cap_max,n", [(300, 1000, 15), (300, 310, 10), (300, 300, 0), (300, 0, 0), (19, 1000, 0), (20, 1000, 1)])
def test_add_draws_n(stubbed, P, cap_max, n):
    stub = stubbed(_Stub(0))
    m = _model()
    if P != 300:
        keep = torch.arange(P)
        for g in m.optimizer.param_groups:
            p = g["params"][0]
            q = torch.nn.Parameter(p.detach()[keep].clone())
            st = m.optimizer.state.pop(p, None)
            if st is not None:
                st["exp_avg"], st["exp_avg_sq"] = st["exp_avg"][keep].clone(), st["exp_avg_sq"][keep].clone()
                m.optimizer.state[q] = st
            g["params"][0] = q
            setattr(m, dg.GROUPS[g["name"]], q)
        for k in ("_degrees", "xyz_gradient_accum", "denom", "max_radii2D"):
            setattr(m, k, getattr(m, k)[keep].clone())
    assert n == max(0, min(cap_max, int(1.05 * P)) - P)
    steps = {g["name"]: m.optimizer.state[g["params"][0]]["step"] for g in m.optimizer.param_groups if g["params"][0] in m.optimizer.state}
    assert mcmc.add_new_gs(m, cap_max) == n
    if n == 0:
        assert stubbed.draws == [] and stub.calls == []
        return
    assert stubbed.draws == [(0, 2 ** 62, (n,), torch.int64)]
    mode, n_emit, table = stub.calls[-1][1]
    assert mode == gsl.MCMC_ADD and n_emit == n
    assert [k for k, _, _ in table] == [0, 0, 0, gsl.MCMC_OPACITY, gsl.DENSIFY_SCALING, 0, 0] + [gsl.MCMC_FRESH] * 3
    for g in m.optimizer.param_groups:
        p = g["params"][0]
        assert p.shape[0] == P + n and p.grad is None and getattr(m, dg.GROUPS[g["name"]]) is p
        if g["name"] in steps:
            assert m.optimizer.state[p]["step"] is steps[g["name"]] and m.optimizer.state[p]["exp_avg"].shape == p.shape
    for k in ("_degrees", "xyz_gradient_accum", "denom", "max_radii2D"):
        assert getattr(m, k).shape[0] == P + n


def test_add_without_weight_changes_nothing(stubbed):
    stub = stubbed(_Stub(0, total=0))
    m = _model()
    ids, _ = _snapshot(m)
    assert mcmc.add_new_gs(m, 1000) == 0
    assert stubbed.draws == [] and [k for k, _ in stub.calls] == ["plan"] and _snapshot(m)[0] == ids


# ------------------------------------------------------------------------------------------------ the restatement vs first principles
def test_sampler_against_brute_force_inverse_cdf():
    g = np.random.default_rng(5)
    o = g.random(300).astype(np.float32)
    o[g.random(300) < 0.2] = 0                                                        # weight 0: never drawn
    o[:3] = [1.0, np.float32(2.0 ** -32), np.float32(2.0 ** -33)]                     # the largest weight, the smallest, one that floors to 0
    cand = g.random(300) < 0.8
    w = rs.weights(o, cand)
    assert w[0] == (1 << 32 if cand[0] else 0) and w[2] == 0
    draws = [int(x) for x in g.integers(0, 1 << 62, 2000, dtype=np.int64)] + [0, (1 << 62) - 1]
    got = rs.sample(w, draws)
    assert np.array_equal(got, rs.sample_brute_force(w, draws))
    assert np.all(w[got] > 0)


@pytest.mark.parametrize("o", [np.float32(0.3), np.float32(1 - 2 ** -23), np.float32(0.006), np.float32(2 ** -20)])
def test_relocation_decimal_identities(o):
    s = [np.float32(0.01), np.float32(2.5), np.float32(1e-4)]
    oc, s1, op, D = rs.relocated_decimal(o, s, 1)
    assert abs(op - Decimal(float(o))) < Decimal(10) ** -45 and abs(D - Decimal(float(o))) < Decimal(10) ** -45
    assert all(abs(a - Decimal(float(b))) <= Decimal(10) ** -45 * Decimal(float(b)) for a, b in zip(s1, s))
    for N in (2, 7, 50):
        _, _, op, _ = rs.relocated_decimal(o, s, N)
        assert abs((1 - (1 - op) ** N) - Decimal(float(o))) < Decimal(10) ** -40


def test_fp32_D_loses_precision():
    """The reason the kernel evaluates D in double: at o = 1 - 2^-23 and N = 50 the fp32 double sum is off by FP32_D_ERROR."""
    _, _, op, D = rs.relocated_decimal(np.float32(1 - 2 ** -23), [1.0, 1.0, 1.0], 50)
    err32 = abs(Decimal(float(rs.D_fp32(float(op), 50))) - D) / D
    Dd, pw, opd = 0.0, 1.0, float(op)                                                 # the kernel's loop in double
    for k in range(50):
        pw *= opd
        term = math.comb(50, k + 1) * pw / math.sqrt(k + 1)
        Dd = Dd - term if k & 1 else Dd + term
    err64 = abs(Decimal(Dd) - D) / D
    assert 0.8 * rs.FP32_D_ERROR <= float(err32) <= 1.2 * rs.FP32_D_ERROR, float(err32)
    assert float(err64) < 1e-12, float(err64)


def test_relocated_torch_matches_decimal_on_cpu():
    o = torch.tensor([0.3, 1 - 2 ** -23, 0.006, 0.9, 0.5], dtype=torch.float32)
    s = torch.tensor([[0.01, 2.5, 1e-4]] * 5, dtype=torch.float32)
    N = torch.tensor([1, 50, 3, 50, 17])
    oc, sc = rs.relocated_torch(o, s, N)
    for i in range(5):
        want_o, want_s, _, _ = rs.relocated_decimal(o[i].item(), s[i].tolist(), int(N[i]))
        ulp = lambda x: np.spacing(np.float32(abs(float(x))))  # noqa: E731
        assert abs(Decimal(float(oc[i])) - want_o) <= Decimal(float(ulp(want_o))), i
        for c in range(3):
            assert abs(Decimal(float(sc[i, c])) - want_s[c]) <= Decimal(float(ulp(want_s[c]))), (i, c)
    assert oc[0] == o[0] and torch.equal(sc[0], s[0])                                   # N = 1 is the identity
