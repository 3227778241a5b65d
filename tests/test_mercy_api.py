"""gs_b200.densify.calculate_redundancy_metric / mercy_points without a GPU: the C ABI's symbols, workspace sizes and argument
errors, the refusals (each leaving the model and the optimizer as they were), the host plumbing against a stub library, and the
torch restatement of the reference's mercy_points against the reference's own goldens (tests/golden/make_golden_mercy.py)."""
import ctypes as C
import glob
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
import mercy_restatement as mr  # noqa: E402
from gs_b200 import densify  # noqa: E402
from gs_b200 import lib as gsl  # noqa: E402

HEADER = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
NEW = ["gsb_redundancy_workspace_bytes", "gsb_redundancy_score", "gsb_mercy_workspace_bytes", "gsb_mercy_plan"]
GOLDENS = sorted(os.path.basename(p)[6:-4] for p in glob.glob(os.path.join(ROOT, "tests", "golden", "mercy_*.npz")))


def load(name):
    return dict(np.load(os.path.join(ROOT, "tests", "golden", f"mercy_{name}.npz")))


def test_symbols_exported():
    L = gsl.lib()
    for s in NEW:
        assert s in gsl.EXPORTED_SYMBOLS
        getattr(L, s)
        assert re.search(rf"GSB_API \w+ {s}\(", HEADER), s
    for name, value in (("GSB_MERCY_REDUNDANCY_OPACITY", gsl.MERCY_REDUNDANCY_OPACITY),
                        ("GSB_MERCY_REDUNDANCY_RANDOM", gsl.MERCY_REDUNDANCY_RANDOM), ("GSB_MERCY_OPACITY", gsl.MERCY_OPACITY),
                        ("GSB_MERCY_REDUNDANCY_OPACITY_OPACITY", gsl.MERCY_REDUNDANCY_OPACITY_OPACITY),
                        ("GSB_MERCY_REDUNDANCY", gsl.MERCY_REDUNDANCY)):
        assert int(re.search(rf"#define {name} (\d+)", HEADER).group(1)) == value, name


def test_workspace_grows():
    L = gsl.lib()
    assert L.gsb_redundancy_workspace_bytes(1000, 30) < L.gsb_redundancy_workspace_bytes(2000, 30)
    assert L.gsb_redundancy_workspace_bytes(1000, 30) < L.gsb_redundancy_workspace_bytes(1000, 64)
    assert L.gsb_redundancy_workspace_bytes(1 << 20, 30) >= 4 * 30 * (1 << 20)
    assert 0 < L.gsb_mercy_workspace_bytes(0) <= L.gsb_mercy_workspace_bytes(1000) < L.gsb_mercy_workspace_bytes(1 << 24)


def test_einval():
    L = gsl.lib()
    f = C.c_void_p(256)
    E = -1
    red = lambda P=10, K=30, n=2, xyz=f, ws=f, out=f, m=f: L.gsb_redundancy_score(  # noqa: E731
        P, xyz, f, f, n, m, f, f, f, 1.0, K, out, f, ws, None)
    for bad in (dict(K=0), dict(K=65), dict(P=-1), dict(P=1 << 30), dict(n=-1), dict(n=1025), dict(xyz=None), dict(ws=None),
                dict(out=None), dict(m=None)):
        assert red(**bad) == E, bad
        assert gsl.lib().gsb_last_error().decode().startswith("redundancy_score")
    assert red(P=0) == 0
    plan = lambda P=10, c=f, o=f, t=0, d=None, nd=-1, ws=f, m=f, th=f, co=f: L.gsb_mercy_plan(  # noqa: E731
        P, c, o, t, 2.0, 2.0, 0.045, d, nd, ws, m, th, co, None)
    for bad in (dict(P=-1), dict(P=1 << 30), dict(t=5), dict(t=-1), dict(ws=None), dict(th=None), dict(co=None), dict(c=None),
                dict(m=None), dict(o=None), dict(t=2, o=None), dict(t=1, d=f), dict(t=1, d=f, nd=-1), dict(t=0, d=f, nd=3)):
        assert plan(**bad) == E, bad
        assert gsl.lib().gsb_last_error().decode().startswith("mercy_plan")


# ------------------------------------------------------------------------------------------------ refusals
def _model():
    m = dg.make_model(dg.load("prune_points"), "cpu")
    P = m._xyz.shape[0]
    m._splatted_num_accum = torch.ones((P, 1, 1), dtype=torch.int32)
    return m


def _fingerprint(m):
    groups = [(g["name"], g["params"][0]) for g in m.optimizer.param_groups]
    state = {id(p): (id(m.optimizer.state[p]), {k: id(v) for k, v in m.optimizer.state[p].items()}) for _, p in groups if p in m.optimizer.state}
    return [(n, id(p)) for n, p in groups], state, {k: id(v) for k, v in vars(m).items()}


def _refused(m, fn, match):
    before = _fingerprint(m)
    with pytest.raises(RuntimeError, match=match):
        fn(m)
    assert _fingerprint(m) == before


def test_refuses_cpu_tensors():
    _refused(_model(), lambda m: densify.mercy_points(m, {}), "CUDA")


@pytest.mark.parametrize("case", ["dtype", "shape", "missing", "noncontig", "list_f_rest", "quantised", "optimizer"])
def test_refusals_leave_everything(case, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    m = _model()
    P = m._xyz.shape[0]
    if case == "dtype":
        m._splatted_num_accum = torch.ones((P, 1, 1), dtype=torch.float32)
    elif case == "shape":
        m._splatted_num_accum = torch.ones((P + 1, 1), dtype=torch.int32)
    elif case == "missing":
        del m._splatted_num_accum
    elif case == "noncontig":
        m._splatted_num_accum = torch.ones((2 * P, 1), dtype=torch.int32)[::2]
    elif case == "list_f_rest":
        m._features_rest = [m._features_rest]
    elif case == "quantised":
        m._codebook_dict = {"x": 1}
    elif case == "optimizer":
        m.optimizer = torch.optim.Adam([{"params": [m._xyz], "name": "xyz"}], lr=0.1)
    d = {}
    _refused(m, lambda m: densify.mercy_points(m, d), "densify")
    assert d == {}


# ------------------------------------------------------------------------------------------------ host plumbing
class _Stub:
    """Records gsb_mercy_plan calls; writes n_redundant = 3 into the counts on every call."""

    def __init__(self):
        self.calls = []

    def gsb_mercy_workspace_bytes(self, P):
        return 1024

    def gsb_mercy_plan(self, P, counts, logits, code, lam, mmin, q, draws, n_draws, ws, mask, thr, cnt, stream):
        self.calls.append(dict(P=P, code=code, lam=lam, mmin=mmin, q=q, draws=draws, n_draws=n_draws))
        C.cast(cnt, C.POINTER(C.c_int64))[0] = 3
        return 0


@pytest.mark.parametrize("mtype,code,q", [("redundancy_opacity", 0, 0.0), ("redundancy_random", 1, 0.0), ("opacity", 2, 0.045),
                                          ("redundancy_opacity_opacity", 3, 0.03), ("something else", 4, 0.0)])
def test_plumbing_against_stub(mtype, code, q, monkeypatch):
    """The arguments reach the library as the C prototype casts them (lambda and q fp32, mercy_minimum fp64), and the random
    type draws torch.rand of the count read back between its two calls."""
    stub = _Stub()
    real = gsl.lib()
    proto = real.gsb_mercy_plan.argtypes
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(gsl, "lib", lambda: stub)
    monkeypatch.setattr(gsl, "current_stream", lambda dev: 0)
    monkeypatch.setattr(gsl, "on_device", lambda dev: __import__("contextlib").nullcontext())
    drawn = []
    real_rand = torch.rand
    monkeypatch.setattr(torch, "rand", lambda shape, **k: drawn.append(tuple(shape)) or real_rand(shape))
    planned = {}
    monkeypatch.setattr(densify, "_plan", lambda *a, **k: planned.update(k) or (None, None, None))
    monkeypatch.setattr(densify, "_emit", lambda *a, **k: None)
    m = _model()
    d = {}
    densify.mercy_points(m, d, lambda_mercy=0.1, mercy_minimum=2.3, mercy_type=mtype)
    assert len(stub.calls) == (2 if code == 1 else 1)
    for c in stub.calls:
        assert c["code"] == code and c["P"] == m._xyz.shape[0]
        cast = lambda t, v: t(v).value  # noqa: E731
        assert cast(proto[4], c["lam"]) == float(np.float32(0.1)) and cast(proto[6], c["q"]) == float(np.float32(q))
        assert cast(proto[5], c["mmin"]) == 2.3
    if code == 1:
        assert drawn == [(3,)]
        assert stub.calls[0]["draws"] is None and stub.calls[1]["n_draws"] == 3 and stub.calls[1]["draws"]
    else:
        assert drawn == [] and stub.calls[0]["draws"] is None
    assert planned["mask"].dtype == torch.uint8
    assert d["n_points_mercied"].dtype == torch.int64 and d["n_points_mercied"].dim() == 0
    assert d["redundancy_threshold"].shape == (1,)
    ot = d["opacity_threshold"]
    assert (ot.shape == () if code == 2 else ot.shape == (1,) if code == 3 else ot == 0 and isinstance(ot, int))


# ------------------------------------------------------------------------------------------------ restatement vs goldens
class _Holder:
    pass


def run_restatement(z):
    m = _Holder()
    P = int(z["P"])
    m._opacity = torch.from_numpy(z["logits"])
    m._splatted_num_accum = torch.from_numpy(z["counts"]).view(P, 1, 1)
    seen = {}
    draws = torch.from_numpy(z["draws"])
    calls = []
    d = {}
    mr.mercy_points(m, d, float(z["lambda"]), int(z["mercy_minimum"]), str(z["type"]),
                    prune_points=lambda mask: seen.__setitem__("mask", mask), rand=lambda shape: calls.append(shape) or draws.view(shape))
    return seen["mask"].reshape(-1), d, calls


def test_goldens_present():
    assert len(GOLDENS) >= 15


@pytest.mark.parametrize("name", GOLDENS)
def test_golden_premise(name):
    """Every exact threshold lies 1e-4 or more from an integer, or std is 0, or there is no variance (P = 1)."""
    z = load(name)
    c = z["counts"].astype(np.float64)
    if c.size < 2 or c.std() == 0:
        return
    t = float(z["exact_threshold"])
    assert abs(t - round(t)) >= 1e-4


@pytest.mark.parametrize("name", GOLDENS)
def test_restatement_reproduces_goldens(name):
    z = load(name)
    mask, d, calls = run_restatement(z)
    assert np.array_equal(mask.numpy().astype(bool), z["mask"])
    assert int(d["n_points_mercied"]) == int(z["n_points_mercied"])
    assert np.array_equal(d["redundancy_threshold"].numpy().view(np.uint32), z["redundancy_threshold"].view(np.uint32))
    ot = d["opacity_threshold"]
    assert torch.is_tensor(ot) == bool(z["opacity_threshold_is_tensor"])
    if torch.is_tensor(ot):
        assert np.array_equal(ot.numpy().view(np.uint32), z["opacity_threshold"].view(np.uint32))
    assert len(calls) == int(z["n_draw_calls"])
