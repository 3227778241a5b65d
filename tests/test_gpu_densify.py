"""gs_b200.densify on the GPU: against the reference's goldens (recorded samples substituted for torch.normal) and against the
torch restatement of the reference run on the same GPU (tests/densify_restatement.py), at P = 100 k and at C3 size (3 M).

Bounds, as observed and documented in DESIGN.md §5g:
  * every copied value, every moment, grad, degree and statistic, the counts, the row order and the generator state: bitwise;
  * split children's scaling (exp / multiply / log): bitwise against torch on the GPU; against the CPU goldens within
    CHILD_TOL of the column's largest magnitude (CPU libm against CUDA);
  * split children's xyz (rotation @ sample + xyz): torch.bmm's rounding depends on the cuBLAS kernel it picks per batch size,
    so against torch within XYZ_TOL of the column's largest magnitude, and against the goldens within CHILD_TOL.
"""
import os
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
from gs_b200.optim import GaussianAdam  # noqa: E402

pytestmark = pytest.mark.gpu
CHILD_TOL = 1e-6
XYZ_TOL = 1e-6


def _run_native(m, z, d):
    op, sg, a = str(z["op"]), bool(z["store_grads"]), dg.args(z)
    if op == "densify_and_prune":
        densify.densify_and_prune(m, a["max_grad"], a["min_opacity"], a["extent"], a["max_screen_size"], d, sg)
    elif op == "prune":
        densify.prune(m, a["min_opacity"], a["extent"], a["max_screen_size"], d, sg)
    elif op == "prune_points":
        densify.prune_points(m, torch.from_numpy(z["mask"]).cuda(), sg)
    else:
        vs = torch.zeros(z["view_grad"].shape, device="cuda", requires_grad=True)
        vs.grad = torch.from_numpy(z["view_grad"]).cuda()
        densify.add_densification_stats(m, vs, torch.from_numpy(z["visibility"]).cuda(), torch.from_numpy(z["radii"]).cuda())


@pytest.mark.parametrize("name", dg.CASES)
def test_against_reference_goldens(name, monkeypatch):
    z = dg.load(name)
    calls = []

    def recorded(mean, std):
        calls.append(tuple(mean.shape))
        return torch.from_numpy(z["samples"]).cuda()

    monkeypatch.setattr(torch, "normal", recorded)
    m, d = dg.make_model(z, "cuda"), {}
    _run_native(m, z, d)
    torch.cuda.synchronize()
    if str(z["op"]) == "densify_and_prune":
        assert calls == [tuple(z["samples"].shape)]
    out = dg.outputs(m)
    if str(z["op"]) == "add_densification_stats":
        # torch.norm on the CPU rounds differently from CUDA; on the GPU the accumulator is bitwise (test below)
        a, b = out.pop("xyz_gradient_accum"), z.pop("out.xyz_gradient_accum")
        assert np.abs(a.astype(np.float64) - b).max() <= CHILD_TOL * np.abs(b).max()
        out["xyz_gradient_accum"], z["out.xyz_gradient_accum"] = b, b
    dg.compare(out, z, computed_tol=CHILD_TOL)
    got = {k: int(v.item()) if torch.is_tensor(v) else v for k, v in d.items()}
    assert got == {k[5:]: int(v) for k, v in z.items() if k.startswith("dict.")}
    assert list(d) == [k[5:] for k in z if k.startswith("dict.")]
    for k, v in d.items():
        if k == "n_points_pruned":
            assert torch.is_tensor(v) and v.dim() == 0 and v.dtype == torch.int64 and v.is_cuda
        else:
            assert type(v) is int


# ------------------------------------------------------------------------------------------------ against torch on the GPU
class Model(dg.Model):
    pass


def synthetic(P, C, seed, opt_cls=torch.optim.Adam, no_state=None, frac=(0.05, 0.05, 0.03)):
    """A model with roughly frac = (cloned, split, pruned) of its rows selected, its optimizer stepped once."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    m = Model()
    m._xyz = torch.nn.Parameter(torch.randn(P, 3, device=dev, generator=g) * 3)
    m._features_dc = torch.nn.Parameter(torch.randn(P, 1, 3, device=dev, generator=g))
    m._features_rest = torch.nn.Parameter(torch.randn(P, C, 3, device=dev, generator=g) * 0.1)
    u = torch.rand(P, device=dev, generator=g)
    m._opacity = torch.nn.Parameter(torch.where(u < frac[2], -7.0, 1.0 + u).unsqueeze(1))
    big = torch.rand(P, device=dev, generator=g) < 0.5
    sc = torch.rand(P, 3, device=dev, generator=g) * 2 - 6
    sc[big] += 3.5                                           # max scale > percent_dense * extent for about half
    sc[torch.rand(P, device=dev, generator=g) < 0.002, 2] = 2.5   # some children pruned by 0.1 * extent
    m._scaling = torch.nn.Parameter(sc)
    m._rotation = torch.nn.Parameter(torch.randn(P, 4, device=dev, generator=g))
    m._degrees = torch.randint(0, 4, (P, 1), device=dev, generator=g, dtype=torch.int32)
    m.percent_dense = 0.01
    groups = [{"params": [getattr(m, a)], "lr": 1e-3, "name": n} for n, a in dg.GROUPS.items()]
    m.optimizer = opt_cls(groups, lr=0.0, eps=1e-15)
    for n, a in dg.GROUPS.items():
        p = getattr(m, a)
        p.grad = None if n == no_state else torch.randn(p.shape, device=dev, generator=g) * 1e-3
    m.optimizer.step()
    hot = torch.rand(P, device=dev, generator=g) < 2 * frac[0]
    m.denom = torch.randint(1, 6, (P, 1), device=dev, generator=g).float()
    m.denom[torch.rand(P, device=dev, generator=g) < 0.01] = 0
    m.xyz_gradient_accum = torch.where(hot.unsqueeze(1), 3e-4, 1e-5) * m.denom
    m.max_radii2D = torch.randint(0, 30, (P,), device=dev, generator=g).float()
    return m


def clone_model(m, opt_cls=torch.optim.Adam):
    c = Model()
    for n, a in dg.GROUPS.items():
        p = getattr(m, a)
        q = torch.nn.Parameter(p.detach().clone())
        if p.grad is not None:
            q.grad = p.grad.clone()
        setattr(c, a, q)
    c.optimizer = opt_cls([{"params": [getattr(c, a)], "lr": 1e-3, "name": n} for n, a in dg.GROUPS.items()], lr=0.0, eps=1e-15)
    for n, a in dg.GROUPS.items():
        st = m.optimizer.state.get(getattr(m, a))
        if st is not None:
            c.optimizer.state[getattr(c, a)] = {k: v.clone() for k, v in st.items()}
    for k in ("_degrees", "xyz_gradient_accum", "denom", "max_radii2D"):
        setattr(c, k, getattr(m, k).clone())
    c.percent_dense = m.percent_dense
    return c


def assert_same(a, b, xyz_tol=XYZ_TOL):
    oa, ob = dg.outputs(a), dg.outputs(b)
    assert sorted(oa) == sorted(ob)
    for k in oa:
        x, y = oa[k], ob[k]
        assert x.shape == y.shape and x.dtype == y.dtype, k
        if k == "xyz":
            err = np.abs(x.astype(np.float64) - y).max(initial=0) / max(np.abs(y).max(initial=0), 1e-30)
            assert err <= xyz_tol, (k, err)
        else:
            assert x.tobytes() == y.tobytes(), f"{k} differs"
    for g1, g2 in zip(a.optimizer.param_groups, b.optimizer.param_groups):
        s1, s2 = a.optimizer.state.get(g1["params"][0]), b.optimizer.state.get(g2["params"][0])
        assert (s1 is None) == (s2 is None)
    if hasattr(b, "density_gradient_accum"):
        assert a.density_gradient_accum.shape == b.density_gradient_accum.shape


@pytest.mark.parametrize("P,C,opt_cls,store_grads,screen", [
    (100_000, 15, torch.optim.Adam, False, None),
    (100_000, 3, GaussianAdam, True, 20),
    (3_000_000, 15, GaussianAdam, False, 20),
])
def test_against_restatement(P, C, opt_cls, store_grads, screen):
    m = synthetic(P, C, seed=P + C, opt_cls=opt_cls, no_state=None if store_grads else "f_dc")
    r = clone_model(m, opt_cls)
    steps = {n: m.optimizer.state[getattr(m, a)]["step"] for n, a in dg.GROUPS.items() if getattr(m, a) in m.optimizer.state}
    d_n, d_r = {}, {}
    torch.manual_seed(123)
    densify.densify_and_prune(m, 0.0002, 0.005, 3.7, screen, d_n, store_grads)
    st_n = torch.cuda.get_rng_state()
    torch.manual_seed(123)
    rs.densify_and_prune(r, 0.0002, 0.005, 3.7, screen, d_r, store_grads)
    st_r = torch.cuda.get_rng_state()
    assert torch.equal(st_n, st_r)
    assert {k: int(v) for k, v in d_n.items()} == {k: int(v) for k, v in d_r.items()}
    assert d_n["n_points_cloned"] > 0 and d_n["n_points_split"] > 0 and int(d_n["n_points_pruned"]) > 0
    print(f"P={P}: cloned {d_n['n_points_cloned'] / P:.3f} split {d_n['n_points_split'] / P:.3f} "
          f"pruned {int(d_n['n_points_pruned']) / P:.3f}")
    assert_same(m, r)
    for n, a in dg.GROUPS.items():
        p = getattr(m, a)
        if n in steps:
            assert m.optimizer.state[p]["step"] is steps[n]
    # 25 more optimizer steps on both models, with the same gradients
    g = torch.Generator(device="cuda").manual_seed(7)
    for _ in range(25):
        for a in dg.GROUPS.values():
            grad = torch.randn(getattr(m, a).shape, device="cuda", generator=g) * 1e-3
            getattr(m, a).grad, getattr(r, a).grad = grad.clone(), grad.clone()
        m.optimizer.step()
        r.optimizer.step()
    assert_same(m, r, xyz_tol=4 * XYZ_TOL)


@pytest.mark.parametrize("seed", [0, 1])
def test_prune_points_and_prune_against_restatement(seed):
    m = synthetic(50_000, 15, seed=seed)
    r = clone_model(m)
    g = torch.Generator(device="cuda").manual_seed(seed)
    mask = torch.rand(50_000, device="cuda", generator=g) < 0.2
    densify.prune_points(m, mask)
    rs.prune_points(r, mask)
    assert_same(m, r, xyz_tol=0)
    # a mercy_points-style mask: the lower half of the opacities among rows over a threshold
    over = torch.rand(m._xyz.shape[0], device="cuda", generator=g) < 0.3
    op = torch.sigmoid(m._opacity).squeeze(1)
    mask = over.clone()
    mask[over.clone()] = op[over] < op[over].median()
    for a in dg.GROUPS.values():                             # store_grads carries the grads the params have now
        grad = torch.randn(getattr(m, a).shape, device="cuda", generator=g)
        getattr(m, a).grad, getattr(r, a).grad = grad.clone(), grad.clone()
    densify.prune_points(m, mask, store_grads=True)
    rs.prune_points(r, mask, store_grads=True)
    assert_same(m, r, xyz_tol=0)
    d1, d2 = {}, {}
    densify.prune(m, 0.3, 3.7, 20, d1)
    rs.prune(r, 0.3, 3.7, 20, d2)
    assert int(d1["n_points_pruned"]) == int(d2["n_points_pruned"]) > 0
    assert_same(m, r, xyz_tol=0)


def test_add_densification_stats_bitwise_and_sync_free():
    P = 200_000
    m = synthetic(P, 3, seed=5)
    r = clone_model(m)
    g = torch.Generator(device="cuda").manual_seed(5)
    for _ in range(10):
        vs = torch.zeros(P, 3, device="cuda", requires_grad=True)
        vis = torch.rand(P, device="cuda", generator=g) < 0.8
        vs.grad = torch.randn(P, 3, device="cuda", generator=g) * 1e-3 * vis.unsqueeze(1)
        radii = (torch.rand(P, device="cuda", generator=g) * 50).int() * vis
        torch.cuda.set_sync_debug_mode("error")
        try:
            densify.add_densification_stats(m, vs, vis, radii)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        rs.add_densification_stats(r, vs, vis, radii)
    for k in ("xyz_gradient_accum", "denom", "max_radii2D"):
        assert getattr(m, k).cpu().numpy().tobytes() == getattr(r, k).cpu().numpy().tobytes(), k


def test_edge_cases():
    # nothing selected, everything pruned
    for kw, want in ((dict(max_grad=1e30, min_opacity=0.0), None), (dict(max_grad=0.0002, min_opacity=1.5), 0)):
        m = synthetic(10_000, 3, seed=11)
        r = clone_model(m)
        d1, d2 = {}, {}
        torch.manual_seed(1)
        densify.densify_and_prune(m, kw["max_grad"], kw["min_opacity"], 3.7, None, d1)
        torch.manual_seed(1)
        rs.densify_and_prune(r, kw["max_grad"], kw["min_opacity"], 3.7, None, d2)
        assert {k: int(v) for k, v in d1.items()} == {k: int(v) for k, v in d2.items()}
        if want is not None:
            assert m._xyz.shape[0] == want
        assert_same(m, r)
    # P = 0
    m = synthetic(1, 3, seed=3)
    densify.prune_points(m, torch.ones(1, dtype=torch.bool, device="cuda"))
    assert m._xyz.shape == (0, 3)
    d = {}
    densify.densify_and_prune(m, 0.0002, 0.005, 3.7, 20, d)
    assert m._xyz.shape == (0, 3) and d["n_points_cloned"] == 0 and int(d["n_points_pruned"]) == 0


def test_stream_and_run_to_run():
    outs = []
    for use_stream in (False, True, True):
        m = synthetic(100_000, 15, seed=21)
        torch.manual_seed(9)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s) if use_stream else torch.cuda.stream(torch.cuda.current_stream()):
            densify.densify_and_prune(m, 0.0002, 0.005, 3.7, 20, {})
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        outs.append({k: v.tobytes() for k, v in dg.outputs(m).items()})
    assert outs[0] == outs[1] == outs[2]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_second_device():
    with torch.cuda.device(1):
        m = synthetic(20_000, 3, seed=4)
    r = clone_model(m)
    assert m._xyz.device.index == 1
    d1, d2 = {}, {}
    torch.cuda.manual_seed_all(3)
    densify.densify_and_prune(m, 0.0002, 0.005, 3.7, None, d1)
    torch.cuda.manual_seed_all(3)
    with torch.cuda.device(1):
        rs.densify_and_prune(r, 0.0002, 0.005, 3.7, None, d2)
    assert_same(m, r)
