"""Golden densification fixtures written by the reference's OWN GaussianModel.densify_and_prune / prune / prune_points /
add_densification_stats (scene/gaussian_model.py:553-695), imported from the reference checkout ($GS_REFERENCE_ROOT) and run on
the CPU of the build container.  Writes tests/golden/densify_<case>.npz.

    python tests/golden/make_golden_densify.py

What is NOT the reference here, and why: the module is imported with the stubs of make_golden_ply.py (no GPU, no extensions);
a TorchFunctionMode sends the reference's `device="cuda"` factory calls to the CPU and records what torch.normal returned, so a
test can substitute the same samples; torch.cuda.empty_cache() is a no-op without a GPU.  The inputs are synthetic and chosen to
hit every branch: a grad exactly at the threshold, denom = 0 (NaN -> 0), a max scale exactly at percent_dense * extent
(_scaling = 0 with percent_dense * extent = 1), children pruned by 0.1 * extent, low opacity, C = 0 and S = 0, max_grad <= 0,
max_screen_size None or 20, store_grads both ways, a group without optimizer state, and f_rest with 15 and 3 coefficients.
"""
import os
import sys

import numpy as np
import torch
from torch.overrides import TorchFunctionMode

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_ply import import_reference_model  # noqa: E402

GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
          "rotation": "_rotation"}


class OnCpu(TorchFunctionMode):
    """Redirects device="cuda" to the CPU and records torch.normal's results."""

    def __init__(self):
        super().__init__()
        self.samples = []

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = dict(kwargs or {})
        if str(kwargs.get("device", "")).startswith("cuda"):
            kwargs["device"] = "cpu"
        out = func(*args, **kwargs)
        if func is torch.normal:
            self.samples.append(out.detach().clone())
        return out


def make_model(gm, P, C, seed, no_state="f_dc", grads_all=False, cold=False):
    g = torch.Generator().manual_seed(seed)
    m = gm.GaussianModel(3)
    m._xyz = torch.nn.Parameter(torch.randn(P, 3, generator=g) * 2)
    m._features_dc = torch.nn.Parameter(torch.randn(P, 1, 3, generator=g))
    m._features_rest = torch.nn.Parameter(torch.randn(P, C, 3, generator=g) * 0.1)
    op = torch.randn(P, 1, generator=g) * 2
    op[:P // 10] = -8.0                                            # sigmoid < 0.005
    m._opacity = torch.nn.Parameter(op)
    sc = torch.rand(P, 3, generator=g) * 4 - 3                     # exp in [0.05, 2.7]: both sides of percent_dense * extent = 1
    sc[P // 10:P // 10 + 6] = 0.0                                  # max scale exactly 1.0 = percent_dense * extent (exp(0) = 1 anywhere)
    sc[P // 5:P // 5 + 8, 1] = 3.3                                 # exp = 27.1 -> children 16.9 > 0.1 * extent = 10: children pruned
    m._scaling = torch.nn.Parameter(sc)
    m._rotation = torch.nn.Parameter(torch.randn(P, 4, generator=g))
    m._degrees = torch.randint(0, 4, (P, 1), generator=g, dtype=torch.int32)
    m.percent_dense = 0.01
    m.optimizer = torch.optim.Adam([{"params": [getattr(m, a)], "lr": 1e-3, "name": n} for n, a in GROUPS.items()], lr=0.0, eps=1e-15)
    for n, a in GROUPS.items():
        p = getattr(m, a)
        p.grad = None if n == no_state else torch.randn(p.shape, generator=g) * 1e-3
    m.optimizer.step()
    for n, a in GROUPS.items():
        p = getattr(m, a)
        p.grad = torch.randn(p.shape, generator=g) * 1e-3 if (grads_all or n != no_state) else None
    acc = (torch.rand(P, 1, generator=g) * 4e-4).float()
    den = torch.randint(0, 5, (P, 1), generator=g).float()
    acc[3:9] = torch.tensor(np.float32(0.0002)).item()             # grad exactly fp32(0.0002) (< the double 0.0002) with denom 1
    den[3:9] = 1.0
    den[9:14] = 0.0                                                # 0 / 0 = NaN -> 0; x / 0 = inf
    acc[9:11] = 0.0
    if cold:                                                       # nothing reaches the threshold: C = S = 0
        acc.zero_()
    m.xyz_gradient_accum, m.denom = acc, den
    m.max_radii2D = torch.randint(0, 40, (P,), generator=g).float()
    return m


def snapshot(m, prefix, out):
    opt = m.optimizer
    for g in opt.param_groups:
        n, p = g["name"], g["params"][0]
        out[f"{prefix}{n}"] = p.detach().numpy().copy()
        st = opt.state.get(p, None)
        out[f"{prefix}{n}.has_state"] = np.array(st is not None)
        if st is not None:
            out[f"{prefix}{n}.exp_avg"] = st["exp_avg"].numpy().copy()
            out[f"{prefix}{n}.exp_avg_sq"] = st["exp_avg_sq"].numpy().copy()
            out[f"{prefix}{n}.step"] = np.array(float(st["step"]))
        out[f"{prefix}{n}.has_grad"] = np.array(p.grad is not None)
        if p.grad is not None:
            out[f"{prefix}{n}.grad"] = p.grad.numpy().copy()
    out[f"{prefix}degrees"] = m._degrees.numpy().copy()
    for k in ("xyz_gradient_accum", "denom", "max_radii2D"):
        out[f"{prefix}{k}"] = getattr(m, k).numpy().copy()
    if hasattr(m, "density_gradient_accum"):
        out[f"{prefix}density_gradient_accum_rows"] = np.array(m.density_gradient_accum.shape[0])


CASES = {
    # name: (P, C, seed, op, kwargs, store_grads, no_state, grads_all)
    "dp_none": (300, 15, 1, "densify_and_prune", dict(max_grad=0.0002, min_opacity=0.005, extent=100.0, max_screen_size=None), False, "f_dc", False),
    "dp_screen_sg": (300, 3, 2, "densify_and_prune", dict(max_grad=0.0002, min_opacity=0.005, extent=100.0, max_screen_size=20), True, "f_dc", True),
    "dp_empty": (150, 15, 3, "densify_and_prune", dict(max_grad=1e9, min_opacity=0.005, extent=100.0, max_screen_size=None), False, None, False),
    "dp_maxgrad0": (200, 3, 4, "densify_and_prune", dict(max_grad=0.0, min_opacity=0.005, extent=100.0, max_screen_size=20), False, "opacity", False),
    "prune_screen_sg": (200, 15, 5, "prune", dict(min_opacity=0.005, extent=100.0, max_screen_size=20), True, "f_dc", False),
    "prune_none": (300, 3, 6, "prune", dict(min_opacity=1 / 255, extent=100.0, max_screen_size=None), False, None, False),
    "prune_points": (200, 15, 7, "prune_points", {}, True, "rotation", False),
    "stats": (200, 3, 8, "add_densification_stats", {}, False, None, False),
}


def run_case(gm, name):
    P, C, seed, op, kw, sg, no_state, grads_all = CASES[name]
    m = make_model(gm, P, C, seed, no_state, grads_all, cold=name == "dp_empty")
    out = {"P": np.array(P), "C": np.array(C), "op": np.array(op), "store_grads": np.array(sg)}
    for k, v in kw.items():
        out[f"arg.{k}"] = np.array(np.nan if v is None else v, dtype=np.float64)
    snapshot(m, "in.", out)
    mode = OnCpu()
    d = {}
    g = torch.Generator().manual_seed(seed + 100)
    with mode:
        if op == "densify_and_prune":
            m.densify_and_prune(kw["max_grad"], kw["min_opacity"], kw["extent"], kw["max_screen_size"], d, store_grads=sg)
        elif op == "prune":
            m.prune(kw["min_opacity"], kw["extent"], kw["max_screen_size"], d, store_grads=sg)
        elif op == "prune_points":
            mask = torch.rand(P, generator=g) < 0.3
            out["mask"] = mask.numpy()
            m.prune_points(mask, store_grads=sg)
        else:
            vs = torch.zeros(P, 3, requires_grad=True)
            vs.grad = torch.randn(P, 3, generator=g) * 1e-3
            vis = torch.rand(P, generator=g) < 0.7
            vs.grad[~vis] = 0.0
            radii = torch.randint(0, 60, (P,), generator=g, dtype=torch.int32)
            radii[~vis] = 0
            out["view_grad"], out["visibility"], out["radii"] = vs.grad.numpy().copy(), vis.numpy(), radii.numpy()
            m.max_radii2D[vis] = torch.max(m.max_radii2D[vis], radii[vis])     # train.py:134
            m.add_densification_stats(vs, vis)
    if mode.samples:
        out["samples"] = mode.samples[0].numpy()
    out["n_normal_calls"] = np.array(len(mode.samples))
    for k, v in d.items():
        out[f"dict.{k}"] = np.array(v.item() if torch.is_tensor(v) else v)
    snapshot(m, "out.", out)
    return out


def main():
    gm = import_reference_model()
    for name in CASES:
        out = run_case(gm, name)
        path = os.path.join(HERE, f"densify_{name}.npz")
        np.savez_compressed(path, **out)
        print(name, {k[5:]: int(v) for k, v in out.items() if k.startswith("dict.")}, int(out["out.xyz"].shape[0]), "rows",
              os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
