"""Loading tests/golden/densify_*.npz into a model on any device, and comparing a model with a golden's outputs."""
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
CASES = ("dp_none", "dp_screen_sg", "dp_empty", "dp_maxgrad0", "prune_screen_sg", "prune_none", "prune_points", "stats")
GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
          "rotation": "_rotation"}


class Model:
    """The attributes of the reference's GaussianModel that densification reads and writes."""
    _codebook_dict = None


def load(name):
    return dict(np.load(os.path.join(GOLDEN, f"densify_{name}.npz")))


def make_model(z, device, optimizer_cls=torch.optim.Adam):
    m = Model()
    t = lambda k: torch.from_numpy(z[k]).to(device)  # noqa: E731
    for n, a in GROUPS.items():
        setattr(m, a, torch.nn.Parameter(t(f"in.{n}")))
    m.optimizer = optimizer_cls([{"params": [getattr(m, a)], "lr": 1e-3, "name": n} for n, a in GROUPS.items()], lr=0.0, eps=1e-15)
    for n, a in GROUPS.items():
        p = getattr(m, a)
        if z[f"in.{n}.has_state"]:
            m.optimizer.state[p] = {"step": torch.tensor(float(z[f"in.{n}.step"])), "exp_avg": t(f"in.{n}.exp_avg"),
                                    "exp_avg_sq": t(f"in.{n}.exp_avg_sq")}
        if z[f"in.{n}.has_grad"]:
            p.grad = t(f"in.{n}.grad")
    m._degrees = t("in.degrees")
    m.xyz_gradient_accum, m.denom, m.max_radii2D = t("in.xyz_gradient_accum"), t("in.denom"), t("in.max_radii2D")
    m.percent_dense = 0.01
    return m


def args(z):
    a = {k[4:]: float(v) for k, v in z.items() if k.startswith("arg.")}
    if "max_screen_size" in a:
        a["max_screen_size"] = None if np.isnan(a["max_screen_size"]) else int(a["max_screen_size"])
    return a


def outputs(m):
    """{key: numpy array} of a model in the golden's "out." naming."""
    out = {}
    for g in m.optimizer.param_groups:
        n, p = g["name"], g["params"][0]
        out[n] = p.detach().cpu().numpy()
        st = m.optimizer.state.get(p, None)
        out[f"{n}.has_state"] = np.array(st is not None)
        if st is not None:
            out[f"{n}.exp_avg"], out[f"{n}.exp_avg_sq"] = st["exp_avg"].cpu().numpy(), st["exp_avg_sq"].cpu().numpy()
            out[f"{n}.step"] = np.array(float(st["step"]))
        out[f"{n}.has_grad"] = np.array(p.grad is not None)
        if p.grad is not None:
            out[f"{n}.grad"] = p.grad.cpu().numpy()
    out["degrees"] = m._degrees.cpu().numpy()
    for k in ("xyz_gradient_accum", "denom", "max_radii2D"):
        out[k] = getattr(m, k).cpu().numpy()
    if hasattr(m, "density_gradient_accum"):
        out["density_gradient_accum_rows"] = np.array(m.density_gradient_accum.shape[0])
    return out


def child_rows(z):
    """Row slice of the split children in the output: they follow the kept originals and the kept clones."""
    n = int(z["out.xyz"].shape[0])
    return slice(n - 2 * _children(z), n)


def _children(z):
    # the children are the rows whose values are not copies: count them from the output's scaling, which for a child is
    # log(exp(s) / 1.6) and so never equals an input row bit for bit in these fixtures
    ins = {r.tobytes() for r in z["in.scaling"]}
    return sum(r.tobytes() not in ins for r in z["out.scaling"]) // 2


def compare(got, z, computed_tol=None):
    """Asserts that every output equals the golden bit for bit; with computed_tol, the split children's xyz and scaling only to
    that bound relative to their largest magnitude (CPU libm / bmm against CUDA)."""
    keys = [k[4:] for k in z if k.startswith("out.")]
    assert sorted(keys) == sorted(got), (sorted(keys), sorted(got))
    kids = child_rows(z) if computed_tol is not None else None
    for k in keys:
        a, b = got[k], z[f"out.{k}"]
        assert a.shape == b.shape and a.dtype == b.dtype, (k, a.shape, b.shape, a.dtype, b.dtype)
        if kids is not None and k in ("xyz", "scaling"):
            ra, rb = a[kids], b[kids]
            err = np.abs(ra.astype(np.float64) - rb).max(initial=0) / max(np.abs(rb).max(initial=0), 1e-30)
            assert err <= computed_tol, (k, err)
            a, b = np.delete(a, np.arange(a.shape[0])[kids], axis=0), np.delete(b, np.arange(b.shape[0])[kids], axis=0)
        assert np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes(), f"{k} differs"
