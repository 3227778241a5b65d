"""Golden mercy fixtures written by the reference's OWN GaussianModel.mercy_points (scene/gaussian_model.py:524-551), imported
from the reference checkout ($GS_REFERENCE_ROOT) and run on the CPU of the build container.  Writes tests/golden/mercy_<case>.npz.

    python tests/golden/make_golden_mercy.py

What is NOT the reference here, and why: the module is imported with the stubs of make_golden_ply.py (no GPU, no extensions);
a TorchFunctionMode sends the reference's `device="cuda"` factory calls to the CPU and records what torch.rand returned, so a
test can substitute the same draws; prune_points is replaced on the instance by a recorder of its mask (the prune itself is
gs_b200.densify.prune_points, checked by the densification goldens).  Every case's exact threshold (mean + lambda * std in
fp64) lies at least 1e-4 from an integer, or std is 0, so fp32 rounding of the statistics cannot move a row (asserted here and
in tests/test_mercy_api.py).
"""
import os
import sys

import numpy as np
import torch
from torch.overrides import TorchFunctionMode

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_ply import import_reference_model  # noqa: E402


class OnCpu(TorchFunctionMode):
    """Redirects device="cuda" to the CPU and records torch.rand's results."""

    def __init__(self):
        super().__init__()
        self.draws = []

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = dict(kwargs or {})
        if str(kwargs.get("device", "")).startswith("cuda"):
            kwargs["device"] = "cpu"
        out = func(*args, **kwargs)
        if func is torch.rand:
            self.draws.append(out.detach().clone())
        return out


def exact_threshold(c, lam):
    c = np.asarray(c, np.float64)
    if c.size < 2:
        return float("nan")
    return c.mean() + lam * c.std(ddof=1)


# name: (P, type, lambda, mercy_minimum, counts spec, logits spec)
CASES = {
    "ro_odd": (301, "redundancy_opacity", 1.0, 2, "poisson", "normal"),
    "ro_even_ties": (400, "redundancy_opacity", 1.0, 2, "poisson", "ties"),
    "ro_min_wins": (300, "redundancy_opacity", 0.1, 6, "poisson", "normal"),
    "random": (500, "redundancy_random", 1.0, 2, "poisson", "normal"),
    "random_none": (200, "redundancy_random", 2.0, 50, "poisson", "normal"),
    "opacity_int_rank": (201, "opacity", 2.0, 2, "poisson", "normal"),
    "opacity_frac_rank": (300, "opacity", 2.0, 2, "poisson", "normal"),
    "opacity_nan": (300, "opacity", 2.0, 2, "poisson", "nan"),
    "roo": (300, "redundancy_opacity_opacity", 1.0, 2, "poisson", "normal"),
    "roo_nan": (300, "redundancy_opacity_opacity", 1.0, 2, "poisson", "nan"),
    "ro_nan": (300, "redundancy_opacity", 1.0, 2, "poisson", "nan"),
    "other": (300, "none", 1.0, 2, "poisson", "normal"),
    "std0": (128, "redundancy_opacity", 2.0, 2, "equal", "normal"),
    "p1": (1, "other", 2.0, 2, "poisson", "normal"),
    "none_redundant": (250, "redundancy_opacity", 2.0, 40, "poisson", "normal"),
}


def make_inputs(name, P, cspec, ospec, lam, seed):
    g = torch.Generator().manual_seed(seed)
    if cspec == "equal":
        c = torch.full((P,), 5, dtype=torch.int32)
    else:
        c = torch.poisson(torch.full((P,), 4.0), generator=g).to(torch.int32) + 1
    logits = torch.randn(P, 1, generator=g) * 2
    if ospec == "ties":
        logits = torch.randint(-3, 4, (P, 1), generator=g).float()      # many equal opacities, also at the median
    if ospec == "nan":
        logits[int(c.argmax())] = float("nan")                        # a redundant row: the median is NaN too
    return c, logits


def run_case(gm, name, spec):
    P, mtype, lam, mmin, cspec, ospec = spec
    seed = 11
    while True:
        c, logits = make_inputs(name, P, cspec, ospec, lam, seed)
        t = exact_threshold(c.numpy(), lam)
        if cspec == "equal" or P < 2 or abs(t - round(t)) >= 1e-4:
            break
        seed += 1
    m = gm.GaussianModel(3)
    m._opacity = torch.nn.Parameter(logits.clone())
    m._splatted_num_accum = c.view(P, 1, 1).clone()
    seen = {}
    m.prune_points = lambda mask, store_grads=False: seen.__setitem__("mask", mask.clone())
    d = {}
    mode = OnCpu()
    with mode:
        m.mercy_points(d, lam, mmin, mtype)
    ot = d["opacity_threshold"]
    out = {"P": np.int64(P), "type": np.array(mtype), "lambda": np.float64(lam), "mercy_minimum": np.float64(mmin),
           "seed": np.int64(seed), "counts": c.numpy(), "logits": logits.numpy(),
           "mask": seen["mask"].reshape(-1).numpy().astype(bool),
           "n_points_mercied": d["n_points_mercied"].numpy(), "redundancy_threshold": d["redundancy_threshold"].numpy(),
           "opacity_threshold_is_tensor": np.bool_(torch.is_tensor(ot)),
           "opacity_threshold": ot.detach().numpy() if torch.is_tensor(ot) else np.float32(ot),
           "draws": mode.draws[0].reshape(-1).numpy() if mode.draws else np.zeros(0, np.float32),
           "n_draw_calls": np.int64(len(mode.draws)),
           "n_redundant": np.int64(int((c.float() > max(float(d["redundancy_threshold"].reshape(-1)[0]), mmin)).sum())),
           "exact_threshold": np.float64(exact_threshold(c.numpy(), lam))}
    np.savez(os.path.join(HERE, f"mercy_{name}.npz"), **out)
    print(f"{name}: P={P} type={mtype} mercied={int(out['n_points_mercied'])} thr={float(out["redundancy_threshold"].reshape(-1)[0]):.6f} "
          f"opacity_thr={out['opacity_threshold']} draws={out['draws'].size} redundant={int(out['n_redundant'])}")


def main():
    gm = import_reference_model()
    for name, spec in CASES.items():
        run_case(gm, name, spec)


if __name__ == "__main__":
    main()
