"""GPU probe: which fp32 formulas reproduce the torch ops of the reference's densification on CUDA bit for bit?

    python tools/probe_torch_densify.py

Covers the ops of GaussianModel.add_densification_stats / densify_and_prune / prune (DESIGN.md §5g): the norm of the first two
columns of the view-space gradient, sigmoid, log next to exp, the division of a tensor by a Python scalar, the comparisons with
Python-double thresholds, torch.normal(mean=zeros, std) against randn * std + 0 from the same seed, and the contraction order of
torch.bmm for [B, 3, 3] x [B, 3, 1] at several B (cuBLAS may choose a different kernel per batch size).  Each torch CUDA result is
compared with candidate formulas evaluated on the CPU (fp32 numpy; fma() is the exactly rounded one of probe_torch_adam.py).
Prints the mismatch count of every candidate; 0 marks torch's arithmetic.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from probe_torch_adam import fma, report  # noqa: E402

f32, f64 = np.float32, np.float64


def wide(rng, n, lo=-30, hi=10, positive=False):
    x = (10.0 ** rng.uniform(lo, hi, n)).astype(f32)
    if not positive:
        x *= rng.choice(np.array([-1, 1], f32), n)
    x[rng.random(n) < 0.02] = 0
    return x


def report_mask(name, got, cands):
    got = got.cpu().numpy()
    for cname, v in cands.items():
        print(f"{name:10s} {cname:40s} mismatches {int((got != v).sum())} / {got.size}", flush=True)


def main():
    assert torch.cuda.is_available(), "the probe needs a GPU"
    dev = torch.device("cuda")
    rng = np.random.default_rng(11)
    n = 2_000_000

    # torch.norm(grad[:, :2], dim=-1, keepdim=True) on the view-space gradient [P, 3] (add_densification_stats)
    g = wide(rng, 3 * n, -20, 5).reshape(n, 3)
    a, b = g[:, 0], g[:, 1]
    out = torch.norm(torch.from_numpy(g).to(dev)[:, :2], dim=-1, keepdim=True)[:, 0]
    report("norm", out, {"sqrt(a*a + b*b) unfused": np.sqrt(a * a + b * b), "sqrt(fma(b, b, a*a))": np.sqrt(fma(b, b, a * a)),
                         "sqrt(fma(a, a, b*b))": np.sqrt(fma(a, a, b * b)),
                         "sqrt(a*a + b*b) in double": np.sqrt(a.astype(f64) ** 2 + b.astype(f64) ** 2).astype(f32)})

    # sigmoid, exp and log (get_opacity, get_scaling, scaling_inverse_activation)
    x = rng.uniform(-20, 20, n).astype(f32)
    X = torch.from_numpy(x).to(dev)
    E = torch.exp(-X).cpu().numpy()
    report("sigmoid", torch.sigmoid(X), {"1 / (1 + torch.exp(-x)) IEEE": f32(1) / (f32(1) + E),
                                          "correctly rounded": (1 / (1 + np.exp(-x.astype(f64)))).astype(f32)})
    report("exp", torch.exp(X), {"correctly rounded": np.exp(x.astype(f64)).astype(f32)})
    pos = wide(rng, n, -30, 30, positive=True) + f32(1e-30)
    report("log", torch.log(torch.from_numpy(pos).to(dev)), {"correctly rounded": np.log(pos.astype(f64)).astype(f32),
                                                               "numpy fp32 log": np.log(pos)})

    # division by a Python scalar (exp(s) / (0.8 * N)) and by a tensor (xyz_gradient_accum / denom)
    s = wide(rng, n, -10, 10, positive=True)
    d = 0.8 * 2
    report("div 1.6", torch.from_numpy(s).to(dev) / d, {"x / fp32(1.6) IEEE": s / f32(d), "x * fp32(1 / fp32(1.6))": s * (f32(1) / f32(d)),
                                                         "x * fp32(1 / 1.6)": s * f32(1 / d)})
    den = rng.integers(0, 50, n).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        report("div tensor", torch.from_numpy(s).to(dev) / torch.from_numpy(den).to(dev), {"x / d IEEE": s / den})

    # comparisons with Python-double thresholds: values around fp32(t) and the double t itself
    for t in (0.0002, 0.01 * 3.7, 0.1 * 3.7, 0.005, 20):
        c = f32(t)
        near = np.concatenate([np.array([np.nextafter(c, f32(-1)), c, np.nextafter(c, f32(1))], f32),
                               (c * (1 + rng.uniform(-1e-6, 1e-6, 1000))).astype(f32)])
        T = torch.from_numpy(near).to(dev)
        for op, fn in ((">=", np.greater_equal), ("<=", np.less_equal), (">", np.greater), ("<", np.less)):
            res = {">=": T >= t, "<=": T <= t, ">": T > t, "<": T < t}[op]
            report_mask(f"x {op} {t:g}", res, {"against fp32(t)": fn(near, c), "against double t": fn(near.astype(f64), t)})

    # torch.normal(mean=zeros, std) against randn * std + 0 drawn from the same generator state
    std = torch.from_numpy(wide(rng, 3 * 200_000, -3, 1, positive=True).reshape(-1, 3)).to(dev)
    torch.manual_seed(5)
    a_ = torch.normal(mean=torch.zeros_like(std), std=std)
    st_a = torch.cuda.get_rng_state()
    torch.manual_seed(5)
    b_ = torch.randn_like(std) * std + 0
    st_b = torch.cuda.get_rng_state()
    report("normal", a_, {"randn * std + 0": b_.cpu().numpy()})
    print(f"normal     generator state after both equal: {bool(torch.equal(st_a, st_b))}", flush=True)

    # bmm [B, 3, 3] x [B, 3, 1] (split children: rots @ samples)
    for B in (1, 2, 3, 17, 100, 1000, 4096, 65536, 150_000, 300_000):
        R = rng.uniform(-1, 1, (B, 3, 3)).astype(f32)
        v = rng.normal(0, 1, (B, 3)).astype(f32) * (10.0 ** rng.uniform(-4, 1, (B, 1))).astype(f32)
        out = torch.bmm(torch.from_numpy(R).to(dev), torch.from_numpy(v).to(dev).unsqueeze(-1)).squeeze(-1)
        r0, r1, r2 = R[:, :, 0], R[:, :, 1], R[:, :, 2]
        x0, x1, x2 = v[:, None, 0], v[:, None, 1], v[:, None, 2]
        report(f"bmm B={B}", out.reshape(-1), {
            "fma(r2,x2, fma(r1,x1, r0*x0))": fma(r2, x2, fma(r1, x1, r0 * x0)).reshape(-1),
            "fma(r2,x2, fma(r1,x1, fma(r0,x0,0)))": fma(r2, x2, fma(r1, x1, fma(r0, x0, f32(0)))).reshape(-1),
            "fma(r0,x0, fma(r1,x1, r2*x2))": fma(r0, x0, fma(r1, x1, r2 * x2)).reshape(-1),
            "(r0*x0 + r1*x1) + r2*x2 unfused": ((r0 * x0 + r1 * x1) + r2 * x2).reshape(-1),
            "double sum, rounded once": (r0.astype(f64) * x0 + r1.astype(f64) * x1 + r2.astype(f64) * x2).astype(f32).reshape(-1)})


if __name__ == "__main__":
    main()
