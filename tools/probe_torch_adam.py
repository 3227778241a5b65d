"""GPU probe: which fp32 formulas reproduce torch.optim.Adam's default (foreach) CUDA step bit for bit?

    python tools/probe_torch_adam.py

Each of the seven foreach passes of torch's _multi_tensor_adam (non-capturable branch) is run on its own over 2 M elements with
exponents from 1e-30 to 1e+10, exact zeros and mixed signs, and compared with candidate formulas evaluated on the CPU (fp32
numpy; a contracted multiply-add is the exactly rounded fma() below: the product of two fp32 values is exact in double, and the
double rounding of the sum is corrected with TwoSum).  Then three whole torch.optim.Adam steps are compared with the chain of
the matching candidates, and with GaussianAdam.  Prints the mismatch count of every candidate; 0 marks torch's arithmetic.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "reduced-3dgs_b200"))
from gs_b200.optim import GaussianAdam  # noqa: E402

f32, f64 = np.float32, np.float64


def fma(a, b, c):
    """Exactly rounded fp32 fma(a, b, c).  a*b is exact in double; s = p + c is not always, and rounding s to fp32 would round
    twice.  Since every fp32 rounding midpoint is a double, RN_double cannot carry the exact sum across one: the two roundings
    differ only when s lands exactly on a midpoint while the exact sum does not.  TwoSum gives the exact error e of s; on a
    midpoint with e != 0, s moves one double ulp towards the exact sum first."""
    p = np.asarray(a, f32).astype(f64) * np.asarray(b, f32).astype(f64)
    c = np.asarray(c, f32).astype(f64)
    with np.errstate(over="ignore", invalid="ignore"):
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        r = s.astype(f32)
        other = np.nextafter(r, np.where(s > r.astype(f64), f32(np.inf), f32(-np.inf)).astype(f32))
        tie = (s != r.astype(f64)) & (s == (r.astype(f64) + other.astype(f64)) * 0.5) & (e != 0)
        s = np.where(tie, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(f32)


def wide(rng, n, positive=False):
    x = (10.0 ** rng.uniform(-30, 10, n)).astype(f32)
    if not positive:
        x *= rng.choice(np.array([-1, 1], f32), n)
    x[rng.random(n) < 0.02] = 0
    return x


def report(name, got, cands):
    got = got.cpu().numpy()
    for cname, v in cands.items():
        bad = int(((v.view(np.uint32) != got.view(np.uint32)) & ~(np.isnan(v) & np.isnan(got))).sum())
        print(f"{name:10s} {cname:40s} mismatches {bad} / {got.size}", flush=True)


def main():
    assert torch.cuda.is_available(), "the probe needs a GPU"
    dev = torch.device("cuda")
    rng = np.random.default_rng(7)
    n = 2_000_000
    g, m, p = wide(rng, n), wide(rng, n), wide(rng, n)
    v = wide(rng, n, positive=True)
    G, M, V, Pt = (torch.from_numpy(a).to(dev) for a in (g, m, v, p))
    beta1, beta2, eps, lr = 0.9, 0.999, 1e-15, 1.6e-4

    for w in (1 - beta1, 1 - 0.3):               # both branches of ATen's lerp (|w| < 0.5 and not)
        out = M.clone()
        torch._foreach_lerp_([out], [G], w)
        wf = f32(w)
        d = g - m
        report(f"lerp w={w:.1f}", out, {"fma(w, g-m, m)": fma(wf, d, m), "m + w*(g-m) unfused": m + wf * d,
                                          "fma(-(g-m), 1-w, g)": fma(-d, f32(1) - wf, g), "g - (g-m)*(1-w) unfused": g - d * (f32(1) - wf)})
    out = V.clone()
    torch._foreach_mul_([out], beta2)
    report("mul", out, {"v*beta2": v * f32(beta2)})
    vb = v * f32(beta2)
    out = torch.from_numpy(vb).to(dev)
    torch._foreach_addcmul_([out], [G], [G], 1 - beta2)
    c = f32(1 - beta2)
    report("addcmul", out, {"fma(c, g*g, v)": fma(c, g * g, vb), "v + c*(g*g) unfused": vb + c * (g * g), "fma(c*g, g, v)": fma(c * g, g, vb)})
    (out,) = torch._foreach_sqrt([V])
    report("sqrt", out, {"sqrt (IEEE)": np.sqrt(v)})
    sq = np.sqrt(v)
    for step in (1, 7, 1000):
        bc2_sqrt = (1 - beta2 ** step) ** 0.5
        out = torch.from_numpy(sq).to(dev)
        torch._foreach_div_([out], [bc2_sqrt])
        report(f"div t={step}", out, {"x / s (IEEE)": sq / f32(bc2_sqrt), "x * fp32(1/fp32(s))": sq * (f32(1) / f32(bc2_sqrt)),
                                      "x * fp32(1/s) (double reciprocal)": sq * f32(1 / bc2_sqrt)})
    out = torch.from_numpy(sq).to(dev)
    torch._foreach_add_([out], eps)
    report("add eps", out, {"x + eps": sq + f32(eps)})
    den = (np.abs(wide(rng, n, positive=True)) + f32(1e-20)).astype(f32)
    for step in (1, 1000):
        step_size = (lr / (1 - beta1 ** step)) * -1
        out = Pt.clone()
        torch._foreach_addcdiv_([out], [M], [torch.from_numpy(den).to(dev)], [step_size])
        s = f32(step_size)
        report(f"addcdiv t={step}", out, {"fma(s, m/d, p)": fma(s, m / den, p), "p + s*(m/d) unfused": p + s * (m / den),
                                          "p + (s*m)/d": p + (s * m) / den})

    # three whole steps: torch.optim.Adam vs the chain of the candidates above vs GaussianAdam
    shape = (n // 4, 4)
    P0, M0 = torch.from_numpy(p).reshape(shape), torch.zeros(shape)
    grads = [torch.from_numpy(wide(rng, n)).reshape(shape) for _ in range(3)]
    ref = P0.to(dev).clone().requires_grad_(True)
    ours = P0.to(dev).clone().requires_grad_(True)
    opt_t = torch.optim.Adam([ref], lr=lr, betas=(beta1, beta2), eps=eps)
    opt_o = GaussianAdam([ours], lr=lr, betas=(beta1, beta2), eps=eps)
    pe, me, ve = P0.numpy().copy(), M0.numpy().copy(), M0.numpy().copy()
    for t, gr in enumerate(grads, 1):
        ref.grad, ours.grad = gr.to(dev), gr.to(dev)
        opt_t.step()
        opt_o.step()
        gn = gr.numpy()
        me = fma(f32(1 - beta1), gn - me, me)
        ve = fma(f32(1 - beta2), gn * gn, ve * f32(beta2))
        d = np.sqrt(ve) / f32((1 - beta2 ** t) ** 0.5) + f32(eps)
        pe = fma(f32((lr / (1 - beta1 ** t)) * -1), me / d, pe)
    st = opt_t.state[ref]
    report("adam x3", ref.detach(), {"param: candidate chain": pe})
    report("adam x3", st["exp_avg"], {"exp_avg: candidate chain": me})
    report("adam x3", st["exp_avg_sq"], {"exp_avg_sq: candidate chain": ve})
    so = opt_o.state[ours]
    report("adam x3", ref.detach(), {"param: GaussianAdam": ours.detach().cpu().numpy()})
    report("adam x3", st["exp_avg"], {"exp_avg: GaussianAdam": so["exp_avg"].cpu().numpy()})
    report("adam x3", st["exp_avg_sq"], {"exp_avg_sq: GaussianAdam": so["exp_avg_sq"].cpu().numpy()})


if __name__ == "__main__":
    main()
