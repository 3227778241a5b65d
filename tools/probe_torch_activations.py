"""GPU probe: which fp32 formulas reproduce the backward of torch's exp() and F.normalize() on CUDA bit for bit?

    python tools/probe_torch_activations.py

`render()` with `pipe.fused_activations` differentiates get_scaling = exp(_scaling) and get_rotation = F.normalize(_rotation)
inside the preprocess backward (DESIGN.md §5h).  Autograd runs ExpBackward0, then for the rotation DivBackward0 (both inputs),
ExpandBackward0 (a sum over the four components), ClampMinBackward0 and LinalgVectorNormBackward0.  Each candidate below is a
restatement in single torch elementwise ops (every op one IEEE fp32 rounding); 0 mismatches marks torch's arithmetic.
Quaternion norms span 1e-30 to 1e+10, with exact zeros and norms below the 1e-12 clamp.
"""
import numpy as np
import torch
import torch.nn.functional as F


def report(name, got, cands):
    for cname, v in cands.items():
        bad = int(((v.view(torch.int32) != got.view(torch.int32)) & ~(torch.isnan(v) & torch.isnan(got))).sum())
        print(f"{name:10s} {cname:52s} mismatches {bad} / {got.numel()}", flush=True)


def main():
    assert torch.cuda.is_available(), "the probe needs a GPU"
    dev = torch.device("cuda")
    print("device:", torch.cuda.get_device_name(dev), "torch", torch.__version__, flush=True)
    gen = torch.Generator().manual_seed(11)
    n = 2_000_000

    # ExpBackward0: grad * result
    x = (torch.rand(n, generator=gen) * 20 - 10).to(dev).requires_grad_()
    g = torch.randn(n, generator=gen).to(dev)
    y = torch.exp(x)
    y.backward(g)
    with torch.no_grad():
        report("exp", x.grad, {"g * exp(x)": g * y, "exp(x) * g": y * g})

    # F.normalize(q, dim=1): q / clamp_min(||q||, 1e-12)
    P = n // 4
    q = torch.randn(P, 4, generator=gen) * torch.pow(10.0, torch.empty(P, 1).uniform_(-30, 10, generator=gen))
    q[: P // 100] = 0
    q[P // 100: P // 50] *= 1e-14 / q[P // 100: P // 50].norm(dim=1, keepdim=True)
    q = q[torch.randperm(P, generator=gen)].to(dev).requires_grad_()
    g = torch.randn(P, 4, generator=gen).to(dev)
    out = F.normalize(q)
    out.backward(g)
    with torch.no_grad():
        nrm = q.norm(dim=1, keepdim=True)
        d = nrm.clamp_min(1e-12)
        report("normalize", out, {"fwd: q / max(norm, 1e-12)": q / d})
        gs = g / d                                                   # DivBackward0, self
        go = -g * ((q / d) / d)                                      # DivBackward0, other
        sums = {"((g0+g1)+g2)+g3": ((go[:, 0] + go[:, 1]) + go[:, 2]) + go[:, 3],
                "(g0+g2)+(g1+g3)": (go[:, 0] + go[:, 2]) + (go[:, 1] + go[:, 3]),
                "(g0+g1)+(g2+g3)": (go[:, 0] + go[:, 1]) + (go[:, 2] + go[:, 3])}
        for sname, s in sums.items():
            gn = torch.where(nrm >= 1e-12, s[:, None], torch.zeros_like(nrm))   # ClampMinBackward0
            cands = {}
            for fname, gq in (("gn * (q / n)", gn * (q / nrm)), ("q * (gn / n)", q * (gn / nrm)), ("(q * gn) / n", (q * gn) / nrm)):
                gq = torch.where(nrm == 0, torch.zeros_like(gq), gq)            # LinalgVectorNormBackward0 masks norm == 0
                cands[f"sum {sname}, {fname}"] = gs + gq
            report("normalize", q.grad, cands)


if __name__ == "__main__":
    main()
