"""A/B timing of gs_b200.mcmc (DESIGN.md §5n) at 1 M and 3 M Gaussians with C3 positions:

  noise   mcmc.inject_noise against the authors' torch block (build_scaling_rotation, L @ L^T, the gate, bmm, add_) on the same draws;
  reloc   mcmc.relocate_gs + mcmc.add_new_gs at about 5 % dead rows against the authors' relocate_gs / add_new_gs in torch
          (nonzero, multinomial, bincount, the relocation in fp32 torch ops, the indexed writes and the optimizer surgery).

CUDA events per step, the arms alternated (benchkit.time_arms), the L2 flushed in front of every step; each step starts from the
same model state.  Prints the card banner and one JSON line per size.

    python tools/bench_mcmc.py [--sizes 1000000 3000000] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import benchkit  # noqa: E402  (puts the repository on sys.path)

from gs_b200 import mcmc, synth  # noqa: E402
from gs_b200.optim import GaussianAdam  # noqa: E402

GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
          "rotation": "_rotation"}


class Model:
    _codebook_dict = None


def make_model(P, dev):
    """C3's scene (positions, scales, rotations, SH) with about 5 % of the opacities below the dead threshold, and Adam state."""
    s = synth.config_scene("C3", P)
    m = Model()
    g = torch.Generator().manual_seed(1)
    op = s.opacity.clone()
    op[torch.rand(P, generator=g) < 0.05] = -7.0
    vals = dict(xyz=s.means3D, f_dc=s.sh[:, :1], f_rest=s.sh[:, 1:16], opacity=op.view(P, 1), scaling=torch.log(s.scales),
                rotation=s.rotations)
    for n, a in GROUPS.items():
        setattr(m, a, torch.nn.Parameter(vals[n].contiguous().to(dev)))
    m.optimizer = GaussianAdam([{"params": [getattr(m, a)], "lr": 1e-3, "name": n} for n, a in GROUPS.items()], lr=0.0, eps=1e-15)
    for n, a in GROUPS.items():
        p = getattr(m, a)
        m.optimizer.state[p] = {"step": torch.tensor(100.0), "exp_avg": torch.randn_like(p) * 1e-4, "exp_avg_sq": torch.rand_like(p) * 1e-8}
    m._degrees = torch.full((P, 1), 3, dtype=torch.int32, device=dev)
    m.xyz_gradient_accum, m.denom = torch.zeros(P, 1, device=dev), torch.zeros(P, 1, device=dev)
    m.max_radii2D = torch.zeros(P, device=dev)
    return m


def fresh(src):
    m = Model()
    for a in GROUPS.values():
        setattr(m, a, torch.nn.Parameter(getattr(src, a).detach().clone()))
    m.optimizer = GaussianAdam([{"params": [getattr(m, a)], "lr": 1e-3, "name": n} for n, a in GROUPS.items()], lr=0.0, eps=1e-15)
    for a in GROUPS.values():
        st = src.optimizer.state[getattr(src, a)]
        m.optimizer.state[getattr(m, a)] = {k: v.clone() for k, v in st.items()}
    for k in ("_degrees", "xyz_gradient_accum", "denom", "max_radii2D"):
        setattr(m, k, getattr(src, k).clone())
    return m


# ------------------------------------------------------------------------------------------------ the authors' torch code
def torch_noise(m, eps, xyz_lr, noise_lr=5e5):
    s, r = torch.exp(m._scaling), torch.nn.functional.normalize(m._rotation)
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = torch.zeros((q.size(0), 3, 3), device=q.device)
    rr, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - rr * z); R[:, 0, 2] = 2 * (x * z + rr * y)   # noqa: E702
    R[:, 1, 0] = 2 * (x * y + rr * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - rr * x)   # noqa: E702
    R[:, 2, 0] = 2 * (x * z - rr * y); R[:, 2, 1] = 2 * (y * z + rr * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)   # noqa: E702
    L = torch.zeros((s.shape[0], 3, 3), device=s.device)
    L[:, 0, 0], L[:, 1, 1], L[:, 2, 2] = s[:, 0], s[:, 1], s[:, 2]
    L = R @ L
    cov = L @ L.transpose(1, 2)
    gate = 1 / (1 + torch.exp(-100 * ((1 - torch.sigmoid(m._opacity)) - 0.995)))
    noise = torch.bmm(cov, (eps * gate * noise_lr * xyz_lr).unsqueeze(-1)).squeeze(-1)
    m._xyz.add_(noise)


def _torch_relocation(o, s, N):
    """The authors' compute_relocation (their CUDA kernel) restated in fp32 torch ops, vectorised over k."""
    op = 1 - torch.pow(1 - o, 1.0 / N)
    k = torch.arange(50, device=o.device, dtype=torch.float32)
    binom = torch.exp(torch.lgamma(N[:, None] + 1) - torch.lgamma(k + 2) - torch.lgamma(N[:, None] - k))
    terms = torch.where(k < N[:, None], binom * (-1) ** k * op[:, None] ** (k + 1) / torch.sqrt(k + 1), torch.zeros(()))
    D = terms.sum(1)
    return op, s * (o / D)[:, None]


def _update_params(m, idx, ratio):
    N = torch.clamp(ratio[idx, 0] + 1, max=50).float()
    op, sc = _torch_relocation(torch.sigmoid(m._opacity)[idx, 0], torch.exp(m._scaling)[idx], N)
    op = torch.clamp(op.unsqueeze(-1), max=1.0 - torch.finfo(torch.float32).eps, min=0.005)
    return (m._xyz[idx], m._features_dc[idx], m._features_rest[idx], torch.log(op / (1 - op)), torch.log(sc), m._rotation[idx])


def _replace(m, tensors, inds):
    for g in m.optimizer.param_groups:
        st = m.optimizer.state.get(g["params"][0])
        st["exp_avg"][inds] = 0
        st["exp_avg_sq"][inds] = 0
        del m.optimizer.state[g["params"][0]]
        g["params"][0] = torch.nn.Parameter(tensors[g["name"]].requires_grad_(True))
        m.optimizer.state[g["params"][0]] = st
        setattr(m, GROUPS[g["name"]], g["params"][0])


def _sample(probs, num, alive=None):
    probs = probs / (probs.sum() + torch.finfo(torch.float32).eps)
    idx = torch.multinomial(probs, num, replacement=True)
    if alive is not None:
        idx = alive[idx]
    return idx, torch.bincount(idx).unsqueeze(-1)


@torch.no_grad()
def torch_relocate_add(m, cap_max):
    dead = (torch.sigmoid(m._opacity) <= 0.005).squeeze(-1)
    dead_idx, alive_idx = dead.nonzero(as_tuple=True)[0], (~dead).nonzero(as_tuple=True)[0]
    idx, ratio = _sample(torch.sigmoid(m._opacity)[alive_idx, 0], dead_idx.shape[0], alive_idx)
    xyz, fdc, frest, op, sc, rot = _update_params(m, idx, ratio)
    m._xyz[dead_idx], m._features_dc[dead_idx], m._features_rest[dead_idx] = xyz, fdc, frest
    m._opacity[dead_idx], m._scaling[dead_idx], m._rotation[dead_idx] = op, sc, rot
    m._opacity[idx], m._scaling[idx] = m._opacity[dead_idx], m._scaling[dead_idx]
    _replace(m, {n: getattr(m, a).detach() for n, a in GROUPS.items()}, idx)
    P = m._opacity.shape[0]
    n = max(0, min(cap_max, int(1.05 * P)) - P)
    idx, ratio = _sample(torch.sigmoid(m._opacity).squeeze(-1), n)
    xyz, fdc, frest, op, sc, rot = _update_params(m, idx, ratio)
    m._opacity[idx], m._scaling[idx] = op, sc
    new = dict(xyz=xyz, f_dc=fdc, f_rest=frest, opacity=op, scaling=sc, rotation=rot)
    for g in m.optimizer.param_groups:                                            # densification_postfix's cat_tensors_to_optimizer
        st = m.optimizer.state[g["params"][0]]
        st["exp_avg"] = torch.cat([st["exp_avg"], torch.zeros_like(new[g["name"]])])
        st["exp_avg_sq"] = torch.cat([st["exp_avg_sq"], torch.zeros_like(new[g["name"]])])
        p = g["params"][0]
        del m.optimizer.state[p]
        g["params"][0] = torch.nn.Parameter(torch.cat([p.detach(), new[g["name"]]]).requires_grad_(True))
        m.optimizer.state[g["params"][0]] = st
        setattr(m, GROUPS[g["name"]], g["params"][0])
    _replace(m, {n: getattr(m, a).detach() for n, a in GROUPS.items()}, idx)
    m._degrees = torch.cat([m._degrees, m._degrees[idx]])
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev = benchkit.device("bench_mcmc")
    benchkit.banner(tool="bench_mcmc")
    flush = benchkit.l2_flush(dev)
    for P in a.sizes:
        base = make_model(P, dev)
        eps = torch.randn(P, 3, device=dev)
        nm, tm = fresh(base), fresh(base)

        def native_noise(i):
            mcmc.inject_noise(nm, 1.6e-4)

        def authors_noise(i):
            with torch.no_grad():
                torch_noise(tm, eps, 1.6e-4)
        noise = benchkit.time_arms({"native": native_noise, "torch": authors_noise}, a.steps, a.warmup, flush)

        def native_reloc(i):
            m = fresh(base)
            torch.cuda.synchronize()
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            mcmc.relocate_gs(m)
            mcmc.add_new_gs(m, 10 * P)
            e1.record()
            return e0, e1

        def authors_reloc(i):
            m = fresh(base)
            torch.cuda.synchronize()
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            torch_relocate_add(m, 10 * P)
            e1.record()
            return e0, e1
        reloc = {"native": [], "torch": []}
        for i in range(a.warmup + a.steps):
            for k, fn in (("native", native_reloc), ("torch", authors_reloc))[:: 1 if i % 2 == 0 else -1]:
                e0, e1 = fn(i)
                torch.cuda.synchronize()
                if i >= a.warmup:
                    reloc[k].append(e0.elapsed_time(e1))
        med = lambda v: round(statistics.median(v), 4)  # noqa: E731
        print(json.dumps({"P": P, "dead_fraction": round(float((torch.sigmoid(base._opacity) <= 0.005).float().mean()), 4),
                          "noise_ms": {k: med(v) for k, v in noise.items()},
                          "relocate_add_ms": {k: med(v) for k, v in reloc.items()}, "steps": a.steps}), flush=True)
        del base, nm, tm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
