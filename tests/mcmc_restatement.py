"""Restatements of gs_b200.mcmc (DESIGN.md §5n) that the tests compare the kernels with.

  * the sampler in Python integers: fixed-point weights, exact prefix, floor(d * total / 2^62), first prefix above it;
  * the relocation values of paper eq. 9 in 50-digit decimal, from the exact fp32 inputs;
  * the fp32 evaluation of D that the kernel avoids (its error is recorded below);
  * the authors' relocate_gs / add_new_gs surgery in torch, fed the sampled indices, with the relocated values evaluated in float64
    in the kernel's operation order.

Why the kernel evaluates D in double: at o = 1 - 2^-23 and N = 50 (o' = 0.2732), the issue's double sum evaluated term by term in
fp32 differs from the decimal value by FP32_D_ERROR = 6.2e-4 (relative; about 10^4 fp32 roundings), while the kernel's double loop
keeps 2.3e-13 (tests/test_mcmc_api.py measures both).
"""
import math
from decimal import Decimal, getcontext

import numpy as np
import torch

N_MAX = 50
FP32_D_ERROR = 6.2e-4        # relative error of the fp32 D at o = 1 - 2^-23, N = 50 (test_mcmc_api.py::test_fp32_D_loses_precision)


# ------------------------------------------------------------------------------------------------ sampler
def weights(o, candidates):
    """W_i = floor(o_i 2^32) (uint64) for candidate rows, 0 for the others.  o: fp32 opacities (numpy)."""
    o = np.asarray(o, dtype=np.float32).astype(np.float64)
    w = np.floor(np.nan_to_num(o, nan=0.0) * 2.0 ** 32).astype(np.uint64)
    return np.where(np.asarray(candidates, dtype=bool), w, np.uint64(0)).astype(np.uint64)


def sample(w, draws):
    """Source row of each draw (Python ints): the first row whose inclusive prefix exceeds floor(d * total / 2^62)."""
    prefix = np.cumsum(w.astype(np.uint64), dtype=np.uint64)
    total = int(prefix[-1])
    t = np.array([((int(d) % (1 << 62)) * total) >> 62 for d in draws], dtype=np.uint64)
    return np.searchsorted(prefix, t, side="right").astype(np.int64)


def sample_brute_force(w, draws):
    """The same draws by walking the CDF row by row (the definition)."""
    total = sum(int(x) for x in w)
    out = []
    for d in draws:
        t = (int(d) * total) >> 62
        acc = 0
        for i, x in enumerate(w):
            acc += int(x)
            if acc > t:
                out.append(i)
                break
    return np.array(out, dtype=np.int64)


# ------------------------------------------------------------------------------------------------ relocation values
def relocated_decimal(o, s, N, digits=50):
    """(o' clamped, [s'0, s'1, s'2], o' unclamped, D) as Decimals from the exact fp32 o and s (paper eq. 9, the double sum)."""
    getcontext().prec = digits
    o, s = Decimal(float(o)), [Decimal(float(x)) for x in s]
    one = Decimal(1)
    op = one - (one - o) ** (one / Decimal(N))
    D = Decimal(0)
    for i in range(1, N + 1):
        for k in range(i):
            D += Decimal(math.comb(i - 1, k)) * (-1) ** k * op ** (k + 1) / Decimal(k + 1).sqrt()
    oc = min(max(op, Decimal(float(np.float32(0.005)))), one - Decimal(2) ** -23)
    return oc, [x * o / D for x in s], op, D


def D_fp32(op, N):
    """The issue's double sum evaluated term by term in fp32 (numpy), as a port of the authors' float kernel would."""
    f = np.float32
    op, D = f(op), f(0)
    for i in range(1, N + 1):
        for k in range(i):
            D = f(D + f(f(math.comb(i - 1, k)) * f(f((-1) ** k) / np.sqrt(f(k + 1))) * f(op ** f(k + 1))))
    return D


def relocated_torch(o, s, N):
    """The kernel's evaluation on torch tensors: o fp32 [n], s fp32 [n, 3], N int64 [n] -> (o' clamped fp32 [n], s' fp32 [n, 3]).
    Every float64 operation is a separate torch kernel (no contraction), in the kernel's order; the binomials C(N, k + 1) are exact."""
    dev = o.device
    od, Nd = o.double(), N.double()
    op = 1.0 - torch.pow(1.0 - od, torch.ones_like(Nd) / Nd)
    table = torch.tensor([[float(math.comb(n, k + 1)) for k in range(N_MAX)] for n in range(N_MAX + 1)], dtype=torch.float64, device=dev)
    D, pw = torch.zeros_like(od), torch.ones_like(od)
    for k in range(N_MAX):
        act = k < N
        pw = torch.where(act, pw * op, pw)
        term = (table[N, k] * pw) / torch.full_like(od, math.sqrt(k + 1))
        D = torch.where(act, D - term if k & 1 else D + term, D)
    coeff = od / D
    oc = torch.clamp(op.float(), min=0.005, max=1.0 - torch.finfo(torch.float32).eps)
    return oc, (coeff.unsqueeze(1) * s.double()).float()


# ------------------------------------------------------------------------------------------------ the authors' surgery
GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
          "rotation": "_rotation"}


def _new_values(model, idx):
    """_update_params: the relocated logits and log-scales of the sampled rows idx (with repeats), N = min(bincount + 1, 50)."""
    P = model._opacity.shape[0]
    ratio = torch.bincount(idx, minlength=P)
    N = torch.clamp(ratio[idx] + 1, max=N_MAX)
    oc, sc = relocated_torch(torch.sigmoid(model._opacity.detach()[idx, 0]), torch.exp(model._scaling.detach()[idx]), N)
    return torch.log(oc / (1 - oc)).unsqueeze(1), torch.log(sc)


def relocate_gs(model, dead_mask, idx):
    """The authors' relocate_gs with the multinomial draw replaced by the source rows idx (one per dead row, in row order)."""
    dead = dead_mask.nonzero(as_tuple=True)[0]
    new_op, new_sc = _new_values(model, idx)
    with torch.no_grad():
        for n, a in GROUPS.items():
            p = getattr(model, a)
            if n == "opacity":
                p[dead] = new_op
                p[idx] = new_op
            elif n == "scaling":
                p[dead] = new_sc
                p[idx] = new_sc
            else:
                p[dead] = p[idx]
        model._degrees[dead] = model._degrees[idx]
    for g in model.optimizer.param_groups:
        st = model.optimizer.state.get(g["params"][0])
        if st is not None:
            st["exp_avg"][idx] = 0
            st["exp_avg_sq"][idx] = 0
        g["params"][0].grad = None


def add_new_gs(model, idx):
    """The authors' add_new_gs with the multinomial draw replaced by the source rows idx; -> n."""
    n = idx.numel()
    new_op, new_sc = _new_values(model, idx)
    new = {}
    with torch.no_grad():
        for name, a in GROUPS.items():
            p = getattr(model, a)
            if name == "opacity":
                p[idx] = new_op
                new[name] = new_op
            elif name == "scaling":
                p[idx] = new_sc
                new[name] = new_sc
            else:
                new[name] = p[idx]
    opt = model.optimizer
    for g in opt.param_groups:
        name, p = g["name"], g["params"][0]
        st = opt.state.get(p)
        q = torch.nn.Parameter(torch.cat([p.detach(), new[name]]).requires_grad_(True))
        if st is not None:
            st["exp_avg"][idx] = 0
            st["exp_avg_sq"][idx] = 0
            st["exp_avg"] = torch.cat([st["exp_avg"], torch.zeros_like(new[name])])
            st["exp_avg_sq"] = torch.cat([st["exp_avg_sq"], torch.zeros_like(new[name])])
            del opt.state[p]
            opt.state[q] = st
        g["params"][0] = q
        setattr(model, GROUPS[name], q)
    model._degrees = torch.cat([model._degrees, model._degrees[idx]])
    for k in ("xyz_gradient_accum", "denom", "max_radii2D", "xyz_gradient_accum_abs"):
        t = getattr(model, k, None)
        if t is not None:
            setattr(model, k, torch.cat([t, torch.zeros((n,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)]))
    return n


def noise_chain(model, eps, xyz_lr, noise_lr):
    """The authors' noise block (train.py): build_scaling_rotation, L @ L^T, the gate, bmm -> the new xyz (not applied)."""
    s, q = torch.exp(model._scaling.detach()), torch.nn.functional.normalize(model._rotation.detach())
    norm = torch.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3])
    r, x, y, z = (q / norm[:, None]).unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    L = R @ torch.diag_embed(s)
    cov = L @ L.transpose(1, 2)
    o = torch.sigmoid(model._opacity.detach())
    gate = 1 / (1 + torch.exp(-100 * ((1 - o) - 0.995)))
    noise = eps * gate * noise_lr * xyz_lr
    return model._xyz.detach() + torch.bmm(cov, noise.unsqueeze(-1)).squeeze(-1)


def noise_float64(xyz, scaling, rotation, logits, eps, xyz_lr, noise_lr):
    """(Delta64, bound term |R| s^2 |R|^T |v|) in float64 from the contract's fp32 o = sigmoid(logits), s = exp(scaling) and
    q = F.normalize(rotation) (torch's fp32 results) and the draws, with noise_lr / xyz_lr as their fp32 casts."""
    a, b = float(np.float32(noise_lr)), float(np.float32(xyz_lr))
    s = torch.exp(scaling).double()
    q = torch.nn.functional.normalize(rotation).double()
    q = q / q.norm(dim=1, keepdim=True)
    r, x, y, z = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    o = torch.sigmoid(logits).double()
    gate = 1 / (1 + torch.exp(-100 * ((1 - o) - 0.995)))
    v = eps.double() * gate * a * b
    S2 = torch.diag_embed(s * s)
    delta = (R @ S2 @ R.transpose(1, 2) @ v.unsqueeze(-1)).squeeze(-1)
    bound = (R.abs() @ S2 @ R.abs().transpose(1, 2) @ v.abs().unsqueeze(-1)).squeeze(-1)
    return delta, bound
