"""A torch restatement of the reference's densification (GaussianModel.densify_and_prune / prune / prune_points /
add_densification_stats and train.py:134), written from the contract in DESIGN.md §5g, on whatever device the model lives.

It is what gs_b200.densify is compared with on the GPU: test_densify_api.py shows on the CPU that it reproduces the goldens the
reference's own code wrote (tests/golden/make_golden_densify.py), so the GPU tests can run it on the same device as the kernels.
A model is any object with the reference's attribute names and a torch.optim.Adam-compatible optimizer with the six named groups.
"""
import torch
from torch import nn

GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
          "rotation": "_rotation"}


def rotation_matrices(q):
    """Unit-quaternion (r, x, y, z) rotation matrices; every elementwise torch op rounds on its own."""
    norm = torch.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3])
    q = q / norm[:, None]
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros((q.size(0), 3, 3), device=q.device)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - r * z)
    R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y)
    R[:, 2, 1] = 2 * (y * z + r * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _params(m):
    return {g["name"]: g["params"][0] for g in m.optimizer.param_groups}


def _set_params(m, params):
    for g in m.optimizer.param_groups:
        g["params"][0] = params[g["name"]]
        setattr(m, GROUPS[g["name"]], params[g["name"]])


def _keep_rows(m, keep, store_grads):
    """Rows `keep` (bool) of every param, its moments (state moved to the new Parameter) and, with state and store_grads, its grad;
    a group without state only gets its param.  _degrees and the three statistics are indexed too."""
    opt, new = m.optimizer, {}
    for name, p in _params(m).items():
        st = opt.state.get(p, None)
        q = nn.Parameter(p.detach()[keep].requires_grad_(True))
        if st is not None:
            st["exp_avg"], st["exp_avg_sq"] = st["exp_avg"][keep], st["exp_avg_sq"][keep]
            if store_grads:
                q.grad = p.grad[keep]
            del opt.state[p]
            opt.state[q] = st
        new[name] = q
    _set_params(m, new)
    m._degrees = m._degrees[keep]
    m.xyz_gradient_accum, m.denom, m.max_radii2D = m.xyz_gradient_accum[keep], m.denom[keep], m.max_radii2D[keep]


def _append_rows(m, ext, store_grads):
    """Appends ext[name] to every param; new rows get zero moments and, with store_grads, zero grads."""
    opt, new = m.optimizer, {}
    for name, p in _params(m).items():
        st = opt.state.get(p, None)
        q = nn.Parameter(torch.cat((p.detach(), ext[name]), dim=0).requires_grad_(True))
        if store_grads:
            q.grad = torch.cat((p.grad, torch.zeros_like(ext[name])), dim=0)
        if st is not None:
            st["exp_avg"] = torch.cat((st["exp_avg"], torch.zeros_like(ext[name])), dim=0)
            st["exp_avg_sq"] = torch.cat((st["exp_avg_sq"], torch.zeros_like(ext[name])), dim=0)
            del opt.state[p]
            opt.state[q] = st
        new[name] = q
    _set_params(m, new)
    m._degrees = torch.cat((m._degrees, ext["degrees"]), dim=0)
    n, dev = m._xyz.shape[0], m._xyz.device
    m.xyz_gradient_accum = torch.zeros((n, 1), device=dev)
    m.density_gradient_accum = torch.zeros((n, 1), device=dev)
    m.denom = torch.zeros((n, 1), device=dev)
    m.max_radii2D = torch.zeros((n), device=dev)


def prune_points(m, mask, store_grads=False):
    _keep_rows(m, ~mask, store_grads)


def prune(m, min_opacity, extent, max_screen_size, d, store_grads=False):
    mask = (torch.sigmoid(m._opacity) < min_opacity).squeeze()
    if max_screen_size:
        mask = mask | (m.max_radii2D > max_screen_size) | (torch.exp(m._scaling).max(dim=1).values > 0.1 * extent)
    d["n_points_pruned"] = mask.sum()
    prune_points(m, mask, store_grads)


def densify_and_prune(m, max_grad, min_opacity, extent, max_screen_size, d, store_grads=False, normal=torch.normal):
    grads = m.xyz_gradient_accum / m.denom
    grads[grads.isnan()] = 0.0
    dev = m._xyz.device
    # clone
    sel = (grads.squeeze(1) >= max_grad) & (torch.exp(m._scaling).max(dim=1).values <= m.percent_dense * extent)
    n_cloned = int(sel.sum().item())
    p = _params(m)
    _append_rows(m, {**{k: v.detach()[sel] for k, v in p.items()}, "degrees": m._degrees[sel]}, store_grads)
    # split, over the rows after the clone with zero grads for the clones
    padded = torch.zeros((m._xyz.shape[0]), device=dev)
    padded[:grads.shape[0]] = grads.squeeze(1)
    sel = (padded >= max_grad) & (torch.exp(m._scaling).max(dim=1).values > m.percent_dense * extent)
    n_split = int(sel.sum().item())
    p = {k: v.detach() for k, v in _params(m).items()}
    stds = torch.exp(p["scaling"])[sel].repeat(2, 1)
    samples = normal(mean=torch.zeros((stds.size(0), 3), device=dev), std=stds)
    rots = rotation_matrices(p["rotation"][sel]).repeat(2, 1, 1)
    ext = {"xyz": torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + p["xyz"][sel].repeat(2, 1),
           "scaling": torch.log(torch.exp(p["scaling"])[sel].repeat(2, 1) / (0.8 * 2)),
           "rotation": p["rotation"][sel].repeat(2, 1), "f_dc": p["f_dc"][sel].repeat(2, 1, 1),
           "f_rest": p["f_rest"][sel].repeat(2, 1, 1), "opacity": p["opacity"][sel].repeat(2, 1), "degrees": m._degrees[sel].repeat(2, 1)}
    _append_rows(m, ext, store_grads)
    # the split parents go; a group without state loses its grad here (prune_points does not carry it)
    prune_points(m, torch.cat((sel, torch.zeros(2 * n_split, device=dev, dtype=torch.bool))), store_grads)
    prune(m, min_opacity, extent, max_screen_size, d, store_grads)
    d["n_points_cloned"] = n_cloned
    d["n_points_split"] = n_split


def add_densification_stats(m, viewspace_point_tensor, update_filter, radii=None):
    if radii is not None:                                     # train.py:134
        m.max_radii2D[update_filter] = torch.max(m.max_radii2D[update_filter], radii[update_filter])
    m.xyz_gradient_accum += torch.norm(viewspace_point_tensor.grad[:, :2], dim=-1, keepdim=True)
    m.denom += update_filter.unsqueeze(1)
