"""GaussianAdam: torch.optim.Adam whose step is one CUDA launch (gsb_adam_step, DESIGN.md §5f).

    optimizer = GaussianAdam(groups, lr=0.0, eps=1e-15)         # the reference's training_setup, unchanged otherwise
    ...
    optimizer.step()                                               # dense: bit-identical to torch.optim.Adam
    optimizer.step(visibility=visibility_filter, degrees=gaussians._degrees)   # sparse

Construction, param groups (lr / betas / eps per group, extra keys such as the reference's "name" kept), state layout
(state[p] = {"step": CPU float32 tensor, "exp_avg", "exp_avg_sq"}), state_dict / load_state_dict and zero_grad are
torch.optim.Adam's own, so the reference's optimizer-state surgery (prune, concatenate, replace) and checkpoints work
unchanged and in both directions.  step() computes what torch 2.11's default (foreach) CUDA path computes, bit for bit:
the bias corrections in Python double exactly as torch does, the elementwise update in one kernel for every tensor.

Sparse modes, for a model whose tensors all have one row per Gaussian (dim 0 = P):
  visibility  bool [P] (render()'s "visibility_filter", or the union over a view batch): row i of every tensor is updated only
              if visibility[i]; other rows keep param, exp_avg and exp_avg_sq bit for bit.
  degrees     int32 [P] or [P, 1] (the active SH degree per Gaussian, clamped to 0..3): in a param group with the key
              "sh_offset": k, an [P, C, 3] tensor whose column c holds SH coefficient k + c, coefficient k + c of row i is updated
              only if k + c < (degrees[i] + 1)^2 (the reference's f_rest: k = 1; f_dc: k = 0).  Other groups ignore degrees.
Updated entries are what dense mode computes.  state["step"] advances on every call for every param with a gradient, as in
torch, and the bias correction uses it.  The masks' row counts are checked against the params that have a gradient only: after
densification or pruning the model's params are new and have none, so such a step does nothing (as torch's does) even though
the render's visibility still has the old row count.  A param with a gradient whose dim 0 differs from a mask's is an error.
Nothing synchronises with the host; the work runs on the current stream of the params' device.
"""
from __future__ import annotations

import torch
from torch.optim.optimizer import _get_scalar_dtype, _get_value

from . import lib as gsl


class GaussianAdam(torch.optim.Adam):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None,
                 maximize=False, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False):
        _check_options(dict(lr=lr, betas=betas, weight_decay=weight_decay, amsgrad=amsgrad, maximize=maximize, capturable=capturable,
                            differentiable=differentiable, fused=fused))
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, foreach=foreach,
                         maximize=maximize, capturable=capturable, differentiable=differentiable, fused=fused,
                         decoupled_weight_decay=decoupled_weight_decay)
        for group in self.param_groups:
            _check_options(group)

    @torch.no_grad()
    def step(self, closure=None, visibility=None, degrees=None):
        """One Adam step over every param with a gradient; see the module docstring for `visibility` and `degrees`."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        P, _ = _rows(visibility, degrees)
        sparse = P is not None
        # validate everything before touching any state, so that a refused step leaves the optimizer as it was
        todo = []                        # (param, group) in group order
        for group in self.param_groups:
            _check_options(group)
            for p in group["params"]:
                if p.grad is None:
                    continue
                _check_tensor(p, p.grad, degrees is not None and group.get("sh_offset") is not None)
                state = self.state.get(p)
                for k in ("exp_avg", "exp_avg_sq") if state else ():
                    s = state[k]
                    if s.shape != p.shape or s.dtype != torch.float32 or s.device != p.device or not s.is_contiguous():
                        raise RuntimeError(f"GaussianAdam: state['{k}'] must be a contiguous fp32 tensor of the param's shape and device")
                # the masks are compared with the params they apply to, not with each other: after densification or pruning
                # the params are new and have no gradient yet, while visibility still has the render's row count
                for name, m in (("visibility", visibility), ("degrees", degrees)):
                    if m is not None and (p.dim() == 0 or p.shape[0] != m.shape[0] or p.device != m.device):
                        raise RuntimeError(f"GaussianAdam: {name} has {m.shape[0]} rows on {m.device}, but a param with a gradient "
                                           f"has shape {tuple(p.shape)} on {p.device}: every such param needs dim 0 = P")
                todo.append((p, group))
        if not todo:
            return loss
        for p, _ in todo:
            state = self.state[p]
            if len(state) == 0:
                state["step"] = torch.tensor(0.0, dtype=_get_scalar_dtype())
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        todo = [(p, self.state[p], group) for p, group in todo]
        # torch's foreach path: every step advances before the bias corrections are formed (_foreach_add_ of a CPU 1.0)
        steps = [st["step"] for _, st, _ in todo]
        if all(s.is_cpu for s in steps):
            torch._foreach_add_(steps, torch.tensor(1.0, device="cpu"), alpha=1.0)
        else:
            torch._foreach_add_(steps, 1)
        per_device = {}
        for p, state, group in todo:
            if p.numel() == 0:
                continue
            beta1, beta2 = group["betas"]
            lr, eps = group["lr"], group["eps"]
            step = _get_value(state["step"])
            # exactly torch.optim.adam._multi_tensor_adam's host arithmetic (Python double), cast to fp32 by the ctypes fields
            # as ATen casts its Scalar arguments
            bias_correction1 = 1 - beta1 ** step
            bias_correction2 = 1 - beta2 ** step
            step_size = (lr / bias_correction1) * -1
            bias_correction2_sqrt = bias_correction2 ** 0.5
            sh = group.get("sh_offset")
            e = gsl.GsbAdamTensor()
            e.param, e.grad = p.data_ptr(), p.grad.data_ptr()
            e.exp_avg, e.exp_avg_sq = state["exp_avg"].data_ptr(), state["exp_avg_sq"].data_ptr()
            e.numel = p.numel()
            e.row_width = p.numel() // P if sparse else 1
            e.sh_offset = int(sh) if (sh is not None and degrees is not None) else -1
            e.one_minus_beta1, e.beta2, e.one_minus_beta2 = 1 - beta1, beta2, 1 - beta2
            e.eps, e.bc2_sqrt, e.step_size = eps, bias_correction2_sqrt, step_size
            per_device.setdefault(p.device, []).append(e)
        vis_ptr = None if visibility is None else visibility.data_ptr()
        deg_ptr = None if degrees is None else degrees.data_ptr()
        L = gsl.lib()
        for dev, entries in per_device.items():
            stream = gsl.current_stream(dev)
            with gsl.on_device(dev):
                for i in range(0, len(entries), gsl.ADAM_MAX_TENSORS):
                    chunk = entries[i:i + gsl.ADAM_MAX_TENSORS]
                    table = (gsl.GsbAdamTensor * len(chunk))(*chunk)
                    gsl.check(L.gsb_adam_step(table, len(chunk), P or 0, vis_ptr, deg_ptr, stream))
        return loss


def _check_options(group):
    """Refuses what the kernel does not implement (everything else of torch.optim.Adam's contract holds)."""
    for key in ("amsgrad", "maximize", "capturable", "differentiable", "fused"):
        if group.get(key):
            raise ValueError(f"GaussianAdam does not support {key}=True")
    if group.get("weight_decay", 0) != 0:
        raise ValueError("GaussianAdam does not support weight_decay != 0")
    if torch.is_tensor(group.get("lr")) or any(torch.is_tensor(b) for b in group.get("betas", ())):
        raise ValueError("GaussianAdam takes lr and betas as Python numbers, not tensors")
    sh = group.get("sh_offset")
    if sh is not None and (isinstance(sh, bool) or not isinstance(sh, int) or sh < 0):
        raise ValueError(f"GaussianAdam: sh_offset must be a non-negative int, got {sh!r}")


def _check_tensor(p, g, banded):
    if g.is_sparse:
        raise RuntimeError("GaussianAdam does not support sparse gradients")
    if p.dtype != torch.float32 or g.dtype != torch.float32:
        raise RuntimeError(f"GaussianAdam: params and grads must be fp32, got {p.dtype} / {g.dtype}")
    if not p.is_contiguous() or not g.is_contiguous() or g.shape != p.shape:
        raise RuntimeError("GaussianAdam: params and grads must be contiguous and of the same shape")
    if not p.is_cuda or not g.is_cuda or g.device != p.device:
        raise RuntimeError("GaussianAdam: params and grads must be CUDA tensors on one device (there is no CPU path)")
    if banded and (p.dim() != 3 or p.shape[2] != 3):
        raise RuntimeError(f"GaussianAdam: a group with sh_offset needs [P, C, 3] tensors, got {tuple(p.shape)}")


def _rows(visibility, degrees):
    """(P, device) of the sparse modes, (None, None) for dense.  Only the masks' own form is checked here; their row counts are
    checked against the params that have a gradient."""
    if visibility is not None:
        if visibility.dtype != torch.bool or visibility.dim() != 1 or not visibility.is_cuda or not visibility.is_contiguous():
            raise RuntimeError("GaussianAdam: visibility must be a contiguous bool CUDA tensor [P]")
    if degrees is not None:
        if (degrees.dtype != torch.int32 or not degrees.is_cuda or not degrees.is_contiguous()
                or not (degrees.dim() == 1 or (degrees.dim() == 2 and degrees.shape[1] == 1))):
            raise RuntimeError("GaussianAdam: degrees must be a contiguous int32 CUDA tensor [P] or [P, 1]")
    m = visibility if visibility is not None else degrees
    return (None, None) if m is None else (m.shape[0], m.device)
