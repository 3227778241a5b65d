"""Native 3DGS-MCMC densification (Kheradmand et al., "3D Gaussian Splatting as Markov Chain Monte Carlo", 2024; DESIGN.md §5n):
the authors' GaussianModel.relocate_gs / add_new_gs and the position noise of their training loop, on the model and its Adam state.

    from gs_b200 import mcmc
    GaussianModel.relocate_gs = mcmc.relocate_gs                    # INTEGRATION.md section I
    GaussianModel.add_new_gs = mcmc.add_new_gs
    GaussianModel.inject_noise = mcmc.inject_noise                  # replaces the L @ L^T / randn / bmm block after optimizer.step()

The signatures are the authors' methods with `self` -> `model`.  The model contract and its refusals are densify's (_validate):
torch.optim.Adam or GaussianAdam with the six groups, no codebooks, no variable-SH lists.  A refusal leaves the model, the optimizer
and the CUDA generator as they were.

Sampling.  The authors draw with torch.multinomial, whose bytes change from run to run.  Here the weights are the fixed-point
opacities floor(o * 2^32) of the candidate rows and one torch.randint(0, 2**62, (n,)) on the model's device drives an exact integer
inverse CDF (gsb_mcmc_plan): the same distribution up to the 2^-32 quantisation, not the same indices as multinomial, and the same
bytes on every run for the same generator state.  The relocated opacity and scales are evaluated in double (paper eq. 9).

Kept quirk of the authors' code (and gsplat's): relocate_gs zeroes the Adam moments of the sampled SOURCE rows; the dead rows that
receive their parameters keep their own moments.

The emit table entries (densify._entry) and add_new_gs's allocation and optimizer surgery (densify._resized) are densify's.
"""
from __future__ import annotations

import ctypes as C
import numbers

import torch

from . import densify
from . import lib as gsl

MIN_OPACITY = 0.005          # the authors' dead threshold: sigmoid(_opacity) <= 0.005
KIND = {"opacity": gsl.MCMC_OPACITY, "scaling": gsl.DENSIFY_SCALING}


def inject_noise(model, xyz_lr, noise_lr=5e5):
    """The authors' noise step (train.py, after optimizer.step()): xyz += R diag(s)^2 R^T (eps * g * noise_lr * xyz_lr) with
    eps = torch.randn_like(_xyz) and the gate g = 1 / (1 + exp(-100 ((1 - o) - 0.995))).  One launch, evaluated in double, in place
    on _xyz; rows whose fp32 gate is 0 keep their bytes.  noise_lr and xyz_lr are used as their fp32 casts and must be finite."""
    lrs = (C.c_float(float(noise_lr)).value, C.c_float(float(xyz_lr)).value)
    if not all(abs(v) < float("inf") for v in lrs):
        raise RuntimeError(f"mcmc: noise_lr ({noise_lr}) and xyz_lr ({xyz_lr}) must be finite in fp32")
    groups, P, dev = densify._validate(model, False)
    p = {name: t for name, _, t, _ in groups}
    draws = torch.randn_like(p["xyz"])
    if P == 0:
        return
    with gsl.on_device(dev):
        gsl.check(gsl.lib().gsb_mcmc_noise(P, p["xyz"].data_ptr(), p["scaling"].data_ptr(), p["rotation"].data_ptr(),
                                           p["opacity"].data_ptr(), draws.data_ptr(), lrs[0], lrs[1], gsl.current_stream(dev)))


def relocate_gs(model, dead_mask=None):
    """The authors' relocate_gs: each dead row (dead_mask, bool [P]; None: sigmoid(_opacity) <= 0.005) takes the xyz, features,
    rotation and _degrees of a live row sampled by opacity, and the relocated opacity and scaling that the sampled row also takes;
    the sampled rows' moments are zeroed in all six groups.  In place (the same Parameters, state dicts and step tensors); every
    param's .grad is set to None.  No dead row, no live row (or live rows that all weigh 0) changes nothing and draws nothing.
    One host read: the dead count."""
    groups, P, dev = densify._validate(model, False)
    if dead_mask is not None and (not torch.is_tensor(dead_mask) or dead_mask.dtype != torch.bool or tuple(dead_mask.shape) != (P,)
                                  or dead_mask.device != dev):
        raise RuntimeError(f"mcmc: dead_mask must be a bool tensor [{P}] on {dev}")
    if P == 0:
        return
    mask = None if dead_mask is None else dead_mask.contiguous()
    ws, counts = _plan(groups, P, dev, gsl.MCMC_RELOCATE, mask)
    n_dead, total = counts.tolist()[:2]
    if n_dead == 0 or total == 0:
        return
    draws = torch.randint(0, 2 ** 62, (n_dead,), dtype=torch.int64, device=dev)
    _plan(groups, P, dev, gsl.MCMC_RELOCATE, mask, ws, draws)
    entries = []
    for name, _, p, state in groups:
        moments = None if state is None else (state["exp_avg"], state["exp_avg_sq"])
        entries.append(densify._entry(p, p, KIND.get(name, gsl.DENSIFY_COPY), moments, moments))
    entries.append(densify._entry(model._degrees, model._degrees, gsl.DENSIFY_COPY))
    if getattr(model, "filter_3D", None) is not None:
        entries.append(densify._entry(model.filter_3D, model.filter_3D, gsl.DENSIFY_COPY))
    _emit(entries, P, dev, gsl.MCMC_RELOCATE, n_dead, ws)
    for _, _, p, _ in groups:
        p.grad = None


def add_new_gs(model, cap_max):
    """The authors' add_new_gs: P' = min(cap_max, int(1.05 * P)) and n = max(0, P' - P) rows sampled by opacity (every row a
    candidate) are appended in sample order, each a copy of its source with the relocated opacity and scaling the source also takes.
    New rows have zero moments, the sampled sources' moments are zeroed; _degrees copies the source, the statistics
    (xyz_gradient_accum, denom, max_radii2D, xyz_gradient_accum_abs) get zero rows.  New Parameters carry the state dicts (as
    densify does) with .grad None.  -> n.  At most one host read (the total weight); n = 0 draws nothing."""
    if isinstance(cap_max, bool) or not isinstance(cap_max, numbers.Integral) or cap_max < 0:
        raise RuntimeError(f"mcmc: cap_max must be a non-negative int, got {cap_max!r}")
    groups, P, dev = densify._validate(model, False)
    n = max(0, min(int(cap_max), int(1.05 * P)) - P)
    if n == 0:
        return 0
    ws, counts = _plan(groups, P, dev, gsl.MCMC_ADD)
    if int(counts[1]) == 0:                                  # every opacity below 2^-32: nothing to sample from
        return 0
    draws = torch.randint(0, 2 ** 62, (n,), dtype=torch.int64, device=dev)
    _plan(groups, P, dev, gsl.MCMC_ADD, None, ws, draws)
    entries, install = densify._resized(model, groups, P + n, dev, KIND, gsl.MCMC_FRESH)
    _emit(entries, P, dev, gsl.MCMC_ADD, n, ws)
    install()
    return n


# ------------------------------------------------------------------------------------------------ internals
def _plan(groups, P, dev, mode, mask=None, ws=None, draws=None):
    """Without draws: a new workspace and the counts (dead rows, total weight) read back, the one host read.  With draws: the
    second phase into `ws`."""
    p = {name: t for name, _, t, _ in groups}
    counts = None
    if draws is None:
        ws = torch.empty(gsl.lib().gsb_mcmc_workspace_bytes(P), dtype=torch.uint8, device=dev)
        counts = torch.empty(gsl.MCMC_COUNTS, dtype=torch.int64, device=dev)
    with gsl.on_device(dev):
        gsl.check(gsl.lib().gsb_mcmc_plan(P, mode, p["opacity"].data_ptr(), p["scaling"].data_ptr(),
                                          None if mask is None else mask.data_ptr(), MIN_OPACITY,
                                          0 if draws is None else draws.numel(), None if draws is None else draws.data_ptr(),
                                          ws.data_ptr(), None if counts is None else counts.data_ptr(), gsl.current_stream(dev)))
    return ws, counts


def _emit(entries, P, dev, mode, n, ws):
    table = (gsl.GsbDensifyTensor * len(entries))(*entries)
    with gsl.on_device(dev):
        gsl.check(gsl.lib().gsb_mcmc_emit(table, len(entries), P, mode, n, ws.data_ptr(), gsl.current_stream(dev)))
