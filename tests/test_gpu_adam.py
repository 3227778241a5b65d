"""GPU: GaussianAdam (gs_b200.optim, gsb_adam_step; DESIGN.md §5f) against torch.optim.Adam, bit for bit unless stated:
dense mode on the reference's six tensor shapes, the visibility and SH-band sparse modes (skipped entries untouched, updated
ones as torch), offset views and odd sizes, the reference's optimizer-state surgery and state_dict in both directions, one
launch per step, run-to-run / stream / device invariance, and training through render()."""
import copy
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "reduced-3dgs_b200"))
from gs_b200 import lib as gsl  # noqa: E402
from gs_b200 import synth  # noqa: E402
from gs_b200.optim import GaussianAdam  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
SHAPES = [("xyz", (3,), 1.6e-4), ("f_dc", (1, 3), 2.5e-3), ("f_rest", (15, 3), 2.5e-3 / 20), ("opacity", (1,), 0.05),
          ("scaling", (3,), 5e-3), ("rotation", (4,), 1e-3)]


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def assert_same(a, b, what=""):
    assert a.shape == b.shape, what
    diff = int((bits(a) != bits(b)).sum())
    assert diff == 0, f"{what}: {diff} of {a.numel()} entries differ"


def make_groups(P, seed, device=DEV, extra_sh=False):
    """The reference's six groups (gaussian_model.py:208-217 shapes, names and per-group learning rates), seeded values.
    extra_sh adds a [P, 16, 3] group with sh_offset 0 (a model that keeps all SH coefficients in one tensor)."""
    g = torch.Generator().manual_seed(seed)
    groups = []
    shapes = SHAPES + ([("features", (16, 3), 2e-3)] if extra_sh else [])
    for name, tail, lr in shapes:
        p = torch.nn.Parameter(torch.randn((P,) + tail, generator=g).to(device))
        grp = {"params": [p], "lr": lr, "name": name}
        if name == "f_rest":
            grp["sh_offset"] = 1
        if name == "features":
            grp["sh_offset"] = 0
        groups.append(grp)
    return groups


def clone_groups(groups, device=None):
    out = []
    for grp in groups:
        c = dict(grp)
        c["params"] = [torch.nn.Parameter(p.detach().clone() if device is None else p.detach().to(device)) for p in grp["params"]]
        out.append(c)
    return out


def hard_grad(shape, gen, device=DEV):
    """randn scaled over 4 decades, with exact zeros, 1e-30, +-1e10 and mixed signs."""
    x = torch.randn(shape, generator=gen) * 10.0 ** (torch.rand(shape, generator=gen) * 4 - 3)
    u = torch.rand(shape, generator=gen)
    x[u < 0.03] = 0.0
    x[(u >= 0.03) & (u < 0.04)] = 1e-30
    x[(u >= 0.04) & (u < 0.045)] = 1e10
    x[(u >= 0.045) & (u < 0.05)] = -1e10
    return x.to(device)


def set_grads(group_lists, seed):
    gen = torch.Generator().manual_seed(seed)
    grads = [hard_grad(grp["params"][0].shape, gen, grp["params"][0].device) for grp in group_lists[0]]
    for groups in group_lists:
        for grp, gr in zip(groups, grads):
            grp["params"][0].grad = gr.to(grp["params"][0].device).clone()


def assert_same_state(opt_a, groups_a, opt_b, groups_b):
    for ga, gb in zip(groups_a, groups_b):
        pa, pb = ga["params"][0], gb["params"][0]
        assert_same(pa, pb, ga["name"] + " param")
        sa, sb = opt_a.state[pa], opt_b.state[pb]
        assert_same(sa["exp_avg"], sb["exp_avg"], ga["name"] + " exp_avg")
        assert_same(sa["exp_avg_sq"], sb["exp_avg_sq"], ga["name"] + " exp_avg_sq")
        assert float(sa["step"]) == float(sb["step"])


def test_dense_is_torch_adam():
    P = 100_003
    ours = make_groups(P, 1)
    theirs = clone_groups(ours)
    kw = dict(lr=0.0, betas=(0.8, 0.99), eps=1e-15)
    opt, ref = GaussianAdam(ours, **kw), torch.optim.Adam(theirs, **kw)
    for t in range(25):
        lr = 1.6e-4 * (0.01 ** (t / 25))                  # the xyz learning rate changes every step (gaussian_model.py:223-229)
        opt.param_groups[0]["lr"] = ref.param_groups[0]["lr"] = lr
        set_grads([ours, theirs], 100 + t)
        opt.step()
        ref.step()
    assert_same_state(opt, ours, ref, theirs)


def _masked_reference(ref, theirs, keep_fn):
    """torch Adam step on every entry, then the entries keep_fn marks as skipped are put back (param and both moments)."""
    before = [(grp["params"][0].detach().clone(), ref.state[grp["params"][0]]["exp_avg"].clone(),
               ref.state[grp["params"][0]]["exp_avg_sq"].clone()) for grp in theirs]
    ref.step()
    with torch.no_grad():
        for grp, (p0, m0, v0) in zip(theirs, before):
            p = grp["params"][0]
            upd = keep_fn(grp, p)
            st = ref.state[p]
            p.copy_(torch.where(upd, p, p0))
            st["exp_avg"].copy_(torch.where(upd, st["exp_avg"], m0))
            st["exp_avg_sq"].copy_(torch.where(upd, st["exp_avg_sq"], v0))


def _band_mask(grp, p, deg):
    if "sh_offset" not in grp:
        return torch.ones_like(p, dtype=torch.bool)
    C = p.shape[1]
    d = deg.view(-1).clamp(0, 3).long()
    coef = grp["sh_offset"] + torch.arange(C, device=p.device)
    return (coef.view(1, C) < ((d + 1) ** 2).view(-1, 1)).unsqueeze(-1).expand_as(p)


def _row_mask(p, vis):
    return vis.view((-1,) + (1,) * (p.dim() - 1)).expand_as(p)


def test_visibility_updates_visible_rows_only():
    P = 50_001
    ours = make_groups(P, 2)
    theirs = clone_groups(ours)
    opt, ref = GaussianAdam(ours, lr=0.0, eps=1e-15), torch.optim.Adam(theirs, lr=0.0, eps=1e-15)
    for t in range(3):                                     # a non-trivial state first
        set_grads([ours, theirs], 200 + t)
        opt.step()
        ref.step()
    gen = torch.Generator().manual_seed(9)
    for t in range(5):
        vis = (torch.rand(P, generator=gen) < 0.6).to(DEV)
        set_grads([ours, theirs], 300 + t)
        before = [(grp["params"][0].detach().clone(), opt.state[grp["params"][0]]["exp_avg"].clone()) for grp in ours]
        opt.step(visibility=vis)
        _masked_reference(ref, theirs, lambda grp, p: _row_mask(p, vis))
        for grp, (p0, m0) in zip(ours, before):          # unvisited rows: untouched
            assert_same(grp["params"][0][~vis], p0[~vis], grp["name"])
            assert_same(opt.state[grp["params"][0]]["exp_avg"][~vis], m0[~vis], grp["name"])
        assert_same_state(opt, ours, ref, theirs)


def test_degrees_update_active_bands_only():
    P = 30_007
    ours = make_groups(P, 3, extra_sh=True)
    theirs = clone_groups(ours)
    opt, ref = GaussianAdam(ours, lr=0.0, eps=1e-15), torch.optim.Adam(theirs, lr=0.0, eps=1e-15)
    for t in range(2):
        set_grads([ours, theirs], 400 + t)
        opt.step()
        ref.step()
    gen = torch.Generator().manual_seed(11)
    for t in range(4):
        deg = torch.randint(0, 4, (P, 1), generator=gen, dtype=torch.int32)         # mixed, not sorted by degree
        deg[:7, 0] = torch.tensor([-3, -1, 4, 9, 0, 3, 2], dtype=torch.int32)      # outside 0..3: clamped
        deg = deg.to(DEV)
        vis = (torch.rand(P, generator=gen) < 0.7).to(DEV) if t >= 2 else None
        set_grads([ours, theirs], 500 + t)
        sh_before = {grp["name"]: grp["params"][0].detach().clone() for grp in ours if "sh_offset" in grp}
        opt.step(visibility=vis, degrees=deg if t % 2 else deg.view(-1))
        _masked_reference(ref, theirs, lambda grp, p: _band_mask(grp, p, deg) & (_row_mask(p, vis) if vis is not None else True))
        for grp in ours:
            if "sh_offset" in grp:
                p = grp["params"][0]
                off = ~_band_mask(grp, p, deg)
                assert bool(off.any())
                assert_same(p[off], sh_before[grp["name"]][off], grp["name"] + " inactive")
        assert_same_state(opt, ours, ref, theirs)


def test_everything_active_is_dense():
    P = 20_011
    ours = make_groups(P, 4)
    dense = clone_groups(ours)
    opt, opt_d = GaussianAdam(ours, lr=0.0, eps=1e-15), GaussianAdam(dense, lr=0.0, eps=1e-15)
    theirs = clone_groups(ours)
    ref = torch.optim.Adam(theirs, lr=0.0, eps=1e-15)
    vis, deg = torch.ones(P, dtype=torch.bool, device=DEV), torch.full((P, 1), 3, dtype=torch.int32, device=DEV)
    for t in range(4):
        set_grads([ours, dense, theirs], 600 + t)
        opt.step(visibility=vis, degrees=deg)
        opt_d.step()
        ref.step()
    assert_same_state(opt, ours, opt_d, dense)
    assert_same_state(opt, ours, ref, theirs)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 7, 13, 1001])
def test_offset_views_and_odd_sizes(n):
    """Storage offsets 0..3 floats for param, grad and both moments (equal: head / 128-bit body / tail; mixed: scalar path)."""
    gen = torch.Generator().manual_seed(n)
    for offs in [(0, 0, 0, 0), (1, 1, 1, 1), (2, 2, 2, 2), (3, 3, 3, 3), (1, 2, 3, 0), (0, 3, 0, 1)]:
        def at(o, src):
            base = torch.zeros(n + 8, device=DEV)
            base[o:o + n] = src
            return base[o:o + n]
        p0, m0, v0 = torch.randn(n, generator=gen), torch.randn(n, generator=gen), torch.rand(n, generator=gen)
        opts, params = [], []
        for cls in (GaussianAdam, torch.optim.Adam):
            p = torch.nn.Parameter(at(offs[0], p0))
            assert p.storage_offset() == offs[0]
            opt = cls([p], lr=1e-2, eps=1e-15)
            opt.state[p] = {"step": torch.tensor(4.0), "exp_avg": at(offs[2], m0), "exp_avg_sq": at(offs[3], v0)}
            opts.append(opt)
            params.append(p)
        for t in range(3):
            g = hard_grad((n,), gen)
            for p, opt in zip(params, opts):
                p.grad = at(offs[1], g)
                opt.step()
        for k in ("exp_avg", "exp_avg_sq"):
            assert_same(opts[0].state[params[0]][k], opts[1].state[params[1]][k], f"{offs} {k}")
        assert_same(params[0], params[1], f"{offs} param")


def test_one_row_empty_model_and_params_without_grad():
    one = make_groups(1, 5)
    theirs = clone_groups(one)
    opt, ref = GaussianAdam(one), torch.optim.Adam(theirs)
    for t in range(3):
        set_grads([one, theirs], 700 + t)
        opt.step(visibility=torch.ones(1, dtype=torch.bool, device=DEV), degrees=torch.full((1,), 3, dtype=torch.int32, device=DEV))
        ref.step()
    assert_same_state(opt, one, ref, theirs)
    # P = 0: no launch, the step still advances
    empty = make_groups(0, 6)
    opt0 = GaussianAdam(empty)
    for grp in empty:
        grp["params"][0].grad = torch.zeros_like(grp["params"][0])
    n0 = gsl.launch_count()
    opt0.step(visibility=torch.zeros(0, dtype=torch.bool, device=DEV), degrees=torch.zeros(0, dtype=torch.int32, device=DEV))
    opt0.step()
    torch.cuda.synchronize()
    assert gsl.launch_count() == n0
    assert float(opt0.state[empty[0]["params"][0]]["step"]) == 2.0
    # a param without a grad keeps its state, the others move on
    frozen = one[2]["params"][0]
    snap = {k: v.clone() for k, v in opt.state[frozen].items()}
    p_snap = frozen.detach().clone()
    set_grads([one], 800)
    frozen.grad = None
    opt.step()
    assert_same(frozen, p_snap, "param without grad")
    for k in ("exp_avg", "exp_avg_sq"):
        assert_same(opt.state[frozen][k], snap[k], k)
    assert float(opt.state[frozen]["step"]) == float(snap["step"]) == 3.0
    with pytest.raises(RuntimeError, match="dim 0"):
        set_grads([one], 801)
        opt.step(visibility=torch.ones(2, dtype=torch.bool, device=DEV))


# ---- the reference's optimizer-state surgery (scene/gaussian_model.py _prune_optimizer / cat_tensors_to_optimizer /
# replace_tensor_to_optimizer), restated: index or extend the moments, re-key the state to a new Parameter ----

def prune(opt, keep):
    for grp in opt.param_groups:
        old = grp["params"][0]
        st = opt.state.get(old, None)
        new = torch.nn.Parameter(old[keep].requires_grad_(True))
        if st is not None:
            st["exp_avg"] = st["exp_avg"][keep]
            st["exp_avg_sq"] = st["exp_avg_sq"][keep]
            del opt.state[old]
            opt.state[new] = st
        grp["params"][0] = new


def cat(opt, extension):
    for grp in opt.param_groups:
        old = grp["params"][0]
        ext = extension[grp["name"]]
        st = opt.state.get(old, None)
        new = torch.nn.Parameter(torch.cat((old, ext), dim=0).requires_grad_(True))
        if st is not None:
            st["exp_avg"] = torch.cat((st["exp_avg"], torch.zeros_like(ext)), dim=0)
            st["exp_avg_sq"] = torch.cat((st["exp_avg_sq"], torch.zeros_like(ext)), dim=0)
            del opt.state[old]
            opt.state[new] = st
        grp["params"][0] = new


def replace(opt, tensor, name):
    for grp in opt.param_groups:
        if grp["name"] == name:
            old = grp["params"][0]
            st = opt.state.get(old, None)
            st["exp_avg"] = torch.zeros_like(tensor)
            st["exp_avg_sq"] = torch.zeros_like(tensor)
            del opt.state[old]
            new = torch.nn.Parameter(tensor.requires_grad_(True))
            opt.state[new] = st
            grp["params"][0] = new


def test_densify_iteration_with_stale_visibility_does_nothing():
    """train.py's order: render (visibility of P rows) -> densify / prune (new params without grad, _degrees resized) -> step.
    The step has no param with a gradient: no launch, no error, no state change, as torch.optim.Adam."""
    P = 10_007
    ours = make_groups(P, 14)
    theirs = clone_groups(ours)
    opt, ref = GaussianAdam(ours, lr=0.0, eps=1e-15), torch.optim.Adam(theirs, lr=0.0, eps=1e-15)
    gen = torch.Generator().manual_seed(15)
    degrees = torch.randint(0, 4, (P, 1), generator=gen, dtype=torch.int32).to(DEV)
    for t in range(2):
        _step_both(opt, ref, 1100 + t)
    old_vis = (torch.rand(P, generator=gen) < 0.8).to(DEV)           # the render's visibility_filter, P rows
    keep = (torch.rand(P, generator=gen) > 0.1).to(DEV)
    for o in (opt, ref):
        prune(o, keep)
    ext = {name: torch.randn((333,) + tail, generator=gen).to(DEV) for name, tail, _ in SHAPES}
    for o in (opt, ref):
        cat(o, ext)
    P2 = opt.param_groups[0]["params"][0].shape[0]
    new_degrees = torch.cat([degrees[keep], torch.zeros(333, 1, dtype=torch.int32, device=DEV)])
    assert P2 != P and new_degrees.shape[0] == P2
    n0 = gsl.launch_count()
    opt.step(visibility=old_vis, degrees=new_degrees)               # every param is new: grad None
    ref.step()
    torch.cuda.synchronize()
    assert gsl.launch_count() == n0
    assert_same_state(opt, opt.param_groups, ref, ref.param_groups)
    assert all(float(opt.state[g["params"][0]]["step"]) == 2.0 for g in opt.param_groups)
    # the next iteration renders the new model: both masks have P2 rows, and the step goes on as torch's
    new_vis = (torch.rand(P2, generator=gen) < 0.8).to(DEV)
    set_grads([opt.param_groups, ref.param_groups], 1200)
    opt.step(visibility=new_vis, degrees=new_degrees)
    _masked_reference(ref, ref.param_groups, lambda grp, p: _row_mask(p, new_vis) & _band_mask(grp, p, new_degrees))
    assert_same_state(opt, opt.param_groups, ref, ref.param_groups)
    # a gradient present while a mask still has the old row count is an error, raised before any state moves
    set_grads([opt.param_groups], 1300)
    snap = [float(opt.state[g["params"][0]]["step"]) for g in opt.param_groups]
    with pytest.raises(RuntimeError, match="dim 0"):
        opt.step(visibility=old_vis, degrees=new_degrees)
    assert [float(opt.state[g["params"][0]]["step"]) for g in opt.param_groups] == snap


@pytest.mark.parametrize("tail,sh_offset", [((1,), None), ((3,), None), ((4,), None), ((5, 3), 1), ((16, 3), 0)])
@pytest.mark.parametrize("mode", ["visibility", "degrees", "both"])
def test_sparse_offset_views(tail, sh_offset, mode):
    """The sparse row / column derivation on tensors whose first element is not 16-byte aligned (a head of 1-3 scalars before the
    128-bit chunks) and on mixed alignments (all scalar): storage offsets 0-3, odd row counts."""
    gen = torch.Generator().manual_seed(len(tail) * 100 + tail[0])
    width = int(np.prod(tail))
    for R in (1, 7, 1001):
        n = R * width
        for offs in [(1, 1, 1, 1), (2, 2, 2, 2), (3, 3, 3, 3), (0, 0, 0, 0), (1, 2, 3, 0)]:
            def at(o, src):
                base = torch.zeros(n + 8, device=DEV)
                base[o:o + n] = src.reshape(-1)
                return base[o:o + n].view((R,) + tail)
            p0, m0, v0 = torch.randn(n, generator=gen), torch.randn(n, generator=gen), torch.rand(n, generator=gen)
            vis = (torch.rand(R, generator=gen) < 0.6).to(DEV) if mode != "degrees" else None
            deg = torch.randint(-1, 5, (R,), generator=gen, dtype=torch.int32).to(DEV) if mode != "visibility" else None
            params, opts = [], []
            for cls in (GaussianAdam, torch.optim.Adam):
                p = torch.nn.Parameter(at(offs[0], p0))
                grp = {"params": [p], "lr": 1e-2, "name": "t"}
                if sh_offset is not None:
                    grp["sh_offset"] = sh_offset
                opt = cls([grp], eps=1e-15)
                opt.state[p] = {"step": torch.tensor(4.0), "exp_avg": at(offs[2], m0), "exp_avg_sq": at(offs[3], v0)}
                params.append(p)
                opts.append(opt)
            assert params[0].storage_offset() == offs[0]
            for t in range(2):
                g = hard_grad((n,), gen)
                params[0].grad = at(offs[1], g)
                params[1].grad = at(offs[1], g)
                before = params[0].detach().clone()
                opts[0].step(visibility=vis, degrees=deg)

                def keep(grp, p):
                    k = torch.ones_like(p, dtype=torch.bool)
                    if vis is not None:
                        k &= _row_mask(p, vis)
                    if deg is not None and "sh_offset" in grp:
                        k &= _band_mask(grp, p, deg)
                    return k
                _masked_reference(opts[1], opts[1].param_groups, keep)
                k = keep(opts[0].param_groups[0], params[0])
                assert_same(params[0][~k], before[~k], f"{tail} {mode} {offs} R={R} skipped")
            what = f"{tail} {mode} {offs} R={R}"
            assert_same(params[0], params[1], what + " param")
            for key in ("exp_avg", "exp_avg_sq"):
                assert_same(opts[0].state[params[0]][key], opts[1].state[params[1]][key], what + " " + key)


def _step_both(opt, ref, seed, vis=None):
    set_grads([opt.param_groups, ref.param_groups], seed)
    if vis is None:
        opt.step()
        ref.step()
    else:
        opt.step(visibility=vis)
        _masked_reference(ref, ref.param_groups, lambda grp, p: _row_mask(p, vis))


def test_state_surgery_and_state_dict_round_trip():
    P = 40_003
    ours = make_groups(P, 7)
    theirs = clone_groups(ours)
    opt, ref = GaussianAdam(ours, lr=0.0, eps=1e-15), torch.optim.Adam(theirs, lr=0.0, eps=1e-15)
    for t in range(3):
        _step_both(opt, ref, 900 + t)
    gen = torch.Generator().manual_seed(12)
    keep = (torch.rand(P, generator=gen) > 0.2).to(DEV)
    prune(opt, keep)
    prune(ref, keep)
    n_new = 3_001
    ext = {name: torch.randn((n_new,) + tail, generator=gen).to(DEV) for name, tail, _ in SHAPES}
    cat(opt, ext)
    cat(ref, ext)
    P2 = opt.param_groups[0]["params"][0].shape[0]
    op = torch.randn(P2, 1, generator=gen).to(DEV)
    replace(opt, op.clone(), "opacity")
    replace(ref, op.clone(), "opacity")
    for t in range(3):
        vis = (torch.rand(P2, generator=gen) < 0.5).to(DEV) if t == 1 else None
        _step_both(opt, ref, 950 + t, vis)
    assert_same_state(opt, opt.param_groups, ref, ref.param_groups)
    # state_dict from either class loads into the other and continues identically
    for src, src_groups in ((opt, opt.param_groups), (ref, ref.param_groups)):
        a_groups = clone_groups(src_groups)
        b_groups = clone_groups(src_groups)
        a = GaussianAdam(a_groups, lr=0.0, eps=1e-15)
        b = torch.optim.Adam(b_groups, lr=0.0, eps=1e-15)
        # deep copies: load_state_dict keeps tensors that already sit on the param's device, so both would share the moments
        a.load_state_dict(copy.deepcopy(src.state_dict()))
        b.load_state_dict(copy.deepcopy(src.state_dict()))
        for t in range(2):
            _step_both(a, b, 990 + t)
        assert_same_state(a, a.param_groups, b, b.param_groups)


def _six_step_snapshot(stream=None, device=DEV):
    groups = make_groups(20_003, 8, device)
    opt = GaussianAdam(groups, lr=0.0, eps=1e-15)
    gen = torch.Generator().manual_seed(13)
    deg = torch.randint(0, 4, (20_003, 1), generator=gen, dtype=torch.int32).to(device)
    vis = (torch.rand(20_003, generator=gen) < 0.5).to(device)
    counts = []
    ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.device(device)
    with ctx:
        for t in range(4):
            set_grads([groups], 1000 + t)
            n0 = gsl.launch_count()
            opt.step(visibility=vis if t % 2 else None, degrees=deg if t >= 2 else None)
            counts.append(gsl.launch_count() - n0)
    torch.cuda.synchronize(device)
    out = []
    for grp in groups:
        p = grp["params"][0]
        out += [p.detach().cpu(), opt.state[p]["exp_avg"].cpu(), opt.state[p]["exp_avg_sq"].cpu()]
    return counts, out


def test_one_launch_same_bytes_streams_and_devices():
    counts, a = _six_step_snapshot()
    assert counts == [1, 1, 1, 1]
    _, b = _six_step_snapshot()
    _, c = _six_step_snapshot(stream=torch.cuda.Stream())
    for x, y, z in zip(a, b, c):
        assert torch.equal(bits(x), bits(y)) and torch.equal(bits(x), bits(z))
    if torch.cuda.device_count() > 1:
        _, d = _six_step_snapshot(device=torch.device("cuda", 1))
        for x, y in zip(a, d):
            assert torch.equal(bits(x), bits(y))


class _Model:
    """The attributes render() reads from the reference's GaussianModel (activations as in scene/gaussian_model.py:141-158)."""

    def __init__(self, scene, dev):
        self._xyz = torch.nn.Parameter(scene.means3D.to(dev).clone())
        self._opacity = torch.nn.Parameter(scene.opacity.to(dev).clone())
        self._log_scaling = torch.nn.Parameter(torch.log(scene.scales.to(dev)))
        self._rotation = torch.nn.Parameter(scene.rotations.to(dev).clone())
        self._features = torch.nn.Parameter(scene.sh.to(dev).clone())
        self._degrees = scene.degrees.to(dev)
        self.active_sh_degree = self.max_sh_degree = 3
        self.per_band_count = [int((scene.degrees == d).sum()) for d in range(4)]

    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: torch.exp(s._log_scaling))
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rotation))
    get_features = property(lambda s: s._features)

    def groups(self):
        return [{"params": [self._xyz], "lr": 2e-4, "name": "xyz"}, {"params": [self._opacity], "lr": 5e-2, "name": "opacity"},
                {"params": [self._log_scaling], "lr": 5e-3, "name": "scaling"}, {"params": [self._rotation], "lr": 1e-3, "name": "rotation"},
                {"params": [self._features], "lr": 1e-2, "name": "features", "sh_offset": 0}]


def test_training_with_sparse_steps_reduces_the_loss():
    from gaussian_renderer import render
    from utils.loss_utils import l1_ssim_loss
    W, H = 256, 192
    target = synth.make_scene(6_000, 71, sh_degree=3, mixed_degrees=True, box=(1.9 * W / H, 1.9, 1.0), log_scale_mean=math.log(0.04), M=16)
    cams = []
    for yaw in (-10.0, 0.0, 10.0):
        th = math.radians(yaw)
        Rc2w = np.array([[math.cos(th), 0, math.sin(th)], [0, 1, 0], [-math.sin(th), 0, math.cos(th)]])
        C = Rc2w @ np.array([0.0, 0.0, -4.0])
        cams.append(synth.make_camera(W, H, Rc2w, -Rc2w.T @ C).to(DEV))
    pipe = SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    bg = torch.tensor([0.1, 0.1, 0.1], device=DEV)
    with torch.no_grad():
        gts = [render(c, _Model(target, DEV), pipe, bg)["render"].clone() for c in cams]
    g = torch.Generator().manual_seed(5)
    start = synth.Scene(target.means3D + 0.01 * torch.randn(target.means3D.shape, generator=g),
                        target.opacity + 0.5 * torch.randn(target.opacity.shape, generator=g),
                        target.scales * torch.exp(0.2 * torch.randn(target.scales.shape, generator=g)),
                        torch.nn.functional.normalize(target.rotations + 0.1 * torch.randn(target.rotations.shape, generator=g)),
                        target.sh + 0.1 * torch.randn(target.sh.shape, generator=g), target.degrees)

    def train(make_opt, sparse):
        model = _Model(start, DEV)
        opt = make_opt(model.groups())
        losses = []
        for it in range(90):
            k = it % len(cams)
            opt.zero_grad(set_to_none=True)
            pkg = render(cams[k], model, pipe, bg)
            loss = l1_ssim_loss(pkg["render"], gts[k], 0.2)
            loss.backward()
            if sparse:
                opt.step(visibility=pkg["visibility_filter"], degrees=model._degrees)
            else:
                opt.step()
            losses.append(float(loss.detach()))
        return sum(losses[:3]) / 3, sum(losses[-3:]) / 3

    first, last = train(GaussianAdam, True)
    assert last < 0.8 * first, (first, last)
    _, last_dense = train(GaussianAdam, False)
    _, last_torch = train(torch.optim.Adam, False)
    assert last_dense < 0.8 * first
    # the render backward's atomics make the two runs differ in the last bits from the first step on
    assert abs(last_dense - last_torch) <= 0.05 * last_torch, (last_dense, last_torch)
