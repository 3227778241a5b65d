"""CPU: GaussianAdam (gs_b200.optim) and gsb_adam_step without a GPU — the C ABI's layout and argument checks, the refused
options, and, with a stub of the library, the tensor table the Python side builds (widths, sh_offset, and the fp32 scalars
against the values torch's own foreach Adam hands to its kernels)."""
import contextlib
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from gs_b200 import lib as gsl
from gs_b200 import optim
from gs_b200.optim import GaussianAdam

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = [f for f, _ in gsl.GsbAdamTensor._fields_]


def test_symbol_and_layout_match_header():
    assert "gsb_adam_step" in gsl.EXPORTED_SYMBOLS and gsl.lib().gsb_adam_step is not None
    text = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
    assert int(re.search(r"#define GSB_ADAM_MAX_TENSORS (\d+)", text).group(1)) == gsl.ADAM_MAX_TENSORS
    T = gsl.GsbAdamTensor
    assert C.sizeof(T) == 4 * 8 + 8 + 4 + 4 + 6 * 4
    assert (T.numel.offset, T.row_width.offset, T.sh_offset.offset, T.one_minus_beta1.offset, T.step_size.offset) == (32, 40, 44, 48, 68)
    assert FIELDS[-6:] == ["one_minus_beta1", "beta2", "one_minus_beta2", "eps", "bc2_sqrt", "step_size"]


def _entry(numel=12, width=3, sh=-1, base=0x10000):
    e = gsl.GsbAdamTensor()
    e.param, e.grad, e.exp_avg, e.exp_avg_sq = base, base + 0x1000, base + 0x2000, base + 0x3000
    e.numel, e.row_width, e.sh_offset = numel, width, sh
    return e


@pytest.mark.parametrize("case", ["n_negative", "n_too_many", "null_table", "P_negative", "numel_negative", "null_pointer",
                                  "sh_offset_below", "sh_width_not_3", "rows_not_P", "width_zero_sparse", "misaligned"])
def test_einval_without_gpu(case):
    """Every one of these is rejected before any CUDA call (fake device addresses are never touched)."""
    L = gsl.lib()
    n, P, vis, deg = 1, 4, None, None
    e = _entry()
    if case == "n_negative":
        n = -1
    elif case == "n_too_many":
        n = gsl.ADAM_MAX_TENSORS + 1
    elif case == "null_table":
        st = L.gsb_adam_step(None, 1, 4, None, None, None)
        assert st == -1 and b"adam" in L.gsb_last_error()
        return
    elif case == "P_negative":
        P = -1
    elif case == "numel_negative":
        e.numel = -5
    elif case == "null_pointer":
        e.exp_avg_sq = None
    elif case == "sh_offset_below":
        e.sh_offset = -2
    elif case == "sh_width_not_3":
        e.sh_offset, e.row_width, e.numel = 1, 4, 16
        deg = 0x40000
    elif case == "rows_not_P":
        e.numel = 13                          # 4 rows of 3 = 12
        vis = 0x40000
    elif case == "width_zero_sparse":
        e.row_width = 0
        deg = 0x40000
    elif case == "misaligned":
        e.grad = e.grad + 2
    table = (gsl.GsbAdamTensor * max(n, 1, gsl.ADAM_MAX_TENSORS + 1))(*([e] * (gsl.ADAM_MAX_TENSORS + 1)))
    st = L.gsb_adam_step(table, n, P, vis, deg, None)
    assert st == -1, case
    assert b"adam_step" in L.gsb_last_error()


def _param(*shape):
    return torch.nn.Parameter(torch.zeros(*shape))


@pytest.mark.parametrize("kw", [dict(amsgrad=True), dict(weight_decay=0.01), dict(maximize=True), dict(capturable=True),
                                dict(differentiable=True), dict(fused=True), dict(lr=torch.tensor(0.1)), dict(betas=(torch.tensor(0.9), 0.999))])
def test_refused_options(kw):
    with pytest.raises(ValueError):
        GaussianAdam([_param(4, 3)], **kw)


def test_refused_group_options_and_sh_offset():
    with pytest.raises(ValueError):
        GaussianAdam([{"params": [_param(4, 3)], "amsgrad": True}])
    with pytest.raises(ValueError):
        GaussianAdam([{"params": [_param(4, 3)], "weight_decay": 1e-4}])
    with pytest.raises(ValueError):
        GaussianAdam([{"params": [_param(4, 15, 3)], "sh_offset": -1}])
    opt = GaussianAdam([_param(4, 3)])
    opt.param_groups[0]["maximize"] = True            # options changed after construction are caught by step()
    opt.param_groups[0]["params"][0].grad = torch.zeros(4, 3)
    with pytest.raises(ValueError):
        opt.step()


def test_refused_tensors():
    p = _param(4, 3)
    opt = GaussianAdam([p])
    p.grad = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="CUDA"):                    # CPU tensors: there is no CPU path
        opt.step()
    p.grad = torch.zeros(4, 3).to_sparse()
    with pytest.raises(RuntimeError, match="sparse"):
        opt.step()
    q = torch.nn.Parameter(torch.zeros(4, 3, dtype=torch.float64))
    q.grad = torch.zeros(4, 3, dtype=torch.float64)
    with pytest.raises(RuntimeError, match="fp32"):
        GaussianAdam([q]).step()
    r = torch.nn.Parameter(torch.zeros(3, 4).t())
    r.grad = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="contiguous"):
        GaussianAdam([r]).step()
    p.grad = torch.zeros(3, 4).t()
    with pytest.raises(RuntimeError, match="contiguous"):
        opt.step()
    p.grad = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="visibility"):
        opt.step(visibility=torch.ones(4, dtype=torch.bool))           # a CPU mask
    with pytest.raises(RuntimeError, match="degrees"):
        opt.step(degrees=torch.zeros(4, dtype=torch.int32))
    assert len(opt.state) == 0                                          # nothing was touched


# ---- with a stub of the library: the Python side's table, on CPU tensors ----

class _StubLib:
    def __init__(self):
        self.calls = []

    def gsb_adam_step(self, table, n, P, vis, deg, stream):
        self.calls.append(dict(P=P, vis=vis, deg=deg, entries=[{f: getattr(table[i], f) for f in FIELDS} for i in range(n)]))
        return 0


@pytest.fixture
def stub(monkeypatch):
    s = _StubLib()
    monkeypatch.setattr(gsl, "lib", lambda: s)
    monkeypatch.setattr(gsl, "current_stream", lambda dev: 0)
    monkeypatch.setattr(gsl, "on_device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(optim, "_check_tensor", lambda p, g, banded: None)     # lets CPU tensors through to the stub
    return s


def _six_groups(P, lr_scale=1.0):
    """The reference's training_setup groups (scene/gaussian_model.py:208-217 shapes and names), own values."""
    shapes = [("xyz", (P, 3), 1.6e-4), ("f_dc", (P, 1, 3), 2.5e-3), ("f_rest", (P, 15, 3), 2.5e-3 / 20), ("opacity", (P, 1), 0.05),
              ("scaling", (P, 3), 5e-3), ("rotation", (P, 4), 1e-3)]
    g = torch.Generator().manual_seed(3)
    groups = []
    for name, shape, lr in shapes:
        p = torch.nn.Parameter(torch.randn(*shape, generator=g))
        grp = {"params": [p], "lr": lr * lr_scale, "name": name}
        if name == "f_rest":
            grp["sh_offset"] = 1
        groups.append(grp)
    return groups


def _set_grads(groups, seed):
    g = torch.Generator().manual_seed(seed)
    for grp in groups:
        p = grp["params"][0]
        p.grad = torch.randn(p.shape, generator=g)


def test_table_of_the_six_group_model_matches_torch_scalars(stub, monkeypatch):
    """widths and sh_offset, and step_size / bc2_sqrt equal (as fp32) to what torch's foreach Adam passes to its kernels."""
    P = 10
    ours = _six_groups(P)
    theirs = _six_groups(P)
    opt = GaussianAdam(ours, lr=0.0, eps=1e-15)
    ref = torch.optim.Adam(theirs, lr=0.0, eps=1e-15, foreach=True)
    seen = {}
    orig_div, orig_addcdiv = torch._foreach_div_, torch._foreach_addcdiv_

    def div_(tensors, other):
        seen["bc2_sqrt"] = list(other)
        return orig_div(tensors, other)

    def addcdiv_(p, m, d, scalars):
        seen["step_size"] = list(scalars)
        return orig_addcdiv(p, m, d, scalars)

    monkeypatch.setattr(torch, "_foreach_div_", div_)
    monkeypatch.setattr(torch, "_foreach_addcdiv_", addcdiv_)
    checked = 0
    rows = optim._rows
    for t in range(1, 1001):
        _set_grads(ours, t)
        _set_grads(theirs, t)
        seen.clear()
        if t == 2:          # the sparse form, with CPU stand-ins for the mask and the degrees
            monkeypatch.setattr(optim, "_rows", lambda v, d: (P, torch.device("cpu")))
            opt.step(visibility=torch.ones(P, dtype=torch.bool), degrees=torch.zeros(P, 1, dtype=torch.int32))
            monkeypatch.setattr(optim, "_rows", rows)
        else:
            opt.step()
        ref.step()          # one group per call of the foreach kernels: `seen` holds the last group's (rotation's) scalars
        call = stub.calls[-1]
        assert len(stub.calls) == t and len(call["entries"]) == 6
        if t in (1, 2, 1000):
            E = call["entries"]
            if t == 2:      # sparse: rows of P, the f_rest group banded from coefficient 1
                assert call["P"] == P
                assert [e["row_width"] for e in E] == [3, 3, 45, 1, 3, 4]
                assert [e["sh_offset"] for e in E] == [-1, -1, 1, -1, -1, -1]
            else:
                assert call["P"] == 0 and [e["sh_offset"] for e in E] == [-1] * 6
            assert [e["numel"] for e in E] == [P * 3, P * 3, P * 45, P, P * 3, P * 4]
            for e, grp in zip(E, ours):
                lr = grp["lr"]
                assert e["step_size"] == float(np.float32((lr / (1 - 0.9 ** t)) * -1))
                assert e["bc2_sqrt"] == float(np.float32((1 - 0.999 ** t) ** 0.5))
                assert e["one_minus_beta1"] == float(np.float32(1 - 0.9)) and e["beta2"] == float(np.float32(0.999))
                assert e["one_minus_beta2"] == float(np.float32(1 - 0.999)) and e["eps"] == float(np.float32(1e-15))
            assert E[-1]["step_size"] == float(np.float32(seen["step_size"][0]))
            assert E[-1]["bc2_sqrt"] == float(np.float32(seen["bc2_sqrt"][0]))
            checked += 1
        assert float(opt.state[ours[0]["params"][0]]["step"]) == t
    assert checked == 3


def test_state_layout_matches_torch_adam(stub):
    p, q = _param(5, 3), _param(5, 3)
    p.grad, q.grad = torch.ones(5, 3), torch.ones(5, 3)
    ours, ref = GaussianAdam([p]), torch.optim.Adam([q])
    ours.step()
    ref.step()
    so, sr = ours.state[p], ref.state[q]
    assert list(so) == list(sr) == ["step", "exp_avg", "exp_avg_sq"]
    for k in so:
        assert so[k].dtype == sr[k].dtype and so[k].shape == sr[k].shape and so[k].device == sr[k].device
    assert so["step"].device.type == "cpu" and so["step"].dtype == torch.float32 and float(so["step"]) == 1.0
    sd_o, sd_r = ours.state_dict(), ref.state_dict()
    assert set(sd_o["param_groups"][0]) == set(sd_r["param_groups"][0])


def test_lr_change_reaches_next_call(stub):
    groups = _six_groups(6)
    opt = GaussianAdam(groups, lr=0.0, eps=1e-15)
    _set_grads(groups, 1)
    opt.step()
    opt.param_groups[0]["lr"] = 0.5                        # what the reference's xyz scheduler does between steps
    opt.step()
    e = stub.calls[-1]["entries"][0]
    assert e["step_size"] == float(np.float32((0.5 / (1 - 0.9 ** 2)) * -1))
    assert stub.calls[-1]["entries"][1]["step_size"] == float(np.float32((2.5e-3 / (1 - 0.9 ** 2)) * -1))


def test_params_without_grad_are_left_out(stub):
    groups = _six_groups(6)
    opt = GaussianAdam(groups)
    _set_grads(groups, 1)
    groups[3]["params"][0].grad = None
    opt.step()
    E = stub.calls[-1]["entries"]
    assert len(E) == 5 and groups[3]["params"][0].data_ptr() not in [e["param"] for e in E]
    assert groups[3]["params"][0] not in opt.state


def test_empty_model_makes_no_call(stub):
    groups = _six_groups(0)
    opt = GaussianAdam(groups)
    _set_grads(groups, 1)
    opt.step()
    assert stub.calls == []
    assert float(opt.state[groups[0]["params"][0]]["step"]) == 1.0          # the step still advances, as in torch


def test_more_tensors_than_the_table_holds_take_several_calls(stub):
    ps = [_param(3, 2) for _ in range(gsl.ADAM_MAX_TENSORS + 3)]
    for p in ps:
        p.grad = torch.ones(3, 2)
    GaussianAdam(ps).step()
    assert [len(c["entries"]) for c in stub.calls] == [gsl.ADAM_MAX_TENSORS, 3]
    assert [e["param"] for c in stub.calls for e in c["entries"]] == [p.data_ptr() for p in ps]


def test_refused_step_leaves_the_optimizer_as_it_was(stub, monkeypatch):
    """A mask whose row count differs from a param with a gradient is refused before any state is created or advanced."""
    groups = _six_groups(10)
    opt = GaussianAdam(groups)
    _set_grads(groups, 1)
    groups[0]["params"][0].grad = None
    opt.step()                                                          # xyz has no state yet, the others step 1
    _set_grads(groups, 2)
    monkeypatch.setattr(optim, "_rows", lambda v, d: (7, torch.device("cpu")))
    with pytest.raises(RuntimeError, match="dim 0"):
        opt.step(visibility=torch.ones(7, dtype=torch.bool))
    assert groups[0]["params"][0] not in opt.state
    assert [float(opt.state[g["params"][0]]["step"]) for g in groups[1:]] == [1.0] * 5
    assert len(stub.calls) == 1
