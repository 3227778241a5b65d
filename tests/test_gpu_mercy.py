"""gs_b200.densify.calculate_redundancy_metric / mercy_points on the GPU against the reference's glue restated in torch over the
same library (tests/mercy_restatement.py), the reference's own records (kn_red.npz, mercy_*.npz) and a torch.sort of the
opacities beyond torch.quantile's 2^24 limit."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "reduced-3dgs_b200"))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import knn_cases as KC  # noqa: E402
import mercy_restatement as mr  # noqa: E402
import refsummary as S  # noqa: E402
from gs_b200 import densify  # noqa: E402
from gs_b200 import lib as gsl  # noqa: E402
from gs_b200.optim import GaussianAdam  # noqa: E402
from test_gpu_densify import assert_same, clone_model, synthetic  # noqa: E402

pytestmark = pytest.mark.gpu
TYPES = ("redundancy_opacity", "redundancy_random", "opacity", "redundancy_opacity_opacity", "anything else")
GOLDENS = sorted(os.path.basename(p)[6:-4] for p in glob.glob(os.path.join(HERE, "golden", "mercy_*.npz")))


def _scene(P, seed=5, kind="C3"):
    """(xyz, scales, rotations) on the GPU, cameras of the t1 tools case."""
    g = torch.Generator().manual_seed(seed)
    if kind == "t1":
        c, scene, cams = KC.red_inputs()
        return scene.means3D.cuda(), scene.scales.cuda(), scene.rotations.cuda(), cams, c["radius_scale"]
    xyz = KC.c3_positions(P)
    scales = torch.exp(np.log(0.004) + 0.6 * torch.randn(P, 3, generator=g))
    q = torch.randn(P, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    _, _, cams = KC.red_inputs()
    return xyz.cuda(), scales.cuda(), q.cuda(), cams, 1.0


def _both(xyz, sc, rot, cams, ps, K, defined=False):
    s = mr.RedScene(xyz, sc, rot, cams)
    ours = densify.calculate_redundancy_metric(s, pixel_scale=ps, num_neighbours=K)
    ref = mr.calculate_redundancy_metric(s, pixel_scale=ps, num_neighbours=K, defined=defined)
    return ours, ref


def _assert_red_equal(ours, ref):
    (m, c), (rm, rc) = ours, ref
    assert m.dtype == torch.int32 and m.shape == rm.shape and c.dtype == torch.float32 and c.shape == rc.shape
    assert torch.equal(m, rm), "min_redundancy differs from the chain"
    assert c.cpu().numpy().tobytes() == rc.cpu().numpy().tobytes(), "cube_size differs from the chain"


@pytest.mark.parametrize("P,K,ps,kind", [(20_000, 30, None, "t1"), (100_000, 1, 1.0, "C3"), (100_000, 30, 0.37, "C3"),
                                         (100_000, 64, 1.0, "C3"), (100_000, 30, 1.0, "C3"), (3_000_000, 30, 1.0, "C3")])
def test_redundancy_against_chain(P, K, ps, kind):
    xyz, sc, rot, cams, rs = _scene(P, kind=kind)
    ours, ref = _both(xyz, sc, rot, cams, rs if ps is None else ps, K)
    _assert_red_equal(ours, ref)
    assert int(ours[0].min()) >= 1 and int(ours[0].max()) <= K + 1


def test_redundancy_against_reference_record():
    ref = S.load_parts("kn_red")
    xyz, sc, rot, cams, ps = _scene(0, kind="t1")
    m, _ = densify.calculate_redundancy_metric(mr.RedScene(xyz, sc, rot, cams), pixel_scale=ps, num_neighbours=30)
    if int(ref["n_ties"]) == 0:
        assert np.array_equal(m.cpu().numpy(), ref["min_redundancy"])
    else:
        pytest.skip("kn_red has neighbours tied at the K-th distance")


@pytest.mark.parametrize("P,K", [(1, 30), (20, 30), (30, 30), (31, 30), (5, 64)])
def test_redundancy_small_defined(P, K):
    xyz, sc, rot, cams, _ = _scene(P)
    ours, ref = _both(xyz[:P].contiguous(), sc[:P].contiguous(), rot[:P].contiguous(), cams, 0.37, K, defined=True)
    _assert_red_equal(ours, ref)


def test_redundancy_empty():
    z = torch.zeros((0, 3), device="cuda")
    _, _, cams = KC.red_inputs()
    m, c = densify.calculate_redundancy_metric(mr.RedScene(z, z, torch.zeros((0, 4), device="cuda"), cams))
    assert m.shape == (0, 1) and c.shape == (0, 1)


def test_redundancy_peak_memory():
    P, K = 1_000_000, 30
    xyz, sc, rot, cams, _ = _scene(P)
    s = mr.RedScene(xyz, sc, rot, cams)
    peaks = {}
    for name, fn in (("chain", lambda: mr.calculate_redundancy_metric(s, num_neighbours=K)),
                     ("native", lambda: densify.calculate_redundancy_metric(s, num_neighbours=K))):
        fn()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del out
    assert peaks["native"] <= peaks["chain"] - P * (K + 1) * 5, peaks


def test_redundancy_deterministic_and_side_stream():
    xyz, sc, rot, cams, _ = _scene(300_000)
    s = mr.RedScene(xyz, sc, rot, cams)
    first = [t.cpu().numpy().tobytes() for t in densify.calculate_redundancy_metric(s)]
    side = torch.cuda.Stream()
    for i in range(5):
        with torch.cuda.stream(side if i % 2 else torch.cuda.current_stream()):
            out = densify.calculate_redundancy_metric(s)
        torch.cuda.synchronize()
        assert [t.cpu().numpy().tobytes() for t in out] == first


# ------------------------------------------------------------------------------------------------ mercy
def _counts(P, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = (torch.poisson(torch.full((P,), 4.0, device="cuda"), generator=g) + 1).to(torch.int32)
    return c


def _mercy_pair(P, mtype, opt_cls, seed=0, lam=1.0, mmin=2):
    m = synthetic(P, 15, seed, opt_cls=opt_cls)
    m._opacity.data.copy_(torch.randn(P, 1, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed + 7)) * 2)
    k = seed
    while True:                                # counts whose exact threshold is at least 1e-4 from an integer
        c = _counts(P, k)
        x = c.double()
        t = float(x.mean() + lam * x.std())
        if abs(t - round(t)) >= 1e-4:
            break
        k += 1
    r = clone_model(m, opt_cls)
    m._splatted_num_accum = c.view(P, 1, 1).clone()
    r._splatted_num_accum = c.view(P, 1, 1).clone()
    torch.cuda.manual_seed(1234)
    d = {}
    densify.mercy_points(m, d, lam, mmin, mtype)
    s_ours = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(1234)
    rd = {}
    mr.mercy_points(r, rd, lam, mmin, mtype, prune_points=lambda mask: densify.prune_points(r, mask))
    s_ref = torch.cuda.get_rng_state()
    return m, d, r, rd, torch.equal(s_ours, s_ref)


def _assert_dict(d, rd):
    assert sorted(d) == sorted(rd)
    for k in d:
        a, b = d[k], rd[k]
        assert type(a) is type(b), k
        if torch.is_tensor(a):                 # the reference's opacity threshold carries a grad_fn; ours is a plain statistic
            a, b = a.detach(), b.detach()
        if not torch.is_tensor(a):
            assert a == b, k
            continue
        assert a.shape == b.shape and a.dtype == b.dtype and a.device == b.device, k
        if k == "redundancy_threshold":       # correctly rounded here, torch's fp32 reduction tree there (DESIGN.md §5k)
            assert torch.allclose(a, b, rtol=2e-6, atol=0), (a, b)
        else:
            assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), (k, a, b)


@pytest.mark.parametrize("opt_cls", [torch.optim.Adam, GaussianAdam])
@pytest.mark.parametrize("mtype", TYPES)
@pytest.mark.parametrize("P", [100_000, 3_000_000])
def test_mercy_against_restatement(P, mtype, opt_cls):
    if P > 100_000 and opt_cls is GaussianAdam and mtype not in ("redundancy_opacity", "redundancy_opacity_opacity"):
        pytest.skip("3 M is run with GaussianAdam for the two median types only")
    m, d, r, rd, same_rng = _mercy_pair(P, mtype, opt_cls)
    assert same_rng, "the CUDA generator state differs from the reference's"
    assert_same(m, r)
    _assert_dict(d, rd)
    assert m._xyz.shape[0] == P - int(d["n_points_mercied"])


def _golden_model(z):
    P = int(z["P"])
    m = synthetic(P, 15, 3)
    m._opacity.data.copy_(torch.from_numpy(z["logits"]).cuda())
    m._splatted_num_accum = torch.from_numpy(z["counts"]).cuda().view(P, 1, 1)
    return m


@pytest.mark.parametrize("name", GOLDENS)
def test_mercy_goldens(name, monkeypatch):
    z = dict(np.load(os.path.join(HERE, "golden", f"mercy_{name}.npz")))
    m = _golden_model(z)
    keep = ~z["mask"]
    want = m._opacity.detach().cpu().numpy()[keep]
    draws = torch.from_numpy(z["draws"]).cuda()
    calls = []
    real = torch.rand
    monkeypatch.setattr(torch, "rand", lambda shape, **k: calls.append(tuple(shape)) or (real(shape, **k).copy_(draws.view(shape))))
    d = {}
    densify.mercy_points(m, d, float(z["lambda"]), int(z["mercy_minimum"]), str(z["type"]))
    assert len(calls) == int(z["n_draw_calls"])
    assert m._opacity.detach().cpu().numpy().tobytes() == want.tobytes()       # NaN logits compare by their bits
    assert int(d["n_points_mercied"]) == int(z["n_points_mercied"])
    rt = d["redundancy_threshold"].cpu().numpy()
    assert rt.shape == z["redundancy_threshold"].shape
    assert np.allclose(rt, z["redundancy_threshold"], rtol=2e-6, atol=0, equal_nan=True)
    ot = d["opacity_threshold"]
    assert torch.is_tensor(ot) == bool(z["opacity_threshold_is_tensor"])
    if torch.is_tensor(ot):
        o = ot.cpu().numpy()
        assert o.shape == z["opacity_threshold"].shape
        # the goldens' lerp ran on the CPU; the CUDA lerp may round the last bit differently
        assert np.allclose(o, z["opacity_threshold"], rtol=3e-7, atol=0, equal_nan=True)


def _plan_direct(counts, logits, code, lam=2.0, mmin=2.0, q=0.045, stream=None):
    P = counts.numel()
    L = gsl.lib()
    ws = torch.empty(L.gsb_mercy_workspace_bytes(P), dtype=torch.uint8, device="cuda")
    mask = torch.empty(P, dtype=torch.uint8, device="cuda")
    thr = torch.empty(2, device="cuda")
    cnt = torch.empty(2, dtype=torch.int64, device="cuda")
    st = (stream or torch.cuda.current_stream()).cuda_stream
    gsl.check(L.gsb_mercy_plan(P, counts.data_ptr(), logits.data_ptr(), code, lam, mmin, q, None, -1, ws.data_ptr(),
                               mask.data_ptr(), thr.data_ptr(), cnt.data_ptr(), st))
    return mask, thr, cnt


def _quantile_by_sort(v, q):
    """torch.quantile's fp32 rank / lerp formula on a torch.sort (no size limit)."""
    s = torch.sort(v)[0]
    n = s.numel()
    r = torch.tensor(q, dtype=torch.float32, device=v.device) * torch.tensor(float(n - 1), dtype=torch.float32, device=v.device)
    lo = r.to(torch.int64)
    w = r - lo
    hi = torch.ceil(r).to(torch.int64)
    return torch.lerp(s[lo], s[hi], w)


def test_opacity_beyond_quantile_limit():
    P = (1 << 24) + 3
    g = torch.Generator(device="cuda").manual_seed(9)
    logits = torch.randn(P, device="cuda", generator=g) * 2
    counts = torch.ones(P, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="too large"):
        torch.sigmoid(logits).quantile(0.045)
    mask, thr, cnt = _plan_direct(counts, logits, gsl.MERCY_OPACITY)
    op = torch.sigmoid(logits)
    want = _quantile_by_sort(op, 0.045)
    assert thr[1].cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
    assert torch.equal(mask.bool(), op < want)
    assert int(cnt[1]) == int((op < want).sum())


def test_mercy_deterministic_and_second_device():
    P = 2_000_000
    g = torch.Generator(device="cuda").manual_seed(4)
    logits = torch.randn(P, device="cuda", generator=g) * 2
    counts = _counts(P, 4)
    first = [t.cpu().numpy().tobytes() for t in _plan_direct(counts, logits, gsl.MERCY_REDUNDANCY_OPACITY_OPACITY, q=0.03)]
    side = torch.cuda.Stream()
    for i in range(5):
        out = _plan_direct(counts, logits, gsl.MERCY_REDUNDANCY_OPACITY_OPACITY, q=0.03, stream=side if i % 2 else None)
        torch.cuda.synchronize()
        assert [t.cpu().numpy().tobytes() for t in out] == first
    if torch.cuda.device_count() > 1:
        with torch.cuda.device(1):
            out = _plan_direct(counts.to("cuda:1"), logits.to("cuda:1"), gsl.MERCY_REDUNDANCY_OPACITY_OPACITY, q=0.03)
            torch.cuda.synchronize()
        assert [t.cpu().numpy().tobytes() for t in out] == first
