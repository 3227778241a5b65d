"""GPU: the contribution statistics (gsb_contributions, DESIGN.md §5p).

  - Per Gaussian against the float64 restatement of tests/contrib64.py on the 16 + 2 boundary scenes of backward_edges.py, t1 and
    the constructed exact fp32 tie: `pixels` exact, `weight_sum` within 1e-5 o64 + 1e-6 (+ the borderline allowance of
    statistics_edges), `weight_max` within (4 + 2 k) ulp, `top_id` equal where the best two weights differ by more than 1e-6
    relative, and the earlier Gaussian on the exact tie.  Anti-aliasing and a non-zero 3D filter against the restatement fed the
    kernel's own records (debug_out).
  - Each path against the path it is bit-identical to: raw = activated, quantised = de-quantised, pruned = compacted (ids
    remapped), zero filter_3D = none, variable_sh_bands = dense.
  - At 1080p with P = 1 M: pixels == the statistics forward's touched_pixels bitwise, sum weight_sum == sum (1 - final_T) to 1e-5,
    and the map-weighted sum == the F = 1 feature backward's dL_dfeatures within 1e-4 relative (or twice that path's run-to-run
    spread, if larger: the backward rebuilds T back to front with MUFU.RCP, so its alpha T is not the forward's).
  - Nothing else moves (colour, radii, maps, features, exports and the deterministic gradients are the same bytes with and without
    contributions); the same bytes on five runs, on a side stream and on a second GPU; a map with -1, 2, NaN and inf gives the bytes
    of its clamped copy; P = 0, R = 0 and all pruned; importance pruning over 8 orbit cameras followed by a training step.
Observed on one H100 80GB HBM3 at its 700 W limit (pytest -s prints the ratios per case): every count of a tight Gaussian exact;
the largest |d weight_sum| 0.029 of its bar (t1), |d weight_max| 0.93 of its bar (dense_12k), top_id equal on every checked pixel;
with AA / a filter 0.017 and 0.51 of the bars (large, filter_3D); at 1080p the weighted sum within 1.0e-5 of the feature backward,
whose own run-to-run spread is 5e-7.  Rounded without the FMAs of pair_power, the restatement puts t1's weight_max at 2.4 of its bar."""
import math

import numpy as np
import pytest
import torch

import backward_edges as BE
import contrib64 as C6
import gs_oracle
import ours as O
from diff_gaussian_rasterization import _C
from gs_b200 import synth
from gs_b200.model import GaussianModelView

pytestmark = pytest.mark.gpu
DEV = "cuda"
_cache = {}


def _fwd(scene, cam, bg=None, aa=False, dbg=None, **kw):
    """_C.rasterize_gaussians of an activated scene -> (args, outputs)."""
    args = O.forward_args(scene, cam, torch.zeros(3) if bg is None else bg)
    return args, _C.rasterize_gaussians(*args, antialiasing=aa, debug_out=dbg, **kw)


def _contrib(out, cam, P, weights=None):
    return _C.contributions(out[3], out[4], out[5], out[0], cam.image_width, cam.image_height, P, pixel_weights=weights)


def _np(c):
    return [t.cpu().numpy() for t in c]


def _same(a, b):
    return all(O.same(x, y) for x, y in zip(a, b))


def _oracle(name):
    if name not in _cache:
        case = C6.build(name)
        o = C6.oracle(case)
        _cache[name] = case, o, C6.restate(o, case.W, case.H), BE.borderline_pairs(o, case.W, case.H)
    return _cache[name]


@pytest.mark.parametrize("name", C6.CASES + [C6.TIE])
def test_per_gaussian_against_contrib64(name):
    case, o, c64, pairs = _oracle(name)
    dbg = {}
    _, out = _fwd(case.scene, case.cam, case.bg, dbg=dbg)
    st = O.state(out, case.cam, case.scene.P)
    assert int(out[0]) == int(o["num_rendered"]) and np.array_equal(out[2].cpu().numpy(), o["radii"])
    assert np.array_equal(st["point_list"].cpu().numpy().astype(np.uint32), o["point_list"])
    got = _np(_contrib(out, case.cam, case.scene.P))
    if name == C6.TIE:
        # the kernel's records are the oracle's bits, so the fp32 tie is the kernel's tie too
        assert np.array_equal(dbg["conic_opacity"].cpu().numpy(), o["conic_opacity"]) and np.array_equal(dbg["means2D"].cpu().numpy(), o["means2D"])
    ratios, failures = C6.compare(name, o, c64, pairs, got, tie_pixel=case.meta.get("tie_pixel"))
    assert not failures, [(what, ids[:8].tolist()) for what, ids in failures]


def _kernel_state(out, dbg, cam, bg):
    """The restatement's input built from the kernel's own records and lists (the oracle's render over them)."""
    st = O.state(out, cam, dbg["means2D"].shape[0])
    o = dict(radii=out[2].cpu().numpy(), means2D=dbg["means2D"].cpu().numpy(), conic_opacity=dbg["conic_opacity"].cpu().numpy(),
             rgb=dbg["rgb"].cpu().numpy(), point_list=st["point_list"].cpu().numpy().astype(np.uint32),
             ranges=st["ranges"].cpu().numpy().astype(np.uint32))
    o.update(gs_oracle.render_forward_stats(o, o, bg, cam.image_width, cam.image_height))
    assert np.array_equal(o["n_contrib"], st["n_contrib"].cpu().numpy().astype(np.uint32))
    return o


@pytest.mark.parametrize("mode", ["aa", "filter_3D"])
@pytest.mark.parametrize("name", ["odd_20x36", "saturation", "dense_4k", "large"])
def test_antialiasing_and_filter_against_the_kernels_records(name, mode):
    case = BE.build(name, aa=mode == "aa")
    dbg = {}
    kw = {}
    if mode == "filter_3D":
        kw["filter_3D"] = (0.3 * case.scene.scales.mean(1) * torch.rand(case.scene.P, generator=torch.Generator().manual_seed(3))).to(DEV)
    _, out = _fwd(case.scene, case.cam, case.bg, aa=mode == "aa", dbg=dbg, **kw)
    o = _kernel_state(out, dbg, case.cam, case.bg)
    c64 = C6.restate(o, case.W, case.H)
    _, failures = C6.compare("%s, %s" % (name, mode), o, c64, BE.borderline_pairs(o, case.W, case.H), _np(_contrib(out, case.cam, case.scene.P)))
    assert not failures, [(what, ids[:8].tolist()) for what, ids in failures]


# ---- the paths that are bit-identical to one another ----------------------------------------------------------------------------

def _render(pc, cam, pipe=None, **kw):
    from gaussian_renderer import render
    from types import SimpleNamespace
    pipe = pipe or SimpleNamespace(debug=False, convert_SHs_python=False, compute_cov3D_python=False)
    with torch.no_grad():
        return render(cam, pc, pipe, torch.tensor([0.2, 0.4, 0.6], device=DEV), contributions=True, **kw)


def _cam(W=160, H=96):
    return O.yaw_cam(W, H, 5.0)


def _map(H, W, seed=1):
    return torch.rand(H, W, generator=torch.Generator().manual_seed(seed)).to(DEV)


def test_raw_equals_activated():
    from test_gpu_fused_activations import Model, _scene, _render as render_fused
    cam = _cam()
    m = Model(_scene(20_000, cam.image_width, cam.image_height, 41), 15)
    w = _map(cam.image_height, cam.image_width)
    with torch.no_grad():
        a = render_fused(m, cam, False, contributions=True, pixel_weights=w)["contributions"]
        b = render_fused(m, cam, True, contributions=True, pixel_weights=w)["contributions"]
    assert int((a.pixels > 0).sum()) > 1000 and _same(a, b)


def test_quantised_equals_dequantised():
    cam = _cam()
    q = synth.quantise_scene(synth.make_scene(20_000, 42, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.02))).to(DEV)
    dense = q.dequantise()
    a = _render(GaussianModelView(dense, DEV, quant=q, requires_grad=False), cam)["contributions"]
    b = _render(GaussianModelView(dense, DEV, requires_grad=False), cam)["contributions"]
    assert int((a.pixels > 0).sum()) > 1000 and _same(a, b)


def test_pruned_equals_compacted():
    cam = _cam()
    scene = synth.make_scene(20_000, 43, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.02))
    pm = synth.prune_mask(scene.P, 7, 0.4).bool()
    keep = torch.nonzero(~pm).view(-1)
    small = synth.Scene(*[t[keep].contiguous() for t in (scene.means3D, scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees)])
    a = _render(GaussianModelView(scene, DEV, prune_mask=pm, requires_grad=False), cam)["contributions"]
    b = _render(GaussianModelView(small, DEV, requires_grad=False), cam)["contributions"]
    kd = keep.to(DEV)
    for x, y in zip(a[:3], b[:3]):
        assert O.same(x[kd], y) and not x[pm.to(DEV)].any()
    assert O.same(a.top_id, torch.where(b.top_id >= 0, kd[b.top_id.clamp(min=0).long()].int(), b.top_id))


def test_zero_filter_equals_none():
    cam = _cam()
    pc = GaussianModelView(synth.make_scene(20_000, 44, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.02)), DEV, requires_grad=False)
    a = _render(pc, cam)["contributions"]
    pc.filter_3D = torch.zeros(pc.get_xyz.shape[0], 1, device=DEV)
    b = _render(pc, cam)["contributions"]
    assert _same(a, b)


def test_variable_sh_bands_equals_dense():
    import cases
    _, scene, cam, _, _, _ = cases.build_inputs("g3")
    cam = cam.to(DEV)
    w = _map(cam.image_height, cam.image_width, 4)
    a = _render(GaussianModelView(scene, DEV, requires_grad=False, variable_sh_bands=True), cam, variable_sh_bands=True, pixel_weights=w)
    b = _render(GaussianModelView(scene, DEV, requires_grad=False), cam, pixel_weights=w)
    assert O.same(a["render"], b["render"]) and _same(a["contributions"], b["contributions"])


# ---- identities at 1080p -------------------------------------------------------------------------------------------------------

def test_identities_at_1080p():
    W, H = 1920, 1080
    cam = synth.make_camera(W, H)
    scene = synth.make_scene(1_000_000, 45, box=(3.0, 1.7, 1.0), log_scale_mean=math.log(0.01))
    args, out = _fwd(scene, cam)
    P = scene.P
    c = _contrib(out, cam, P)
    # the statistics forward's count
    touched = torch.empty(P, 1, dtype=torch.int32, device=DEV)
    tsum = torch.empty(P, 1, device=DEV)
    _C._forward(*args, statistics=(touched, tsum))
    assert int((c.pixels > 0).sum()) > 100_000 and O.same(c.pixels, touched.view(-1))
    # the weights of a pixel add up to its opacity
    st = O.state(out, cam, P)
    total = float((1.0 - st["final_T"].double()).sum())
    assert abs(float(c.weight_sum.double().sum()) - total) <= 1e-5 * total
    # the map-weighted sum is the F = 1 feature backward's dL_dfeatures (sum alpha T dL_dout)
    w = _map(H, W, 5)
    cw = _contrib(out, cam, P, w)
    ones = torch.ones(P, 1, device=DEV)
    runs = [O.backward(args, out, torch.zeros(3, H, W), features=ones, dL_dfeatures_out=w.view(1, H, W))[-1].view(-1).double()
            for _ in range(2)]
    scale = runs[0].abs() + 1e-6
    spread = float(((runs[0] - runs[1]).abs() / scale).max())
    err = float(((cw.weight_sum.double() - runs[0]).abs() / scale).max())
    print("\n[1080p, 1M] weight_sum vs feature backward: max rel err %.3g, the feature backward's own run-to-run spread %.3g" % (err, spread))
    assert err <= max(2.0 * spread, 1e-4)


# ---- nothing else moves; the same bytes everywhere --------------------------------------------------------------------------

def test_nothing_else_moves():
    from test_gpu_fused_activations import Model, _scene, _render as render_fused
    cam = _cam()
    base = Model(_scene(20_000, cam.image_width, cam.image_height, 46), 15)
    feats = torch.rand(base._xyz.shape[0], 3, device=DEV)
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        res = []
        for contrib in (False, True):
            m = base.clone()
            pkg = render_fused(m, cam, True, return_maps=True, features=feats, **(dict(contributions=True) if contrib else {}))
            (pkg["render"].sum() + pkg["invdepth"].sum() + 2 * pkg["alpha"].sum()).backward()
            res.append(([pkg[k] for k in ("render", "radii", "invdepth", "alpha", "features")], [t.grad for t in m.leaves()], pkg))
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    (o0, g0, _), (o1, g1, pkg) = res
    assert "contributions" in pkg and all(O.same(a, b) for a, b in zip(o0, o1)) and all(O.same(a, b) for a, b in zip(g0, g1))
    # the forward's exports are unchanged by the pass
    scene = synth.make_scene(20_000, 47, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.02))
    _, out = _fwd(scene, cam, return_maps=True)
    s0 = O.state(out, cam, scene.P)
    _contrib(out, cam, scene.P, _map(cam.image_height, cam.image_width))
    s1 = O.state(out, cam, scene.P)
    assert all(O.same(s0[k], s1[k]) for k in s0)


def test_same_bytes_on_every_run_stream_and_device():
    cam = _cam()
    scene = synth.make_scene(50_000, 48, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.02))
    _, out = _fwd(scene, cam)
    w = _map(cam.image_height, cam.image_width, 6)
    for weights in (None, w):
        first = _contrib(out, cam, scene.P, weights)
        for _ in range(4):
            assert _same(first, _contrib(out, cam, scene.P, weights))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            again = _contrib(out, cam, scene.P, weights)
        side.synchronize()
        assert _same(first, again)
        if torch.cuda.device_count() > 1:
            with torch.cuda.device(1):
                args = O.forward_args(scene, cam, torch.zeros(3), dev="cuda:1")
                out1 = _C.rasterize_gaussians(*args)
                c1 = _C.contributions(out1[3], out1[4], out1[5], out1[0], cam.image_width, cam.image_height, scene.P,
                                      pixel_weights=None if weights is None else weights.to("cuda:1"))
            assert _same(first, [t.to(DEV) for t in c1])


def test_map_is_clamped_on_read():
    cam = _cam()
    scene = synth.make_scene(20_000, 49, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.02))
    _, out = _fwd(scene, cam)
    w = (3.0 * _map(cam.image_height, cam.image_width, 7) - 1.0)
    w.view(-1)[::5] = -1.0
    w.view(-1)[1::5] = 2.0
    w.view(-1)[2::7] = float("nan")
    w.view(-1)[3::11] = float("inf")
    w.view(-1)[4::13] = float("-inf")
    clamped = torch.where(torch.isnan(w), torch.zeros_like(w), w.clamp(0.0, 1.0))
    assert _same(_contrib(out, cam, scene.P, w), _contrib(out, cam, scene.P, clamped))
    assert _same(_contrib(out, cam, scene.P, w.view(1, *w.shape)), _contrib(out, cam, scene.P, clamped))


def test_edge_cases():
    empty, culled = O.empty_and_culled_scenes()
    cam = synth.make_camera(33, 17)
    for scene in (empty, culled):
        _, out = _fwd(scene, cam)
        c = _contrib(out, cam, scene.P, _map(17, 33))
        assert not any(t.any() for t in c[:3]) and bool((c.top_id == -1).all()) and tuple(c.top_id.shape) == (17, 33)
    scene = synth.make_scene(5_000, 50, box=(3.0, 1.9, 1.0), log_scale_mean=math.log(0.03))
    _, out = _fwd(scene, cam, prune_mask=torch.ones(scene.P, dtype=torch.bool, device=DEV))
    c = _contrib(out, cam, scene.P)
    assert int(out[0]) == 0 and not any(t.any() for t in c[:3]) and bool((c.top_id == -1).all())


def test_importance_pruning_over_orbit_cameras_then_a_training_step():
    from test_gpu_fused_activations import Model, _adam, _scene, _render as render_fused
    from gs_b200 import densify
    W, H = 160, 96
    m = Model(_scene(30_000, W, H, 51), 15)
    m.optimizer = _adam(m)
    P = m._xyz.shape[0]
    m.xyz_gradient_accum, m.denom, m.max_radii2D = torch.zeros(P, 1, device=DEV), torch.zeros(P, 1, device=DEV), torch.zeros(P, device=DEV)
    cams = synth.orbit_cameras(8, W, H, radius=4.0)
    score = torch.zeros(P, device=DEV)
    with torch.no_grad():
        for cam in cams:
            score += render_fused(m, cam.to(DEV), True, contributions=True)["contributions"].weight_sum
    assert int((score > 0).sum()) > P // 4
    prune = torch.zeros(P, dtype=torch.bool, device=DEV)
    prune[torch.argsort(score)[:int(0.3 * P)]] = True
    densify.prune_points(m, prune)
    assert m._xyz.shape[0] == P - int(0.3 * P)
    gt = torch.rand(3, H, W, device=DEV)
    pkg = render_fused(m, cams[0].to(DEV), True)
    loss = (pkg["render"] - gt).abs().mean()
    loss.backward()
    m.optimizer.step()
    assert math.isfinite(float(loss.detach())) and all(torch.isfinite(t).all() for t in m.leaves())
