"""GPU: the deterministic SH-culling statistics and k-means (DESIGN.md §5j).
  1. statistics: touched_pixels equal to the default path's, transmittance_sum within 1e-6 of it (both paths against the oracle:
     test_gpu_statistics_edges.py), the t1 / t1_large golden bars (2e-5) through calculate_colours_variance under torch's
     flag, five identical runs of all three outputs at 1920x1080 (1 M Gaussians, 8 cameras) also on a side stream and a second GPU,
     and the edges P = 0, R = 0 and everything outside the view;
  2. k-means: 0 iterations give the default ids; after 1 iteration and at convergence the centres are bit-identical to the float32
     restatement (oracle/kmeans_det_order.py) and the last iteration is the restatement's; the ids are the assignment for the returned
     centres; the k1 / k1_large golden checks; five identical runs on 9 M values for skewed and degenerate inputs;
  3. end to end: a reduced-3dgs run (training with densification, SH-band culling, redundancy pruning, 20 codebooks, the quantised
     PLY) twice under torch.use_deterministic_algorithms(True) gives the same degrees, codebooks and PLY bytes."""
import contextlib
import math
import os
import sys

import numpy as np
import pytest
import torch

import ours as O
import test_gpu_tools as T
from test_gpu_statistics_edges import stats_forward
from diff_gaussian_rasterization import _C
from gs_b200 import densify, ply, synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
sys.path.insert(0, os.path.join(HERE, "golden"))
import cases  # noqa: E402
import kmeans_det_order as KD  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


@contextlib.contextmanager
def torch_flag(on=True):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


# ---- 1. statistics -------------------------------------------------------------------------------------------------------------
def test_statistics_match_the_default_path():
    c, scene, cams, nb = cases.build_tools_inputs("t1")
    cam = cams[0]
    R0, r0, t0, s0, _ = stats_forward(scene, cam, False)
    R1, r1, t1, s1, _ = stats_forward(scene, cam, True)
    assert R0 == R1 and torch.equal(r0, r1)
    assert torch.equal(t0, t1) and int(t1.sum()) > 0
    s0, s1 = s0.cpu().numpy().reshape(-1), s1.cpu().numpy().reshape(-1)
    assert np.abs(s1.astype(np.float64) - s0).max() <= 1e-6 * np.abs(s0).max()
    assert np.all((s1 == 0) == (t1.cpu().numpy().reshape(-1) == 0))


def test_colour_variance_goldens_under_the_torch_flag():
    """test_gpu_tools' t1 and t1_large checks (2e-5 on the three colour-variance outputs) with the flag on: None follows it."""
    with torch_flag():
        for name in [n for n in cases.TOOLS_CASES if os.path.isfile(os.path.join(T.GOLD, n + ".npz"))]:
            T.test_tools_against_reference_goldens(name)
        T.test_tools_against_live_reference()


def _dense_views(n, W=1920, H=1080):
    cams = [O.yaw_cam(W, H, yaw) for yaw in np.linspace(-20.0, 20.0, n)]
    return dict(positions=torch.stack([c.camera_center for c in cams]), views=torch.stack([c.world_view_transform for c in cams]),
                projs=torch.stack([c.full_proj_transform for c in cams]),
                tanx=torch.tensor([math.tan(c.FoVx * 0.5) for c in cams]), tany=torch.tensor([math.tan(c.FoVy * 0.5) for c in cams]),
                H=torch.full((n,), H, dtype=torch.int32), W=torch.full((n,), W, dtype=torch.int32))


def _variance(sc, ct, **kw):
    return _C.calculate_colours_variance(ct["positions"], sc.means3D, sc.opacity, sc.scales, sc.rotations, ct["views"], ct["projs"],
                                         ct["tanx"], ct["tany"], ct["H"], ct["W"], sc.sh, sc.degrees, 3, **kw)


def test_statistics_reproducible_at_1080p():
    scene = synth.make_scene(1_000_000, 23, sh_degree=3, box=(1.9 * 1920 / 1080, 1.9, 1.0), log_scale_mean=math.log(0.01))
    runs = {}
    for dev in [f"cuda:{i}" for i in range(min(torch.cuda.device_count(), 2))]:
        sc = scene.to(dev)
        ct = {k: v.to(dev) for k, v in _dense_views(8).items()}
        outs = [_variance(sc, ct, deterministic=True) for _ in range(5)]
        side = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(side):
            outs.append(_variance(sc, ct, deterministic=True))
        side.synchronize()
        for o in outs[1:]:
            for a, b in zip(outs[0], o):
                assert O.same(a, b)
        runs[dev] = [t.cpu() for t in outs[0]]
        # against the default path: the same values to the float atomics' rounding
        ref = _variance(sc, ct, deterministic=False)
        for a, b in zip(outs[0], ref):
            a, b = a.cpu().numpy(), b.cpu().numpy()
            assert np.array_equal(np.isnan(a), np.isnan(b))
            m = ~np.isnan(a)
            assert np.abs(a[m].astype(np.float64) - b[m]).max() <= 2e-5 * np.abs(b[m]).max()
    vals = list(runs.values())
    for other in vals[1:]:
        for a, b in zip(vals[0], other):
            assert O.same(a, b)


def test_statistics_edges():
    c, scene, cams, nb = cases.build_tools_inputs("t1")
    cam = cams[0]
    # P = 0 through the C ABI
    empty = synth.Scene(*[t[:0] for t in (scene.means3D, scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees)])
    R, radii, touched, tsum, _ = stats_forward(empty, cam, True)
    assert R == 0 and radii.numel() == 0 and touched.numel() == 0
    # R = 0: everything far outside the view (culled by the frustum test)
    for shift in (torch.tensor([1e4, 0.0, 0.0]), torch.tensor([0.0, -1e4, 0.0])):
        moved = synth.Scene(scene.means3D + shift, scene.opacity, scene.scales, scene.rotations, scene.sh, scene.degrees)
        R, radii, touched, tsum, _ = stats_forward(moved, cam, True)
        assert R == 0 and int(touched.abs().sum()) == 0 and float(tsum.abs().sum()) == 0.0
    # the Python entry point with no camera and with P = 0
    sc = scene.to(DEV)
    ct = {k: v.to(DEV) for k, v in cases.tools_camera_tensors(cams).items()}
    d, v, m = _C.calculate_colours_variance(ct["positions"][:0], sc.means3D, sc.opacity, sc.scales, sc.rotations, ct["views"][:0],
                                            ct["projs"][:0], ct["tanx"][:0], ct["tany"][:0], ct["H"][:0], ct["W"][:0], sc.sh, sc.degrees, 3,
                                            deterministic=True)
    assert d.shape == (scene.P, 3) and bool(torch.isnan(d).all())


# ---- 2. k-means ------------------------------------------------------------------------------------------------------------------
def _km(values, centres, tol, it, det=True):
    ids, c = _C.kmeans_cuda(torch.as_tensor(values).reshape(-1, 1).to(DEV), torch.as_tensor(centres).to(DEV), tol, it, deterministic=det)
    return ids.cpu().numpy().reshape(-1), c.cpu().numpy()


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _kmeans_case(name, n, K, rng):
    if name == "normal":
        v = rng.normal(size=n).astype(np.float32)
    elif name == "uniform":
        v = rng.uniform(-1, 1, size=n).astype(np.float32)
    elif name == "zeros70":
        v = (0.05 * rng.normal(size=n)).astype(np.float32)
        v[rng.random(n) < 0.7] = 0.0
    elif name == "nonfinite":
        v = rng.normal(size=n).astype(np.float32)
        v[rng.random(n) < 0.01] = np.nan
        v[rng.random(n) < 0.005] = np.inf
        v[rng.random(n) < 0.005] = -np.inf
    else:
        raise ValueError(name)
    centres = v[rng.integers(0, n, K)].copy()
    centres[~np.isfinite(centres)] = 0.5
    return v, centres


@pytest.mark.parametrize("name,n,K,tol", [("normal", 50_000, 64, 1e-4), ("zeros70", 60_000, 32, 1e-4), ("nonfinite", 40_000, 16, 1e-3),
                                          ("uniform", 20_000, 1, 1e-4), ("normal", 1_000, 256, 1e-4), ("uniform", 9, 4, 1e-4)])
def test_kmeans_matches_the_restatement(name, n, K, tol):
    rng = np.random.default_rng(n + K)
    v, c0 = _kmeans_case(name, n, K, rng)
    ids0, cc0 = _km(v, c0, tol, 0)
    assert np.array_equal(ids0, _km(v, c0, tol, 0, det=False)[0]) and np.array_equal(ids0, KD.assign(v, c0))
    assert _bits(cc0).tolist() == _bits(c0).tolist()
    r_ids1, r_c1, r_it1 = KD.kmeans(v, c0, tol, 1)
    ids1, c1 = _km(v, c0, tol, 1)
    assert r_it1 == 1 and _bits(c1).tolist() == _bits(r_c1).tolist() and np.array_equal(ids1, r_ids1)
    r_ids, r_c, r_it = KD.kmeans(v, c0, tol, 500)
    ids, c = _km(v, c0, tol, 500)
    assert _bits(c).tolist() == _bits(r_c).tolist(), name
    assert np.array_equal(ids, r_ids) and np.array_equal(ids, KD.assign(v, c))
    # the iteration count: stopping one iteration earlier gives the restatement's centres of that iteration, which differ from the
    # final ones whenever the last iteration moved a centre
    if r_it > 1:
        _, r_prev, _ = KD.kmeans(v, c0, tol, r_it - 1)
        _, prev = _km(v, c0, tol, r_it - 1)
        assert _bits(prev).tolist() == _bits(r_prev).tolist()
        if _bits(r_prev).tolist() != _bits(r_c).tolist():
            assert _bits(prev).tolist() != _bits(c).tolist()
    print(f"{name}: n={n} K={K} {r_it} iterations")


def test_kmeans_goldens_under_the_torch_flag():
    """test_gpu_tools' k1 and k1_large checks with the flag on: kmeans_cuda's None follows it."""
    with torch_flag():
        for name in [n for n in cases.KMEANS_CASES if os.path.isfile(os.path.join(T.GOLD, n + ".npz"))]:
            T.test_kmeans_against_reference_goldens(name)
        T.test_kmeans_against_live_reference_and_edges()


@pytest.mark.parametrize("case", ["zeros70", "duplicate_centres", "equal_centres", "nonfinite", "k1", "k1024"])
def test_kmeans_reproducible_on_9m_values(case):
    n = 9_000_000
    rng = np.random.default_rng(11)
    base = {"zeros70": "zeros70", "nonfinite": "nonfinite"}.get(case, "normal")
    v, c = _kmeans_case(base, n, 1024 if case == "k1024" else 256, rng)
    if case == "duplicate_centres":
        c[1::2] = c[0::2]
    elif case == "equal_centres":
        c[:] = 0.25
    elif case == "k1":
        c = c[:1]
    vd, cd = torch.from_numpy(v).view(-1, 1).to(DEV), torch.from_numpy(c).to(DEV)
    outs = [_C.kmeans_cuda(vd, cd, 1e-4, 500, deterministic=True) for _ in range(4)]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.empty(12345, device=DEV)                                        # another workspace address
        outs.append(_C.kmeans_cuda(vd, cd, 1e-4, 500, deterministic=True))
    side.synchronize()
    for ids, cc in outs[1:]:
        assert torch.equal(ids, outs[0][0]) and O.same(cc, outs[0][1])
    ids, cc = outs[0]
    assert torch.equal(ids, _C.kmeans_cuda(vd, cc, 1e-4, 0, deterministic=False)[0])     # the assignment for the returned centres


# ---- 3. end to end ---------------------------------------------------------------------------------------------------------------
def _cam_tensors(cams):
    """gaussian_model.py:729-735: the stacked camera tensors (tan of the half field of view taken on the device)."""
    fx = torch.tensor([c.FoVx for c in cams], device=DEV, dtype=torch.float32)
    fy = torch.tensor([c.FoVy for c in cams], device=DEV, dtype=torch.float32)
    return dict(positions=torch.stack([c.camera_center for c in cams]), views=torch.stack([c.world_view_transform for c in cams]),
                projs=torch.stack([c.full_proj_transform for c in cams]), tanx=torch.tan(fx * 0.5), tany=torch.tan(fy * 0.5),
                H=torch.tensor([c.image_height for c in cams], device=DEV, dtype=torch.int32),
                W=torch.tensor([c.image_width for c in cams], device=DEV, dtype=torch.int32))


def _cull_sh_bands(m, cams, threshold, std_threshold):
    """gaussian_model.py:728-760 cull_sh_bands with _low_variance_colour_culling / _low_distance_colour_culling (:696-726)."""
    ct = _cam_tensors(cams)

    def run():
        return _C.calculate_colours_variance(ct["positions"], m.get_xyz, m._opacity, m.get_scaling, m.get_rotation, ct["views"], ct["projs"],
                                             ct["tanx"], ct["tany"], ct["H"], ct["W"], m.get_features, m._degrees, m.active_sh_degree)

    with torch.no_grad():
        _, weighted_variance, weighted_mean = run()
        std = weighted_variance.sqrt()
        std[std.isnan()] = 0
        std = std.mean(dim=2).squeeze()
        std_mask = std < std_threshold
        m._features_dc[std_mask] = (weighted_mean[std_mask] - 0.5) / 0.28209479177387814
        m._degrees[std_mask] = 0
        m._features_rest[std_mask] = 0
        colour_distances, _, _ = run()
        colour_distances[colour_distances.isnan()] = 0
        for sh_degree in range(m.active_sh_degree - 1, 0, -1):
            coeffs_num = (sh_degree + 1) ** 2 - 1
            mask = colour_distances[:, sh_degree] < threshold
            m._degrees[mask] = torch.min(torch.tensor([sh_degree], device=DEV, dtype=int), m._degrees[mask]).int()
            m._features_rest[mask, coeffs_num:] = 0


def _mercy(m, cams, num_neighbours=30, lambda_mercy=2, mercy_minimum=2):
    """scene/__init__.py:142-174 calculate_redundancy_metric and gaussian_model.py:524-551 mercy_points ('redundancy_opacity')."""
    from simple_knn._C import distIndex2
    fp = torch.stack([c.full_proj_transform for c in cams])
    inv = torch.stack([c.full_proj_transform.double().cpu().inverse().float() for c in cams]).to(DEV)
    H = torch.tensor([c.image_height for c in cams], device=DEV, dtype=torch.int32)
    W = torch.tensor([c.image_width for c in cams], device=DEV, dtype=torch.int32)
    with torch.no_grad():
        cube = _C.find_minimum_projected_pixel_size(fp, inv, m._xyz, H, W)
        half = cube * torch.sqrt(torch.tensor([3], device=DEV)) / 2
        _, idx = distIndex2(m.get_xyz, num_neighbours)
        idx = idx.view(-1, num_neighbours)
        red, inter = _C.sphere_ellipsoid_intersection(m._xyz, m.get_scaling, m.get_rotation, idx, half, num_neighbours)
        red += 1
        P = m._xyz.shape[0]
        idx = torch.cat((torch.arange(P, device=DEV, dtype=torch.int).view(-1, 1), idx), dim=1)
        inter = torch.cat((torch.ones_like(m._opacity, dtype=bool), inter), dim=1)
        acc = _C.allocate_minimum_redundancy_value(red, idx, inter, num_neighbours + 1)[0].unsqueeze(1)
        mean = acc.squeeze().float().mean(dim=0, keepdim=True)
        std = acc.squeeze().float().var(dim=0, keepdim=True).sqrt()
        threshold = max((mean + lambda_mercy * std).item(), mercy_minimum)
        mask = (acc > threshold).squeeze()
        opacity = torch.sigmoid(m._opacity)
        mask[mask.clone()] = opacity[mask].squeeze() < opacity[mask].median()
    densify.prune_points(m, mask)
    return int(mask.sum())


def _codebook(values, inverse=lambda x: x, num_clusters=256, tol=0.0001):
    """gaussian_model.py:36-45 generate_codebook -> (u8 ids in the shape of values, centres after the inverse activation)."""
    shape = values.shape
    values = values.flatten().view(-1, 1)
    centers = values[torch.randint(values.shape[0], (num_clusters, 1), device=DEV).squeeze()].view(-1, 1)
    ids, centers = _C.kmeans_cuda(values, centers.squeeze(), tol, 500)
    return ids.byte().squeeze().view(shape), inverse(centers.view(-1, 1))


def _pipeline(out_dir, tag):
    from test_gpu_deterministic import _train
    m, _ = _train(lambda it: it % 2 == 0)
    cams = [O.yaw_cam(256, 192, yaw) for yaw in (-10.0, 0.0, 10.0)]
    deg_before = m._degrees.clone()
    # thresholds from the statistics themselves, so that a good share of the Gaussians loses bands
    with torch.no_grad():
        ct = _cam_tensors(cams)
        d, v, _ = _C.calculate_colours_variance(ct["positions"], m.get_xyz, m._opacity, m.get_scaling, m.get_rotation, ct["views"],
                                                ct["projs"], ct["tanx"], ct["tany"], ct["H"], ct["W"], m.get_features, m._degrees, 3)
        d = torch.nan_to_num(d)
        threshold = float(d[:, 1].sort().values[int(0.3 * d.shape[0])])
        std = torch.nan_to_num(v.sqrt()).mean(dim=2).squeeze()
        std_threshold = float(std.sort().values[int(0.02 * std.shape[0])])
    _cull_sh_bands(m, cams, threshold, std_threshold)
    lost = float((m._degrees < deg_before).float().mean())
    degrees = m._degrees.clone()
    n_mercied = _mercy(m, cams)
    P = m._xyz.shape[0]
    with torch.no_grad():
        cb = [_codebook(m._features_dc.detach()[:, 0], tol=0.001)]
        cb += [_codebook(m._features_rest.detach()[:, k]) for k in range(15)]
        cb.append(_codebook(torch.sigmoid(m._opacity.detach()), lambda x: torch.log(x / (1 - x))))
        cb.append(_codebook(torch.exp(m._scaling.detach()), torch.log))
        rot = torch.nn.functional.normalize(m._rotation.detach())
        cb.append(_codebook(rot[:, 0:1]))
        cb.append(_codebook(rot[:, 1:]))
    q = synth.QuantScene(m._xyz.detach(), m._degrees.view(-1, 1).int(), cb[0][0].view(P, 3),
                         torch.stack([cb[1 + k][0].view(P, 3) for k in range(15)], dim=1), cb[16][0].view(-1), cb[17][0].view(P, 3),
                         torch.cat((cb[18][0].view(P, 1), cb[19][0].view(P, 3)), dim=1),
                         torch.stack([c.view(-1) for _, c in cb]))
    paths = []
    for half in (False, True):
        p = os.path.join(out_dir, f"{tag}_quantised{'_half' if half else ''}.ply")
        ply.save_reduced_ply(p, q, half_float=half)
        paths.append(p)
    return dict(degrees=degrees.cpu(), lost=lost, mercied=n_mercied, centers=q.centers.cpu(), paths=paths)


def test_reduced_3dgs_run_is_reproducible(tmp_path):
    with torch_flag():
        torch.manual_seed(0)
        a = _pipeline(str(tmp_path), "a")
        torch.manual_seed(0)
        b = _pipeline(str(tmp_path), "b")
    print(f"bands lost by {100 * a['lost']:.1f} % of the Gaussians, {a['mercied']} mercied")
    assert a["lost"] >= 0.10
    assert torch.equal(a["degrees"], b["degrees"])
    assert O.same(a["centers"], b["centers"])
    for pa, pb in zip(a["paths"], b["paths"]):
        with open(pa, "rb") as fa, open(pb, "rb") as fb:
            assert fa.read() == fb.read(), os.path.basename(pa)
