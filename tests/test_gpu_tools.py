"""GPU: the reduced-3dgs tools around the rasterizer (SURVEY §8(f) rows 2-3: SH-culling statistics, redundancy score)
through the drop-in `_C` entry points, against (a) the golden outputs of the reference itself (tests/golden/t1.npz),
(b) the CPU oracle and (c) the reference's golden record of a larger case (tests/golden/t1_large.npz).  The statistics forward
and the colour statistics are checked per Gaussian against the oracle in test_gpu_statistics_edges.py.

Tolerances: integers / masks exact (oracle: except pairs the oracle flags as within rounding of a threshold, because host powf
and MUFU-based powf differ in the last ulp); floats 2e-5 relative to the array's scale — the reference's own run-to-run noise
(float atomics) is recorded in the golden as noise_*."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import cases  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(HERE, "golden")


def _C():
    from diff_gaussian_rasterization import _C as c
    return c


def _close(a, b, tol, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.array_equal(np.isnan(a), np.isnan(b)), what + ": NaN pattern"
    m = ~np.isnan(a)
    scale = np.abs(b[m]).max() + 1e-30
    err = np.abs(a[m] - b[m]).max() / scale
    assert err <= tol, (what, err)


def _run_ours(c, scene, cams, nb, dev="cuda"):
    C = _C()
    ct = {k: v.to(dev) for k, v in cases.tools_camera_tensors(cams).items()}
    sc = scene.to(dev)
    P, knn = scene.P, c["knn"]
    out = {}
    d, v, m = C.calculate_colours_variance(ct["positions"], sc.means3D, sc.opacity, sc.scales, sc.rotations, ct["views"], ct["projs"],
                                           ct["tanx"], ct["tany"], ct["H"], ct["W"], sc.sh, sc.degrees, 3)
    out.update(cv_distance=d, cv_variance=v, cv_mean=m)
    px = C.find_minimum_projected_pixel_size(ct["projs"], ct["inv_projs"], sc.means3D, ct["H"], ct["W"])
    out["pixel_size"] = px
    half = px * c["radius_scale"] * torch.sqrt(torch.tensor([3.0], device=dev)) / 2
    red, mask = C.sphere_ellipsoid_intersection(sc.means3D, sc.scales, sc.rotations, nb.to(dev), half, knn)
    out.update(half_diagonal=half, redundancy=red, intersection_mask=mask)
    idx = torch.cat((torch.arange(P, device=dev, dtype=torch.int).view(-1, 1), nb.to(dev)), dim=1)
    mk = torch.cat((torch.ones((P, 1), device=dev, dtype=torch.bool), mask), dim=1)
    out["min_redundancy"] = C.allocate_minimum_redundancy_value(red + 1, idx, mk, knn + 1)[0]
    return {k: v.cpu().numpy() for k, v in out.items()}


def _check(ours, ref, exact_floats=True):
    for k in ("cv_distance", "cv_variance", "cv_mean"):
        _close(ours[k], ref[k], 2e-5, k)
    if exact_floats:
        assert np.array_equal(ours["pixel_size"], ref["pixel_size"]), "pixel_size is expected bit-identical (same operation order)"
    _close(ours["pixel_size"], ref["pixel_size"], 1e-6, "pixel_size")
    assert ours["redundancy"].dtype == np.int32 and ours["intersection_mask"].dtype == np.bool_
    assert np.array_equal(ours["intersection_mask"], ref["intersection_mask"])
    assert np.array_equal(ours["redundancy"], ref["redundancy"])
    assert np.array_equal(ours["min_redundancy"], ref["min_redundancy"])


@pytest.mark.parametrize("name", [n for n in cases.TOOLS_CASES if os.path.isfile(os.path.join(GOLD, n + ".npz"))])
def test_tools_against_reference_goldens(name):
    c, scene, cams, nb = cases.build_tools_inputs(name)
    ref = dict(np.load(os.path.join(GOLD, name + ".npz")))
    _check(_run_ours(c, scene, cams, nb), ref)


def test_tools_against_live_reference():
    """A larger case (60 k Gaussians, four views up to 640x512) against the reference's golden record (t1_large.npz: digests of the
    exact outputs, a sample of the statistics, see golden/refsummary.py)."""
    import make_golden_fullsize as MG
    import refsummary as S
    ref = S.load("t1_large")
    ours = _run_ours(*MG.tools_large_inputs())
    for k in ("cv_distance", "cv_variance", "cv_mean"):
        assert S.digest(np.isnan(ours[k])) == ref[k + "_nan"], k + ": NaN pattern"
        x, y, scale = S.sampled(ref, k, ours[k])
        m = ~np.isnan(y)
        assert np.abs(x[m].astype(np.float64) - y[m]).max() / (scale + 1e-30) <= 2e-5, k
    assert S.digest(ours["pixel_size"]) == ref["pixel_size"], "pixel_size is expected bit-identical (same operation order)"
    assert ours["redundancy"].dtype == np.int32 and ours["intersection_mask"].dtype == np.bool_
    for k in ("intersection_mask", "redundancy", "min_redundancy"):
        assert S.digest(ours[k]) == ref[k], k


def test_tools_edge_cases():
    C = _C()
    dev = "cuda"
    # no camera sees the point -> 10000; knn = 0; P = 0
    xyz = torch.tensor([[0.0, 0.0, -50.0], [0.0, 0.0, 0.0]], device=dev)
    cam = cases.synth.make_camera(64, 48).to(dev)
    px = C.find_minimum_projected_pixel_size(cam.full_proj_transform[None], cam.full_proj_transform.inverse()[None], xyz,
                                             torch.tensor([48], dtype=torch.int32, device=dev), torch.tensor([64], dtype=torch.int32, device=dev))
    assert px.shape == (2, 1) and float(px[0]) == 10000.0 and 0 < float(px[1]) < 1
    red, mask = C.sphere_ellipsoid_intersection(xyz, torch.ones(2, 3, device=dev), torch.tensor([[1.0, 0, 0, 0]] * 2, device=dev),
                                                torch.empty((2, 0), dtype=torch.int32, device=dev), torch.ones(2, 1, device=dev), 0)
    assert red.shape == (2, 1) and int(red.abs().sum()) == 0 and mask.shape == (2, 0)
    e = torch.empty((0, 3), device=dev)
    assert C.find_minimum_projected_pixel_size(cam.full_proj_transform[None], cam.full_proj_transform[None], e,
                                               torch.tensor([48], dtype=torch.int32), torch.tensor([64], dtype=torch.int32)).shape == (0, 1)
    out = C.allocate_minimum_redundancy_value(torch.tensor([[3], [1]], dtype=torch.int32, device=dev),
                                              torch.tensor([[0, 1], [1, 0]], dtype=torch.int32, device=dev),
                                              torch.tensor([[True, True], [True, False]], device=dev), 2)[0]
    assert out.cpu().tolist() == [[2], [1]]          # initial value P = 2 caps index 0; index 1 takes min(3, 1)
    with pytest.raises(RuntimeError):
        C.calculate_colours_variance(torch.zeros(1, 3, device=dev), torch.zeros(4, 3, device=dev), torch.zeros(4, 1, device=dev),
                                     torch.ones(4, 3, device=dev), torch.ones(4, 4, device=dev), torch.eye(4, device=dev)[None],
                                     torch.eye(4, device=dev)[None], torch.ones(1), torch.ones(1), torch.tensor([8]), torch.tensor([8]),
                                     torch.zeros(4, 16, 3, device=dev), torch.zeros(4, 1, dtype=torch.int32, device=dev), 2)


# ---- codebook k-means (reduced_3dgs.cu:289-338) -----------------------------------------------------------------------
def _kmeans_cost(v, ids, cc):
    return float(np.abs(v.reshape(-1).astype(np.float64) - cc.astype(np.float64)[ids.reshape(-1)]).mean())


def _kmeans_checks(c, v, centers, ref):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
    import gs_oracle as O
    C = _C()
    vd, cd = v.cuda(), centers.cuda()
    # (1) zero iterations = the assignment rule alone: exact, centres unchanged
    ids0, c0 = C.kmeans_cuda(vd, cd, c["tol"], 0)
    assert ids0.dtype == torch.int32 and tuple(ids0.shape) == (v.shape[0], 1) and tuple(c0.shape) == (c["k"],)
    assert np.array_equal(c0.cpu().numpy(), centers.numpy())
    assert np.array_equal(ids0.cpu().numpy(), ref["ids_iter0"])
    # (2) one iteration: same partition -> same sizes, centres equal up to float summation order
    ids1, c1 = C.kmeans_cuda(vd, cd, 0.0, 1)
    # (both sides add ~6 000 floats per centre with float atomics in an arbitrary order: a few 1e-6 relative is their own run-to-run
    # noise — a 2e-6 bound here failed about one run in five against the LIVE reference)
    assert np.abs(c1.cpu().numpy() - ref["centers_iter1"]).max() <= 2e-5 * (np.abs(ref["centers_iter1"]).max() + 1e-30) + 1e-6
    mism = (ids1.cpu().numpy() != ref["ids_iter1"]).mean()
    assert mism <= 1e-4, mism                                    # a value within an ulp of a boundary may flip with the summation order
    # (3) to convergence: the returned ids are EXACTLY the assignment for the returned centres, and the quantisation cost
    #     matches the reference's (trajectories differ by summation-order noise, so centres are compared loosely)
    idsf, cf = C.kmeans_cuda(vd, cd, c["tol"], c["max_iterations"])
    idsf, cf = idsf.cpu().numpy(), cf.cpu().numpy()
    assert np.array_equal(idsf.reshape(-1), O.kmeans_update_ids(v.numpy(), cf))
    cost = _kmeans_cost(v.numpy(), idsf, cf)
    assert abs(cost - float(ref["cost_final"])) <= max(2e-3 * float(ref["cost_final"]), 4 * float(ref["noise_cost_final"])), (cost, float(ref["cost_final"]))
    assert np.abs(np.sort(cf) - np.sort(ref["centers_final"])).max() <= max(2e-2, 10 * float(ref["noise_centers_final"]))


@pytest.mark.parametrize("name", [n for n in cases.KMEANS_CASES if os.path.isfile(os.path.join(GOLD, n + ".npz"))])
def test_kmeans_against_reference_goldens(name):
    c, v, centers = cases.build_kmeans_inputs(name)
    _kmeans_checks(c, v, centers, dict(np.load(os.path.join(GOLD, name + ".npz"))))


def test_kmeans_against_live_reference_and_edges():
    C = _C()
    import make_golden_fullsize as MG
    import refsummary as S
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
    import gs_oracle as O
    # 1.5 M values against the reference's golden record (k1_large.npz): the id arrays are stored as digests; the assignment rule
    # is exact (argmin, checked against the oracle below), so they are rebuilt from the stored centres and checked against those
    ref = S.load("k1_large")
    c, v, centers = cases.build_kmeans_inputs("k1", n=MG.KMEANS_LARGE_N)
    for it in ("0", "1"):
        ids = O.kmeans_update_ids(v.numpy(), ref["centers_iter" + it]).reshape(-1, 1)
        assert S.digest(ids) == ref["ids_iter" + it], "ids_iter" + it
        ref["ids_iter" + it] = ids
    _kmeans_checks(c, v, centers, ref)
    # n % 256 != 0: the reference's trailing partial block is undefined (cases.KMEANS_CASES); everything before it must agree
    c2, v2, centers2 = cases.build_kmeans_inputs("k1", n=MG.KMEANS_PARTIAL_N)
    ids_our, _ = C.kmeans_cuda(v2.cuda(), centers2.cuda(), 0.0, 0)
    full = MG.KMEANS_PARTIAL_N - MG.KMEANS_PARTIAL_N % 256
    assert S.digest(ids_our[:full]) == ref["partial_ids_full_blocks"]
    assert np.array_equal(ids_our.cpu().numpy().reshape(-1), O.kmeans_update_ids(v2.numpy(), centers2.numpy()))
    # all centres equal -> the first iteration puts everything into index 0; the empty clusters become 0 (NaN -> 0, reduced_3dgs.cu:323)
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
    import gs_oracle as O2
    v = torch.linspace(-1, 1, 1000, device="cuda").view(-1, 1)
    ids, cc = C.kmeans_cuda(v, torch.full((256,), 0.25, device="cuda"), 0.0, 1)
    assert abs(float(cc[0]) - float(v.mean())) < 1e-6 and float(cc[1:].abs().sum()) == 0.0
    assert np.array_equal(ids.cpu().numpy().reshape(-1), O2.kmeans_update_ids(v.cpu().numpy(), cc.cpu().numpy()))
    # ties: a value exactly between two centres takes the lower INDEX (strict `<` in kmeans.cu:96), wherever that centre lies
    ids, _ = C.kmeans_cuda(torch.tensor([[0.0], [0.0]], device="cuda"), torch.tensor([1.0, -1.0, 5.0], device="cuda"), 0.0, 0)
    assert ids.view(-1).tolist() == [0, 0]
    ids, _ = C.kmeans_cuda(torch.tensor([[0.0]], device="cuda"), torch.tensor([5.0, 1.0, -1.0], device="cuda"), 0.0, 0)
    assert ids.view(-1).tolist() == [1]
    # empty input
    ids, cc = C.kmeans_cuda(torch.empty((0, 1), device="cuda"), torch.arange(4, dtype=torch.float32, device="cuda"), 0.1, 5)
    assert tuple(ids.shape) == (0, 1) and cc.tolist() == [0.0, 1.0, 2.0, 3.0]


# ---- loss side of the step: L1 + D-SSIM (utils/loss_utils.py, train.py:110-115) --------------------------------------------
def test_loss_against_reference_golden_and_oracle():
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
    import gs_oracle as O
    import make_golden_loss as M
    from utils import loss_utils as LU
    ref = dict(np.load(os.path.join(GOLD, "loss1.npz")))
    img, gt = M.inputs()
    lam = float(ref["lambda_dssim"])
    x = img.cuda().requires_grad_(True)
    loss = LU.l1_ssim_loss(x, gt.cuda(), lam)
    loss.backward()
    assert abs(float(loss.detach()) - float(ref["loss"])) < 2e-6
    assert np.abs(x.grad.cpu().numpy() - ref["grad"]).max() <= 2e-4 * np.abs(ref["grad"]).max()
    # the reference's call pattern: two functions, combined by autograd (train.py:110-115)
    x2 = img.cuda().requires_grad_(True)
    Ll1, s = LU.l1_loss(x2, gt.cuda()), LU.ssim(x2, gt.cuda())
    assert abs(float(Ll1.detach()) - float(ref["l1"])) < 1e-7 and abs(float(s.detach()) - float(ref["ssim"])) < 2e-5
    ((1.0 - lam) * Ll1 + lam * (1.0 - s)).backward()
    assert np.abs(x2.grad.cpu().numpy() - ref["grad"]).max() <= 2e-4 * np.abs(ref["grad"]).max()
    x3 = img.cuda().requires_grad_(True)
    LU.ssim(x3, gt.cuda()).backward()
    assert np.abs(x3.grad.cpu().numpy() - ref["grad_ssim_only"]).max() <= 2e-4 * np.abs(ref["grad_ssim_only"]).max()
    # full size, non-trivial upstream gradient, against the float64 oracle
    g = torch.Generator().manual_seed(3)
    a, b = torch.rand(3, 1080, 1920, generator=g), torch.rand(3, 1080, 1920, generator=g)
    xa = a.cuda().requires_grad_(True)
    (2.5 * LU.l1_ssim_loss(xa, b.cuda(), 0.2)).backward()
    l1, ss, lo, gr = O.l1_ssim(a, b, 0.2)
    assert np.abs(xa.grad.cpu().numpy() - 2.5 * gr).max() <= 1e-4 * np.abs(2.5 * gr).max()
    with pytest.raises(NotImplementedError):
        LU.ssim(x, gt.cuda(), window_size=7)
