"""GPU: the SH-culling statistics per Gaussian against the oracle (tests/statistics_edges.py) on the rasterizer's boundary scenes
(the 16 of tests/backward_edges.py and t1's first camera):
  - the statistics forward (render_forward_kernel<STATS = true>, and its fixed-point twin with `deterministic`): radii, point list
    and ranges equal to the oracle's first, then per Gaussian `touched_pixels` exact and `transmittance_sum` within 1e-5 o64 + 1e-6
    of the oracle's fp64 sum (+ 1/254 per borderline pixel behind a pair near alpha 1/255), the Gaussians near a borderline
    decision within the count of their borderline pixels, culled ones exactly zero (the outputs are poisoned before the call, so
    an unwritten row shows);
  - calculate_colours_variance (the statistics forward + sh_stats_update_kernel per camera) on three cameras, with appended faint,
    unseen and one-camera Gaussians, against gs_oracle.colours_variance: the NaN pattern exact, rows within 2e-5 max|row| + 1e-7
    (1e-3 of the array's scale for Gaussians near or behind a borderline decision); `deterministic` gives the same bytes twice.
Observed in two runs on one H100 80GB HBM3 at its 700 W limit (pytest -s prints the ratios per case): every count of a tight
Gaussian exact in both paths; the largest |d tsum| of a tight Gaussian 0.032 of its bar outside `large`, and in `large` 0.41 on
the default path and 0.21 in fixed point.  There the 600 px Gaussian 20013 flips at one pixel where its alpha is 1/255 within 2e-9:
its count is 1 lower and its sum within 0.3 of its bar, and the two Gaussians composited behind it there, of 215 and 351 pixels,
are 2.4e-5 and 1.3e-5 of their sums higher (statistics_edges.FLIP).  The colour statistics within 0.112 of their bar (the mean of
`large`), the rows near or behind a borderline decision within 1e-7 of the scale.  The file takes ~25 s.
Each of these one-line edits fails the file on that H100: the ballot on the alpha test instead of on the contribution (36 of 46
tests), T * (1 - alpha) summed instead of T, the sum without the contribution guard (all 46), sh_stats_update_kernel without its
isnan(coef) guard or with the pre-update mean in the variance term (14: the colour-statistics tests)."""
import math

import numpy as np
import pytest
import torch

import backward_edges as BE
import ours
import statistics_edges as SE
from diff_gaussian_rasterization import _C

pytestmark = pytest.mark.gpu
DEV = "cuda"
_cache = {}


def stats_forward(scene, cam, det, dev=DEV):
    """The statistics forward of `scene` on `cam` (zero background), fixed point with `det`; touched_pixels and transmittance_sum
    are filled with -7 and the fixed-point workspace with 0xA5 first -> (R, radii, touched, tsum, raw outputs of _C._forward)."""
    sc = scene.to(dev)
    W, H = cam.image_width, cam.image_height
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    touched = torch.full((scene.P, 1), -7, dtype=torch.int32, device=dev)
    tsum = torch.full((scene.P, 1), -7.0, device=dev)
    kw = {}
    if det:
        kw["statistics_workspace"] = torch.full((int(_C._lib.lib().gsb_statistics_workspace_bytes(scene.P)),), 0xA5, dtype=torch.uint8,
                                                device=dev)
    E = torch.empty(0)
    out = _C._forward(torch.zeros(3, device=dev), sc.means3D, E, sc.opacity, sc.scales, sc.rotations, 1.0, E,
                      cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev), tx, ty, H, W, sc.sh, sc.degrees,
                      cam.camera_center.to(dev), False, False, statistics=(touched, tsum), **kw)
    return out[0], out[2], touched, tsum, out


def _oracle(name):
    if name not in _cache:
        case = SE.build(name)
        o = SE.oracle(case.scene, case.cam, case.bg)
        _cache[name] = case, o, BE.borderline_pairs(o, case.W, case.H)
    return _cache[name]


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("name", SE.CASES)
def test_statistics_forward_per_gaussian_against_oracle(name, deterministic):
    case, o, pairs = _oracle(name)
    R, radii, touched, tsum, out = stats_forward(case.scene, case.cam, deterministic)
    st = ours.state(out, case.cam, case.scene.P)
    assert int(R) == int(o["num_rendered"])
    assert np.array_equal(radii.cpu().numpy(), o["radii"]), "radii"
    assert np.array_equal(st["point_list"].cpu().numpy().astype(np.uint32), o["point_list"]), "point_list"
    assert np.array_equal(st["ranges"].cpu().numpy().astype(np.uint32).reshape(-1), o["ranges"].reshape(-1)), "ranges"
    t, s = touched.cpu().numpy().reshape(-1), tsum.cpu().numpy().reshape(-1)
    _, failures = SE.compare("%s%s" % (name, ", deterministic" if deterministic else ""), o, pairs, t, s)
    assert not failures, "\n" + SE.describe(failures, o, t, s)


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("name", SE.VAR_CASES)
def test_colours_variance_against_oracle(name, deterministic):
    key = "variance " + name
    if key not in _cache:
        vc = SE.variance_case(name)
        _cache[key] = vc, SE.variance_oracle(vc)
    vc, (ref, _, loose) = _cache[key]
    args = [a.to(DEV) if torch.is_tensor(a) else a for a in SE.variance_args(vc)]
    got = _C.calculate_colours_variance(*args, deterministic=deterministic)
    if deterministic:
        again = _C.calculate_colours_variance(*args, deterministic=True)
        assert all(ours.same(a, b) for a, b in zip(got, again)), "the deterministic statistics give the same bytes on every run"
    got = [g.cpu().numpy() for g in got]
    _, failures = SE.compare_variance("%s%s" % (name, ", deterministic" if deterministic else ""), ref, got, loose)
    assert not failures, "\n".join("%s: %s: rows %s" % (n, what, rows[:8].tolist()) for n, what, rows in failures)
