"""GPU: the anti-aliased CUDA forward and backward (antialiasing=True, DESIGN.md §5e) against the fp64 oracle, element by element,
on the boundary scenes of tests/backward_edges.py (the 16 BE.CASES built for AA) and on the AA scenes: needle-thin splats on both
sides of the clamp of q = det0 / det1 and right at it (aa_needles), and sub-pixel splats with s << 1 (aa_subpixel).
  - forward: radii, keys, point_list, ranges and n_contrib (off borderline pixels) equal the oracle's, and o^ = sigmoid * s is
    within ULP_OPACITY ulp of it (the kernel's exponential is MUFU.EX2, the oracle's exp2f);
  - backward, default and deterministic=True: backward_edges.compare with the bars of test_gpu_backward_edges.py, and the second
    pass with dL = 0 on the borderline pixels;
  - camera gradients (AA off, the same 16 scenes): the kernel's view / proj / campos gradients against the float64 chain
    (camera_chain.py) of the fp64 oracle's screen-space gradients, 2e-4 of sum |c_i| per entry; the `large` scene's frustum-clamp
    Gaussians are in it.
On aa_needles (backward_edges.compare_aa) every array is checked per element on the 72 needles with a c / det0 < 1e2 (the 48
bisected to within 1e-3 of the clamp, 25 clamped ones: the clamp decision and the gradient through q reach dL_dcov3D, dL_dscales,
dL_dmeans3D and dL_drotations there), and all but dL_dmeans3D / dL_drotations, which are ill-conditioned in fp32, on the others;
aa_subpixel and the 16 scenes check every array.
Observed maxima are printed (pytest -s)."""
import math
import time

import numpy as np
import pytest
import torch

import backward_edges as BE
import gs_oracle
import ours
from camera_chain import chain, check

pytestmark = pytest.mark.gpu

ULP_OPACITY = 4


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.parametrize("name", BE.AA_CASES + BE.CASES)
def test_aa_forward_and_backward_per_element_against_fp64_oracle(name):
    case = BE.build(name, aa=True)
    t0 = time.perf_counter()
    o, o64, o32 = BE.oracle(case, aa=True)
    excl = BE.excluded(case, o)
    BE.assert_reaches(case, o, excl)
    args, out, fwd = ours.run_forward(case.scene, case.cam, case.bg, aa=True)
    assert int(fwd["num_rendered"]) == int(o["num_rendered"])
    for k in ("radii", "keys", "point_list", "ranges"):
        assert np.array_equal(np.asarray(o[k]).reshape(-1), fwd[k].reshape(-1)), k
    nb = ~o["borderline"]
    assert np.array_equal(o["n_contrib"][nb], fwd["n_contrib"][nb]), "n_contrib"
    vis = o["radii"] > 0
    u = _ulps(fwd["conic_opacity"][vis, 3], o["conic_opacity"][vis, 3])
    print("\n[%s, aa] o^: max %d ulp from the oracle's, %d of %d bit-identical" % (name, int(u.max()), int((u == 0).sum()), int(vis.sum())))
    assert int(u.max()) <= ULP_OPACITY
    bar = BE.BAR_CASE.get(name, (BE.R_REL, BE.A_ABS))
    dL_masked = None
    if excl.any():
        dL_masked = case.dL.clone()
        dL_masked[:, torch.from_numpy(o["borderline"])] = 0.0
        _, m64, m32 = BE.oracle(case, dL=dL_masked, fwd=o, aa=True)
    for det in (False, True):
        label = "%s, aa%s" % (name, ", deterministic" if det else "")
        got = ours.run_backward(args, out, case.dL, case.lam, aa=True, deterministic=det)
        failures = BE.compare_aa(label, case, o, o64, o32, got, ~excl, glob=(excl, BE.EXCLUDED_BAR), bar=bar)
        assert not failures, "\n" + BE.describe(failures, o, o64, got, case.W, case.H)
        if dL_masked is not None:
            mgot = ours.run_backward(args, out, dL_masked, case.lam, aa=True, deterministic=det)
            failures = BE.compare_aa(label + ", borderline dL = 0", case, o, m64, m32, mgot, np.ones_like(excl), bar=bar)
            assert not failures, "\n" + BE.describe(failures, o, m64, mgot, case.W, case.H)
    print("[%s, aa] total %.2f s" % (name, time.perf_counter() - t0))


@pytest.mark.parametrize("name", BE.CASES)
def test_camera_grads_against_the_chain_of_the_fp64_oracle(name):
    case = BE.build(name)
    kw = case.cam_kw()
    s = case.scene
    o = gs_oracle.forward(s.means3D, s.opacity, s.scales, s.rotations, s.sh, s.degrees, bg=case.bg, **kw)
    ob = gs_oracle.backward(o, case.dL, s.means3D, s.scales, s.rotations, s.sh, s.degrees, bg=case.bg, f64=True, **kw)
    args, out = ours.forward(s, case.cam, case.bg.cuda())
    assert np.array_equal(out[2].cpu().numpy(), o["radii"])
    g = ours.backward(args, out, case.dL, camera_grads=True)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    vis = out[2] > 0
    per = chain(case.cam.world_view_transform, case.cam.full_proj_transform, case.cam.camera_center, case.W, case.H, kw["tan_fovx"],
                kw["tan_fovy"], s.means3D, t(o["cov3D"]), s.sh, s.degrees, t(o["clamped"]), vis, t(ob["dL_dmeans2D"]),
                t(ob["dL_dconic"]), t(ob["dL_dcolors"]))
    check(g[8:], per, 2e-4, name + " vs fp64 oracle")
    if name == "large":
        assert int(BE.clamp_branch(case, o).sum()) >= 8, "the frustum-clamp Gaussians are in the chain"
