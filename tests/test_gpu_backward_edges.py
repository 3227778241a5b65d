"""GPU: the CUDA backward (render_backward_kernel + the preprocess backward) against the fp64 oracle, element by element, on
scenes built to reach the kernel's boundaries (tests/backward_edges.py):
  - a staircase of list lengths 1..1000 per tile (stash flushes at 16 / 17, partial and exact 64-entry batches, the staging
    ring's first wrap and parity flip, lists many times the ring), and the same with one tile of equal depths;
  - odd and tiny images (1x1 .. 33x1): partial tiles and warps whose lanes 4..7 or rows 2..3 lie outside the image, a last
    tile column 1 pixel wide, a background != 0;
  - Gaussians of 100..600 px radius far from the warps they touch on 1920x1080 under a random signed dL (the moment shift),
    some centred beyond the frustum clamp;
  - opaque stacks that terminate pixels partway down the list, alpha clamped at 0.99, SH colours clamped at 0;
  - the dense sort-path tiles of test_gpu_parity (2 048 .. 40 000 entries), one with faint opacities so that `hi` > 8 192.
Every case feeds the oracle's own forward state to its fp64 and fp32 backwards; integers are asserted equal first.
Bar per element (backward_edges.compare): |ours - o64| <= max(8 E32, 1e-4 |o64|_row, 1e-6 max|o64|), with E32 and |o64|_row
the largest |o32 - o64| and |o64| of the Gaussian's row of that array; Gaussians an exponential ulp may move at a borderline pixel
(backward_edges.excluded) are held to 1e-3 of the array's scale and checked per element on a second backward with dL = 0 on the
borderline pixels; culled ones get exactly zero.
Observed on one H100 (pytest -s prints, per case and array, max e / max(E32, 1e-4 |o64|_row, 1e-6 max|o64|) and max e / bar):
at most 0.58 of the bar in every case but dense_faint, whose deep faint stacks reach 3.97e-4 of the row in dL_dconic, 2.47e-4 in
dL_dscales and 1.6e-4 in dL_drotations, and its smallest gradients 4e-6 of the array's scale; that case's bar is
max(8 E32, 1e-3 |o64|_row, 1e-5 max|o64|) (backward_edges.BAR_CASE).  The file takes ~12 s."""
import time

import numpy as np
import pytest
import torch

import backward_edges as BE
import ours

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", BE.CASES)
def test_backward_per_element_against_fp64_oracle(name):
    assert ours.GRAD_NAMES == BE.GRAD_NAMES
    case = BE.build(name)
    t0 = time.perf_counter()
    o, o64, o32 = BE.oracle(case)
    excl = BE.excluded(case, o)
    t1 = time.perf_counter()
    BE.assert_reaches(case, o, excl)
    args, out, fwd = ours.run_forward(case.scene, case.cam, case.bg)
    assert int(fwd["num_rendered"]) == int(o["num_rendered"])
    for k in ("radii", "keys", "point_list", "ranges"):
        assert np.array_equal(np.asarray(o[k]).reshape(-1), fwd[k].reshape(-1)), k
    nb = ~o["borderline"]
    assert np.array_equal(o["n_contrib"][nb], fwd["n_contrib"][nb]), "n_contrib"
    got = ours.run_backward(args, out, case.dL, case.lam)
    ratios, failures = BE.compare(name, o, o64, o32, got, ~excl, glob=(excl, BE.EXCLUDED_BAR),
                                  bar=BE.BAR_CASE.get(name, (BE.R_REL, BE.A_ABS)))
    assert not failures, "\n" + BE.describe(failures, o, o64, got, case.W, case.H)
    if excl.any():
        # with dL/dpixel = 0 on the borderline pixels no flipped decision reaches a gradient: every Gaussian per element
        dL = case.dL.clone()
        dL[:, torch.from_numpy(o["borderline"])] = 0.0
        _, m64, m32 = BE.oracle(case, dL=dL, fwd=o)
        mgot = ours.run_backward(args, out, dL, case.lam)
        _, failures = BE.compare(name + ", borderline dL = 0", o, m64, m32, mgot, np.ones_like(excl), bar=BE.BAR_CASE.get(name, (BE.R_REL, BE.A_ABS)))
        assert not failures, "\n" + BE.describe(failures, o, m64, mgot, case.W, case.H)
    print("[%s] oracle %.2f s, total %.2f s" % (name, t1 - t0, time.perf_counter() - t0))
    if name == "large":
        # the Gaussians of the frustum-clamp branch were checked per element, dL_dmeans3D included
        clamp = BE.clamp_branch(case, o) & ~excl
        assert clamp.sum() >= 4 and np.abs(o64["dL_dmeans3D"][clamp]).min() > 0
