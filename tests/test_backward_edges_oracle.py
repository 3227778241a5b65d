"""CPU: the scenes of tests/backward_edges.py reach the render backward's boundaries they are built for, and the per-element
comparison of test_gpu_backward_edges.py catches near-misses made with the fp64 oracle itself that the global 2e-4-of-scale bar
of test_gpu_parity.test_against_oracle_midsize lets through.  Only the oracle runs here: no GPU."""
import time

import numpy as np
import pytest

import backward_edges as BE

_cache = {}


def _run(name):
    if name not in _cache:
        case = BE.build(name)
        t = time.perf_counter()
        o, o64, o32 = BE.oracle(case)
        excl = BE.excluded(case, o)
        print("\n[%s] oracle %.2f s; %d visible, %d excluded, %d borderline pixels" % (
            name, time.perf_counter() - t, int((o["radii"] > 0).sum()), int(excl.sum()), int(o["borderline"].sum())))
        _cache[name] = case, o, o64, o32, excl
    return _cache[name]


def _global_ok(o64, got):
    return all(np.abs(np.asarray(got[n], np.float64).reshape(-1) - np.asarray(o64[n], np.float64).reshape(-1)).max()
               <= BE.GLOBAL * np.abs(o64[n]).max() for n in BE.ARRAYS if o64[n].size)


@pytest.mark.parametrize("name", BE.CASES)
def test_scene_reaches_its_boundary(name):
    case, o, o64, o32, excl = _run(name)
    BE.assert_reaches(case, o, excl)
    # the oracle's fp32 backward passes its own net (K >= 1): the bar is not tighter than the reference's arithmetic
    ratios, failures = BE.compare(name, o, o64, o32, o32, ~excl, glob=(excl, BE.EXCLUDED_BAR), verbose=False)
    assert not failures, BE.describe(failures, o, o64, o32, case.W, case.H)


def test_odd_sizes_cover_partial_warps_and_tiles():
    """Warps (8x4 pixels) with lanes 4..7 or rows 2..3 outside the image, and a last tile column 1 pixel wide."""
    Ws, Hs = [w for w, h in BE.ODD_SIZES], [h for w, h in BE.ODD_SIZES]
    assert any(0 < w % 8 <= 4 for w in Ws) and any(0 < h % 4 <= 2 for h in Hs)
    assert any(w % 8 > 4 for w in Ws) and any(h % 4 == 3 for h in Hs)
    assert any(w % 16 == 1 for w in Ws) and (1, 1) in BE.ODD_SIZES
    for w, h in BE.ODD_SIZES:
        case, o, o64, o32, excl = _run("odd_%dx%d" % (w, h))
        # Gaussians listed in the last tile column / row receive gradient
        gx, gy = (w + 15) // 16, (h + 15) // 16
        t = np.arange(gx * gy)
        edge = (t % gx == gx - 1) | (t // gx == gy - 1)
        ids = np.concatenate([o["point_list"][o["ranges"][i, 0]:o["ranges"][i, 1]] for i in t[edge]]).astype(np.int64)
        assert np.abs(o64["dL_dopacity"][ids]).max() > 0


def test_per_element_check_rejects_what_the_global_bar_accepts():
    accepted_globally = []
    # 1. one tile's n_contrib lowered by one on a single pixel (staircase, the 17-entry tile: a stash flush + 1)
    case, o, o64, o32, excl = _run("staircase")
    t = BE.STAIRCASE.index(17)
    y0, x0 = 16 * (t // 6), 16 * (t % 6)
    nc = o["n_contrib"][y0:y0 + 16, x0:x0 + 16]
    ok = (nc > 0) & ~o["borderline"][y0:y0 + 16, x0:x0 + 16]
    y, x = np.unravel_index(np.argmax(np.where(ok, nc, 0)), nc.shape)
    bad = dict(o)
    bad["n_contrib"] = o["n_contrib"].copy()
    bad["n_contrib"][y0 + y, x0 + x] -= 1
    _, m64, _ = BE.oracle(case, fwd=bad)
    _, failures = BE.compare("n_contrib - 1", o, o64, o32, m64, ~excl)
    assert failures, "a pair dropped at one pixel must be caught"
    accepted_globally.append(_global_ok(o64, m64))
    # 2. dL zeroed on the inside pixels of a partial warp at the right edge (17x15: the last tile column is 1 pixel wide)
    case, o, o64, o32, excl = _run("odd_17x15")
    dL = case.dL.clone()
    dL[:, 4:8, 16] = 0.0
    _, m64, _ = BE.oracle(case, dL=dL)
    _, failures = BE.compare("partial warp dL = 0", o, o64, o32, m64, ~excl)
    assert failures, "the contribution of a partial warp's inside lanes must be caught"
    accepted_globally.append(_global_ok(o64, m64))
    # 3. one Gaussian's dL_dmeans2D.x scaled by 1.001 (a mid-sized one whose x component is its largest and where the
    #    reference's own error is far smaller)
    case, o, o64, o32, excl = _run("odd_20x36")
    a = np.abs(o64["dL_dmeans2D"][:, 0])
    e32 = np.abs(o32["dL_dmeans2D"] - o64["dL_dmeans2D"]).max(axis=1)
    cand = np.nonzero((o["radii"] > 0) & ~excl & (a > 0.01 * a.max()) & (a < 0.1 * a.max()) & (e32 < 1e-6 * a) &
                      (a >= np.abs(o64["dL_dmeans2D"][:, 1])))[0]
    assert cand.size
    m64 = {k: v.copy() for k, v in o64.items()}
    m64["dL_dmeans2D"][cand[0], 0] *= 1.001
    _, failures = BE.compare("dL_dmeans2D.x * 1.001", o, o64, o32, m64, ~excl)
    assert failures and failures[0][0] == "dL_dmeans2D" and failures[0][2].tolist() == [cand[0]]
    accepted_globally.append(_global_ok(o64, m64))
    print("\naccepted by the global bar:", accepted_globally)
    assert any(accepted_globally)
