"""CPU: the statistics cases of tests/statistics_edges.py reach what they are built for, and the per-Gaussian comparison of
test_gpu_statistics_edges.py rejects near-misses made with the oracle itself, some of which the older whole-array rule (counts off
on up to 4 Gaussians per borderline pixel, sums within 1e-3 of the scale once a pixel is borderline) accepts.  Only the oracle
runs here: no GPU."""
import numpy as np
import pytest

import backward_edges as BE
import gs_oracle
import statistics_edges as SE

_cache = {}


def _run(name):
    if name not in _cache:
        case = SE.build(name)
        o = SE.oracle(case.scene, case.cam, case.bg)
        pairs = BE.borderline_pairs(o, case.W, case.H)
        vis = o["radii"] > 0
        print("\n[%s] %d visible, %d near a borderline decision, %d behind one, %d borderline pixels" % (
            name, int(vis.sum()), int(pairs[0].sum()), int((pairs[2] > 0).sum()), int(o["borderline"].sum())))
        _cache[name] = case, o, pairs
    return _cache[name]


def _variance(name):
    key = "variance " + name
    if key not in _cache:
        vc = SE.variance_case(name)
        _cache[key] = vc, SE.variance_oracle(vc)
    return _cache[key]


def _tiles_with_outside_lanes(W, H):
    """Tiles whose 8x4 warps have lanes outside the W x H image."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tx, ty = np.meshgrid(np.arange(gx), np.arange(gy))
    return ((16 * (tx + 1) > W) & (W % 8 != 0)) | ((16 * (ty + 1) > H) & (H % 4 != 0))


@pytest.mark.parametrize("name", SE.CASES)
def test_case_reaches_its_boundary(name):
    case, o, pairs = _run(name)
    BE.assert_reaches(case, o, BE.excluded(case, o))
    vis = o["radii"] > 0
    loose = pairs[0] | (pairs[2] > 0)
    assert loose[vis].mean() <= SE.NEAR_MAX, (name, loose[vis].mean())
    assert o["touched_pixels"].sum() > 0 and np.all(o["transmittance_sum"][o["touched_pixels"] == 0] == 0)
    # the oracle's own sum rounded to fp32 (what the kernel returns) passes: the bar is not tighter than the output's precision
    _, failures = SE.compare(name, o, pairs, o["touched_pixels"], o["transmittance_sum"].astype(np.float32), verbose=False)
    assert not failures, SE.describe(failures, o, o["touched_pixels"], o["transmittance_sum"])


def test_cases_cover_the_statistics_forward_boundaries():
    counts = {n: (_run(n)[1]["ranges"][:, 1] - _run(n)[1]["ranges"][:, 0]).astype(np.int64) for n in SE.CASES}
    # lists across the 32-entry chunk and the 256-entry batch, and many batches long
    assert any(((c % 32 != 0) & (c > 32)).any() for c in counts.values())
    assert any((c > 256).any() for c in counts.values()) and any((c > 2048).any() for c in counts.values())
    # partial warps: lanes outside the image in tiles whose listed Gaussians do touch pixels
    for w, h in BE.ODD_SIZES:
        case, o, _ = _run("odd_%dx%d" % (w, h))
        part = _tiles_with_outside_lanes(w, h).reshape(-1)
        if not part.any():
            continue
        ids = np.concatenate([o["point_list"][o["ranges"][t, 0]:o["ranges"][t, 1]] for t in np.nonzero(part)[0]]).astype(np.int64)
        assert (o["touched_pixels"][ids] > 0).any(), (w, h)
    assert sum(_tiles_with_outside_lanes(w, h).any() for w, h in BE.ODD_SIZES) >= 5


@pytest.mark.parametrize("name", SE.VAR_CASES)
def test_variance_case_reaches_its_groups(name):
    vc, ((d, v, m), per, loose) = _variance(name)
    gr = vc.groups
    assert vc.scene.sh.shape[1] == 16 and set(vc.scene.degrees.view(-1).tolist()) == {0, 1, 2, 3}
    assert len(vc.cams) == 3 and all(gr[k].size == SE.GROUP_SIZE for k in gr)
    radii = np.stack([p["radii"] for p in per])
    touched = np.stack([p["touched_pixels"] for p in per])
    # (a) present in every camera, touched nowhere: wSum = 0, so NaN distance and variance and a zero mean
    assert (radii[:, gr["faint"]] > 0).all() and (touched[:, gr["faint"]] == 0).all()
    assert np.isnan(d[gr["faint"]]).all() and np.isnan(v[gr["faint"]]).all() and (m[gr["faint"]] == 0).all()
    # (b) never present
    assert (radii[:, gr["outside"]] == 0).all() and np.isnan(d[gr["outside"]]).all() and (m[gr["outside"]] == 0).all()
    # (c) present in exactly one camera, most of them touched there
    one = radii[:, gr["one"]] > 0
    assert (one.sum(0) == 1).all()
    assert (touched[:, gr["one"]][one] > 0).sum() >= SE.GROUP_SIZE // 3
    # and every other row is finite: the scene's visible Gaussians carry statistics
    fin = ~np.isnan(d).any(1)
    assert fin.sum() >= 0.2 * vc.scene.P and not np.isnan(m).any()
    print("\n[%s] %d of %d Gaussians near or behind a borderline decision in some camera" % (name, int(loose.sum()), loose.size))
    assert loose.mean() <= SE.NEAR_MAX
    if name == "t1":
        WH = [(c.image_width, c.image_height) for c in vc.cams]
        assert any(w > h for w, h in WH) and any(w == h for w, h in WH) and any(w < h for w, h in WH)


def test_per_gaussian_check_rejects_what_the_old_rule_accepts():
    accepted = {}

    def caught(label, o, pairs, touched, tsum):
        _, failures = SE.compare(label, o, pairs, touched, tsum, verbose=False)
        assert failures, label + " must be caught"
        accepted[label] = SE.old_rule_ok(o, touched, tsum)

    case, o, pairs = _run("large")
    near, count, _ = pairs
    vis, t_o, s_o = o["radii"] > 0, o["touched_pixels"], o["transmittance_sum"]
    # 1. one count off by one on a Gaussian away from every borderline pixel
    g = int(np.nonzero(vis & ~near & (count == 0) & (t_o > 0))[0][0])
    t = t_o.copy()
    t[g] += 1
    caught("touched + 1", o, pairs, t, s_o)
    # 2. one sum 1e-4 too large, on a Gaussian of thousands of pixels
    g = int(np.nonzero(vis & ~near & (count == 0) & (t_o >= 2000))[0][0])
    s = s_o.copy()
    s[g] *= 1.0 + 1e-4
    caught("tsum * (1 + 1e-4)", o, pairs, t_o, s)
    # 3. the pixels of partial warps outside the image counted (a warp's `inside` ignored): odd_17x15 rendered as 32x16 on the same
    #    tile lists
    case, o, pairs = _run("odd_17x15")
    pad = gs_oracle.render_forward_stats(o, o, case.bg, 32, 16)
    caught("off-image pixels counted", o, pairs, pad["touched_pixels"], pad["transmittance_sum"])
    # 4. the pair that stops a saturated pixel counted as a contributor (the ballot on the alpha test, not on `contributes`)
    case, o, pairs = _run("saturation")
    t = o["touched_pixels"].copy()
    gx = (case.W + 15) // 16
    for y in range(case.H):
        for x in range(case.W):
            tile = (y // 16) * gx + x // 16
            ids = o["point_list"][o["ranges"][tile, 0]:o["ranges"][tile, 1]].astype(np.int64)
            power, a = BE._pair_alpha(o, ids, x, y)
            n = int(o["n_contrib"][y, x])
            after = np.nonzero(((power <= 0) & (a >= 1.0 / 255.0))[n:])[0]
            if after.size:
                t[ids[n + after[0]]] += 1
    caught("terminating pair counted", o, pairs, t, o["transmittance_sum"])
    # 5. calculate_colours_variance without the reference's aliasing of the old and the new mean
    vc, (ref, _, loose) = _variance("odd_17x15")
    (d, v, m), _, _ = SE.variance_oracle(vc, alias_mean=False)
    _, failures = SE.compare_variance("mean_old not aliased", ref, (d, v, m), loose, verbose=False)
    assert failures and {n for n, _, _ in failures} == {"variance"}
    accepted["mean_old not aliased"] = SE.old_variance_rule_ok(ref, (d, v, m))
    print("\naccepted by the old rule:", accepted)
    assert any(accepted.values())
