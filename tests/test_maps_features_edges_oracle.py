"""CPU: the fp64 compositions of tests/maps_features64.py (the inverse-depth / alpha maps' backward and the feature channels'
backward, from the colour oracle) reach the render and feature backwards' boundaries on the scenes of tests/backward_edges.py, and
the per-element comparison of test_gpu_maps_features_edges.py catches near-misses made with the oracle itself, some of which the
1e-4-of-the-array's-scale bar of test_gpu_maps.py lets through.  Only the oracle runs here: no GPU."""
import time

import numpy as np
import pytest

import backward_edges as BE
import maps_features64 as MF

_cache = {}
FEAT_SEED, GRAD_SEED = 31, 37


def _run(name, aa=False):
    """-> (case, forward state, excluded, maps-only (o64, o32), maps' dL_dinvdepth / dL_dalpha)."""
    key = (name, aa)
    if key not in _cache:
        case = BE.build(name, aa=aa)
        aa = case.meta["aa"]
        t = time.perf_counter()
        o = _forward(case, aa)
        excl = BE.excluded(case, o)
        Gd, Ga = MF.map_gradients(case.W, case.H, GRAD_SEED)
        maps = MF.compose(case, o, maps=(Gd, Ga), aa=aa)
        print("\n[%s%s] maps oracle %.2f s" % (name, ", aa" if aa else "", time.perf_counter() - t))
        _cache[key] = case, o, excl, maps, (Gd, Ga)
    return _cache[key]


def _forward(case, aa):
    import gs_oracle
    s = case.scene
    return gs_oracle.forward(s.means3D, s.opacity, s.scales, s.rotations, s.sh, s.degrees, bg=case.bg, antialiasing=aa, **case.cam_kw())


def _features(P, F):
    return np.random.default_rng(FEAT_SEED).standard_normal((P, F)).astype(np.float32)


def _global_ok(o64, got, arrays):
    """test_gpu_maps' bar: 1e-4 of each array's largest |o64|."""
    return all(np.abs(np.asarray(got[n], np.float64) - np.asarray(o64[n], np.float64)).max() <= 1e-4 * np.abs(o64[n]).max()
               for n in arrays if np.asarray(o64[n]).size)


def _partial_warp_pixels(W, H):
    """Pixels in warps (8x4) that are cut by the image's right or bottom edge, and pixels of a last tile column 1 pixel wide."""
    ys, xs = np.mgrid[0:H, 0:W]
    cut = ((W % 8 != 0) & (xs >= W - W % 8)) | ((H % 4 != 0) & (ys >= H - H % 4)) | ((W % 16 == 1) & (xs == W - 1))
    return cut


@pytest.mark.parametrize("name", ["odd_%dx%d" % s for s in BE.ODD_SIZES if s[0] % 8 or s[1] % 4 or s[0] % 16 == 1])
def test_maps_reach_the_partial_warps_and_the_last_tile_column(name):
    """dL_dinvdepth and dL_dalpha reach the Gaussians of the partial warps' pixels: masking them there moves those Gaussians'
    gradients by more than the per-element bar."""
    case, o, excl, (m64, m32), (Gd, Ga) = _run(name)
    BE.assert_reaches(case, o, excl)
    cut = _partial_warp_pixels(case.W, case.H) & (o["n_contrib"] > 0)
    assert cut.any(), "a partial warp holds contributing pixels"
    for which in (0, 1):
        g = [Gd.copy(), Ga.copy()]
        g[which][cut] = 0.0
        b64, _ = MF.compose(case, o, maps=tuple(g))
        _, failures = BE.compare("%s, %s masked on partial warps" % (name, ("dL_dinvdepth", "dL_dalpha")[which]), o, m64, m32, b64,
                                 ~excl, verbose=False)
        assert failures, (name, which)
    # ... and the oracle's own fp32 composition passes the net: the bar is not tighter than the reference's arithmetic
    _, failures = BE.compare(name, o, m64, m32, m32, ~excl, glob=(excl, BE.EXCLUDED_BAR), verbose=False)
    assert not failures, BE.describe(failures, o, m64, m32, case.W, case.H)


def test_the_direct_depth_term_carries_some_gaussians():
    """On some checked Gaussians the direct term -dinvd / z^2 (V[2], V[6], V[10]) is at least half of |dL_dmeans3D|."""
    for name in ("staircase", "odd_20x36", "saturation"):
        case, o, excl, (m64, _), _ = _run(name)
        V = case.cam.world_view_transform.numpy().astype(np.float64).reshape(-1)
        vis = o["radii"] > 0
        z = np.where(vis, o["depths"].astype(np.float64), 1.0)
        direct = np.abs(m64["dinvd"] / (z * z))[:, None] * np.abs(np.array([V[2], V[6], V[10]]))[None, :]
        share = direct.max(1) / np.maximum(np.abs(m64["dL_dmeans3D"]).max(1), 1e-300)
        n = int((vis & ~excl & (share >= 0.5)).sum())
        print("\n[%s] %d checked Gaussians whose direct depth term is >= half of |dL_dmeans3D|" % (name, n))
        assert n >= 10, name


def test_the_alpha_map_term_is_significant_where_final_T_is_small():
    """saturation: Gaussians all of whose pixels end with final_T < 1e-2 still get an alpha-map share of dL_dopacity above the
    per-element bar (T_final / (1 - alpha) is small there, the term is not)."""
    case, o, excl, (m64, m32), (Gd, Ga) = _run("saturation")
    a64, _ = MF.compose(case, o, maps=(np.zeros_like(Gd), Ga))
    W, H = case.W, case.H
    gx = (W + 15) // 16
    small = np.zeros(o["radii"].shape[0], bool)
    big_T = np.zeros_like(small)
    for y in range(H):
        for x in range(W):
            t = (y // 16) * gx + x // 16
            ids = o["point_list"][o["ranges"][t, 0]:o["ranges"][t, 0] + o["n_contrib"][y, x]].astype(np.int64)
            (small if o["final_T"][y, x] < 1e-2 else big_T)[ids] = True
    sel = small & ~big_T & (o["radii"] > 0) & ~excl
    share = np.abs(a64["dL_dopacity"][:, 0]) / np.maximum(np.abs(m64["dL_dopacity"][:, 0]), 1e-300)
    n = int((sel & (share > 10 * BE.R_REL)).sum())
    print("\n[saturation] %d Gaussians under final_T < 1e-2 only; %d with an alpha-map share of dL_dopacity > %g" % (
        int(sel.sum()), n, 10 * BE.R_REL))
    assert n >= 20


def test_features_reach_the_batch_boundaries_and_long_lists():
    """dL_dfeatures and the feature geometry reach the entries at the 256-entry batch boundaries of features_backward_kernel
    (staircase tiles of 255 / 256 / 257 and 511 / 512 / 513 entries) and, on dense_faint, lists of more than 8 192 entries."""
    case, o, excl, _, _ = _run("staircase")
    P = o["radii"].shape[0]
    A, h, _ = MF.rank3(17, case.H, case.W, GRAD_SEED)
    f64, f32 = MF.compose(case, o, features=(_features(P, 17), (A, h)))
    for k in (255, 256, 257, 511, 512, 513):
        t = BE.STAIRCASE.index(k)
        r0 = int(o["ranges"][t, 0])
        for pos in {254, 255, 256, 510, 511, 512} & set(range(k)):
            g = int(o["point_list"][r0 + pos])
            assert np.abs(f64["dL_dfeatures"][g]).max() > 0 and np.abs(f64["dL_dopacity"][g]).max() > 0, (k, pos)
    _, failures = BE.compare("staircase, F = 17 rank 3", o, f64, f32, f32, ~excl, glob=(excl, BE.EXCLUDED_BAR), verbose=False,
                             arrays=BE.ARRAYS + ["dL_dfeatures"])
    assert not failures
    case = BE.build("dense_faint")
    o = _forward(case, False)
    P = o["radii"].shape[0]
    hi = BE.tile_hi(o, case.W, case.H)
    t = int(np.argmax(hi))
    assert hi[t] > 8192
    A, h, _ = MF.rank3(9, case.H, case.W, GRAD_SEED)
    f64, _ = MF.compose(case, o, features=(_features(P, 9), (A, h)))
    deep = o["point_list"][int(o["ranges"][t, 0]) + 8192:int(o["ranges"][t, 0]) + int(hi[t])].astype(np.int64)
    assert (np.abs(f64["dL_dfeatures"][deep]).max(1) > 0).sum() >= 100


def test_per_element_check_rejects_what_the_global_bar_accepts():
    accepted_globally = []
    # 1. the alpha-map term dropped at one pixel of a partial warp (17x15: the last tile column is 1 pixel wide)
    case, o, excl, (m64, m32), (Gd, Ga) = _run("odd_17x15")
    arrays = BE.ARRAYS
    bad = Ga.copy()
    cut = _partial_warp_pixels(case.W, case.H) & (o["n_contrib"] > 0) & ~o["borderline"]
    cut[:, :case.W - 1] = False                                                    # the 1-pixel tile column
    ys, xs = np.nonzero(cut)
    y, x = int(ys[len(ys) // 2]), int(xs[len(xs) // 2])
    bad[y, x] = 0.0
    b64, _ = MF.compose(case, o, maps=(Gd, bad))
    _, failures = BE.compare("alpha-map term dropped at pixel (%d, %d)" % (x, y), o, m64, m32, b64, ~excl)
    assert failures, "the alpha-map term of one pixel must be caught"
    accepted_globally.append(("alpha-map term at one pixel", _global_ok(m64, b64, arrays)))
    # 2. 1/depth of the wrong Gaussian for one row (odd_20x36: the next visible Gaussian's)
    case, o, excl, (m64, m32), (Gd, Ga) = _run("odd_20x36")
    vis = np.nonzero((o["radii"] > 0) & ~excl)[0]
    rgb = MF.invdepth_colours(o)
    i, j = next((a, b) for a, b in zip(vis[:-1], vis[1:]) if abs(rgb[a, 0] / rgb[b, 0] - 1.0) > 0.05)
    rgb[i, 0] = rgb[j, 0]
    real = MF.invdepth_colours
    MF.invdepth_colours = lambda o_: rgb
    try:
        b64, _ = MF.compose(case, o, maps=(Gd, Ga))
    finally:
        MF.invdepth_colours = real
    _, failures = BE.compare("1/depth of Gaussian %d for row %d" % (j, i), o, m64, m32, b64, ~excl)
    assert failures, "a wrong Gaussian's 1/depth must be caught"
    accepted_globally.append(("1/depth of the wrong Gaussian", _global_ok(m64, b64, arrays)))
    # 3. the direct depth term omitted for one Gaussian (one where it is a small part of its dL_dmeans3D)
    V = case.cam.world_view_transform.numpy().astype(np.float64).reshape(-1)
    z = np.where(o["radii"] > 0, o["depths"].astype(np.float64), 1.0)
    direct = (-m64["dinvd"] / (z * z))[:, None] * np.array([V[2], V[6], V[10]])[None, :]
    share = np.abs(direct).max(1) / np.maximum(np.abs(m64["dL_dmeans3D"]).max(1), 1e-300)
    cand = vis[(share[vis] > 0.01) & (share[vis] < 0.2)]
    assert cand.size
    g = int(cand[np.argmax(np.abs(m64["dL_dmeans3D"][cand]).max(1))])
    b64 = {k: np.array(v, copy=True) for k, v in m64.items()}
    b64["dL_dmeans3D"][g] -= direct[g]
    _, failures = BE.compare("direct depth term of Gaussian %d omitted" % g, o, m64, m32, b64, ~excl)
    assert failures and failures[0][0] == "dL_dmeans3D" and failures[0][2].tolist() == [g]
    accepted_globally.append(("direct depth term of one Gaussian", _global_ok(m64, b64, arrays)))
    # 4. F = 17: the second 16-channel chunk's (channel 16's) geometry terms dropped on one tile
    case, o, excl, _, _ = _run("staircase")
    P = o["radii"].shape[0]
    feat = _features(P, 17)
    G = MF.full_rank(17, case.H, case.W, GRAD_SEED)
    f64, f32 = MF.compose(case, o, features=(feat, G))
    t = BE.STAIRCASE.index(65)
    Gb = G.copy()
    Gb[16, 16 * (t // 6):16 * (t // 6) + 16, 16 * (t % 6):16 * (t % 6) + 16] = 0.0
    b64, _ = MF.compose(case, o, features=(feat, Gb))
    b64["dL_dfeatures"] = f64["dL_dfeatures"]                                      # only the geometry terms are dropped
    _, failures = BE.compare("F = 17, channel 16's geometry dropped on tile %d" % t, o, f64, f32, b64, ~excl,
                             arrays=BE.ARRAYS + ["dL_dfeatures"])
    assert failures, "one chunk's geometry terms on one tile must be caught"
    accepted_globally.append(("second chunk's geometry on one tile", _global_ok(f64, b64, BE.ARRAYS + ["dL_dfeatures"])))
    print("\naccepted by test_gpu_maps' bar (1e-4 of each array's scale):", accepted_globally)
    assert any(ok for _, ok in accepted_globally)


def test_maps_composition_pins_the_absgrad_restatement():
    """absgrad64.pair_sums with the maps' gradients: its signed sums are the maps composition's dL_dmeans2D."""
    import absgrad64
    for name in ("odd_17x15", "saturation", "aa_needles"):
        case, o, excl, _, (Gd, Ga) = _run(name)
        m64, _ = MF.compose(case, o, colour=BE.oracle(case, fwd=o, aa=case.meta["aa"])[1:], maps=(Gd, Ga), aa=case.meta["aa"])
        signed, ab = absgrad64.pair_sums(o, case.bg.numpy(), case.dL.numpy(), case.W, case.H, dL_dinvdepth=Gd, dL_dalpha=Ga)
        ref = np.asarray(m64["dL_dmeans2D"], np.float64)[:, :2]
        vis = o["radii"] > 0
        chk = vis & ~excl
        err = np.abs(signed - ref).max(axis=1)
        row = np.maximum(np.abs(ref).max(axis=1), ab.max(axis=1))
        bar = np.maximum(1e-5 * row, 1e-8 * np.abs(ref).max())
        assert (err[chk] <= bar[chk]).all(), (name, float((err[chk] / np.maximum(row[chk], 1e-30)).max()))
        assert (ab + 1e-12 * ab.max() >= np.abs(signed)).all() and (ab[~vis] == 0).all()
