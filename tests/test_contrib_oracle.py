"""CPU: the contribution cases of tests/contrib64.py reach what they are built for, the float64 restatement agrees with the oracle's
statistics forward, and the per-Gaussian comparison of test_gpu_contrib.py rejects near-misses made with the restatement itself.
Only the oracle runs here: no GPU."""
import numpy as np
import pytest

import backward_edges as BE
import contrib64 as C6
import gs_oracle

_cache = {}


def _run(name):
    if name not in _cache:
        case = C6.build(name)
        o = C6.oracle(case)
        _cache[name] = case, o, C6.restate(o, case.W, case.H), BE.borderline_pairs(o, case.W, case.H)
    return _cache[name]


def _got(c, f32=True):
    t = np.float32 if f32 else np.float64
    return c["weight_sum"].astype(t), c["weight_max"].astype(t), c["pixels"], c["top_id32"]


@pytest.mark.parametrize("name", C6.CASES + [C6.TIE])
def test_restatement_against_the_oracle(name):
    case, o, c, pairs = _run(name)
    near = pairs[0]
    vis = o["radii"] > 0
    # the count is the statistics forward's touched_pixels away from borderline decisions, and zero for culled Gaussians
    assert np.array_equal(c["pixels"][vis & ~near], o["touched_pixels"][vis & ~near].astype(np.int64))
    assert not c["pixels"][~vis].any() and not c["weight_sum"][~vis].any() and not c["weight_max"][~vis].any()
    # sum_i sum_p alpha T = sum_p (1 - final_T): the weights of a pixel add up to its opacity
    total = (1.0 - o["final_T"].astype(np.float64)).sum()
    assert abs(c["weight_sum"].sum() - total) <= 1e-6 * max(total, 1.0), (c["weight_sum"].sum(), total)
    assert np.array_equal(c["top_id"] >= 0, o["n_contrib"] > 0)
    # the restatement rounded to fp32 (what the kernel returns) passes: the bars are not tighter than the outputs' precision
    _, failures = C6.compare(name, o, c, pairs, _got(c), tie_pixel=case.meta.get("tie_pixel"), verbose=False)
    assert not failures, failures


def test_cases_cover_the_pass_boundaries():
    his = {n: BE.tile_hi(_run(n)[1], _run(n)[0].W, _run(n)[0].H) for n in C6.CASES}
    # walks past one 256-entry batch and past 8 192 entries
    assert any((h > 256).any() for h in his.values()) and any((h > 8192).any() for h in his.values())
    # terminated pixels: a passing pair behind n_contrib
    case, o, _, _ = _run("saturation")
    gx = (case.W + 15) // 16
    terminated = 0
    for y in range(case.H):
        for x in range(case.W):
            r0, r1 = (int(v) for v in o["ranges"][(y // 16) * gx + x // 16])
            power, a = BE._pair_alpha(o, o["point_list"][r0:r1].astype(np.int64), x, y)
            terminated += int(((power <= 0) & (a >= 1.0 / 255.0))[int(o["n_contrib"][y, x]):].any())
    assert terminated >= case.W * case.H // 4
    # partial warps (lanes outside the image) and 1-pixel tile columns, with contributing pairs there
    for name in ("odd_17x15", "odd_33x1", "odd_3x7", "odd_20x36"):
        case, o, c, _ = _run(name)
        assert (case.W % 8 or case.H % 4) and (c["top_id"] >= 0).any(), name
    assert any(_run(n)[0].W % 16 == 1 and (_run(n)[2]["top_id"][:, -1] >= 0).any() for n in ("odd_17x15", "odd_33x1"))
    # visible Gaussians with no contributing pair (every pair below 1/255, or behind n_contrib)
    assert sum(int(((_run(n)[1]["radii"] > 0) & (_run(n)[2]["pixels"] == 0)).sum()) for n in C6.CASES) >= 10


def test_the_tie_is_exact_in_fp32():
    case, o, c, _ = _run(C6.TIE)
    x, y = case.meta["tie_pixel"]
    assert int(o["n_contrib"][y, x]) == 2 and list(o["point_list"]) == [0, 1]
    assert np.array_equal(o["means2D"], [[x, y], [x, y]])
    oa, ob = o["conic_opacity"][:, 3].astype(np.float32)
    assert ob * (np.float32(1.0) - oa) == oa, "w_B == w_A in fp32"
    assert c["top_id32"][y, x] == 0 and c["gap"][y, x] < C6.TOP_GAP


def test_map_clamp_and_nan():
    case, o, c, pairs = _run("odd_20x36")
    rng = np.random.default_rng(5)
    m = rng.uniform(-1.0, 2.0, (case.H, case.W)).astype(np.float32)
    m.reshape(-1)[::7] = np.nan
    m.reshape(-1)[3::11] = np.inf
    m.reshape(-1)[5::13] = -np.inf
    assert (m < 0).any() and (m > 1).any() and np.isnan(m).any()
    cm = C6.restate(o, case.W, case.H, weights=m)
    cc = C6.restate(o, case.W, case.H, weights=C6.clamp_map(m))
    assert np.array_equal(cm["weight_sum"], cc["weight_sum"])
    assert (cm["weight_sum"] < c["weight_sum"]).any() and (cm["weight_sum"] <= c["weight_sum"] + 1e-12).all()
    for k in ("weight_max", "pixels", "top_id"):
        assert np.array_equal(cm[k], c[k]), k


def test_per_gaussian_check_rejects_near_misses():
    def caught(label, case, o, c, pairs, got, **kw):
        _, failures = C6.compare(label, o, c, pairs, got, verbose=False, **kw)
        assert failures, label + " must be caught"

    case, o, c, pairs = _run("large")
    near, count, _ = pairs
    vis = o["radii"] > 0
    ws, wm, px, top = _got(c)
    # 1. one count + 1 on a Gaussian away from every borderline pixel
    g = int(np.nonzero(vis & ~near & (count == 0) & (c["pixels"] > 0))[0][0])
    px1 = px.copy()
    px1[g] += 1
    caught("pixels + 1", case, o, c, pairs, (ws, wm, px1, top))
    # 2. the pair that terminates a saturated pixel counted
    case, o, c, pairs = _run("saturation")
    t = C6.restate(o, case.W, case.H, miss="terminating")
    caught("terminating pair counted", case, o, c, pairs, (_got(c)[0], _got(c)[1], t["pixels"], c["top_id"]))
    # 3. the maximum taken over the pairs the alpha test skips
    case, o, c, pairs = _run("dense_faint")
    t = C6.restate(o, case.W, case.H, miss="skipped")
    assert (t["weight_max"] != c["weight_max"]).any()
    caught("maximum over a skipped pair", case, o, c, pairs, (_got(c)[0], t["weight_max"].astype(np.float32), c["pixels"], c["top_id"]))
    # 4. the exact tie broken to the later Gaussian
    case, o, c, pairs = _run(C6.TIE)
    x, y = case.meta["tie_pixel"]
    top = c["top_id32"].copy()
    top[y, x] = 1
    caught("tie to the later Gaussian", case, o, c, pairs, (_got(c)[0], _got(c)[1], c["pixels"], top), tie_pixel=(x, y))
    # 5. a map read without the clamp
    case, o, c, pairs = _run("odd_20x36")
    m = np.random.default_rng(6).uniform(-1.0, 2.0, (case.H, case.W))
    cm = C6.restate(o, case.W, case.H, weights=m)
    un = C6.restate(o, case.W, case.H, weights=m, clamp=False)
    caught("unclamped map", case, o, cm, pairs, _got(un))
    # 6. the pixels of partial warps outside the image counted: odd_17x15 restated as 32 x 16 on the same tile lists
    case, o, c, pairs = _run("odd_17x15")
    pad = dict(o, n_contrib=gs_oracle.render_forward_stats(o, o, case.bg, 32, 16)["n_contrib"])
    cp = C6.restate(pad, 32, 16)
    caught("off-image pixels counted", case, o, c, pairs, (cp["weight_sum"].astype(np.float32), cp["weight_max"].astype(np.float32),
                                                             cp["pixels"], cp["top_id"][:case.H, :case.W]))
