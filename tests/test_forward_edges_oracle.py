"""CPU: the scenes of tests/forward_edges.py reach the render forward's boundaries in every variant, the oracle's fp32 forward is
within the per-pixel bars of its own fp64 render (so the bars are not below the fp32 floor), and the per-pixel check of
test_gpu_forward_edges.py rejects near-misses made from the oracle state, each a plausible kernel bug, one of which today's 1e-4
colour bar accepts.  Only the oracle runs here: no GPU."""
import numpy as np
import pytest

import forward_edges as FE

_cache = {}


def _run(name, variant, F=None):
    key = (name, variant, F)
    if key not in _cache:
        case = FE.build(name, variant)
        inp = FE.inputs(case, variant, F=F)
        o, images = FE.oracle_forward(case, variant, inp)
        _cache[key] = case, o, images
    return _cache[key]


def _variants():
    return [pytest.param(v, F, id=v if F is None else "%s-%d" % (v, F))
            for v in FE.VARIANTS for F in (FE.FEATURE_F if v == "features" else [None])]


@pytest.mark.parametrize("variant, F", _variants())
@pytest.mark.parametrize("name", FE.SCENES)
def test_scene_reaches_its_boundaries_and_the_fp32_oracle_meets_the_bars(name, variant, F):
    case, o, images = _run(name, variant, F)
    r = FE.assert_reaches(case, variant, o)
    # the fp32 oracle against its fp64 render off the borderline pixels, array by array
    nb = ~o["borderline"]
    worst = {}
    for k, (a32, a64) in images.items():
        e = np.abs(a32.astype(np.float64) - a64).max(axis=0)
        worst[k] = float(e[nb].max() / FE.BARS[k]) if nb.any() else 0.0
        assert worst[k] <= FE.FP64_SLACK.get((name, variant), 1.0), (name, variant, k, worst[k])
    print("\n[%s, %s%s] reach %s; fp32 oracle |o32 - o64| / bar: %s" % (
        name, variant, "" if F is None else " F = %d" % F, r, ", ".join("%s %.3g" % kv for kv in worst.items())))


def test_odd_sizes_cover_partial_warps_tiles_and_the_background():
    """Partial warp blocks (8x4) and tiles on both axes, a last tile column 1 pixel wide, 1x1 and 33x1, and a background seen
    through final_T > 0.5 on a partial tile somewhere among the scenes."""
    sizes = [(int(n[4:].split("x")[0]), int(n[4:].split("x")[1])) for n in FE.SCENES if n.startswith("odd_")]
    assert any(w % 8 for w, h in sizes) and any(h % 4 for w, h in sizes)
    assert any(w % 16 == 1 for w, h in sizes) and (1, 1) in sizes and (33, 1) in sizes
    seen = [n for n in FE.SCENES if FE.REACH[n].get("bg_partial", 0) > 0]
    assert seen, "a background visible through final_T > 0.5 on a partial tile"


# ---- near-misses -------------------------------------------------------------------------------------------------------------

def _walk(w, i, rgb, bg, skip=None, alpha_of=None):
    """The fp64 walk of pixel i of tile walk `w` -> (colour [C], final T, n_contrib): `skip` drops one list entry, `alpha_of`
    (an index map over the entries) composites each entry with the alpha of another one (colour only)."""
    passes = w["passes"][i].copy()
    if skip is not None:
        passes[skip] = False
    alpha = w["alpha"][i]
    T, C, last = 1.0, np.zeros(rgb.shape[1]), 0
    for k in np.nonzero(passes)[0]:
        nt = T * (1.0 - alpha[k])
        if nt < 1e-4:
            break
        a = alpha[alpha_of[k]] if alpha_of is not None else alpha[k]
        C += rgb[w["ids"][k]] * a * T
        T, last = nt, int(k) + 1
    return C + T * bg, T, last


def _reject(label, case, o, images, bad_images, bad_nc=None):
    got = dict(n_contrib=o["n_contrib"] if bad_nc is None else bad_nc, **{k: v[0] for k, v in images.items()})
    got.update(bad_images)
    _, failures = FE.compare(label, o, images, got, case.W, case.H)
    assert failures, label + ": must be rejected"
    print(FE.describe(failures, o, images, got, case.W, case.H, limit=1))
    return got


def test_near_miss_faint_pair_skipped_at_low_T():
    """1. One faint pair (alpha < 2/255) skipped where T < 0.02, not the last contributor: the colour moves by less than 1e-4,
    so today's bar accepts it; final_T moves by alpha T >= T / 255."""
    case, o, images = _run("saturation", "plain")
    W, H = case.W, case.H
    rgb = o["rgb"].astype(np.float64)
    bg = case.bg.numpy().astype(np.float64)
    for t in range(FE._tiles(W, H)):
        w = FE.tile_walk(o, W, H, t)
        for i, (x, y) in enumerate(w["xy"]):
            n = int(o["n_contrib"][y, x])
            if o["borderline"][y, x] or n < 2:
                continue
            cand = np.nonzero(w["passes"][i, :n - 1] & (w["front"][i, :n - 1] < 0.02) & (w["alpha"][i, :n - 1] < 2.0 / 255.0) &
                              (w["front"][i, :n - 1] * w["alpha"][i, :n - 1] > 2e-5))[0]
            if not cand.size:
                continue
            c0, T0, n0 = _walk(w, i, rgb, bg)
            c1, T1, n1 = _walk(w, i, rgb, bg, skip=int(cand[0]))
            if n1 != n0 or np.abs(c1 - c0).max() >= FE.OLD_COLOR_BAR:
                continue
            color, final_T = images["color"][0].copy(), images["final_T"][0].copy()
            color[:, y, x] += (c1 - c0).astype(np.float32)
            final_T[0, y, x] += np.float32(T1 - T0)
            got = _reject("faint pair skipped at T %.3g" % w["front"][i, cand[0]], case, o, images,
                          dict(color=color, final_T=final_T))
            assert FE.old_color_ok(o, got), "today's 1e-4 colour bar accepts it"
            return
    raise AssertionError("no pixel with a faint pair at T < 0.02 in front of its last contributor")


def _terminated_pixel(case, o):
    """A pixel off the borderline stopped by T < 1e-4 with at least two contributors -> (tile walk, index, x, y)."""
    W, H = case.W, case.H
    for t in range(FE._tiles(W, H)):
        w = FE.tile_walk(o, W, H, t)
        for i, (x, y) in enumerate(w["xy"]):
            if w["stop"][i] >= 0 and not o["borderline"][y, x] and o["n_contrib"][y, x] >= 2:
                return w, i, x, y
    raise AssertionError("no terminated pixel")


def test_near_miss_final_T_one_pair_early():
    """2. final_T taken in front of the last contributor on a terminated pixel."""
    case, o, images = _run("saturation", "plain")
    w, i, x, y = _terminated_pixel(case, o)
    n = int(o["n_contrib"][y, x])
    final_T = images["final_T"][0].copy()
    final_T[0, y, x] = np.float32(o["final_T"][y, x] / (1.0 - w["alpha"][i, n - 1]))
    _reject("final_T one pair early", case, o, images, dict(final_T=final_T))


def test_near_miss_background_with_the_neighbours_T():
    """3. The background added with the T of the neighbouring pixel (the other row of its pair) of the warp block, in a partial
    warp block (8x4 pixels reaching past the image) of an odd-sized scene."""
    best = None
    for name in [n for n in FE.SCENES if n.startswith("odd_")]:
        case, o, images = _run(name, "plain")
        W, H = case.W, case.H
        T = o["final_T"].astype(np.float64)
        for y in range(H):
            for x in range(W):
                partial = (x // 8) * 8 + 8 > W or (y // 4) * 4 + 4 > H
                ny = y ^ 1
                if partial and ny < H and not o["borderline"][y, x]:
                    d = abs(T[ny, x] - T[y, x]) * float(np.abs(case.bg.numpy()).max())
                    if best is None or d > best[0]:
                        best = (d, name, x, y, ny)
    d, name, x, y, ny = best
    assert d > 10 * FE.BARS["color"], best
    case, o, images = _run(name, "plain")
    color = images["color"][0].copy()
    color[:, y, x] = color[:, y, x] + case.bg.numpy().astype(np.float32) * (o["final_T"][ny, x] - o["final_T"][y, x])
    _reject("%s: background with the neighbour's T" % name, case, o, images, dict(color=color))


def test_near_miss_n_contrib_one_early():
    """4. n_contrib - 1 on a terminated pixel."""
    case, o, images = _run("saturation", "plain")
    _, _, x, y = _terminated_pixel(case, o)
    nc = o["n_contrib"].copy()
    nc[y, x] -= 1
    _reject("n_contrib - 1", case, o, images, {}, bad_nc=nc)


def test_near_miss_invdepth_with_the_previous_alpha():
    """5. The inverse depth composited with the colour's alpha of the previous pair."""
    case, o, images = _run("odd_20x36", "maps")
    W, H = case.W, case.H
    invd = (np.float32(1.0) / o["depths"].astype(np.float32)).astype(np.float64)[:, None]
    for t in range(FE._tiles(W, H)):
        w = FE.tile_walk(o, W, H, t)
        for i, (x, y) in enumerate(w["xy"]):
            if o["borderline"][y, x] or o["n_contrib"][y, x] < 3:
                continue
            p = np.nonzero(w["passes"][i])[0]
            prev = np.arange(w["ids"].size)
            prev[p[1:]] = p[:-1]
            d0, _, _ = _walk(w, i, invd, np.zeros(1))
            d1, _, _ = _walk(w, i, invd, np.zeros(1), alpha_of=prev)
            if abs(d1[0] - d0[0]) < 1e-4:
                continue
            inv = images["invdepth"][0].copy()
            inv[0, y, x] += np.float32(d1[0] - d0[0])
            _reject("invdepth with the previous alpha", case, o, images, dict(invdepth=inv))
            return
    raise AssertionError("no pixel with three contributors")
