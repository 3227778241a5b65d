"""The render forward (render_forward_kernel, gsb_render.cu, and features_forward_kernel, gsb_features.cu) per pixel against the
oracle on the boundary scenes of tests/backward_edges.py, for every forward variant.

Shared by test_forward_edges_oracle.py (CPU: every scene x variant reaches the boundaries it is built for, the fp32 oracle stays
within the bars of its own fp64 render, and the per-pixel check rejects near-misses the older 1e-4 colour bar accepts) and
test_gpu_forward_edges.py (the CUDA forward against the oracle, pixel by pixel).

The scenes are the 16 backward_edges.CASES, the two AA_CASES and t1 of statistics_edges on each of its three cameras (W > H,
W = H, W < H).  The variants:
  plain     the case's own background (!= 0 on the odd sizes), antialiasing off;
  aa        the scene built for antialiasing (backward_edges.build(aa=True)), antialiasing on;
  filter3d  Mip-Splatting's 3D filter with zero, moderate, small-c3 and flat rows (filter3d_restatement.edge_rows): the oracle
            renders the filtered scales with the opacity fl32(sigmoid * c3) (times s with AA);
  quant     the scene quantised to the codebook layout (SH padded to 16 coefficients), against the de-quantised scene;
  pruned    a prune mask over 30 % of the Gaussians (the oracle's prune_mask argument);
  maps      the inverse-depth map (the oracle's colour render with colours fl32(1 / depth), background 0) and alpha = 1 - final_T;
  features  F in FEATURE_F feature channels: one oracle colour render per 3 channels, background 0.
The anti-aliased scenes (AA_CASES) keep antialiasing on in every variant but `plain`.

The check, per pixel and array (color, final_T, invdepth, alpha, features), against the oracle's fp32 forward o32 (the reference's
operation order, which the kernels follow instruction for instruction):
  - n_contrib exact, off the borderline pixels;
  - |ours - o32| <= BARS[array] off the borderline pixels;
  - on a borderline pixel (an ulp of the GPU's exponential can flip a decision there): BARS[array] + allowance(pixel), where each
    pair near a threshold at that pixel (alpha 1/255 or 0.99, power 0, the pair that terminates the pixel) adds
    (alpha + FLIP) * T in front of it, times (1 + 2 max|value|) of the pixel's values: a flipped pair adds or drops alpha * T * c
    and scales everything behind it by at most 1 / (1 - 1/255)."""
import numpy as np
import torch

import backward_edges as BE
import cases
import filter3d_restatement as F3
import gs_oracle
import statistics_edges as SE
from gs_b200 import synth

T1_VIEWS = cases.TOOLS_CASES["t1"]["views"]
T1 = ["t1_%dx%d" % (W, H) for W, H, _ in T1_VIEWS]
SCENES = BE.CASES + BE.AA_CASES + T1
VARIANTS = ["plain", "aa", "filter3d", "quant", "pruned", "maps", "features"]
FEATURE_F = [1, 17]
ARRAYS = ["color", "final_T", "invdepth", "alpha", "features"]
PRUNE_FRAC = 0.3
OLD_COLOR_BAR = 1e-4                         # test_gpu_parity's colour bar, |d| absolute

# The per-pixel bars, |ours - o32| off the borderline pixels.  The oracle agrees with the reference to 2.4e-7 in colour and
# final_T on the goldens (DESIGN.md §3); the kernels run the same operations, and only the exponential (MUFU.EX2 against
# exp2f, <= 2 ulp) differs.  An exp ulp moves alpha by 1.2e-7 of itself, and T and the colour sums by about that much per pair
# once the roundings that follow drift apart.
BARS = {
    "color": 2e-6,          # colour in [0, ~3]: 8 x 2.4e-7 (the fp32 oracle itself is 1.09e-6 from fp64 on dense_12k, filter3d)
    "final_T": 1e-6,        # T in [1e-4, 1]: 4 x 2.4e-7
    "invdepth": 1e-6,       # 1 / depth <= 0.4 on these scenes: the colour's bar
    "alpha": 1e-6,          # 1 - final_T: final_T's bar
    "features": 4e-6,       # standard-normal channels (|f| up to ~4.5): the colour's bar on twice its range
}
FLIP = SE.FLIP
# The fp32 oracle's own distance from its fp64 render, in units of BARS, where it exceeds 1 (test_forward_edges_oracle.py): the
# needles of aa_needles rendered without antialiasing keep a conic whose power -0.5 (A dx^2 + C dy^2) - B dx dy cancels, so the
# fp32 alpha of the reference arithmetic is off by ~1e-5 of itself there: its colour is 2.7 bars and final_T 7.8 bars from fp64.  The
# kernels follow that arithmetic: the GPU test compares with the fp32 oracle at the tight bar.
FP64_SLACK = {("aa_needles", "plain"): 10.0}


class Inputs:
    """What a variant feeds the kernel and the oracle: `scene` is the oracle's (de-quantised, filtered scales), `kernel_scene` the
    one the kernel gets (the unfiltered scales with `filt`), `prune` / `quant` / `filt` / `features` the optional inputs."""

    def __init__(self, scene, aa, bg, kernel_scene=None, prune=None, quant=None, filt=None, c3=None, maps=False, features=None):
        self.scene, self.aa, self.bg = scene, aa, bg
        self.kernel_scene = scene if kernel_scene is None else kernel_scene
        self.prune, self.quant, self.filt, self.c3, self.maps, self.features = prune, quant, filt, c3, maps, features


def build(name, variant="plain"):
    """The case `name` as built for `variant` (the `aa` variant: the scene meant for antialiasing)."""
    if name in T1:
        _, scene, cams, _ = cases.build_tools_inputs("t1")
        i = T1.index(name)
        case = BE.Case(name, scene, cams[i], torch.tensor([0.3, 0.1, 0.2]), None)
        case.meta["aa"] = False
        return case
    return BE.build(name, aa=(variant == "aa"))


def _pad_sh16(scene):
    P, M = scene.sh.shape[:2]
    sh = torch.zeros(P, 16, 3)
    sh[:, :M] = scene.sh
    return synth.Scene(scene.means3D, scene.opacity, scene.scales, scene.rotations, sh.contiguous(), scene.degrees)


def _copy(scene):
    return synth.Scene(*[getattr(scene, k).clone() for k in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])


def inputs(case, variant, dev="cpu", F=None):
    """The variant's inputs on `case` (built by build(name, variant)); `dev` de-quantises the `quant` variant where the kernel
    will (torch's exp and normalize there), `F` is the features variant's channel count."""
    aa = variant == "aa" or (variant != "plain" and case.meta.get("aa", False))
    s = case.scene
    idx = SCENES.index(case.name)
    if variant in ("plain", "aa"):
        return Inputs(s, aa, case.bg)
    if variant == "filter3d":
        ks = _copy(s)
        f, _ = F3.edge_rows(ks, 531 + idx)
        sp, c3 = F3.filtered(ks.scales, f)
        return Inputs(synth.Scene(ks.means3D, ks.opacity, sp.contiguous(), ks.rotations, ks.sh, ks.degrees), aa, case.bg,
                      kernel_scene=ks, filt=f, c3=c3)
    if variant == "quant":
        q = synth.quantise_scene(_pad_sh16(s), seed=idx)
        d = q.to(dev).dequantise()
        deq = synth.Scene(*[getattr(d, k).cpu().contiguous() for k in ("means3D", "opacity", "scales", "rotations", "sh", "degrees")])
        return Inputs(deq, aa, case.bg, quant=q)
    if variant == "pruned":
        return Inputs(s, aa, case.bg, prune=synth.prune_mask(s.P, 600 + idx, PRUNE_FRAC))
    if variant == "maps":
        return Inputs(s, aa, case.bg, maps=True)
    if variant == "features":
        feat = np.random.default_rng(700 + 10 * idx + F).standard_normal((s.P, F)).astype(np.float32)
        return Inputs(s, aa, case.bg, features=feat)
    raise ValueError(variant)


def _render_pair(o, rgb, bg, W, H):
    """-> (fp32 colour [3,H,W], fp64 colour [3,H,W]) of the oracle's render of `o`'s lists with colours `rgb` [P,3]."""
    g = dict(o)
    g["rgb"] = np.ascontiguousarray(rgb, np.float32)
    r32 = gs_oracle.render_forward(g, o, bg, W, H)
    r64 = gs_oracle.render_forward(g, o, bg, W, H, f64=True)
    return r32["color"], r64["color64"]


def oracle_forward(case, variant, inp, o_hat=None):
    """The oracle's fp32 forward state for `variant` (inputs `inp`), with its fp64 render beside it: -> (o, images) where images
    maps each array of the variant to (o32 [C,H,W], o64 [C,H,W]).  `o_hat` ([P], filter3d only) replaces the oracle's own
    fl32(sigmoid * c3) (* s) by the kernel's, which the GPU test holds to it within a few ulp."""
    s, W, H = inp.scene, case.W, case.H
    kw = case.cam_kw()
    o = gs_oracle.forward(s.means3D, s.opacity, s.scales, s.rotations, s.sh, s.degrees, bg=inp.bg, antialiasing=inp.aa,
                          prune_mask=inp.prune, **kw)
    if inp.filt is not None:
        sig = (o["aa_sigmoid"] if inp.aa else o["conic_opacity"][:, 3]).astype(np.float32)
        sc = (sig * inp.c3.numpy()).astype(np.float32)
        o["o_hat_oracle"] = (sc * o["aa_s"]).astype(np.float32) if inp.aa else sc
        o["conic_opacity"][:, 3] = o["o_hat_oracle"] if o_hat is None else o_hat
        o.update(gs_oracle.render_forward(o, o, inp.bg, W, H))
    bg = np.asarray(inp.bg, np.float32)
    zero = np.zeros(3, np.float32)
    r64 = gs_oracle.render_forward(o, o, bg, W, H, f64=True)
    images = dict(color=(o["color"], r64["color64"]), final_T=(o["final_T"][None], r64["final_T64"][None]))
    if inp.maps:
        with np.errstate(divide="ignore"):
            invd = np.float32(1.0) / o["depths"].astype(np.float32)
        c32, c64 = _render_pair(o, np.repeat(invd[:, None], 3, 1), zero, W, H)
        images["invdepth"] = (c32[:1], c64[:1])
        images["alpha"] = ((np.float32(1.0) - o["final_T"])[None], 1.0 - r64["final_T64"][None])
    if inp.features is not None:
        F = inp.features.shape[1]
        parts32, parts64 = [], []
        for c0 in range(0, F, 3):
            rgb = np.zeros((s.P, 3), np.float32)
            rgb[:, :min(3, F - c0)] = inp.features[:, c0:c0 + 3]
            c32, c64 = _render_pair(o, rgb, zero, W, H)
            parts32.append(c32[:min(3, F - c0)])
            parts64.append(c64[:min(3, F - c0)])
        images["features"] = (np.concatenate(parts32), np.concatenate(parts64))
    return o, images


# ---- the pair walk ---------------------------------------------------------------------------------------------------------------

def tile_walk(o, W, H, t):
    """The oracle's walk of tile `t`'s list, for all its pixels inside the image, in float64 from the fp32 pair arithmetic ->
    dict(xy [n, 2] pixels, r0 list start, ids [L], a [n, L] alpha before the clamp, alpha [n, L] after it, power [n, L], passes
    [n, L] (the alpha test), front [n, L] T in front of each entry (0 after the termination), stop [n] the terminating entry or
    -1)."""
    gx = (W + 15) // 16
    x0, y0 = 16 * (t % gx), 16 * (t // gx)
    ys, xs = np.mgrid[y0:min(y0 + 16, H), x0:min(x0 + 16, W)]
    xs, ys = xs.reshape(-1), ys.reshape(-1)
    r0, r1 = (int(v) for v in o["ranges"][t])
    ids = o["point_list"][r0:r1].astype(np.int64)
    m = o["means2D"][ids].astype(np.float32)
    co = o["conic_opacity"][ids].astype(np.float32)
    dx = m[None, :, 0] - xs[:, None].astype(np.float32)
    dy = m[None, :, 1] - ys[:, None].astype(np.float32)
    power = (np.float32(-0.5) * (co[:, 0] * dx * dx + co[:, 2] * dy * dy) - co[:, 1] * dx * dy).astype(np.float64)
    a = co[:, 3].astype(np.float64) * np.exp(power)
    alpha = np.minimum(0.99, a)
    passes = (power <= 0) & (alpha >= 1.0 / 255.0)
    after = np.cumprod(np.where(passes, 1.0 - alpha, 1.0), axis=1)
    ends = passes & (after < 1e-4)
    stop = np.where(ends.any(axis=1), np.argmax(ends, axis=1), -1)
    front = np.concatenate([np.ones((xs.size, 1)), after[:, :-1]], axis=1) if ids.size else after
    front = np.where(np.arange(ids.size)[None, :] > np.where(stop >= 0, stop, ids.size)[:, None], 0.0, front)
    return dict(xy=np.stack([xs, ys], 1), r0=r0, ids=ids, a=a, alpha=alpha, power=power, passes=passes, front=front, stop=stop)


def _tiles(W, H):
    return ((W + 15) // 16) * ((H + 15) // 16)


def allowance(o, W, H, values):
    """[H, W] allowance of the borderline pixels (0 elsewhere): per pair near a threshold (alpha 1/255 or 0.99, power 0) or
    ending the pixel (its last contributor and its terminating pair), (alpha + FLIP) * T in front of it, times 1 + 2 max|value|
    of the pixel (`values` [C,H,W], the oracle's image); a power-0 pair counts every passing pair of the pixel."""
    out = np.zeros((H, W))
    border = o["borderline"]
    if not border.any():
        return out
    vmax = np.abs(values).max(axis=0)
    gx = (W + 15) // 16
    for t in np.unique((np.nonzero(border)[0] // 16) * gx + np.nonzero(border)[1] // 16):
        w = tile_walk(o, W, H, int(t))
        for i, (x, y) in enumerate(w["xy"]):
            if not border[y, x]:
                continue
            a, power, passes = w["a"][i], w["power"][i], w["passes"][i]
            near = (power <= 1e-6) & ((np.abs(a * 255.0 - 1.0) < 1e-5) | (np.abs(a / 0.99 - 1.0) < 1e-5) | (np.abs(power) < 1e-6))
            sel = near.copy()
            if (near & (np.abs(power) < 1e-6)).any():
                sel |= passes
            n = int(o["n_contrib"][y, x])
            if n > 0:
                sel[n - 1] = True
            if w["stop"][i] >= 0:
                sel[w["stop"][i]] = True
            after = np.nonzero(passes[n:])[0]
            if after.size:
                sel[n + after[0]] = True
            out[y, x] = float(((w["alpha"][i] + FLIP) * w["front"][i])[sel].sum()) * (1.0 + 2.0 * float(vmax[y, x]))
    return out


# ---- the comparison ------------------------------------------------------------------------------------------------------------

def compare(label, o, images, got, W, H, verbose=True, allow=None):
    """The per-pixel check of `got` (n_contrib [H,W] and the arrays of `images`, each [C,H,W]) against the oracle's o32 ->
    (ratios, failures).  ratios[array] = largest |ours - o32| / BARS[array] off the borderline pixels, and on them largest
    |ours - o32| / (bar + allowance).  failures: (array, what, pixel mask)."""
    border = o["borderline"]
    failures, ratios = [], {}
    nc = np.asarray(got["n_contrib"]).reshape(H, W).astype(np.int64)
    bad = ~border & (nc != o["n_contrib"].astype(np.int64))
    if bad.any():
        failures.append(("n_contrib", "exact off the borderline pixels", bad))
    allow = {} if allow is None else allow
    for n, (a32, _) in images.items():
        g = np.asarray(got[n], np.float64).reshape(a32.shape)
        e = np.abs(g - a32.astype(np.float64)).max(axis=0)
        e = np.where(np.isnan(e), np.inf, e)
        bar = BARS[n]
        q = e / bar
        if border.any():
            if n not in allow:
                allow[n] = allowance(o, W, H, a32.astype(np.float64))
            qb = e / (bar + allow[n])
        else:
            qb = np.zeros_like(q)
        ratios[n] = (float(q[~border].max()) if (~border).any() else 0.0, float(qb[border].max()) if border.any() else 0.0)
        bad = np.where(border, qb > 1.0, q > 1.0)
        if bad.any():
            failures.append((n, "within %g (+ the borderline allowance)" % bar, bad))
    if verbose:
        print("\n[%s] %d pixels, %d borderline; max e / bar (borderline: e / (bar + allowance)): %s" % (
            label, W * H, int(border.sum()), ", ".join("%s %.3g %.3g" % (k, *v) for k, v in ratios.items())))
    return ratios, failures


def old_color_ok(o, got):
    """test_gpu_parity's rule: colour within 1e-4 absolute off the borderline pixels."""
    nb = ~o["borderline"]
    return bool(np.abs(np.asarray(got["color"], np.float64) - o["color"])[:, nb].max() <= OLD_COLOR_BAR)


def describe(failures, o, images, got, W, H, limit=4):
    """Where the failures are: per array the first pixels, with tile, both n_contrib (list positions), both values, and the
    oracle's T after its last contributor and in front of ours."""
    gx = (W + 15) // 16
    lines = []
    nc = np.asarray(got["n_contrib"]).reshape(H, W)
    gT = np.asarray(got["final_T"]).reshape(H, W)
    for n, what, mask in failures:
        ys, xs = np.nonzero(mask)
        lines.append("%s: %s: %d pixels" % (n, what, ys.size))
        for y, x in list(zip(ys, xs))[:limit]:
            w = tile_walk(o, W, H, (y // 16) * gx + x // 16)
            i = int(np.nonzero((w["xy"][:, 0] == x) & (w["xy"][:, 1] == y))[0][0])
            k = int(nc[y, x])
            L = w["ids"].size
            t_at = float(w["front"][i, k]) if k < L else float(o["final_T"][y, x])
            val = ""
            if n in images:
                val = " oracle %s ours %s;" % (images[n][0][:, y, x].tolist(), np.asarray(got[n]).reshape(images[n][0].shape)[:, y, x].tolist())
            lines.append("  pixel (%d, %d) tile %d (list %d + [0, %d)), borderline %s:%s n_contrib oracle %d ours %d; final_T oracle %.9g "
                         "ours %.9g; the oracle's T (fp64 walk) after list position %d: %.9g" % (
                             x, y, (y // 16) * gx + x // 16, w["r0"], L, bool(o["borderline"][y, x]), val,
                             int(o["n_contrib"][y, x]), k, float(o["final_T"][y, x]), float(gT[y, x]), k, t_at))
    return "\n".join(lines)


# ---- what each scene reaches ---------------------------------------------------------------------------------------------------

def reach(case, o):
    """Counts of what the forward's boundaries see in the state `o`:
      list_256 / list_8192: tiles whose list has more than 256 / 8 192 entries;
      terminated: pixels stopped by T < 1e-4 partway down their list; clamped: pixels with a pair whose alpha clamps at 0.99;
      partial_warp: rendered pixels (n_contrib > 0) in a warp block (8x4) that reaches past the image;
      thin_column: rendered pixels in a last tile column 1 pixel wide;
      faint_tail: pixels whose last contributor sees T < 0.025 with a pair skipped at alpha < 1/255 in front of it;
      bg_partial: pixels of a partial tile with final_T > 0.5 and a background != 0."""
    W, H = case.W, case.H
    counts = (o["ranges"][:, 1].astype(np.int64) - o["ranges"][:, 0])
    nc = o["n_contrib"].astype(np.int64)
    r = dict(list_256=int((counts > 256).sum()), list_8192=int((counts > 8192).sum()))
    gx = (W + 15) // 16
    xs, ys = np.meshgrid(np.arange(W), np.arange(H))
    warp_edge = ((xs // 8) * 8 + 8 > W) | ((ys // 4) * 4 + 4 > H)
    r["partial_warp"] = int((warp_edge & (nc > 0)).sum())
    r["thin_column"] = int(((W % 16 == 1) & (xs == W - 1) & (nc > 0)).sum())
    tile_edge = ((xs // 16) * 16 + 16 > W) | ((ys // 16) * 16 + 16 > H)
    bg_nonzero = bool(np.any(np.asarray(case.bg) != 0)) if case.bg is not None else False
    r["bg_partial"] = int((tile_edge & (o["final_T"] > 0.5)).sum()) if bg_nonzero else 0
    terminated = clamped = faint = 0
    # the pair walks: every tile of small images, a fixed sample of 300 tiles of the large ones
    tiles = np.arange(_tiles(W, H))
    if tiles.size > 300:
        tiles = np.sort(np.random.default_rng(0).choice(tiles, 300, replace=False))
    for t in tiles:
        if o["ranges"][t, 1] == o["ranges"][t, 0]:
            continue
        w = tile_walk(o, W, H, int(t))
        n = nc[w["xy"][:, 1], w["xy"][:, 0]]
        pos = np.arange(w["ids"].size)[None, :]
        inside = pos < n[:, None]
        terminated += int((w["stop"] >= 0).sum())
        clamped += int((w["passes"] & inside & (w["a"] >= 0.99)).any(axis=1).sum())
        last_T = np.where(n > 0, w["front"][np.arange(n.size), np.maximum(n - 1, 0)], 1.0)
        skipped = inside & (w["power"] <= 0) & (w["a"] < 1.0 / 255.0) & (w["a"] > 0.5 / 255.0)
        faint += int(((n > 0) & (last_T < 0.025) & skipped.any(axis=1)).sum())
    r.update(terminated=terminated, clamped=clamped, faint_tail=faint)
    return r


# The predicates each scene must reach, as minimum counts of reach() (measured on the oracle state of every variant; the pruned
# variant loses 30 % of the Gaussians, the anti-aliased one lowers every opacity by s).
REACH = {
    "staircase": dict(list_256=4), "staircase_ties": dict(list_256=4),
    "odd_1x1": dict(partial_warp=1, thin_column=1), "odd_3x7": dict(partial_warp=1, faint_tail=1), "odd_8x4": dict(faint_tail=1),
    "odd_15x17": dict(partial_warp=1, faint_tail=1), "odd_17x15": dict(partial_warp=1, thin_column=1, faint_tail=1),
    "odd_20x36": dict(partial_warp=1, faint_tail=1), "odd_33x1": dict(partial_warp=1, thin_column=1, faint_tail=1),
    "large": dict(bg_partial=1000, faint_tail=10),
    "saturation": dict(terminated=1000, clamped=30, faint_tail=1000),
    "dense_4k": dict(list_256=1, terminated=100, faint_tail=100),
    "dense_12k": dict(list_8192=1, terminated=100, faint_tail=100),
    "dense_40k": dict(list_8192=1, terminated=100, faint_tail=100),
    "dense_ties": dict(list_256=1),
    "dense_faint": dict(list_8192=1),
    "aa_needles": dict(),
    "aa_subpixel": dict(),
    "t1_200x120": dict(bg_partial=1), "t1_160x160": dict(), "t1_96x128": dict(),
}
# (scene, variant): the predicates that variant changes.  With antialiasing the dense scenes' 0.01 splats have s ~ 0.1: their
# opacities drop tenfold and almost no pixel terminates.
REACH_VARIANT = {("dense_4k", "aa"): dict(terminated=0, faint_tail=0), ("dense_12k", "aa"): dict(terminated=0, faint_tail=0),
                 ("dense_40k", "aa"): dict(terminated=1, faint_tail=100)}


def predicates(name, variant):
    p = dict(REACH[name])
    p.update(REACH_VARIANT.get((name, variant), {}))
    return p


def assert_reaches(case, variant, o):
    r = reach(case, o)
    need = predicates(case.name, variant)
    short = {k: (r[k], v) for k, v in need.items() if r[k] < v}
    assert not short, (case.name, variant, short, r)
    return r
