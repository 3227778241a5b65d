"""The contribution statistics (gsb_contributions, DESIGN.md §5p) restated in float64 from the oracle's forward state, and their
per-Gaussian comparison.

Shared by test_contrib_oracle.py (CPU: the cases reach what they are built for, and the comparison rejects near-misses planted in
the restatement) and test_gpu_contrib.py (the CUDA pass against the restatement, Gaussian by Gaussian).

The restatement walks every pixel's tile list of the oracle's fp32 forward state (gs_oracle, the reference's arithmetic): a pair
(p, i) at list position k contributes when k < n_contrib(p), power <= 0 and alpha >= 1/255 (alpha = min(0.99, opacity exp(power)));
T is the float64 product of (1 - alpha) over the contributing pairs in front, and w = alpha T.  With m = the map clamped to [0, 1]
(NaN -> 0) it returns weight_sum = sum m w, weight_max = max w, pixels, top_id (the first maximum in list order, -1 where none),
the gap between each pixel's best and second-best w, and for each Gaussian the number of contributing pairs in front of it at the
pixel of its maximum.  The exponent is rounded as the kernels round it (pair_power), so alpha differs from the kernel's only by the
exponential's few ulp.  It also keeps an fp32 twin of w (alpha and T rounded as the kernel rounds them) for the exact-tie rule.

The comparison, per Gaussian, reuses statistics_edges.compare for the sum and the count (the borderline-pixel machinery of
backward_edges.borderline_pairs): `pixels` exact and `weight_sum` within R_REL o64 + A_ABS (+ 1/254 per borderline pixel behind
a pair near alpha 1/255) on the Gaussians away from borderline decisions, the others within their borderline pixels' count,
culled ones zero.  `weight_max` within (4 + 2 k) ulp of o64 (k: the contributing pairs in front at its maximum, each of which
rounds the kernel's T twice) on the Gaussians away from borderline pixels, within 1/254 (+ that) on those behind one.  `top_id`
equal on every pixel that is not borderline and whose best two weights differ by more than TOP_GAP relative."""
import math

import numpy as np
import torch

import backward_edges as BE
import gs_oracle
import statistics_edges as SE
from gs_b200 import synth

CASES = SE.CASES                            # the 16 + 2 boundary scenes of backward_edges and t1's first camera
TIE = "tie_17x15"
R_REL, A_ABS = SE.R_REL, SE.A_ABS
MAX_ULP = 4
TOP_GAP = 1e-6
F32_099 = float(np.float32(0.99))


def build(name):
    """The case `name`: statistics_edges' cases, or the constructed exact tie."""
    return tie_case() if name == TIE else SE.build(name)


def oracle(case):
    """The oracle's forward state of `case` (preprocess, binning, render; touched_pixels and transmittance_sum included)."""
    return SE.oracle(case.scene, case.cam, case.bg)


def clamp_map(weights):
    """The kernel's read of a pixel-weight map: NaN -> 0, then clamped to [0, 1]."""
    w = np.asarray(weights, np.float64)
    return np.where(np.isnan(w), 0.0, np.clip(w, 0.0, 1.0))


def _fma32(a, b, c):
    """fl32(a b + c) with one rounding (the product of two fp32 values is exact in float64)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def pair_power(A, B, C, dx, dy):
    """The exponent of a pair as the kernels and the reference's contracted SASS round it (gsb_common.cuh pair_power):
    fma(fma(dx, A dx, (C dy) dy), -0.5, -((B dx) dy)).  A plain fp32 restatement differs by an ulp of power, which exp turns into
    |power| ulp of alpha."""
    f = np.float32
    q = _fma32(dx, f(A) * dx, (f(C) * dy) * dy)
    return _fma32(q, f(-0.5), -((f(B) * dx) * dy))


def restate(o, W, H, weights=None, clamp=True, miss=None):
    """-> dict of the four outputs in float64 (see the module doc), from the oracle's state `o`.  `weights` [H, W] or None.
    Near-misses: clamp=False reads the map unclamped; miss="terminating" also counts each pixel's first passing pair behind
    n_contrib, miss="skipped" also takes the maximum over the pairs skipped by the alpha test alone."""
    P = o["radii"].shape[0]
    m = np.ones((H, W)) if weights is None else (clamp_map(weights) if clamp else np.asarray(weights, np.float64))
    ws, wmax, pixels = np.zeros(P), np.zeros(P), np.zeros(P, np.int64)
    front = np.zeros(P, np.int64)
    top, top32 = np.full((H, W), -1, np.int64), np.full((H, W), -1, np.int64)
    gap = np.full((H, W), np.inf)
    gx = (W + 15) // 16
    means, co = o["means2D"].astype(np.float32), o["conic_opacity"].astype(np.float32)
    nc = o["n_contrib"].astype(np.int64)
    for t in range(o["ranges"].shape[0]):
        tx, ty = t % gx, t // gx
        ys, xs = np.mgrid[16 * ty:min(16 * ty + 16, H), 16 * tx:min(16 * tx + 16, W)]
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        r0, r1 = (int(v) for v in o["ranges"][t])
        for c0 in range(0, xs.size, 64):                   # 64 pixels at a time bound the [pixels, list] arrays
            _pixels(o, means, co, nc, r0, r1, xs[c0:c0 + 64], ys[c0:c0 + 64], m, ws, wmax, pixels, front, top, top32, gap, miss)
    return dict(weight_sum=ws, weight_max=wmax, pixels=pixels, top_id=top, top_id32=top32, gap=gap, front=front)


def _pixels(o, means, co, nc, r0, r1, xs, ys, m, ws, wmax, pixels, front, top, top32, gap, miss):
    """restate() on the pixels (xs, ys) of one tile whose list is [r0, r1)."""
    n = nc[ys, xs]
    hi = int(n.max()) if n.size else 0
    if hi == 0:
        return
    if miss == "terminating":
        hi = r1 - r0                                         # the whole list: the terminating pair lies behind n_contrib
    ids = o["point_list"][r0:r0 + hi].astype(np.int64)
    dx = means[ids, 0][None, :] - xs.astype(np.float32)[:, None]
    dy = means[ids, 1][None, :] - ys.astype(np.float32)[:, None]
    c = co[ids]
    power = pair_power(c[:, 0], c[:, 1], c[:, 2], dx, dy).astype(np.float64)
    a = c[:, 3].astype(np.float64) * np.exp(power)
    alpha = np.minimum(F32_099, a)
    ok = (np.arange(hi)[None, :] < n[:, None]) & (power <= 0) & (a >= 1.0 / 255.0)
    ones = np.ones((xs.size, 1))
    T = np.concatenate([ones, np.cumprod(np.where(ok, 1.0 - alpha, 1.0), axis=1)[:, :-1]], axis=1)
    w = np.where(ok, alpha * T, 0.0)
    ws[ids] += (m[ys, xs][:, None] * w).sum(0)
    pixels[ids] += ok.sum(0)
    if miss == "terminating":
        after = (np.arange(hi)[None, :] >= n[:, None]) & (power <= 0) & (a >= 1.0 / 255.0)
        first = after & (np.cumsum(after, axis=1) == 1)
        pixels[ids] += first.sum(0)
    if miss == "skipped":
        skipped = (np.arange(hi)[None, :] < n[:, None]) & (power <= 0) & (a < 1.0 / 255.0)
        w = np.where(skipped, alpha * T, w)
    # the fp32 twin: alpha and T rounded to fp32 as the kernel rounds them, T a sequential fp32 product (the exact-tie rule)
    a32 = np.minimum(np.float32(0.99), c[:, 3][None, :] * np.exp(power).astype(np.float32)).astype(np.float32)
    f32 = np.where(ok, np.float32(1.0) - a32, np.float32(1.0)).astype(np.float32)
    T32 = np.concatenate([ones.astype(np.float32), np.cumprod(f32, axis=1, dtype=np.float32)[:, :-1]], axis=1)
    w32 = np.where(ok, a32 * T32, np.float32(0.0))
    # per Gaussian: the maximum, and the contributing pairs in front of it at the pixel where it is reached
    cols = np.arange(hi)
    at = np.argmax(w, axis=0)
    best = w[at, cols]
    nfront = (np.cumsum(ok, axis=1) - ok)[at, cols]
    upd = best > wmax[ids]
    wmax[ids] = np.where(upd, best, wmax[ids])
    front[ids] = np.where(upd, nfront, front[ids])
    # per pixel: the first maximum in list order, and the relative gap to the second best
    rows = np.arange(xs.size)
    k = np.argmax(w, axis=1)
    bw = w[rows, k]
    top[ys, xs] = np.where(bw > 0, ids[k], -1)
    k32 = np.argmax(w32, axis=1)
    top32[ys, xs] = np.where(w32[rows, k32] > 0, ids[k32], -1)
    if hi > 1:
        second = np.partition(w, hi - 2, axis=1)[:, hi - 2]
        gap[ys, xs] = np.where(bw > 0, (bw - second) / np.maximum(bw, 1e-300), np.inf)


def compare(name, o, c64, pairs, got, tie_pixel=None, verbose=True):
    """The per-Gaussian check of `got` (weight_sum, weight_max, pixels [P], top_id [H, W]) against the restatement `c64` of `o`;
    `pairs` = backward_edges.borderline_pairs(o); `tie_pixel` (x, y): a pixel of an exact fp32 tie, where top_id must follow the
    fp32 twin (the earlier pair) -> (ratios, failures)."""
    ws, wm, px, top = (np.asarray(g) for g in got)
    ws, wm, px = ws.reshape(-1).astype(np.float64), wm.reshape(-1).astype(np.float64), px.reshape(-1).astype(np.int64)
    as_stats = dict(radii=o["radii"], touched_pixels=c64["pixels"], transmittance_sum=c64["weight_sum"])
    ratios, failures = SE.compare(name, as_stats, pairs, px, ws, verbose=False)
    near, _, behind = pairs
    vis = o["radii"] > 0
    ulp = np.spacing(np.float32(np.maximum(c64["weight_max"], 1e-30))).astype(np.float64)
    bar = (MAX_ULP + 2 * c64["front"]) * ulp + np.where(behind > 0, c64["weight_max"] / 254.0, 0.0)
    dm = np.abs(wm - c64["weight_max"])
    chk = vis & ~near
    q = np.where(chk, dm / bar, 0.0)
    if (chk & (dm > bar)).any():
        failures.append(("weight_max within (4 + 2 k) ulp", np.nonzero(chk & (dm > bar))[0]))
    if (~vis & (wm != 0)).any():
        failures.append(("culled Gaussians carry a zero weight_max", np.nonzero(~vis & (wm != 0))[0]))
    sel = ~o["borderline"] & (c64["gap"] > TOP_GAP)
    bad = sel & (top != c64["top_id"])
    if bad.any():
        failures.append(("top_id", np.flatnonzero(bad)))
    if tie_pixel is not None and top[tie_pixel[1], tie_pixel[0]] != c64["top_id32"][tie_pixel[1], tie_pixel[0]]:
        failures.append(("top_id at the exact tie: the earlier pair", np.array([tie_pixel[1] * top.shape[1] + tie_pixel[0]])))
    ratios.update(weight_max=float(q.max()) if q.size else 0.0, top_checked=int(sel.sum()))
    if verbose:
        print("\n[%s] %d visible, %d tight: max |d pixels| %d, |d weight_sum| / bar %.3g, |d weight_max| / bar %.3g; top_id on %d of %d "
              "pixels" % (name, int(vis.sum()), int(chk.sum()), ratios["touched"], ratios["tsum"], ratios["weight_max"], int(sel.sum()),
                          sel.size))
    return ratios, failures


# ---- the constructed exact fp32 tie --------------------------------------------------------------------------------------------

def _on_axis(cam, depths, logits):
    """Gaussians on the optical axis of `cam` (exactly the pixel ((W - 1) / 2, (H - 1) / 2) for odd W, H): power 0 there."""
    n = len(depths)
    z = np.asarray(depths, np.float64) - 4.0                   # synth.make_camera's camera sits at z = -4 looking +z
    means = torch.tensor(np.stack([np.zeros(n), np.zeros(n), z], 1), dtype=torch.float32)
    scales = torch.full((n, 3), 0.01, dtype=torch.float32)
    rots = torch.tensor([[1.0, 0.0, 0.0, 0.0]] * n, dtype=torch.float32)
    sh = torch.zeros(n, 1, 3)
    return synth.Scene(means, torch.tensor(logits, dtype=torch.float32).view(n, 1), scales, rots, sh,
                       torch.zeros(n, 1, dtype=torch.int32))


def tie_case():
    """Two Gaussians on the axis of a 17 x 15 camera, A at depth 2 in front of B at depth 3, whose weights at the centre pixel (8, 7)
    are equal in fp32: fl(o_B fl(1 - o_A)) == o_A, with the opacities as the oracle's preprocess rounds them (found by search).
    The kernel must report A (the earlier in the list) there."""
    cam = synth.make_camera(17, 15)
    la = math.log(0.25 / 0.75)
    target = 0.25 / 0.75
    cand = np.log(target / (1 - target)) + np.linspace(-2e-5, 2e-5, 4001)
    probe = _on_axis(cam, [2.0] + [3.0] * cand.size, [la] + cand.tolist())
    op = SE._preprocess(probe, cam)["conic_opacity"][:, 3].astype(np.float32)
    oa = op[0]
    hit = np.nonzero(op[1:] * (np.float32(1.0) - oa) == oa)[0]
    assert hit.size, "no exact fp32 tie among the candidates"
    lb = float(cand[hit[hit.size // 2]])
    scene = _on_axis(cam, [2.0, 3.0], [la, lb])
    return BE.Case(TIE, scene, cam, torch.zeros(3), None, tie_pixel=(8, 7))
