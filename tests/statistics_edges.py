"""The SH-culling statistics on the rasterizer's boundary scenes, and their per-Gaussian comparison with the oracle.

Shared by test_statistics_edges_oracle.py (CPU: every case reaches what it is built for, and the comparison rejects near-misses
made with the oracle itself that the older whole-array rule accepts) and test_gpu_statistics_edges.py (the CUDA statistics
forward and calculate_colours_variance against the oracle, Gaussian by Gaussian).

Two kernels produce the statistics: the statistics forward (render_forward_kernel<STATS = true>, also in fixed point), which
counts for each Gaussian the pixels it contributes to (`touched_pixels`) and sums the transmittance in front of it there
(`transmittance_sum`), and sh_stats_update_kernel, which turns them into calculate_colours_variance's distances, variance and
mean once per camera.

The statistics forward, per Gaussian, against the oracle's renderCUDA restatement (int32 counts, fp64 sums):
  - Gaussians without a pair near a threshold or next to a termination at a borderline pixel (backward_edges.borderline_pairs):
    `touched_pixels` exact and |tsum - o64| <= R_REL * o64 + A_ABS, plus FLIP = 1/254 for each borderline pixel where the
    Gaussian passes behind a pair near alpha 1/255: that pair may flip in the GPU's exponential, and a flip scales T from there on
    by 1 / (1 - 1/255).  On one H100 the 600 px Gaussian 20013 of `large` does flip at one pixel (alpha 1/255 within 2e-9), and
    the two Gaussians composited behind it there, of 215 and 351 pixels, then differ by 2.4e-5 and 1.3e-5 of their sums;
  - the others: |d touched| at most the number of borderline pixels where their pair passes the alpha test (a flipped decision
    moves one count by 1 there) and |d tsum| at most that number (T <= 1) plus the tight bar's rounding; their share of the
    visible Gaussians is bounded per case (NEAR_MAX);
  - culled Gaussians: exactly zero.
calculate_colours_variance on three cameras against gs_oracle.colours_variance (fp32, the reference's order): the NaN pattern
exact; rows of Gaussians neither near a borderline decision nor behind one in any camera within VAR_R_REL * max|row| +
VAR_A_ABS, the others within VAR_LOOSE of the array's scale."""
import math

import numpy as np
import torch

import backward_edges as BE
import cases
import gs_oracle
import ours

CASES = BE.CASES + ["t1"]
R_REL, A_ABS = 1e-5, 1e-6
FLIP = 1.0 / 254.0
# the largest share of a case's Gaussians near or behind a borderline decision (observed: 1.5e-3 of `large` in the forward,
# 2.2e-3 of its variance case over three cameras; none elsewhere)
NEAR_MAX = 0.005

VAR_CASES = ["staircase", "odd_17x15", "large", "saturation", "dense_12k", "t1"]
VAR_NAMES = ["distance", "variance", "mean"]
VAR_R_REL, VAR_A_ABS = 2e-5, 1e-7
VAR_LOOSE = 1e-3
YAW = 2.0                                    # the two extra cameras of a variance case, degrees about y
GROUP_SIZE = 24                              # Gaussians per appended group


def build(name):
    """The statistics case `name`: a backward_edges case, or `t1` on its first camera (its three cameras in meta["cams"])."""
    if name != "t1":
        return BE.build(name)
    _, scene, cams, _ = cases.build_tools_inputs("t1")
    return BE.Case("t1", scene, cams[0], torch.zeros(3), None, cams=cams)


def oracle(scene, cam, bg):
    """The oracle's statistics forward of `scene` on `cam`: preprocess, binning and render state with touched_pixels and
    transmittance_sum."""
    W, H = cam.image_width, cam.image_height
    o = _preprocess(scene, cam)
    o.update(gs_oracle.bin_and_sort(o, W, H))
    o.update(gs_oracle.render_forward_stats(o, o, bg, W, H))
    return o


def _preprocess(scene, cam):
    return gs_oracle.preprocess(scene.means3D, scene.scales, 1.0, scene.rotations, scene.opacity, scene.sh, scene.degrees, None, None,
                                cam.world_view_transform, cam.full_proj_transform, cam.camera_center, cam.image_width,
                                cam.image_height, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5))


def compare(name, o, pairs, touched, tsum, verbose=True):
    """The per-Gaussian check of a statistics forward (`touched`, `tsum` [P] or [P,1]) against the oracle's `o`; `pairs` = (near,
    count, behind) of backward_edges.borderline_pairs -> (ratios, failures).  ratios: `touched` the largest |d touched| of a tight
    Gaussian, `tsum` the largest |d tsum| / bar of one, `near` the largest |d touched| / count and |d tsum| / bar of the others."""
    near, count, behind = pairs
    vis = o["radii"] > 0
    t_o, s_o = o["touched_pixels"].astype(np.int64), o["transmittance_sum"]
    t_g, s_g = np.asarray(touched).reshape(-1).astype(np.int64), np.asarray(tsum, np.float64).reshape(-1)
    dt, ds = np.abs(t_g - t_o), np.abs(s_g - s_o)
    chk, loose = vis & ~near, vis & near
    rounding = R_REL * s_o + A_ABS
    q = ds / (rounding + behind * FLIP)
    qn = ds / (rounding + count)
    failures = []

    def fail(what, bad):
        if bad.any():
            failures.append((what, np.nonzero(bad)[0]))
    fail("touched_pixels exact", chk & (dt != 0))
    fail("transmittance_sum within %g o64 + %g (+ 1/254 per borderline pixel behind a flip)" % (R_REL, A_ABS), chk & ~(q <= 1.0))
    fail("touched_pixels within the borderline pixels' count", loose & (dt > count))
    fail("transmittance_sum within the borderline pixels' count + %g o64 + %g" % (R_REL, A_ABS), loose & ~(qn <= 1.0))
    fail("culled Gaussians carry exact zeros", ~vis & ((t_g != 0) | (s_g != 0)))
    with np.errstate(divide="ignore", invalid="ignore"):
        mx = lambda a, m: float(a[m].max()) if m.any() else 0.0
        ratios = dict(touched=mx(dt, chk), tsum=mx(q, chk),
                      near=(mx(np.where(count > 0, dt / count, np.where(dt > 0, np.inf, 0.0)), loose), mx(qn, loose)))
    if verbose:
        print("\n[%s] %d of %d visible Gaussians tight (%d behind a pair near a threshold): max |d touched| %d, max |d tsum| / bar "
              "%.3g; %d near a borderline decision: max |d touched| / count %.3g, |d tsum| / bar %.3g" % (
                  name, int(chk.sum()), int(vis.sum()), int((chk & (behind > 0)).sum()), ratios["touched"], ratios["tsum"],
                  int(loose.sum()), *ratios["near"]))
    return ratios, failures


def old_rule_ok(o, touched, tsum):
    """The whole-array rule the per-Gaussian check replaces: counts may differ on 4 Gaussians per borderline pixel, sums within
    1e-5 of the array's scale (1e-3 once any pixel is borderline)."""
    t_o, t_g = o["touched_pixels"], np.asarray(touched).reshape(-1)
    nb = int(o["borderline"].sum())
    if (nb == 0 and not np.array_equal(t_o, t_g)) or (t_o != t_g).sum() > 4 * nb:
        return False
    a, b = np.asarray(tsum, np.float64).reshape(-1), o["transmittance_sum"].astype(np.float32).astype(np.float64)
    return bool(np.abs(a - b).max() / (np.abs(b).max() + 1e-30) <= (1e-5 if nb == 0 else 1e-3))


def describe(failures, o, touched, tsum, limit=5):
    t_g, s_g = np.asarray(touched).reshape(-1), np.asarray(tsum).reshape(-1)
    lines = []
    for what, ids in failures:
        lines.append("%s: %d Gaussians" % (what, ids.size))
        for g in ids[:limit]:
            lines.append("  id %d: oracle %d %.9g, ours %d %.9g" % (g, o["touched_pixels"][g], o["transmittance_sum"][g], t_g[g], s_g[g]))
    return "\n".join(lines)


# ---- calculate_colours_variance on three cameras -------------------------------------------------------------------------------

class VarianceCase:
    def __init__(self, name, scene, cams, groups):
        self.name, self.scene, self.cams, self.groups = name, scene, cams, groups

    def cam_tensors(self):
        ct = cases.tools_camera_tensors(self.cams)
        return [ct[k] for k in ("positions", "views", "projs", "tanx", "tany", "H", "W")]


def variance_case(name):
    """The geometry of case `name` with random 16-coefficient SH (degrees cycling 0, 1, 2, 3) on three cameras: the case's and two
    copies yawed by +-YAW degrees (t1: its own W > H, W = H and W < H cameras), plus three appended groups of GROUP_SIZE:
      faint:   in view, opacity 1/300: present, but no pair reaches alpha 1/255 (wSum stays 0: NaN distance and variance, mean 0);
      outside: behind, too near or far beside every camera: radius 0 everywhere (NaN rows);
      one:     visible (radius > 0) in exactly one camera, picked from candidates around the views with the oracle's preprocess."""
    base = build(name)
    cam, W, H = base.cam, base.W, base.H
    cams = base.meta.get("cams") or [cam, ours.yaw_cam(W, H, -YAW, dev="cpu"), ours.yaw_cam(W, H, YAW, dev="cpu")]
    g = torch.Generator().manual_seed(9000 + CASES.index(name))
    n = GROUP_SIZE
    u = torch.rand(n, 4, generator=g, dtype=torch.float64).numpy()
    faint = BE.pixel_scene(cam, W * (0.3 + 0.4 * u[:, 0]), H * (0.3 + 0.4 * u[:, 1]), 3.0 + 3.0 * u[:, 2], 1.0 + 2.0 * u[:, 3],
                           np.full(n, BE._logit(1.0 / 300.0)), np.zeros((n, 1, 3)), g)
    side = np.arange(n) % 3                   # behind the camera, closer than the near plane, far to the side
    depth = np.where(side == 0, -3.0, np.where(side == 1, 0.1, 4.0))
    outside = BE.pixel_scene(cam, np.where(side == 2, -20.0 * W, W * u[:, 0]), H * u[:, 1], depth, 2.0 * np.ones(n), np.full(n, 2.0),
                             np.zeros((n, 1, 3)), g)
    m = 4000
    v = torch.rand(m, 4, generator=g, dtype=torch.float64).numpy()
    cand = BE.pixel_scene(cam, W * (-1.0 + 3.0 * v[:, 0]), H * v[:, 1], 3.0 + 3.0 * v[:, 2], 0.7 + 1.5 * v[:, 3], np.full(m, 1.0),
                          np.zeros((m, 1, 3)), g)
    seen = np.stack([_preprocess(cand, c)["radii"] > 0 for c in cams], 1)
    pick = np.nonzero(seen.sum(1) == 1)[0]
    # as many of each camera as there are, round robin
    by_cam = [pick[seen[pick, i]] for i in range(len(cams))]
    order = [ids[k] for k in range(max(len(b) for b in by_cam)) for ids in by_cam if k < len(ids)]
    one = torch.as_tensor(order[:n], dtype=torch.int64)
    parts = [base.scene, faint, outside, BE.synth.Scene(*[t[one] for t in (cand.means3D, cand.opacity, cand.scales, cand.rotations,
                                                                            cand.sh, cand.degrees)])]
    P0, P = base.scene.P, sum(s.P for s in parts)
    cat = lambda k: torch.cat([getattr(s, k) for s in parts]).contiguous()
    sh = torch.randn(P, 16, 3, generator=g)
    sh[:, 1:] *= 0.3
    degrees = (torch.arange(P, dtype=torch.int32) % 4).view(P, 1)
    scene = BE.synth.Scene(cat("means3D"), cat("opacity"), cat("scales"), cat("rotations"), sh.contiguous(), degrees)
    idx = np.arange(P)
    return VarianceCase(name, scene, cams, dict(faint=idx[P0:P0 + n], outside=idx[P0 + n:P0 + 2 * n], one=idx[P0 + 2 * n:]))


def variance_args(vc):
    """The positional arguments of calculate_colours_variance (and gs_oracle.colours_variance) for the case, on the CPU."""
    pos, views, projs, tx, ty, H, W = vc.cam_tensors()
    s = vc.scene
    return (pos, s.means3D, s.opacity, s.scales, s.rotations, views, projs, tx, ty, H, W, s.sh, s.degrees, 3)


def variance_oracle(vc, alias_mean=True):
    """-> ((distance, variance, mean), per-camera states, loose): gs_oracle.colours_variance on the case's cameras; `loose` marks
    the Gaussians near or behind a borderline decision in some camera (backward_edges.borderline_pairs)."""
    d, v, m, per = gs_oracle.colours_variance(*variance_args(vc), alias_mean=alias_mean)
    loose = np.zeros(vc.scene.P, bool)
    for st, c in zip(per, vc.cams):
        near, _, behind = BE.borderline_pairs(st, c.image_width, c.image_height)
        loose |= near | (behind > 0)
    return (d, v, m), per, loose


def compare_variance(name, ref, got, loose, verbose=True):
    """calculate_colours_variance's (distance, variance, mean) `got` against the oracle's `ref` -> (ratios, failures): the NaN
    pattern exact; a row (a Gaussian's elements of one array) within VAR_R_REL * max|row| + VAR_A_ABS unless `loose`, those within
    VAR_LOOSE of the array's scale.  ratios[array] = (largest e / bar on the tight rows, largest e / scale on the loose ones)."""
    ratios, failures = {}, []
    for n, a, b in zip(VAR_NAMES, ref, got):
        P = loose.shape[0]
        a, b = np.asarray(a, np.float64).reshape(P, -1), np.asarray(b, np.float64).reshape(P, -1)
        na, nb = np.isnan(a), np.isnan(b)
        if not np.array_equal(na, nb):
            failures.append((n, "NaN pattern", np.nonzero((na != nb).any(1))[0]))
        ok = ~na & ~nb
        a0, b0 = np.where(ok, a, 0.0), np.where(ok, b, 0.0)
        e = np.abs(b0 - a0)
        scale = float(np.abs(a0).max())
        bar = VAR_R_REL * np.abs(a0).max(axis=1, keepdims=True) + VAR_A_ABS
        q = e / bar
        tight = ~loose
        ratios[n] = (float(q[tight].max()) if tight.any() else 0.0, float(e[loose].max()) / scale if loose.any() and scale > 0 else 0.0)
        bad = tight[:, None] & (e > bar)
        if bad.any():
            failures.append((n, "%g of max|row| + %g" % (VAR_R_REL, VAR_A_ABS), np.unique(np.nonzero(bad)[0])))
        bad = loose[:, None] & (e > VAR_LOOSE * scale)
        if bad.any():
            failures.append((n, "%g of scale (rows near a borderline decision)" % VAR_LOOSE, np.unique(np.nonzero(bad)[0])))
    if verbose:
        print("\n[%s, colours variance] %d of %d Gaussians tight; max e / bar, max e / scale (loose): %s" % (
            name, int((~loose).sum()), loose.size, ", ".join("%s %.3g %.3g" % (k, *v) for k, v in ratios.items())))
    return ratios, failures


def old_variance_rule_ok(ref, got):
    """test_gpu_tools' rule for the colour-variance outputs: the NaN pattern, then 2e-5 of the array's scale."""
    for a, b in zip(ref, got):
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        if not np.array_equal(np.isnan(a), np.isnan(b)):
            return False
        m = ~np.isnan(a)
        if m.any() and np.abs(a[m] - b[m]).max() / (np.abs(a[m]).max() + 1e-30) > 2e-5:
            return False
    return True
