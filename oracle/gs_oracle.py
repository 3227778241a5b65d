"""ctypes front-end of the CPU oracle (oracle/gs_oracle.cpp) — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` legs may import
this module.  It restates, stage by stage, the reference pipeline
(diff-gaussian-rasterization/cuda_rasterizer/rasterizer_impl.cu:359-504 forward, :508-630 backward) and
returns every intermediate as a numpy array so parity tests can compare them one by one.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "gs_oracle.cpp")
LIB = os.path.join(HERE, "libgs_oracle.so")
_lib = None

f32p = C.POINTER(C.c_float)
f64p = C.POINTER(C.c_double)
i32p = C.POINTER(C.c_int32)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
u8p = C.POINTER(C.c_uint8)


def build(force: bool = False) -> str:
    if force or not os.path.isfile(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
               "-fvisibility=hidden", "-o", LIB, SRC]
        subprocess.run(cmd, check=True)
    return LIB


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.gso_inclusive_sum.restype = C.c_uint32
        _lib.gso_higher_msb.restype = C.c_uint32
        _lib.gso_num_threads.restype = C.c_int
    return _lib


def _p(a, t):
    if a is None:
        return C.cast(None, t)
    assert a.flags["C_CONTIGUOUS"], "oracle wants contiguous arrays"
    return a.ctypes.data_as(t)


def _np(x, dtype=None):
    if x is None:
        return None
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    x = np.ascontiguousarray(x)
    if dtype is not None and x.dtype != dtype:
        x = x.astype(dtype)
    return x


def num_threads() -> int:
    return int(lib().gso_num_threads())


def higher_msb(n: int) -> int:
    return int(lib().gso_higher_msb(C.c_uint32(n)))


def mark_visible(means3D, viewmatrix):
    means3D, viewmatrix = _np(means3D, np.float32), _np(viewmatrix, np.float32)
    P = means3D.shape[0]
    out = np.zeros(P, np.uint8)
    lib().gso_mark_visible(P, _p(means3D, f32p), _p(viewmatrix, f32p), _p(out, u8p))
    return out.astype(bool)


def preprocess(means3D, scales, scale_modifier, rotations, opacities, shs, degrees, cov3D_precomp, colors_precomp,
               viewmatrix, projmatrix, campos, W, H, tan_fovx, tan_fovy, packed=None, antialiasing=False):
    """forward.cu:354-456 (or :246-350 with packed=(coeffs_num, per_band_count, cumsum)).  `antialiasing`: conic_opacity[:, 3] is
    o^ = sigmoid * s (the product's gsb_preprocess.cu, DESIGN.md §5e), and aa_sigmoid / aa_s / aa_q [P] hold sigmoid, s and q."""
    means3D = _np(means3D, np.float32)
    P = means3D.shape[0]
    scales, rotations = _np(scales, np.float32), _np(rotations, np.float32)
    opacities = _np(opacities, np.float32)
    shs = _np(shs, np.float32)
    degrees = _np(degrees, np.int32)
    cov3D_precomp, colors_precomp = _np(cov3D_precomp, np.float32), _np(colors_precomp, np.float32)
    viewmatrix, projmatrix, campos = _np(viewmatrix, np.float32), _np(projmatrix, np.float32), _np(campos, np.float32)
    M = 0
    if shs is not None and packed is None:
        M = shs.shape[1]
    out = dict(radii=np.zeros(P, np.int32), means2D=np.zeros((P, 2), np.float32), depths=np.zeros(P, np.float32),
               cov3D=np.zeros((P, 6), np.float32), rgb=np.zeros((P, 3), np.float32),
               conic_opacity=np.zeros((P, 4), np.float32), tiles_touched=np.zeros(P, np.uint32),
               clamped=np.zeros((P, 3), np.uint8))
    if antialiasing:
        out.update(aa_sigmoid=np.zeros(P, np.float32), aa_s=np.zeros(P, np.float32), aa_q=np.zeros(P, np.float32))
    aa = lambda k: _p(out.get(k), f32p)
    if packed is not None:
        cn, pbc, cs = [_np(a, np.int32) for a in packed]
    else:
        cn = pbc = cs = None
    lib().gso_preprocess(P, M, _p(means3D, f32p), _p(scales, f32p), C.c_float(scale_modifier), _p(rotations, f32p),
                         _p(opacities, f32p), _p(shs, f32p), _p(degrees, i32p), _p(cov3D_precomp, f32p),
                         _p(colors_precomp, f32p), _p(viewmatrix, f32p), _p(projmatrix, f32p), _p(campos, f32p),
                         W, H, C.c_float(tan_fovx), C.c_float(tan_fovy),
                         0 if packed is None else 1, _p(cn, i32p), _p(pbc, i32p), _p(cs, i32p),
                         _p(out["radii"], i32p), _p(out["means2D"], f32p), _p(out["depths"], f32p), _p(out["cov3D"], f32p),
                         _p(out["rgb"], f32p), _p(out["conic_opacity"], f32p), _p(out["tiles_touched"], u32p),
                         _p(out["clamped"], u8p), 1 if antialiasing else 0, aa("aa_sigmoid"), aa("aa_s"), aa("aa_q"))
    if colors_precomp is not None:
        out["rgb"] = colors_precomp
    if cov3D_precomp is not None:
        out["cov3D"] = cov3D_precomp
    return out


def bin_and_sort(geom, W, H):
    """rasterizer_impl.cu:441-482: scan, duplicateWithKeys, SortPairs, identifyTileRanges."""
    L = lib()
    P = geom["radii"].shape[0]
    offsets = np.zeros(P, np.uint32)
    R = int(L.gso_inclusive_sum(P, _p(geom["tiles_touched"], u32p), _p(offsets, u32p))) if P > 0 else 0
    keys_u = np.zeros(R, np.uint64)
    vals_u = np.zeros(R, np.uint32)
    L.gso_duplicate_with_keys(P, _p(geom["means2D"], f32p), _p(geom["depths"], f32p), _p(offsets, u32p),
                              _p(geom["radii"], i32p), W, H, _p(keys_u, u64p), _p(vals_u, u32p))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    bit = higher_msb(gx * gy)
    keys = np.zeros(R, np.uint64)
    vals = np.zeros(R, np.uint32)
    L.gso_sort_pairs(C.c_int64(R), _p(keys_u, u64p), _p(vals_u, u32p), _p(keys, u64p), _p(vals, u32p), 32 + bit)
    ranges = np.zeros((gx * gy, 2), np.uint32)
    L.gso_identify_tile_ranges(C.c_int64(R), _p(keys, u64p), gx * gy, _p(ranges, u32p))
    return dict(point_offsets=offsets, num_rendered=R, keys_unsorted=keys_u, point_list_unsorted=vals_u,
                keys=keys, point_list=vals, ranges=ranges, sort_bits=32 + bit)


def render_forward(geom, binning, bg, W, H, f64=False):
    bg = _np(bg, np.float32)
    colors = _np(geom["rgb"], np.float32)
    if f64:
        out = np.zeros((3, H, W), np.float64)
        final_T = np.zeros((H, W), np.float64)
        lib().gso_render_forward_f64(W, H, _p(binning["ranges"], u32p), _p(binning["point_list"], u32p),
                                     _p(geom["means2D"], f32p), _p(colors, f32p), _p(geom["conic_opacity"], f32p),
                                     _p(bg, f32p), _p(out, f64p), _p(final_T, f64p))
        return dict(color64=out, final_T64=final_T)
    final_T = np.zeros((H, W), np.float32)
    n_contrib = np.zeros((H, W), np.uint32)
    color = np.zeros((3, H, W), np.float32)
    borderline = np.zeros((H, W), np.uint8)
    lib().gso_render_forward(W, H, _p(binning["ranges"], u32p), _p(binning["point_list"], u32p),
                             _p(geom["means2D"], f32p), _p(colors, f32p), _p(geom["conic_opacity"], f32p), _p(bg, f32p),
                             _p(final_T, f32p), _p(n_contrib, u32p), _p(color, f32p), _p(borderline, u8p))
    return dict(final_T=final_T, n_contrib=n_contrib, color=color, borderline=borderline.astype(bool))


def render_forward_stats(geom, binning, bg, W, H):
    """renderCUDA with calculate_mean_transmittance (forward.cu:560-564): render_forward() + touched_pixels int32 [P] and
    transmittance_sum float64 [P] (the reference accumulates in fp32 with atomics in arbitrary order)."""
    bg = _np(bg, np.float32)
    colors = _np(geom["rgb"], np.float32)
    P = colors.shape[0]
    final_T = np.zeros((H, W), np.float32)
    n_contrib = np.zeros((H, W), np.uint32)
    color = np.zeros((3, H, W), np.float32)
    borderline = np.zeros((H, W), np.uint8)
    touched = np.zeros(P, np.int32)
    tsum = np.zeros(P, np.float64)
    lib().gso_render_forward_stats(W, H, _p(binning["ranges"], u32p), _p(binning["point_list"], u32p),
                                   _p(geom["means2D"], f32p), _p(colors, f32p), _p(geom["conic_opacity"], f32p), _p(bg, f32p),
                                   _p(final_T, f32p), _p(n_contrib, u32p), _p(color, f32p), _p(borderline, u8p),
                                   _p(touched, i32p), _p(tsum, f64p))
    return dict(final_T=final_T, n_contrib=n_contrib, color=color, borderline=borderline.astype(bool),
                touched_pixels=touched, transmittance_sum=tsum)


def sh_colours(means3D, campos, shs, degrees):
    """reduced_3dgs/sh_culling.cu:6-57: colours [P,4,3]; slot k of a Gaussian is written only for k <= its degree (else 0)."""
    means3D, shs = _np(means3D, np.float32), _np(shs, np.float32)
    degrees = _np(degrees, np.int32).reshape(-1)
    campos = _np(campos, np.float32).reshape(3)
    P, M = shs.shape[0], shs.shape[1]
    out = np.zeros((P, 4, 3), np.float32)
    lib().gso_sh_colours(P, M, _p(degrees, i32p), _p(means3D, f32p), _p(campos, f32p), _p(shs, f32p), _p(out, f32p))
    return out


def colours_variance(cam_positions, means3D, opacity, scales, rotations, viewmatrices, projmatrices, tan_fovxs, tan_fovys,
                     image_height, image_width, sh, degrees, max_sh_deg=3, alias_mean=True):
    """Reduced3DGS::calculateColourVariance (reduced_3dgs.cu:41-203) restated with numpy fp32 in the reference's op order.
    Returns (colour distances / wSum [P,3], variance / wSum [P,1,3], mean [P,1,3]) plus, per camera, the statistics and the
    whole forward state (preprocess, binning, render) for tests.  `alias_mean=False` takes the pre-update mean in one factor of
    the variance term: what reduced_3dgs.cu:185-200 reads as, not what it computes (a near-miss for tests)."""
    assert max_sh_deg == 3
    means3D = _np(means3D, np.float32)
    P = means3D.shape[0]
    sh = _np(sh, np.float32)
    degrees = _np(degrees, np.int32).reshape(-1)
    f = np.float32
    wsum, wsumsq = np.zeros((P, 1), f), np.zeros((P, 1), f)
    dist_acc = np.zeros((P, 3), f)
    mean, variance = np.zeros((P, 1, 3), f), np.zeros((P, 1, 3), f)
    per_cam = []
    with np.errstate(invalid="ignore", divide="ignore"):
        for i in range(len(cam_positions)):
            H, W = int(image_height[i]), int(image_width[i])
            campos = _np(cam_positions[i], np.float32)
            geom = preprocess(means3D, scales, 1.0, rotations, opacity, sh, degrees, None, None, _np(viewmatrices[i], np.float32),
                              _np(projmatrices[i], np.float32), campos, W, H, float(tan_fovxs[i]), float(tan_fovys[i]), None)
            binning = bin_and_sort(geom, W, H)
            img = render_forward_stats(geom, binning, np.zeros(3, np.float32), W, H)
            present = geom["radii"] > 0
            touched = img["touched_pixels"]
            t = (img["transmittance_sum"] / np.maximum(touched, 1)).astype(f).reshape(P, 1)          # :154
            wsum = wsum + t                                                                       # :155
            wsumsq = wsumsq + t * t
            colours = sh_colours(means3D, campos, sh, degrees)                                    # :158-164
            colours[~present] = 0                                                                 # :165
            for d in range(3):                                                                    # :167-181
                diff = colours[:, 3:4] - colours[:, d:d + 1]
                dist = np.sqrt((diff * diff).sum(axis=2, dtype=f)).astype(f)
                dist[np.isnan(dist)] = 0
                dist_acc[:, d:d + 1] = dist_acc[:, d:d + 1] + t * dist
            colour = colours[:, 3:4]                                                              # :184
            mean_old = mean.copy()                   # value before the update (the reference's `mean_old` ALIASES `mean`, :185)
            coef = t / wsum
            coef[np.isnan(coef)] = 0
            mean[present] = mean_old[present] + coef[present].reshape(-1, 1, 1) * (colour[present] - mean_old[present])
            # `auto mean_old = mean;` shares storage: after the in-place index_put_ both factors use the NEW mean (:196-200)
            second = mean if alias_mean else mean_old
            variance[present] = variance[present] + t[present].reshape(-1, 1, 1) * (colour[present] - mean[present]) * (colour[present] - second[present])
            per_cam.append(dict(geom, **binning, **img))
        return dist_acc / wsum, variance / wsum.reshape(-1, 1, 1), mean, per_cam


def min_projected_pixel_size(w2ndc, w2ndc_inv, means3D, image_height, image_width):
    """Reduced3DGS::calculatePixelSize (reduced_3dgs.cu:246-268) -> float32 [P,1]."""
    means3D = _np(means3D, np.float32)
    P = means3D.shape[0]
    out = np.full((P, 1), 10000, np.float32)
    for i in range(len(w2ndc)):
        lib().gso_pixel_size_camera(P, _p(means3D, f32p), _p(_np(w2ndc[i], np.float32), f32p), _p(_np(w2ndc_inv[i], np.float32), f32p),
                                    int(image_height[i]), int(image_width[i]), _p(out, f32p))
    return out


def sphere_ellipsoid_intersection(means3D, scales, rotations, neighbours, sphere_radius, knn, dots=False):
    """Reduced3DGS::intersectionTest (reduced_3dgs.cu:205-243) -> (redundancy int32 [P,1], mask bool [P,knn], borderline bool [P]),
    and with dots=True also each pair's `dot` (float32 [P,knn]): a hit is dot < 1."""
    means3D, scales, rotations = _np(means3D, np.float32), _np(scales, np.float32), _np(rotations, np.float32)
    neighbours, sphere_radius = _np(neighbours, np.int32), _np(sphere_radius, np.float32).reshape(-1)
    P = means3D.shape[0]
    red, mask, bl = np.zeros((P, 1), np.int32), np.zeros((P, knn), np.uint8), np.zeros(P, np.uint8)
    dot = np.zeros((P, knn), np.float32) if dots else None
    lib().gso_sphere_ellipsoid(P, _p(means3D, f32p), _p(scales, f32p), _p(rotations, f32p), _p(neighbours, i32p), _p(sphere_radius, f32p),
                               int(knn), _p(red, i32p), _p(mask, u8p), _p(bl, u8p), _p(dot, f32p))
    return (red, mask.astype(bool), bl.astype(bool)) + ((dot,) if dots else ())


def min_redundancy_value(redundancy_values, neighbours, intersection_mask, knn):
    """Reduced3DGS::assignFinalRedundancyValue (reduced_3dgs.cu:270-287) -> int32 [P,1]."""
    red = _np(redundancy_values, np.int32).reshape(-1)
    nb, mask = _np(neighbours, np.int32), _np(intersection_mask).astype(np.uint8)
    P = red.shape[0]
    out = np.full((P, 1), P, np.int32)
    lib().gso_min_redundancy(P, _p(red, i32p), _p(nb, i32p), _p(mask, u8p), int(knn), _p(out, i32p))
    return out


def kmeans_update_ids(values, centers):
    """reduced_3dgs/kmeans.cu:70-107 updateIdsCUDA: argmin_i sqrt((c_i - v)^2) in fp32, first index on ties."""
    v = _np(values, np.float32).reshape(-1)
    c = _np(centers, np.float32).reshape(-1)
    ids = np.empty(v.shape[0], np.int32)
    for a in range(0, v.shape[0], 1 << 16):
        d = c[None, :] - v[a:a + (1 << 16), None]
        d = np.sqrt(d * d)
        d = np.where(np.isnan(d), np.float32(np.inf), d)      # `dist < min_dist` is false for NaN
        ids[a:a + (1 << 16)] = np.argmin(d, axis=1)
    return ids


def kmeans(values, centers, tol, max_iterations):
    """Reduced3DGS::kmeans (reduced_3dgs.cu:289-338).  The cluster sums are taken in double (the reference adds floats with
    atomics in arbitrary order).  Returns (ids int32 [n,1], centers float32 [k], iterations)."""
    v = _np(values, np.float32).reshape(-1)
    new = _np(centers, np.float32).reshape(-1).copy()
    K = new.shape[0]
    it = 0
    with np.errstate(invalid="ignore", divide="ignore"):
        for it in range(1, max_iterations + 1):
            ids = kmeans_update_ids(v, new)
            old = new.copy()
            sums = np.bincount(ids, weights=v.astype(np.float64), minlength=K).astype(np.float32)
            sizes = np.bincount(ids, minlength=K).astype(np.float32)
            new = (sums / sizes).astype(np.float32)
            new[np.isnan(new)] = 0
            if np.abs(old - new).sum(dtype=np.float32) < tol:
                break
    return kmeans_update_ids(v, new).reshape(-1, 1), new, it


def _ssim_window():
    """gaussian(11, 1.5) of utils/loss_utils.py:23-25 in float32, as float64 array."""
    import math
    g = np.array([math.exp(-(x - 5) ** 2 / (2 * 1.5 ** 2)) for x in range(11)], np.float32)
    return (g / g.sum(dtype=np.float32)).astype(np.float64)


def _sepconv(a, w):
    """zero-padded 'same' separable correlation of [C,H,W] with the 11-tap window along H and W (== conv2d(padding=5, groups=C))."""
    C, H, W = a.shape
    p = np.zeros((C, H + 10, W + 10), np.float64)
    p[:, 5:5 + H, 5:5 + W] = a
    t = sum(w[k] * p[:, :, k:k + W] for k in range(11))
    return sum(w[k] * t[:, k:k + H, :] for k in range(11))


def l1_ssim(image, gt, lambda_dssim=0.2):
    """utils/loss_utils.py:17-18 l1_loss, :33-65 ssim / _ssim and their combination of train.py:110-115, in float64, with the
    analytic gradient of the combined loss w.r.t. `image`.  Returns (l1, ssim, loss, dloss_dimage)."""
    x, y = _np(image, np.float64), _np(gt, np.float64)
    w = _ssim_window()
    N = x.size
    mu1, mu2 = _sepconv(x, w), _sepconv(y, w)
    exx, eyy, exy = _sepconv(x * x, w), _sepconv(y * y, w), _sepconv(x * y, w)
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    A1, A2 = 2 * mu1 * mu2 + C1, 2 * (exy - mu1 * mu2) + C2
    B1, B2 = mu1 ** 2 + mu2 ** 2 + C1, (exx - mu1 ** 2) + (eyy - mu2 ** 2) + C2
    smap = A1 * A2 / (B1 * B2)
    l1, ssim = np.abs(x - y).mean(), smap.mean()
    d_mu = 2 * mu2 * (A2 - A1) / (B1 * B2) - smap * 2 * mu1 * (B2 - B1) / (B1 * B2)
    d_xx = -smap / B2
    d_xy = 2 * A1 / (B1 * B2)
    dssim = (_sepconv(d_mu, w) + 2 * x * _sepconv(d_xx, w) + y * _sepconv(d_xy, w)) / N
    grad = (1 - lambda_dssim) * np.sign(x - y) / N - lambda_dssim * dssim
    return l1, ssim, (1 - lambda_dssim) * l1 + lambda_dssim * (1 - ssim), grad


def forward(means3D, opacities, scales=None, rotations=None, shs=None, degrees=None, colors_precomp=None,
            cov3D_precomp=None, *, viewmatrix, projmatrix, campos, bg, W, H, tan_fovx, tan_fovy, scale_modifier=1.0,
            packed=None, prune_mask=None, antialiasing=False):
    """Whole reference forward (rasterizer_impl.cu:359-504).  `prune_mask` (1 = pruned) is applied with the
    reference-equivalent semantics of SURVEY §8(b): run on the compacted set, scatter per-Gaussian outputs
    back to the original indices."""
    means3D = _np(means3D, np.float32)
    P = means3D.shape[0]
    if prune_mask is not None:
        keep = ~_np(prune_mask).astype(bool)
        idx = np.nonzero(keep)[0]
        sub = lambda a: None if a is None else np.ascontiguousarray(_np(a)[keep])
        out = forward(sub(means3D), sub(opacities), sub(scales), sub(rotations), sub(shs), sub(degrees), sub(colors_precomp),
                      sub(cov3D_precomp), viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos, bg=bg, W=W, H=H,
                      tan_fovx=tan_fovx, tan_fovy=tan_fovy, scale_modifier=scale_modifier, antialiasing=antialiasing)
        full = {}
        for k in ("radii", "means2D", "depths", "cov3D", "rgb", "conic_opacity", "tiles_touched", "clamped", "aa_sigmoid", "aa_s", "aa_q"):
            if k not in out:
                continue
            a = out[k]
            z = np.zeros((P,) + a.shape[1:], a.dtype)
            z[idx] = a
            full[k] = z
        full["point_list"] = idx[out["point_list"]].astype(np.uint32)
        full["point_list_unsorted"] = idx[out["point_list_unsorted"]].astype(np.uint32)
        for k in ("num_rendered", "keys", "keys_unsorted", "ranges", "final_T", "n_contrib", "color", "borderline", "sort_bits"):
            full[k] = out[k]
        full["point_offsets"] = np.cumsum(full["tiles_touched"], dtype=np.uint64).astype(np.uint32)
        return full
    bgn = _np(bg, np.float32)
    if P == 0:
        # rasterize_points.cu:184-185: P == 0 returns the zero-initialised image (no background)
        return dict(num_rendered=0, color=np.zeros((3, H, W), np.float32), radii=np.zeros(0, np.int32))
    geom = preprocess(means3D, scales, scale_modifier, rotations, opacities, shs, degrees, cov3D_precomp, colors_precomp,
                      viewmatrix, projmatrix, campos, W, H, tan_fovx, tan_fovy, packed, antialiasing)
    binning = bin_and_sort(geom, W, H)
    img = render_forward(geom, binning, bgn, W, H)
    out = {}
    out.update(geom)
    out.update(binning)
    out.update(img)
    return out


def backward(fwd, dL_dpix, means3D, scales, rotations, shs, degrees, *, viewmatrix, projmatrix, campos, bg, W, H,
             tan_fovx, tan_fovy, scale_modifier=1.0, lambda_sh_sparsity=0.0, f64=False, colors_precomp=None,
             cov3D_precomp=None, antialiasing=False):
    """Whole reference backward (rasterizer_impl.cu:508-630) from the forward state `fwd`.
    Returns the 8 gradients of rasterize_points.cu:304 (+ dL_dconic).  `antialiasing` needs a forward with antialiasing=True: the
    backward differentiates o^ = sigmoid * s at that forward's fp32 sigmoid, s and q (DESIGN.md §5e)."""
    L = lib()
    means3D = _np(means3D, np.float32)
    P = means3D.shape[0]
    scales, rotations = _np(scales, np.float32), _np(rotations, np.float32)
    shs, degrees = _np(shs, np.float32), _np(degrees, np.int32)
    viewmatrix, projmatrix, campos = _np(viewmatrix, np.float32), _np(projmatrix, np.float32), _np(campos, np.float32)
    bg = _np(bg, np.float32)
    dL_dpix = _np(dL_dpix, np.float32)
    M = shs.shape[1] if shs is not None else 0
    rt = np.float64 if f64 else np.float32
    rp = f64p if f64 else f32p
    g = dict(dL_dmeans2D=np.zeros((P, 3), rt), dL_dconic=np.zeros((P, 4), rt), dL_dopacity=np.zeros((P, 1), rt),
             dL_dcolors=np.zeros((P, 3), rt), dL_dmeans3D=np.zeros((P, 3), rt), dL_dcov3D=np.zeros((P, 6), rt),
             dL_dsh=np.zeros((P, M, 3), rt), dL_dscales=np.zeros((P, 3), rt), dL_drotations=np.zeros((P, 4), rt))
    colors = _np(fwd["rgb"], np.float32)
    cov3D = _np(fwd["cov3D"], np.float32)
    rb = L.gso_render_backward_f64 if f64 else L.gso_render_backward
    rb(W, H, _p(fwd["ranges"], u32p), _p(fwd["point_list"], u32p), _p(bg, f32p), _p(fwd["means2D"], f32p),
       _p(fwd["conic_opacity"], f32p), _p(colors, f32p), _p(fwd["final_T"], f32p), _p(fwd["n_contrib"], u32p),
       _p(dL_dpix, f32p), P, _p(g["dL_dmeans2D"], rp), _p(g["dL_dconic"], rp), _p(g["dL_dopacity"], rp), _p(g["dL_dcolors"], rp))
    mult = 0.0
    if lambda_sh_sparsity != 0.0:
        n_vis = int((fwd["radii"] > 0).sum())                                  # rasterizer_impl.cu:549-571
        mult = float(np.float32(lambda_sh_sparsity) / np.float32(n_vis * 15 * 3))
    pb = L.gso_preprocess_backward_f64 if f64 else L.gso_preprocess_backward
    pb(P, M, _p(means3D, f32p), _p(fwd["radii"], i32p), _p(shs, f32p), _p(degrees, i32p), _p(fwd["clamped"], u8p),
       _p(scales, f32p), _p(rotations, f32p), C.c_float(scale_modifier), _p(cov3D, f32p), _p(viewmatrix, f32p),
       _p(projmatrix, f32p), W, H, C.c_float(tan_fovx), C.c_float(tan_fovy), _p(campos, f32p),
       _p(g["dL_dmeans2D"], rp), _p(fwd["conic_opacity"], f32p), _p(g["dL_dconic"], rp), _p(g["dL_dopacity"], rp),
       _p(g["dL_dcolors"], rp), _p(g["dL_dmeans3D"], rp), _p(g["dL_dcov3D"], rp), _p(g["dL_dsh"], rp),
       _p(g["dL_dscales"], rp), _p(g["dL_drotations"], rp), C.c_float(mult),
       *[_p(fwd[k] if antialiasing else None, f32p) for k in ("aa_sigmoid", "aa_s", "aa_q")])
    return g


def psnr(img1, img2) -> float:
    """utils/image_utils.py:17-19: 20*log10(1/sqrt(mse)) over all channels."""
    mse = float(np.mean((np.asarray(img1, np.float64) - np.asarray(img2, np.float64)) ** 2))
    return float("inf") if mse == 0 else 20.0 * np.log10(1.0 / np.sqrt(mse))
