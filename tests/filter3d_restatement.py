"""Restatements of Mip-Splatting's 3D smoothing filter (DESIGN.md §5o), shared by test_filter3d_api.py (CPU) and
test_gpu_filter3d.py: compute_3D_filter in float64 and as Mip-Splatting's per-camera torch loop in fp32, the filtered scales and
opacity factor, and the camera objects the library's compute_3D_filter reads."""
import math
from types import SimpleNamespace

import numpy as np
import torch

F64 = torch.float64
SQRT_02 = 0.2 ** 0.5


def camera(view, W, H, fovx, fovy):
    """An object with the attributes gs_b200.mip.compute_3D_filter reads; `view` is the transposed 4 x 4 world_view_transform."""
    return SimpleNamespace(world_view_transform=view, image_width=W, image_height=H, FoVx=fovx, FoVy=fovy)


def focals(cam):
    """(fx, fy) in double, Mip-Splatting's fov2focal."""
    return cam.image_width / (2.0 * math.tan(cam.FoVx / 2.0)), cam.image_height / (2.0 * math.tan(cam.FoVy / 2.0))


def _view_space(xyz, view, dtype):
    v = view.to(dtype)
    return xyz.to(dtype) @ v[:3, :3] + v[3, :3]


def _fma32(a, b, c):
    """fl32(a * b + c) for fp32 tensors (the product is exact in float64; the sum is rounded twice, which differs from one rounding
    only in rare ties)."""
    return (a.double() * b.double() + c.double()).float()


def view_space_fp32(xyz, view):
    """The rasterizer's xform_row in fp32, row i: fl(fl(fma(z, m[8+i], fma(x, m[i], fl(y m[4+i])))) + m[12+i]) of the transposed
    view matrix: the preprocess's own depth."""
    m = view.to(xyz.device, torch.float32).reshape(-1)
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    rows = []
    for i in range(3):
        t = y * m[4 + i]
        t = _fma32(x, m[i].expand_as(x), t)
        t = _fma32(z, m[8 + i].expand_as(x), t)
        rows.append(t + m[12 + i])
    return torch.stack(rows, 1)


def filter_fp64(xyz, cams):
    """compute_3D_filter in float64 throughout -> (f [P] float64, seen [P] bool, dist [P] float64 with inf where unseen)."""
    P = xyz.shape[0]
    dist = torch.full((P,), math.inf, dtype=F64)
    F = 0.0
    for c in cams:
        fx, fy = focals(c)
        F = max(F, fx)
        t = _view_space(xyz, c.world_view_transform, F64)
        z = t[:, 2]
        zc = z.clamp(min=0.001)
        u = t[:, 0] / zc * fx + c.image_width / 2.0
        v = t[:, 1] / zc * fy + c.image_height / 2.0
        W, H = c.image_width, c.image_height
        ok = (z > 0.2) & (u >= -0.15 * W) & (u <= 1.15 * W) & (v >= -0.15 * H) & (v <= 1.15 * H)
        dist = torch.where(ok, torch.minimum(dist, z), dist)
    seen = torch.isfinite(dist)
    if not bool(seen.any()):
        return torch.zeros(P, dtype=F64), seen, dist
    d = torch.where(seen, dist, dist[seen].max())
    return d / F * SQRT_02, seen, dist


def filter_torch_fp32(xyz, cams):
    """Mip-Splatting's compute_3D_filter loop in torch fp32 on the device of `xyz`: its view transform is the rasterizer's
    (view_space_fp32), the rest are its ops: clamp, divide, multiply-add, the +-15 % screen test, the min, the max over the seen
    rows, distance / focal * sqrt(0.2).  No seen row gives zeros where Mip-Splatting raises.  -> f [P] fp32."""
    dev = xyz.device
    P = xyz.shape[0]
    distance = torch.full((P,), math.inf, device=dev)
    valid_points = torch.zeros(P, dtype=torch.bool, device=dev)
    focal_length = 0.0
    for c in cams:
        t = view_space_fp32(xyz.float(), c.world_view_transform)
        valid_depth = t[:, 2] > 0.2
        x, y, z = t[:, 0], t[:, 1], t[:, 2]
        z = torch.clamp(z, min=0.001)
        fx, fy = focals(c)
        x = x / z * fx + c.image_width / 2.0
        y = y / z * fy + c.image_height / 2.0
        in_screen = torch.logical_and(torch.logical_and(x >= -0.15 * c.image_width, x <= c.image_width * 1.15),
                                      torch.logical_and(y >= -0.15 * c.image_height, y <= 1.15 * c.image_height))
        valid = torch.logical_and(valid_depth, in_screen)
        distance[valid] = torch.min(distance[valid], t[:, 2][valid])
        valid_points = torch.logical_or(valid_points, valid)
        focal_length = max(focal_length, fx)
    if not bool(valid_points.any()):
        return torch.zeros(P, device=dev)
    distance[~valid_points] = distance[valid_points].max()
    return distance / focal_length * SQRT_02


def boundary_ulps(xyz, cams):
    """Per centre, the smallest distance over all cameras from a visibility boundary (z = 0.2 and the four screen bounds), in ulps
    of the compared fp32 quantity, evaluated in float64."""
    P = xyz.shape[0]
    best = torch.full((P,), math.inf, dtype=F64)
    ulp = lambda a: torch.from_numpy(np.spacing(np.abs(a.numpy()).astype(np.float32)).astype(np.float64))  # noqa: E731
    for c in cams:
        fx, fy = focals(c)
        t = _view_space(xyz, c.world_view_transform, F64)
        z = t[:, 2]
        zc = z.clamp(min=0.001)
        u = t[:, 0] / zc * fx + c.image_width / 2.0
        v = t[:, 1] / zc * fy + c.image_height / 2.0
        W, H = c.image_width, c.image_height
        cand = [(z - 0.2).abs() / ulp(z)]
        for val, lo, hi in ((u, -0.15 * W, 1.15 * W), (v, -0.15 * H, 1.15 * H)):
            cand += [(val - lo).abs() / ulp(val), (val - hi).abs() / ulp(val)]
        best = torch.minimum(best, torch.stack(cand).min(0).values)
    return best


def filtered(s, f):
    """torch's get_scaling_with_3D_filter and get_opacity_with_3D_filter factor in fp32: (sqrt(s^2 + f^2), sqrt(det1 / det2)),
    s [P, 3], f [P].  Rows with f == 0 keep s and a factor of 1 (the kernels' zero-filter rule)."""
    s2 = torch.square(s)
    after = s2 + torch.square(f)[:, None]
    det1 = s2[:, 0] * s2[:, 1] * s2[:, 2]
    det2 = after[:, 0] * after[:, 1] * after[:, 2]
    zero = (f == 0)
    return torch.where(zero[:, None], s, torch.sqrt(after)), torch.where(zero, torch.ones_like(f), torch.sqrt(det1 / det2))


def filtered64(s, f):
    """The same in float64 (differentiable): (s', c3)."""
    after = s * s + (f * f)[:, None]
    return torch.sqrt(after), torch.sqrt(torch.prod(s * s, 1) / torch.prod(after, 1))


def c3_of(s, f):
    """c3 in float64 of numpy scales [P, 3] and filter [P]."""
    s = np.asarray(s, np.float64)
    f = np.asarray(f, np.float64)[:, None]
    return np.prod(s / np.sqrt(s * s + f * f), 1)


def filter_for_c3(s, target):
    """Per row the filter f whose c3 equals `target` (bisection in float64 on the monotone c3(f)) -> f [P] float32."""
    s = np.asarray(s, np.float64)
    lo, hi = np.zeros(len(s)), np.full(len(s), 1e4 * max(float(s.max()), 1e-30))
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        big = c3_of(s, mid) > target
        lo, hi = np.where(big, mid, lo), np.where(big, hi, mid)
    return (0.5 * (lo + hi)).astype(np.float32)


EDGE_KINDS = ("zero", "moderate", "strong", "flat", "flat0")


def edge_rows(scene, seed):
    """Adds a filter to `scene` (a synth.Scene, changed in place) with rows of five kinds, by row index:
      zero      f = 0 (the unfiltered arithmetic);
      moderate  f = half the mean scale (c3 ~ 0.3 .. 0.7);
      strong    c3 drawn in [5e-3, 0.05] and the logit raised to 6 (sigmoid 0.9975), so that sigmoid * c3 stays above 1/255 and the
                row composites in the small-c3 regime;
      flat      the smallest axis set to 1e-6, c3 drawn in [0.05, 0.5] (f of the order of 1e-6) and the logit at least 3;
      flat0     the first axis exactly 0: c3 = 0, the row composites nothing and every gradient is 0 (only every 16th such row, so
                the scene keeps its other content).
    -> (f [P] float32 tensor, kind [P] int array of EDGE_KINDS indices)."""
    g = np.random.default_rng(seed)
    s = scene.scales.numpy().astype(np.float64).copy()
    logit = scene.opacity.numpy().reshape(-1).copy()
    P = len(s)
    kind = np.arange(P) % 4
    kind[(np.arange(P) % 64) == 3] = 4
    f = np.zeros(P, np.float32)
    m = kind == 1
    f[m] = (0.5 * s[m].mean(1)).astype(np.float32)
    m = kind == 2
    f[m] = filter_for_c3(s[m], np.exp(g.uniform(np.log(5e-3), np.log(0.05), int(m.sum()))))
    logit[m] = 6.0
    m = kind == 3
    s[m, np.argmin(s[m], 1)] = 1e-6
    f[m] = filter_for_c3(s[m], g.uniform(0.05, 0.5, int(m.sum())))
    logit[m] = np.maximum(logit[m], 3.0)
    m = kind == 4
    s[m, 0] = 0.0
    f[m] = (0.5 * s[m, 1:].mean(1)).astype(np.float32)
    scene.scales = torch.from_numpy(s.astype(np.float32))
    scene.opacity = torch.from_numpy(logit.astype(np.float32)).view(-1, 1)
    return torch.from_numpy(f), kind
