"""Scenes that put the per-Gaussian preprocess, forward (preprocess_kernel, gsb_preprocess.cu) and backward
(preprocess_backward_kernel, gsb_backward.cu), on the inputs real models use, and the comparisons that hold it to float64.

Every scene is seen by `general_camera`: fx != fy (independent FoVx and FoVy), a rotation about all three axes, a centre off
the axes and an odd, non-square image.  With synth.make_camera (R = I, fx == fy) a swapped focal_x / focal_y, a swapped W / H or
a transposed view-matrix index gives the same numbers as the right code.

Shared by test_preprocess_edges_oracle.py (CPU: every scene reaches what it is built for, and the comparisons reject planted
near-misses made with the oracle's own gradients) and test_gpu_preprocess_edges.py (the CUDA kernels against the oracle and
against the float64 chain below).

`restate_chain` is the third reference.  It does not go through gs_oracle.cpp.  It is torch float64 autograd of restate64, per
Gaussian: the SH colour, the 3D covariance, screen_cov with the 0.3 dilation and the conic, and the NDC position.  It is
contracted with screen-space gradients (dL_dconic, dL_dmeans2D, dL_dcolors under the clamp mask) handed in by the caller.  The
GPU test hands in the kernel's own, so the render backward's error drops out of the comparison.  It encodes the reference's
conventions: dL_dscales is d/d(mod * s) (no factor of mod), the frustum clamp holds t constant (restate64.screen_cov), the conic
chain carries 1 / (det^2 + 1e-7) instead of 1 / det^2, and the SH-sparsity term is sign(v) lambda / (45 n_vis) with sign(0) = 0
and n_vis = #(radii > 0), on the active coefficients k >= 1 only."""
import math

import numpy as np
import torch

import backward_edges as BE
import gs_oracle
import restate64 as R64
from gs_b200 import synth

F64 = torch.float64
CASES = ["sh3", "mixed_unsorted", "sh2_in_16", "mod", "precomp", "quant", "raw"]
W_GEN, H_GEN = 333, 197
FOVY_DEG = 57.0
FX_OVER_FY = 1.08                    # fx = 1.08 fy: FoVx follows from it, not from FoVy and the aspect ratio
CAM_ANGLES = (19.0, -34.0, 23.0)     # camera-to-world rotation about x, then y, then z (degrees)
CAM_TARGET = np.array([0.7, -0.4, 0.9])
CAM_DIST = 4.0
MOD = 0.7
LAMBDA = 300.0                       # SH sparsity: lambda / (45 n_vis) is a few % of a typical dL_dsh row (assert_reaches)
# reference 3, per element: |ours - chain| <= max(R3 * |chain|_row, A3 * max|chain|) (see test_gpu_preprocess_edges.py)
R3, A3 = 1e-5, 1e-6
# the SH direction term of dL_dmeans3D on its own: |ours - chain| <= DIR_ULP ulp of the total + DIR_REL * |term|_row
DIR_ULP, DIR_REL = 2.0, 1e-5
SH_ARRAYS = ["dL_dsh", "dL_dmeans3D", "dL_dcov3D", "dL_dscales", "dL_drotations"]


def _rot(axis, deg):
    c, s = math.cos(math.radians(deg)), math.sin(math.radians(deg))
    return {"x": np.array([[1, 0, 0], [0, c, -s], [0, s, c]]), "y": np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]]),
            "z": np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])}[axis]


def general_camera(W=W_GEN, H=H_GEN):
    """A COLMAP-like pinhole camera: fx = 1.08 fy, rotated about x, y and z, centred off the axes.  Its matrices are built by
    synth's restatement of the reference's camera code (_world2view2, _projection), so they round as the reference's do."""
    fovy = math.radians(FOVY_DEG)
    fy = H / (2.0 * math.tan(0.5 * fovy))
    fovx = 2.0 * math.atan(W / (2.0 * FX_OVER_FY * fy))
    Rc2w = _rot("z", CAM_ANGLES[2]) @ _rot("y", CAM_ANGLES[1]) @ _rot("x", CAM_ANGLES[0])
    C = CAM_TARGET - CAM_DIST * Rc2w[:, 2]                 # the camera looks along its z axis at CAM_TARGET
    T = -Rc2w.T @ C
    znear, zfar = 0.01, 100.0
    wvt = torch.tensor(synth._world2view2(Rc2w, T)).transpose(0, 1).contiguous()
    proj = synth._projection(znear, zfar, fovx, fovy).transpose(0, 1)
    full = (wvt.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0).contiguous()
    center = wvt.inverse()[3, :3].contiguous()
    return synth.Camera(W, H, fovx, fovy, znear, zfar, wvt, full, center)


def focal(cam):
    """(fx, fy) as the kernels form them."""
    return cam.image_width / (2.0 * math.tan(cam.FoVx * 0.5)), cam.image_height / (2.0 * math.tan(cam.FoVy * 0.5))


def _case(name, scene, cam, g_seed, lam, mod=1.0, **meta):
    c = BE.Case(name, scene, cam, torch.tensor([0.3, 0.15, 0.45]), synth.grad_image(cam.image_width, cam.image_height, g_seed),
                lam=lam, **meta)
    c.mod = mod
    return c


def _inside(g, n, W, H):
    """n Gaussians over the image and 10 px around it: (px, py, depth, sigma, aniso, logits)."""
    u = torch.rand(n, 5, generator=g, dtype=F64).numpy()
    px, py = -10 + (W + 20) * u[:, 0], -10 + (H + 20) * u[:, 1]
    depth = 1.2 + 2.8 * u[:, 2]
    sigma = 1.5 + 8.5 * u[:, 3]
    aniso = 0.4 + 1.2 * torch.rand(n, 3, generator=g, dtype=F64).numpy()
    logits = 2.0 * torch.randn(n, generator=g, dtype=F64).numpy()
    return px, py, depth, sigma, aniso, logits


def _sh3_scene(cam, g):
    """P = 32 * 40 + 13 Gaussians of degree 3 (the last warp holds 13): strong rest coefficients (0.6 N(0,1)), DC channels of a
    sixth of them at -3 (clamped at 0), 6 % of the rest coefficients exactly 0; 24 centred beyond 1.3 tan(fovx / 2) only and 24
    beyond 1.3 tan(fovy / 2) only, wide enough to reach into the image."""
    W, H = cam.image_width, cam.image_height
    No = 24
    Ni = 32 * 40 + 13 - 2 * No
    px, py, depth, sigma, aniso, logits = _inside(g, Ni, W, H)
    v = torch.rand(2 * No, 5, generator=g, dtype=F64).numpy()
    side = np.arange(No) % 2
    ox = np.where(side == 0, -0.15 * W - 25 - 50 * v[:No, 0], 1.15 * W + 25 + 50 * v[:No, 0])
    oy = 0.15 * H + 0.7 * H * v[:No, 1]
    yx = 0.15 * W + 0.7 * W * v[No:, 0]
    yy = np.where(side == 0, -0.15 * H - 15 - 30 * v[No:, 1], 1.15 * H + 15 + 30 * v[No:, 1])
    px, py = np.concatenate([px, ox, yx]), np.concatenate([py, oy, yy])
    depth = np.concatenate([depth, 2.0 + 2.0 * v[:, 2]])
    sigma = np.concatenate([sigma, 60.0 + 30.0 * v[:, 3]])
    P = px.size
    aniso = np.concatenate([aniso, 0.7 + 0.6 * v[:, 4:5] * np.ones((1, 3))])
    logits = np.concatenate([logits, -1.0 + 2.0 * v[:, 4]])
    sh = torch.randn(P, 16, 3, generator=g).numpy()
    sh[:, 1:] *= 0.6
    u = torch.rand(P, 16, 3, generator=g).numpy()
    sh[:, 0][u[:, 0] < 1.0 / 6.0] = -3.0
    sh[:, 1:][u[:, 1:] < 0.06] = 0.0
    scene = BE.pixel_scene(cam, px, py, depth, sigma, logits, sh, g, aniso)
    return scene, dict(out_x=np.arange(Ni, Ni + No), out_y=np.arange(Ni + No, P))


def _warp_mixed_degrees(n, degs, g):
    """Degrees `degs` cycled and shuffled within every warp of 32: each warp (the partial last one too) holds all of them."""
    d = np.zeros(n, np.int32)
    for w0 in range(0, n, 32):
        k = min(32, n - w0)
        d[w0:w0 + k] = np.asarray(degs)[np.arange(k) % len(degs)][torch.randperm(k, generator=g).numpy()]
    return d


def _mixed_scene(cam, g, P, degs, junk):
    """P Gaussians over the image with M = 16 and degrees `degs` mixed in every warp; the inactive coefficients hold non-zero
    junk (`junk`) or zeros."""
    W, H = cam.image_width, cam.image_height
    px, py, depth, sigma, aniso, logits = _inside(g, P, W, H)
    sh = torch.randn(P, 16, 3, generator=g).numpy()
    sh[:, 1:] *= 0.6
    deg = _warp_mixed_degrees(P, degs, g)
    inactive = np.arange(16)[None, :] >= ((deg + 1) ** 2)[:, None]
    if junk:
        j = torch.randn(P, 16, 3, generator=g).numpy()
        sh[inactive] = (np.sign(j) * (0.2 + np.abs(j)))[inactive]
    else:
        sh[inactive] = 0.0
    scene = BE.pixel_scene(cam, px, py, depth, sigma, logits, sh, g, aniso)
    scene.degrees = torch.from_numpy(deg).view(P, 1)
    return scene


def build(name):
    cam = general_camera()
    if name in ("sh3", "mod", "precomp", "raw"):
        g = torch.Generator().manual_seed(9100)
        scene, meta = _sh3_scene(cam, g)
        if name == "sh3":
            return _case(name, scene, cam, 9101, LAMBDA, **meta)
        if name == "mod":
            return _case(name, scene, cam, 9101, LAMBDA, mod=MOD, **meta)
        if name == "precomp":
            cov = R64.cov3D_from(scene.scales.double(), scene.rotations.double()).float().contiguous()
            col = torch.rand(scene.P, 3, generator=torch.Generator().manual_seed(9102))
            return _case(name, scene, cam, 9101, 0.0, precomp=(cov, col), **meta)
        # the model's leaf parameters: log-scales and rotations of norm 0.5 .. 1.7; the oracle sees their activations
        u = 0.5 + 1.2 * torch.rand(scene.P, 1, generator=torch.Generator().manual_seed(9103))
        raw = (scene.sh[:, :1].contiguous(), scene.sh[:, 1:].contiguous(), torch.log(scene.scales), (scene.rotations * u).contiguous())
        case = _case(name, scene, cam, 9101, LAMBDA, raw=raw, **meta)
        activate_raw(case)
        return case
    if name in ("mixed_unsorted", "quant"):
        g = torch.Generator().manual_seed(9200)
        scene = _mixed_scene(cam, g, 32 * 30 + 13, (0, 1, 2, 3), junk=True)
        if name == "mixed_unsorted":
            return _case(name, scene, cam, 9201, LAMBDA)
        q = synth.quantise_scene(scene)
        return _case(name, q.dequantise(), cam, 9201, LAMBDA, quant=q)
    if name == "sh2_in_16":
        g = torch.Generator().manual_seed(9300)
        return _case(name, _mixed_scene(cam, g, 32 * 25 + 13, (0, 1, 2), junk=False), cam, 9301, LAMBDA)
    raise ValueError(name)


def activate_raw(case, dev="cpu"):
    """The raw case's activated scene, exp(scaling) and F.normalize(rotation), computed on `dev` (the GPU test: on the device, where
    the kernels' activations are bit-identical to torch's)."""
    dc, rest, ls, rot = case.meta["raw"]
    s = case.scene
    case.scene = synth.Scene(s.means3D, s.opacity, torch.exp(ls.to(dev)).cpu(), torch.nn.functional.normalize(rot.to(dev)).cpu(),
                             torch.cat([dc, rest], 1).contiguous(), s.degrees)


# ---- the oracle's side -------------------------------------------------------------------------------------------------------

def oracle(case, dL=None):
    """-> (forward state, fp64 backward, fp32 backward) of the oracle on the case's (activated) scene, with its scale_modifier,
    precomputed inputs and lambda; for the raw case the scale and rotation gradients are chained to the leaf parameters in
    float64 (chain_raw)."""
    s = case.scene
    kw = case.cam_kw()
    pre = case.meta.get("precomp")
    if pre is not None:
        o = gs_oracle.forward(s.means3D, s.opacity, None, None, None, None, colors_precomp=pre[1], cov3D_precomp=pre[0], bg=case.bg,
                              scale_modifier=case.mod, **kw)
        args = (s.means3D, None, None, None, None)
    else:
        o = gs_oracle.forward(s.means3D, s.opacity, s.scales, s.rotations, s.sh, s.degrees, bg=case.bg, scale_modifier=case.mod, **kw)
        args = (s.means3D, s.scales, s.rotations, s.sh, s.degrees)
    bkw = dict(bg=case.bg, lambda_sh_sparsity=case.lam, scale_modifier=case.mod, **kw)
    dL = case.dL if dL is None else dL
    o64 = gs_oracle.backward(o, dL, *args, f64=True, **bkw)
    o32 = gs_oracle.backward(o, dL, *args, f64=False, **bkw)
    if "raw" in case.meta:
        o64, o32 = chain_raw(case, o64), chain_raw(case, o32)
    return o, o64, o32


def chain_raw(case, g):
    """The activated scene's dL_dscales / dL_drotations chained to the leaf log-scales and rotations in float64:
    d/dlog s = s d/ds, d/dq = (I - n n^T) / |q| d/dn with n = q / |q|."""
    _, _, ls, rot = case.meta["raw"]
    s = np.exp(ls.double().numpy())
    q = rot.double().numpy()
    nq = np.linalg.norm(q, axis=1, keepdims=True)
    n = q / nq
    gn = np.asarray(g["dL_drotations"], np.float64)
    out = dict(g)
    out["dL_dscales"] = np.asarray(g["dL_dscales"], np.float64) * s
    out["dL_drotations"] = (gn - n * (n * gn).sum(1, keepdims=True)) / nq
    return out


# ---- the third reference: float64 autograd of restate64 ------------------------------------------------------------------------

def _flip_dx(term, x, y, z):
    """A zero-valued correction whose derivative is -2 d term / dx at fixed (y, z): added to the colour it negates that one term's
    contribution to dRx (a planted near-miss)."""
    xd, yd, zd = x.detach(), y.detach(), z.detach()
    return -2.0 * (term(x, yd, zd) - term(xd, yd, zd))


def sh_colour(sh, deg, d, flip_dRx=False):
    """restate64.sh_colour; `flip_dRx` negates the x-derivative of the degree-3 term of coefficient 10 (C31 x y z)."""
    col = R64.sh_colour(sh, deg, d)
    if flip_dRx:
        x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
        w = (deg.view(-1, 1) > 2) * R64.SH_C3[1] * sh[:, 10]
        col = col + _flip_dx(lambda x, y, z: w * x * y * z, x, y, z)
    return col


def restate_chain(case, vis, clamped, g_m2, g_con, g_col, swap_focal=False, transpose_view=False, flip_dRx=False,
                  drop_sparsity=False):
    """Per-Gaussian float64 gradients of the preprocess inputs from screen-space gradients: g_m2 [P,2+] (dL_dmeans2D, w.r.t. the NDC
    position), g_con [P,4] (dL_dconic of want_conic), g_col [P,3] (dL_dcolors; the `clamped` [P,3] channels carry none) on the
    Gaussians of `vis`.  -> dict of numpy [P, ...] arrays named as the backward's outputs (the raw case: dL_dscales / dL_drotations
    of the leaf log-scales / rotations, dL_dsh of cat(features_dc, features_rest)).  The keyword flags plant near-misses: fx and fy
    swapped, the view matrix's rotation block transposed, one dRx term negated, the sparsity term dropped."""
    s = case.scene
    P = s.P
    idx = torch.from_numpy(np.nonzero(np.asarray(vis))[0])
    t = lambda a: torch.as_tensor(np.asarray(a.detach().cpu() if torch.is_tensor(a) else a), dtype=F64)[idx]
    kw = case.cam_kw()
    tanx, tany = kw["tan_fovx"], kw["tan_fovy"]
    view = kw["viewmatrix"].to(F64).clone()
    if transpose_view:
        view[:3, :3] = view[:3, :3].t().clone()
    proj, campos = kw["projmatrix"].to(F64), kw["campos"].to(F64)
    means = t(s.means3D).requires_grad_()
    pre, raw = case.meta.get("precomp"), case.meta.get("raw")
    leaves = {"dL_dmeans3D": means}
    if pre is not None:
        cov = t(pre[0]).requires_grad_()
    else:
        if raw is not None:
            ls, q_raw = t(raw[2]).requires_grad_(), t(raw[3]).requires_grad_()
            s_eff = case.mod * torch.exp(ls)
            q = q_raw / q_raw.norm(dim=1, keepdim=True)
            leaves.update(dL_dscales=ls, dL_drotations=q_raw)
        else:
            s_eff = (case.mod * t(s.scales)).requires_grad_()
            q = t(s.rotations).requires_grad_()
            leaves.update(dL_dscales=s_eff, dL_drotations=q)
        cov = R64.cov3D_from(s_eff, q)
        cov.retain_grad()
    W, H = case.W, case.H
    if swap_focal:
        W, H = case.H * tanx / tany, case.W * tany / tanx         # fx' = fy, fy' = fx; the clamp keeps tan_fovx / tan_fovy
    mh, tz, a, b, c = R64.screen_cov(means, view, cov, W, H, tanx, tany)
    a, c = a + 0.3, c + 0.3
    det = a * c - b * b
    k = (det * det / (det * det + 1e-7)).detach()                # the kernels' 1 / (det^2 + 1e-7)
    gc = t(g_con)
    loss = k * (gc[:, 0] * (c / det) + 2.0 * gc[:, 1] * (-b / det) + gc[:, 3] * (a / det))
    hom = mh @ proj
    m_w = 1.0 / (hom[:, 3] + 1e-7)
    gm = t(g_m2)
    loss = loss + gm[:, 0] * hom[:, 0] * m_w + gm[:, 1] * hom[:, 1] * m_w
    sh = None
    if pre is None:
        sh = t(s.sh).requires_grad_()
        deg = t(s.degrees.view(-1)).long()
        d = means - campos
        d = d / d.norm(dim=1, keepdim=True)
        col = sh_colour(sh, deg, d, flip_dRx)
        loss = loss + (t(g_col) * col * (1.0 - t(clamped))).sum(1)
    loss.sum().backward()
    res = {n: v.grad for n, v in leaves.items()}
    res["dL_dcov3D"] = cov.grad
    if sh is not None:
        g = sh.grad.clone()
        if case.lam != 0.0 and not drop_sparsity:
            active = torch.arange(sh.shape[1])[None, :] < ((deg + 1) ** 2)[:, None]
            active[:, 0] = False
            g = g + (case.lam / (45.0 * idx.numel())) * torch.sign(sh.detach()) * active[:, :, None]
        res["dL_dsh"] = g
    out = {}
    for n, v in res.items():
        full = np.zeros((P,) + tuple(v.shape[1:]), np.float64)
        full[idx.numpy()] = v.detach().numpy()
        out[n] = full
    return out


def sh_direction_term(case, vis, clamped, g_col):
    """The SH colour's share of dL_dmeans3D alone (through the view direction), float64 [P,3], from dL_dcolors `g_col`."""
    if case.meta.get("precomp") is not None:
        return np.zeros((case.scene.P, 3))
    s = case.scene
    idx = np.nonzero(np.asarray(vis))[0]
    t = lambda a: torch.as_tensor(np.asarray(a.detach().cpu() if torch.is_tensor(a) else a), dtype=F64)[idx]
    means = t(s.means3D).requires_grad_()
    d = means - case.cam.camera_center.to(F64)
    d = d / d.norm(dim=1, keepdim=True)
    col = R64.sh_colour(t(s.sh), t(s.degrees.view(-1)).long(), d)
    (t(g_col) * col * (1.0 - t(clamped))).sum().backward()
    out = np.zeros((s.P, 3))
    out[idx] = means.grad.numpy()
    return out


def compare_restated(name, vis, ref, got, arrays=SH_ARRAYS, bar=(R3, A3), verbose=True):
    """|got - ref| <= max(R * |ref|_row, A * max|ref|) per element on the visible Gaussians; culled ones must carry exactly zero.
    -> (ratios {array: max e / bar}, failures [(array, what, rows)])."""
    vis = np.asarray(vis)
    P = vis.shape[0]
    r_rel, a_abs = bar
    ratios, failures = {}, []
    for n in arrays:
        if n not in ref or got.get(n) is None:
            continue
        a = np.asarray(ref[n], np.float64).reshape(P, -1)
        b = np.asarray(got[n], np.float64).reshape(P, -1)
        if a.size == 0:
            continue
        scale = float(np.abs(a).max())
        e = np.abs(b - a)
        bar_ = np.maximum(r_rel * np.abs(a).max(axis=1, keepdims=True), a_abs * scale)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = np.where(bar_ > 0, e / bar_, np.where(e > 0, np.inf, 0.0))
        ratios[n] = float(q[vis].max()) if vis.any() else 0.0
        bad = vis[:, None] & (e > bar_)
        if bad.any():
            failures.append((n, "per-element (restated chain)", np.unique(np.nonzero(bad)[0])))
        if (b[~vis] != 0).any():
            failures.append((n, "culled Gaussians must carry exactly zero", np.unique(np.nonzero((b != 0) & ~vis[:, None])[0])))
    if verbose:
        print("\n[%s] restated chain: max e / max(%.0e |ref|_row, %.0e max|ref|): %s" % (
            name, r_rel, a_abs, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    return ratios, failures


# ---- what each scene is built to reach ----------------------------------------------------------------------------------------

def clamp_sides(case, o):
    """(visible Gaussians beyond 1.3 tan(fovx / 2) only, beyond 1.3 tan(fovy / 2) only), in fp32 as the preprocess computes t."""
    v = case.cam.world_view_transform.numpy().astype(np.float32).reshape(-1)
    m = case.scene.means3D.numpy().astype(np.float32)
    tx = v[0] * m[:, 0] + v[4] * m[:, 1] + v[8] * m[:, 2] + v[12]
    ty = v[1] * m[:, 0] + v[5] * m[:, 1] + v[9] * m[:, 2] + v[13]
    tz = v[2] * m[:, 0] + v[6] * m[:, 1] + v[10] * m[:, 2] + v[14]
    kw = case.cam_kw()
    bx = np.abs(tx / tz) > np.float32(1.3) * np.float32(kw["tan_fovx"])
    by = np.abs(ty / tz) > np.float32(1.3) * np.float32(kw["tan_fovy"])
    vis = o["radii"] > 0
    return vis & bx & ~by, vis & by & ~bx


# the SH direction term is >= 10 % of dL_dmeans3D's row for this many Gaussians (observed with the oracle: 366, 270, 366, 145)
MIN_DIR_SHARE, MIN_DIR_COUNT = 0.1, {"sh3": 300, "mod": 200, "raw": 300, "mixed_unsorted": 120}


def assert_reaches(case, o, o64=None):
    """What the case is built for, from the oracle's forward state (and, given o64, its gradients), so that a change to synth or
    to the scenes cannot quietly drop coverage."""
    cam, s = case.cam, case.scene
    vis = o["radii"] > 0
    P = s.P
    fx, fy = focal(cam)
    assert 1.05 <= fx / fy <= 1.10, fx / fy
    V = cam.world_view_transform.numpy()[:3, :3]
    assert np.abs(V[~np.eye(3, dtype=bool)]).min() >= 0.2, V
    assert np.abs(cam.camera_center.numpy()).min() >= 0.3, cam.camera_center
    assert case.W % 2 == 1 and case.H % 2 == 1 and case.W != case.H
    assert vis.sum() >= 0.6 * P, (int(vis.sum()), P)
    deg = s.degrees.view(-1).numpy()
    pre = case.meta.get("precomp")
    if pre is None:
        assert s.sh.shape[1] == 16
    if case.name in ("sh3", "mod", "precomp", "raw"):
        assert P % 32 == 13 and (deg == 3).all()
        bx, by = clamp_sides(case, o)
        assert bx.sum() >= 8 and by.sum() >= 8, (int(bx.sum()), int(by.sum()))
        assert np.array_equal(np.nonzero(bx)[0], np.intersect1d(np.nonzero(bx)[0], case.meta["out_x"]))
        assert np.array_equal(np.nonzero(by)[0], np.intersect1d(np.nonzero(by)[0], case.meta["out_y"]))
    if case.name in ("sh3", "mod", "raw"):
        assert o["clamped"][vis].any(axis=1).sum() >= 50, "colour channels clamped at 0"
        assert (s.sh.numpy()[vis][:, 1:] == 0).sum() >= 100, "active coefficients exactly 0"
    if case.name == "mod":
        assert case.mod != 1.0
    if case.name == "precomp":
        assert pre[0].shape == (P, 6) and pre[1].shape == (P, 3)
    if case.name == "raw":
        n = case.meta["raw"][3].norm(dim=1)
        assert float((n - 1).abs().min()) < 0.2 and float(n.min()) < 0.6 and float(n.max()) > 1.5
    if case.name in ("mixed_unsorted", "quant", "sh2_in_16"):
        degs = (0, 1, 2) if case.name == "sh2_in_16" else (0, 1, 2, 3)
        assert P % 32 != 0
        for w0 in range(0, P, 32):
            assert set(deg[w0:w0 + 32].tolist()) == set(degs), "every warp mixes the degrees"
    if case.name == "mixed_unsorted":
        inactive = np.arange(16)[None, :] >= ((deg + 1) ** 2)[:, None]
        assert (s.sh.numpy()[inactive] != 0).all(), "junk in every inactive band"
    if case.name == "quant":
        q = case.meta["quant"]
        inactive = np.arange(1, 16)[None, :] >= ((deg + 1) ** 2)[:, None]
        assert (q.ids_rest.numpy()[inactive] != 0).mean() > 0.9, "the inactive bands' ids point at non-zero centres"
    if o64 is None or pre is not None:
        return
    # the SH direction term is a visible share of dL_dmeans3D, and the sparsity term of a dL_dsh row
    term = sh_direction_term(case, vis, o["clamped"], o64["dL_dcolors"])
    tot = np.abs(np.asarray(o64["dL_dmeans3D"], np.float64)).max(axis=1)
    share = np.abs(term).max(axis=1) / np.maximum(tot, 1e-30)
    if case.name in MIN_DIR_COUNT:
        assert (vis & (share >= MIN_DIR_SHARE)).sum() >= MIN_DIR_COUNT[case.name], int((vis & (share >= MIN_DIR_SHARE)).sum())
    if case.lam:
        mult = case.lam / (45.0 * vis.sum())
        rows = np.abs(np.asarray(o64["dL_dsh"], np.float64)[vis]).reshape(int(vis.sum()), -1).max(axis=1)
        assert mult >= 0.01 * np.median(rows), (mult, float(np.median(rows)))
