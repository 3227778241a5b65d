"""Float64 torch restatement of the anti-aliased forward (DESIGN.md §5e), differentiable by autograd: the AA preprocess
(restate64.py) and front-to-back compositing with the reference's skip, saturate and stop rules, and the maps.  Shared by
test_gpu_antialias.py (against the kernels) and test_antialias_edges_oracle.py (against the fp64 oracle); it runs on the device
of its inputs."""
import math

import torch

import restate64 as R64

F64 = torch.float64
H_DIL = 0.3
AA_MIN_RATIO = 2.5e-5


def render64(x, cam, bg, vis, tiles, at=None):
    """float64 AA forward of the visible Gaussians.  x: dict of float64 leaves (means, logit, view, proj, campos, and scales + rots or
    cov3D, sh + deg or colors).  tiles: per 16x16 tile the depth-sorted Gaussian ids to composite.  `at` (optional): the fp32
    forward's own sigmoid, s and q [P] (float64 tensors); the effective opacity then takes those values, with the derivatives
    sigmoid (1 - sigmoid) and dq / (2 s) at them and none through q where q <= 2.5e-5, which is the point an fp32 backward
    differentiates at; with at["cov3D"] the 3D covariance takes the forward's values too (its derivatives stay float64), and with
    at["means2D"] [P,2], at["conic_opacity"] [P,4], at["rgb"] [P,3] and at["final_T"] [H,W] so do the screen positions (each pair's
    offset from its pixel then rounded to fp32, as the forward forms it), conic, o^, colours and every pixel's transmittance (T scaled
    by final_T / T_final, a constant).  -> (colour, invdepth, alpha, n_contrib, intermediates, margins)."""
    pin = lambda v, k: v if at is None or k not in at else v + (at[k] - v).detach()
    dev = x["means"].device
    W, H = cam.image_width, cam.image_height
    m = x["means"]
    cov = x["cov3D"] if "cov3D" in x else R64.cov3D_from(x["scales"], x["rots"])
    if at is not None and "cov3D" in at:
        cov = cov + (at["cov3D"] - cov).detach()
    mh, tz, a, b, c = R64.screen_cov(m, x["view"], cov, W, H, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5))
    det0 = a * c - b * b
    A, C = a + H_DIL, c + H_DIL
    det1 = A * C - b * b
    con = torch.stack([C / det1, -b / det1, A / det1], 1)
    if at is not None and "conic_opacity" in at:
        con = con + (at["conic_opacity"][:, :3] - con).detach()
    logit = x["logit"].view(-1)
    q = det0 / det1
    if at is None:
        o_hat = torch.sigmoid(logit) * torch.sqrt(torch.clamp_min(q, AA_MIN_RATIO))
    else:
        sig_f, s_f, q_f = at["sigmoid"], at["s"], at["q"]
        sig = sig_f + (logit - logit.detach()) * (sig_f * (1.0 - sig_f))
        s = s_f + torch.where(q_f > AA_MIN_RATIO, (q - q.detach()) / (2.0 * s_f), torch.zeros_like(q))
        o_hat = sig * s
        if "conic_opacity" in at:
            o_hat = o_hat + (at["conic_opacity"][:, 3] - o_hat).detach()
    hom = mh @ x["proj"]
    m_w = 1.0 / (hom[:, 3] + 1e-7)
    ndc = hom[:, :2] * m_w[:, None]
    ndc.retain_grad()
    pix = pin(torch.stack([((ndc[:, 0] + 1.0) * W - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5], 1), "means2D")
    if "colors" in x:
        rgb = x["colors"]
    else:
        d = m - x["campos"]
        d = d / d.norm(dim=1, keepdim=True)
        rgb = torch.clamp_min(R64.sh_colour(x["sh"], x["deg"], d), 0.0)
        rgb.retain_grad()
    rgb_mid, rgb = rgb, pin(rgb, "rgb")
    invd = 1.0 / tz
    colour = torch.zeros(3, H, W, dtype=F64, device=dev)
    invdepth = torch.zeros(H, W, dtype=F64, device=dev)
    alpha_map = torch.zeros(H, W, dtype=F64, device=dev)
    n_contrib = torch.zeros(H, W, dtype=torch.int64, device=dev)
    margin_a, margin_t = math.inf, math.inf
    gx = (W + 15) // 16
    for tile, ids in enumerate(tiles):
        x0, y0 = (tile % gx) * 16, (tile // gx) * 16
        ys, xs = torch.meshgrid(torch.arange(y0, min(y0 + 16, H), device=dev), torch.arange(x0, min(x0 + 16, W), device=dev), indexing="ij")
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        if ids.numel() == 0:
            colour[:, ys, xs] = bg.to(dev, F64)[:, None]
            continue
        assert bool(vis[ids].all())
        dx = pix[ids, 0][None, :] - xs[:, None].to(F64)
        dy = pix[ids, 1][None, :] - ys[:, None].to(F64)
        if at is not None and "means2D" in at:
            dx = dx + ((pix[ids, 0].detach().float()[None, :] - xs[:, None].float()).to(F64) - dx).detach()
            dy = dy + ((pix[ids, 1].detach().float()[None, :] - ys[:, None].float()).to(F64) - dy).detach()
        cc = con[ids]
        power = -0.5 * (cc[:, 0] * dx * dx + cc[:, 2] * dy * dy) - cc[:, 1] * dx * dy
        raw = o_hat[ids][None, :] * torch.exp(power)
        # the reference's backward differentiates alpha = o G through the 0.99 clamp
        alpha = raw + (torch.clamp_max(raw, 0.99) - raw).detach()
        with torch.no_grad():
            keep = (power <= 0) & (alpha >= 1.0 / 255.0)
            margin_a = min(margin_a, float((alpha - 1.0 / 255.0).abs()[power <= 0].min()))
            a_eff = torch.where(keep, alpha, torch.zeros_like(alpha))
            test_T = torch.cumprod(1.0 - a_eff, 1)
            stop = keep & (test_T < 1e-4)
            done = torch.cumsum(stop.int(), 1) > 0
            use = keep & ~done
            if bool(keep.any()):
                margin_t = min(margin_t, float((test_T - 1e-4).abs()[keep].min()))
            pos = torch.arange(1, ids.numel() + 1, device=dev)[None, :]
            n_contrib[ys, xs] = (use * pos).max(1).values
        a_use = torch.where(use, alpha, torch.zeros_like(alpha))
        T_after = torch.cumprod(1.0 - a_use, 1)
        T_before = torch.cat([torch.ones_like(T_after[:, :1]), T_after[:, :-1]], 1)
        w = a_use * T_before
        T_final = T_after[:, -1]
        if at is not None and "final_T" in at:
            r = (at["final_T"][ys, xs] / T_final).detach()
            w, T_final = w * r[:, None], T_final * r
        colour[:, ys, xs] = (w @ rgb[ids]).T + T_final[None, :] * bg.to(dev, F64)[:, None]
        invdepth[ys, xs] = w @ invd[ids]
        alpha_map[ys, xs] = 1.0 - T_final
    return colour, invdepth[None], alpha_map[None], n_contrib, dict(ndc=ndc, rgb=rgb_mid, cov=cov), (margin_a, margin_t)
