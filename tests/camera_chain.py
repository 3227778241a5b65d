"""The float64 chain of the camera gradients, shared by test_gpu_camera.py and test_gpu_antialias_edges.py: screen-space gradients
(dL_dmeans2D, dL_dconic, dL_dcolors) contracted with the restatement of the preprocess (restate64.py) w.r.t. view, proj and campos
as independent tensors, and the bar a kernel's camera gradients are held to against it."""
import torch

import restate64 as R64

F64 = torch.float64


def chain(view, proj, campos, W, H, tanx, tany, means, cov3D, sh, deg, clamped, vis, g_m2, g_con, g_col, dev="cuda", g_invd=None,
          aa=None):
    """Per-Gaussian camera gradients (float64): the screen-space gradients contracted with the restatement of the preprocess
    (screen_cov, cov2D + 0.3, conic, ndc, SH colour).  view / proj / campos are independent.  -> ([P,4,4], [P,4,4], [P,3])
    per visible Gaussian, whose sums are the camera gradients and whose absolute sums are the scales of the bars.
    `g_invd` [P]: the inverse-depth map's dinvd = sum alpha T dL_dinvdepth per Gaussian, which adds dinvd / tz (tz from the view
    row).  `aa` = (g_ohat, sigmoid, q_clamped) [P] each: with anti-aliasing o^ = sigmoid * sqrt(det0 / det1) (DESIGN.md §5e),
    g_ohat = dL/do^, and the Gaussians whose q = det0 / det1 the forward clamped carry no gradient through it."""
    idx = torch.nonzero(vis).view(-1)
    P = idx.numel()
    f = lambda t: t.to(device=dev, dtype=F64)[idx]
    m, cov, gm, gc = f(means), f(cov3D), f(g_m2), f(g_con)
    V = view.to(dev, F64).detach().expand(P, 4, 4).clone().requires_grad_(True)
    Pm = proj.to(dev, F64).detach().expand(P, 4, 4).clone().requires_grad_(True)
    cp = campos.to(dev, F64).detach().expand(P, 3).clone().requires_grad_(True)
    mh, tz, a, b, c = R64.screen_cov(m, V, cov, W, H, tanx, tany)
    det0 = a * c - b * b
    a, c = a + 0.3, c + 0.3
    det = a * c - b * b
    loss = gc[:, 0] * (c / det) + 2.0 * gc[:, 1] * (-b / det) + gc[:, 3] * (a / det)
    if g_invd is not None:
        loss = loss + f(g_invd) / tz
    if aa is not None:
        g_ohat, sig, q_clamped = aa
        clamp = f(q_clamped).bool()
        s = torch.sqrt(torch.where(clamp, torch.ones_like(det0), det0 / det))      # no NaN from a det0 <= 0 in the unused branch
        loss = loss + torch.where(clamp, torch.zeros_like(s), f(g_ohat) * f(sig) * s)
    hom = torch.einsum("pr,prc->pc", mh, Pm)
    m_w = 1.0 / (hom[:, 3] + 1e-7)
    loss = loss + gm[:, 0] * hom[:, 0] * m_w + gm[:, 1] * hom[:, 1] * m_w
    if sh is not None:
        d = m - cp
        d = d / d.norm(dim=1, keepdim=True)
        col = R64.sh_colour(f(sh), deg.to(dev)[idx], d)
        loss = loss + (f(g_col) * col * (1.0 - f(clamped.float()))).sum(1)
    loss.sum().backward()
    return V.grad, Pm.grad, cp.grad


def check(got, per, bar, label):
    """got: kernel (view, proj, campos); per: per-Gaussian contributions.  |got - sum| <= bar * sum |c_i| per entry -> max ratio."""
    worst = 0.0
    for n, k, p in zip(("view", "proj", "campos"), got, per):
        k = k.to(F64).reshape(-1)
        if p is None:
            continue
        p = p.reshape(p.shape[0], -1)
        tot, scale = p.sum(0), p.abs().sum(0)
        zero = scale == 0
        assert float(k[zero].abs().max()) == 0.0 if bool(zero.any()) else True, (label, n)
        r = ((k - tot).abs() / torch.where(zero, torch.ones_like(scale), scale))[~zero]
        worst = max(worst, float(r.max()))
        assert float(r.max()) <= bar, (label, n, float(r.max()), k.tolist(), tot.tolist())
    print(f"\n[camera chain] {label}: max |kernel - chain| / sum|c_i| = {worst:.3e} (bar {bar:g})")
    return worst
