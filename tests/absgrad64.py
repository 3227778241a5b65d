"""Float64 restatement of the render backward's per-pair screen-space terms (DESIGN.md §5m), for the absolute gradient of AbsGS.

For pixel p and Gaussian i of p's list, the reference adds (backward.cu:561-589)
    g_x = 0.5 W o w (-(a dx + b dy)),   g_y = 0.5 H o w (-(b dx + c dy)),   w = G dL/dalpha
to dL_dmeans2D[i], with (a, b, c, o) = conic_opacity[i], (dx, dy) = means2D[i] - p, G = exp(power) and dL/dalpha including the
background term.  This walks each pixel's list with the forward's rules (power > 0 and alpha < 1/255 skip, alpha saturates at
0.99, the list ends at n_contrib) and returns both the signed sums, which must equal the oracle's dL_dmeans2D, and the sums of
the absolute values, which the kernels' absgrad output is checked against.  The skip decisions take the fp32 power, as the
kernels do; everything after that is float64.
"""
import numpy as np


def pair_sums(state, bg, dL, W, H, dL_dinvdepth=None, dL_dalpha=None):
    """state: means2D [P,2], conic_opacity [P,4], rgb [P,3], point_list, ranges [tiles,2], n_contrib [H,W] (any array-likes).
    bg [3], dL [3,H,W].  -> (signed [P,2], absolute [P,2]) float64, with the factors 0.5 W / 0.5 H applied.
    With the maps' gradients (DESIGN.md §5c; [H,W] each, `state` then also needs depths [P]): dL_dinvdepth is that of one more
    channel of colour 1/depth (the IEEE fp32 quotient) and background 0, dL_dalpha that of one of colour 0 and background -1
    (alpha = 1 - final_T)."""
    m2 = np.asarray(state["means2D"], np.float32)
    co = np.asarray(state["conic_opacity"], np.float32)
    rgb = np.asarray(state["rgb"], np.float64)
    pl = np.asarray(state["point_list"]).astype(np.int64)
    ranges = np.asarray(state["ranges"]).astype(np.int64).reshape(-1, 2)
    nc = np.asarray(state["n_contrib"]).astype(np.int64).reshape(H, W)
    bg = np.asarray(bg, np.float64)
    dL = np.asarray(dL, np.float64).reshape(3, H, W)
    if dL_dinvdepth is not None or dL_dalpha is not None:
        # two more channels: colour 1/depth with background 0 under dL_dinvdepth, colour 0 with background -1 under dL_dalpha
        d = np.asarray(state["depths"], np.float32)
        inv = np.zeros(d.shape, np.float32)
        inv[d != 0] = np.float32(1.0) / d[d != 0]
        rgb = np.concatenate([rgb, inv.astype(np.float64)[:, None], np.zeros((rgb.shape[0], 1))], 1)
        bg = np.concatenate([bg, [0.0, -1.0]])
        zero = np.zeros((H, W))
        dL = np.concatenate([dL, np.stack([zero if m is None else np.asarray(m, np.float64).reshape(H, W)
                                           for m in (dL_dinvdepth, dL_dalpha)])], 0)
    P = m2.shape[0]
    signed = np.zeros((P, 2), np.float64)
    absol = np.zeros((P, 2), np.float64)
    gx = (W + 15) // 16
    for t in range(ranges.shape[0]):
        r0, r1 = int(ranges[t, 0]), int(ranges[t, 1])
        if r1 <= r0:
            continue
        tx, ty = (t % gx) * 16, (t // gx) * 16
        ys, xs = np.meshgrid(np.arange(ty, min(ty + 16, H)), np.arange(tx, min(tx + 16, W)), indexing="ij")
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        n = nc[ys, xs]
        hi = int(n.max()) if n.size else 0
        if hi == 0:
            continue
        ids = pl[r0:r0 + hi]
        # fp32 power, as forward.cu:538 / the kernels: fma(fma(dx, A dx, (C dy) dy), -0.5, -((B dx) dy))
        dx = m2[ids, 0][None, :] - xs.astype(np.float32)[:, None]
        dy = m2[ids, 1][None, :] - ys.astype(np.float32)[:, None]
        A, B, Cc, o = co[ids, 0][None, :], co[ids, 1][None, :], co[ids, 2][None, :], co[ids, 3][None, :]
        power = (np.float32(-0.5) * (dx * (A * dx) + (Cc * dy) * dy) - (B * dx) * dy).astype(np.float64)
        G = np.exp(power)
        alpha = np.minimum(0.99, o.astype(np.float64) * G)
        j = np.arange(hi)[None, :]
        valid = (j < n[:, None]) & ~(power > 0) & ~(alpha < 1.0 / 255.0)
        a = np.where(valid, alpha, 0.0)
        one_m = 1.0 - a
        T = np.cumprod(np.concatenate([np.ones((a.shape[0], 1)), one_m[:, :-1]], axis=1), axis=1)     # T in front of entry j
        T_final = T[:, -1] * one_m[:, -1]
        dLp = dL[:, ys, xs].T                                                                          # [pixels, C]
        k = dLp @ rgb[ids].T                                                                           # colour . dL/dpixel
        contrib = k * a * T
        S = np.cumsum(contrib[:, ::-1], axis=1)[:, ::-1] - contrib                                     # entries behind j
        bgd = T_final * (dLp @ bg)
        dLda = T * k - (S + bgd[:, None]) / one_m
        w = np.where(valid, G * dLda, 0.0)
        dx64, dy64 = dx.astype(np.float64), dy.astype(np.float64)
        A64, B64, C64, o64 = (v.astype(np.float64) for v in (A, B, Cc, o))
        tx_ = 0.5 * W * o64 * w * -(A64 * dx64 + B64 * dy64)
        ty_ = 0.5 * H * o64 * w * -(B64 * dx64 + C64 * dy64)
        np.add.at(signed[:, 0], ids, tx_.sum(axis=0))
        np.add.at(signed[:, 1], ids, ty_.sum(axis=0))
        np.add.at(absol[:, 0], ids, np.abs(tx_).sum(axis=0))
        np.add.at(absol[:, 1], ids, np.abs(ty_).sum(axis=0))
    return signed, absol
