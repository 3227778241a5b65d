"""The fp64 oracle of the inverse-depth / alpha maps' backward and of the feature channels' backward, composed from the colour
oracle (gs_oracle.backward) on the scenes of tests/backward_edges.py.  Both extras are linear in quantities the colour oracle
already handles, so the compositions are exact:

  - maps (DESIGN.md §5c): invdepth is a fourth colour channel of colour 1/depth and no background, and alpha = 1 - final_T is the
    colour of a zero-colour render with background -1.  Their backward is the sum of the colour backward, a backward with
    rgb := (1/depth, 0, 0), bg = 0, dL/dpixel = (dL_dinvdepth, 0, 0), and one with rgb := 0, bg = (-1, 0, 0), dL/dpixel =
    (dL_dalpha, 0, 0); the second one's dL_dcolors[:, 0] is dinvd = sum alpha T dL_dinvdepth, whose direct depth term
    -dinvd / z^2 (V[2], V[6], V[10]) adds to dL_dmeans3D.  dL_dcolors and dL_dsh are the colour backward's alone.
  - features (DESIGN.md §5l): a feature channel is a colour channel with bg = 0.  Each group of 3 channels is one backward with
    rgb := features[:, 3k:3k+3] (zero-padded) and no SH; its dL_dcolors is the group's dL_dfeatures, its geometry adds to the colour
    backward's.  ceil(F / 3) backwards are slow on the big scenes, so an upstream gradient of rank 3, G[c] = sum_k A[c, k] h_k
    (`rank3`), takes one: rgb := features @ A and dL/dpixel := h give the exact geometry gradients, and dL_dfeatures =
    dL_dcolors @ A^T.  The oracle reads rgb and dL/dpixel in fp32, so `features @ A` and the kernel's G = A h are rounded once
    (~1e-7 relative), three orders of magnitude under the per-element bar.

`compose` returns (o64, o32) shaped like backward_edges.oracle's, plus dL_dfeatures [P, F] when features are given and `dinvd`
[P] (the per-Gaussian sum alpha T dL_dinvdepth, for the camera chain) when maps are, so backward_edges.compare / compare_aa /
describe work unchanged.  Anti-aliasing passes through (`aa`)."""
import numpy as np

import gs_oracle
from gs_b200 import synth

GRAD_NAMES = ["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations",
              "dL_dconic"]
OWN = ("dL_dcolors", "dL_dsh")                # the colour backward's alone


def _pair(case, o, rgb, bg, dL, aa):
    """(fp64, fp32) oracle backwards of the fp32 forward state `o` with its colours replaced by `rgb` and no SH."""
    s = case.scene
    fwd = dict(o)
    fwd["rgb"] = np.ascontiguousarray(rgb, np.float32)
    kw = dict(bg=np.asarray(bg, np.float32), antialiasing=aa, **case.cam_kw())
    dL = np.ascontiguousarray(dL, np.float32)
    return tuple(gs_oracle.backward(fwd, dL, s.means3D, s.scales, s.rotations, None, s.degrees, f64=f64, **kw) for f64 in (True, False))


def _channel0(img, H, W):
    out = np.zeros((3, H, W), np.float32)
    out[0] = np.asarray(img, np.float32).reshape(H, W)
    return out


def invdepth_colours(o):
    """(1/depth, 0, 0) per Gaussian, an IEEE fp32 division of the forward's depth, 0 for culled rows."""
    d = np.asarray(o["depths"], np.float32)
    vis = o["radii"] > 0
    rgb = np.zeros((d.shape[0], 3), np.float32)
    rgb[vis, 0] = np.float32(1.0) / d[vis]
    return rgb


def rank3(F, H, W, seed):
    """A rank-3 upstream gradient of an F-channel feature image -> (A [F,3], h [3,H,W], G = A h [F,H,W] in fp32), scaled so that
    sum_c f_c G_c of N(0, 1) features has the size of a colour channel's dL/dalpha."""
    rng = np.random.default_rng(seed)
    A = (rng.standard_normal((F, 3)) / np.sqrt(F)).astype(np.float32)
    h = rng.standard_normal((3, H, W)).astype(np.float32)
    G = (A.astype(np.float64) @ h.reshape(3, -1).astype(np.float64)).astype(np.float32).reshape(F, H, W)
    return A, h, G


def full_rank(F, H, W, seed):
    """An upstream gradient [F, H, W] of full rank, with the scale of `rank3`'s."""
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((F, H, W)) / np.sqrt(F)).astype(np.float32)


def map_gradients(W, H, seed):
    """dL_dinvdepth, dL_dalpha [H, W] of the size of a colour channel's (1/depth ~ 0.15..0.4 on these scenes: x 4)."""
    return 4.0 * synth.grad_image(W, H, seed)[0].numpy(), synth.grad_image(W, H, seed + 1)[1].numpy()


def compose(case, o, colour=None, maps=None, features=None, aa=False):
    """-> (o64, o32) of the backward whose loss is the colour loss of `colour` (the (o64, o32) of backward_edges.oracle on the same
    state `o`, or None: no colour loss), plus the maps' with `maps` = (dL_dinvdepth, dL_dalpha) [H, W] each, plus the feature
    image's with `features` = (features [P, F], G), G the [F, H, W] upstream gradient (ceil(F / 3) backwards) or (A, h) of `rank3`
    (one backward)."""
    W, H = case.W, case.H
    P = o["radii"].shape[0]
    M = case.scene.sh.shape[1]
    outs = [{k: np.zeros(v.shape, t) for k, v in _zero_shapes(P, M).items()} for t in (np.float64, np.float32)]

    def add(pair):
        for out, g in zip(outs, pair):
            for k in GRAD_NAMES:
                if k not in OWN:
                    out[k] = out[k] + g[k].astype(out[k].dtype)

    zero_rgb = np.zeros((P, 3), np.float32)
    if maps is not None:
        Gd, Ga = maps
        inv = _pair(case, o, invdepth_colours(o), np.zeros(3), _channel0(Gd, H, W), aa)
        add(inv)
        add(_pair(case, o, zero_rgb, np.array([-1.0, 0.0, 0.0]), _channel0(Ga, H, W), aa))
        V = case.cam.world_view_transform.numpy().astype(np.float32).reshape(-1)
        vis = o["radii"] > 0
        z = np.asarray(o["depths"], np.float32)
        for out, g, t in zip(outs, inv, (np.float64, np.float32)):
            dinvd = np.asarray(g["dL_dcolors"][:, 0], t)
            zz = np.where(vis, z.astype(t), t(1.0))
            dz = np.where(vis, -dinvd / (zz * zz), t(0.0)).astype(t)
            out["dL_dmeans3D"] = out["dL_dmeans3D"] + dz[:, None] * np.array([V[2], V[6], V[10]], t)[None, :]
            out["dinvd"] = dinvd
    if features is not None:
        feat, G = features
        feat = np.asarray(feat, np.float32)
        F = feat.shape[1]
        d64, d32 = np.zeros((P, F), np.float64), np.zeros((P, F), np.float32)
        if isinstance(G, tuple):
            A, h = G
            rgb = (feat.astype(np.float64) @ np.asarray(A, np.float64)).astype(np.float32)
            pair = _pair(case, o, rgb, np.zeros(3), h, aa)
            add(pair)
            d64[:] = pair[0]["dL_dcolors"] @ np.asarray(A, np.float64).T
            d32[:] = (pair[1]["dL_dcolors"].astype(np.float32) @ np.asarray(A, np.float32).T).astype(np.float32)
        else:
            G = np.asarray(G, np.float32)
            for c0 in range(0, F, 3):
                n = min(3, F - c0)
                rgb = np.zeros((P, 3), np.float32)
                rgb[:, :n] = feat[:, c0:c0 + n]
                dL = np.zeros((3, H, W), np.float32)
                dL[:n] = G[c0:c0 + n]
                pair = _pair(case, o, rgb, np.zeros(3), dL, aa)
                add(pair)
                d64[:, c0:c0 + n] = pair[0]["dL_dcolors"][:, :n]
                d32[:, c0:c0 + n] = pair[1]["dL_dcolors"][:, :n]
        outs[0]["dL_dfeatures"], outs[1]["dL_dfeatures"] = d64, d32
    return with_colour((outs[0], outs[1]), colour) if colour is not None else (outs[0], outs[1])


def with_colour(extra, colour):
    """The (o64, o32) composition `extra` (of `compose`, without colour loss) plus the colour backward `colour` = (o64, o32):
    dL_dcolors and dL_dsh are the colour backward's, every other gradient the sum."""
    res = []
    for e, c in zip(extra, colour):
        r = dict(e)
        for k in GRAD_NAMES:
            r[k] = np.asarray(c[k], e[k].dtype) if k in OWN else e[k] + np.asarray(c[k], e[k].dtype)
        res.append(r)
    return tuple(res)


def _zero_shapes(P, M):
    return dict(dL_dmeans2D=np.zeros((P, 3)), dL_dcolors=np.zeros((P, 3)), dL_dopacity=np.zeros((P, 1)), dL_dmeans3D=np.zeros((P, 3)),
                dL_dcov3D=np.zeros((P, 6)), dL_dsh=np.zeros((P, M, 3)), dL_dscales=np.zeros((P, 3)), dL_drotations=np.zeros((P, 4)),
                dL_dconic=np.zeros((P, 4)))


def masked(img, borderline):
    """A copy of the [C, H, W] (or [H, W]) image with the borderline pixels zeroed."""
    out = np.array(img, np.float32, copy=True)
    out[..., borderline] = 0.0
    return out
