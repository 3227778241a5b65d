"""Scenes that put the compositing backward (render_backward_kernel, gsb_render.cu, and the preprocess backward it feeds) on its
batch, ring, stash, tile and geometry boundaries, and the per-element comparison of a backward against the fp64 oracle.

Shared by test_backward_edges_oracle.py (CPU: every scene reaches what it is built for, and the comparison rejects near-misses
the global bar accepts) and test_gpu_backward_edges.py (the CUDA backward against the oracle, element by element).

The comparison, for each gradient array and each element, with o64 the oracle's fp64 backward and o32 its fp32 one (the
reference's expression order) from the same fp32 forward state, e = |ours - o64| and, per Gaussian (row of the array),
E32 = max |o32 - o64| (the reference arithmetic's own error) and |o64|_row = max |o64|:
    e <= max(K * E32, R_REL * |o64|_row, A_ABS * max|o64|)
Gaussians whose gradient a MUFU.EX2-vs-expf ulp can legitimately change (see `excluded`) are held to EXCLUDED_BAR of the
array's scale instead, and checked per element on a second backward whose dL/dpixel is zero on the borderline pixels; culled
ones must carry exactly zero."""
import math

import numpy as np
import torch

import gs_oracle
import restate64 as R64
from gs_b200 import synth

GRAD_NAMES = ["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations"]
ARRAYS = GRAD_NAMES + ["dL_dconic"]
K, R_REL, A_ABS = 8.0, 1e-4, 1e-6          # the per-element bar (see test_gpu_backward_edges.py for what was observed)
GLOBAL = 2e-4                               # test_gpu_parity.test_against_oracle_midsize's bar, of each array's scale
# a flipped pair at the 1/255 rim of a 600 px Gaussian carries dx ~ 600 px: on one H100 it moved that Gaussian's dL_drotations by
# 0.052 of 130 (between 2e-4 and 4e-4 of the array's scale); the excluded Gaussians are checked per element on a masked dL instead
EXCLUDED_BAR = 1e-3
# dense_faint: in its 30 000-entry lists of faint Gaussians the small gradients carry up to 4e-4 of their row's magnitude and
# 4e-6 of the array's scale (dL_dconic; 2.5e-4 / 2.5e-6 in dL_dscales) on one H100, while the fp32 reference stays well below
# that; the kernel recovers T with MUFU.RCP, not an IEEE division.  Every other case stays below 0.6 of the default bar.
BAR_CASE = {"dense_faint": (1e-3, 1e-5)}                 # (R_REL, A_ABS)
# aa_needles: on a needle whose det0 cancels (a c / det0 >= 1e2) dL_dmeans3D and dL_drotations are ill-conditioned in fp32: the
# reference arithmetic itself errs by up to 8.5e-3 / 0.35 of the row there, and on one H100 the dL_drotations of a needle with
# a c / det0 = 6e4 moved by 7 % between two runs (the render backward's atomic order), and one of 278 by 1.7e-3 of its row.  Those
# two arrays of those needles are not checked per element (compare_aa); every other array of every needle is, and every array of
# the 72 well-conditioned ones (a c / det0 < 1e2: the 48 bisected to the clamp, 25 clamped ones).
AA_WELL_CONDITIONED = 1e2
ILL_CONDITIONED_ARRAYS = ["dL_dmeans3D", "dL_drotations"]

STAIRCASE = [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 320, 511, 512, 513, 1000]
TIE_TILE = STAIRCASE.index(129)             # the tile of the tie variant whose Gaussians all share one depth
ODD_SIZES = [(1, 1), (3, 7), (8, 4), (15, 17), (17, 15), (20, 36), (33, 1)]
DENSE = ["dense_4k", "dense_12k", "dense_40k", "dense_ties", "dense_faint"]
CASES = (["staircase", "staircase_ties"] + ["odd_%dx%d" % s for s in ODD_SIZES] + ["large", "saturation"] + DENSE)
# anti-aliased only (antialiasing=True, DESIGN.md §5e): needle-thin splats around the clamp of s, and sub-pixel splats (s << 1)
AA_CASES = ["aa_needles", "aa_subpixel"]
AA_MIN_RATIO = np.float32(2.5e-5)           # the clamp of q = det0 / det1 under s = sqrt(max(2.5e-5, q))
# the share of the visible Gaussians a case may hold to the global bar instead of the per-element one (observed: see the CPU test)
EXCLUDED_MAX = {"large": 0.02, "dense_4k": 0.10, "dense_12k": 0.10, "dense_40k": 0.10, "dense_ties": 0.10, "dense_faint": 0.10}
EXCLUDED_DEFAULT = 0.05
# with anti-aliasing (observed: see test_antialias_edges_oracle.py): odd_20x36's 420 small splats put 18 % of them next to a
# borderline pixel once o^ = sigmoid * s is lower
EXCLUDED_MAX_AA = {"odd_20x36": 0.20}


class Case:
    def __init__(self, name, scene, cam, bg, dL, lam=0.0, **meta):
        self.name, self.scene, self.cam, self.bg, self.dL, self.lam, self.meta = name, scene, cam, bg, dL, lam, meta
        self.W, self.H = cam.image_width, cam.image_height

    def cam_kw(self):
        c = self.cam
        return dict(viewmatrix=c.world_view_transform, projmatrix=c.full_proj_transform, campos=c.camera_center, W=self.W, H=self.H,
                    tan_fovx=math.tan(c.FoVx * 0.5), tan_fovy=math.tan(c.FoVy * 0.5))


def pixel_scene(cam, px, py, depth, sigma_px, logits, sh, g, aniso=None, rots=None):
    """Gaussians placed by their screen centre (px, py), view-space depth and screen-space standard deviation (before the 0.3
    low-pass), on `cam`; random rotations unless `rots` [P,4] gives them (their 3D scales are `sigma_px * depth / focal` times
    `aniso`)."""
    P = len(px)
    W, H = cam.image_width, cam.image_height
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    depth = np.asarray(depth, np.float64)
    xv = ((2.0 * np.asarray(px, np.float64) + 1.0) / W - 1.0) * depth * tx
    yv = ((2.0 * np.asarray(py, np.float64) + 1.0) / H - 1.0) * depth * ty
    view = np.stack([xv, yv, depth, np.ones(P)], 1)
    world = view @ np.linalg.inv(cam.world_view_transform.double().numpy())         # row vectors: p_view = p_world @ V^T
    focal = H / (2.0 * ty)
    s = np.asarray(sigma_px, np.float64) * depth / focal
    scales = s[:, None] * (np.ones((P, 3)) if aniso is None else np.asarray(aniso, np.float64))
    q = torch.randn(P, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=1, keepdim=True)
    if rots is not None:
        q = torch.as_tensor(np.asarray(rots), dtype=torch.float64)
    sh = torch.as_tensor(np.asarray(sh), dtype=torch.float32)
    deg = int(round(math.sqrt(sh.shape[1]))) - 1
    return synth.Scene(torch.from_numpy(world[:, :3]).float().contiguous(), torch.as_tensor(np.asarray(logits), dtype=torch.float32).view(P, 1),
                       torch.from_numpy(scales).float().contiguous(), q.float().contiguous(), sh.contiguous(),
                       torch.full((P, 1), deg, dtype=torch.int32))


def _logit(p):
    return math.log(p / (1.0 - p))


def _aa_isotropic_s(sigma):
    """s = sqrt(det0 / det1) of an isotropic splat of `sigma` px: sigma^2 / (sigma^2 + 0.3)."""
    return sigma * sigma / (sigma * sigma + 0.3)


def _staircase(ties, aa=False):
    """Tile t of a 6x4-tile image gets exactly STAIRCASE[t] faint Gaussians (2D radius <= 6 px, centred in the tile +-2 px, so
    their rect is that tile alone); opacity 0.0068..0.0082 keeps T above 2.7e-4 after 1 000 of them, so every tile's largest
    n_contrib (`hi`) is its list length.  With `aa` the sigmoid is divided by s (isotropic estimate), so o^ stays in that range."""
    W, H = 96, 64
    cam = synth.make_camera(W, H)
    g = torch.Generator().manual_seed(1001 if ties else 1000)
    tiles = np.repeat(np.arange(len(STAIRCASE)), STAIRCASE)
    P = tiles.size
    u = torch.rand(P, 6, generator=g, dtype=torch.float64).numpy()
    px = 16 * (tiles % 6) + 8 + 4 * (u[:, 0] - 0.5)
    py = 16 * (tiles // 6) + 8 + 4 * (u[:, 1] - 0.5)
    depth = 3.0 + 3.0 * u[:, 2]
    if ties:
        depth[tiles == TIE_TILE] = 4.25                    # exactly representable: the view-space depths are bit-identical
    sigma = 0.8 + 0.6 * u[:, 3]
    logits = _logit(0.0068) + (_logit(0.0082) - _logit(0.0068)) * u[:, 4]
    if aa:
        logits = np.log(1.0 / (1.0 + np.exp(-logits)) / _aa_isotropic_s(sigma))
        logits = logits - np.log1p(-np.exp(logits))
    sh = torch.randn(P, 4, 3, generator=g).numpy()
    sh[:, 1:] *= 0.15
    scene = pixel_scene(cam, px, py, depth, sigma, logits, sh, g)
    return Case("staircase_ties" if ties else "staircase", scene, cam, torch.tensor([0.2, 0.3, 0.1]), synth.grad_image(W, H, 1002),
                tile_k=np.array(STAIRCASE))


def _odd(W, H):
    """Gaussians of 0.7..5 px standard deviation centred over the image and 6 px around it, any opacity, background != 0."""
    cam = synth.make_camera(W, H)
    g = torch.Generator().manual_seed(2000 + 100 * W + H)
    P = 60 + (W * H) // 2
    u = torch.rand(P, 6, generator=g, dtype=torch.float64).numpy()
    px, py = -6 + (W + 12) * u[:, 0], -6 + (H + 12) * u[:, 1]
    depth = 2.5 + 4.0 * u[:, 2]
    sigma = 0.7 + 4.3 * u[:, 3]
    aniso = 0.4 + 1.2 * torch.rand(P, 3, generator=g, dtype=torch.float64).numpy()
    logits = 2.0 * torch.randn(P, generator=g).numpy()
    sh = torch.randn(P, 9, 3, generator=g).numpy()
    sh[:, 1:] *= 0.2
    scene = pixel_scene(cam, px, py, depth, sigma, logits, sh, g, aniso)
    return Case("odd_%dx%d" % (W, H), scene, cam, torch.tensor([0.3, 0.6, 0.15]), synth.grad_image(W, H, 2001), lam=0.05)


def _large():
    """36 Gaussians of 35..200 px standard deviation (2D radii ~100..600 px) over 20 000 small ones on 1920x1080, random signed
    dL.  12 of the large ones are centred beyond 1.3 tan(fov / 2) left, right or below the image, with a radius that reaches in:
    the preprocess backward's frustum clamp zeroes their screen-x (or y) chain term."""
    W, H = 1920, 1080
    cam = synth.make_camera(W, H)
    g = torch.Generator().manual_seed(3000)
    Ns, Nl, No = 20_000, 24, 12
    u = torch.rand(Ns, 5, generator=g, dtype=torch.float64).numpy()
    px, py = W * u[:, 0], H * u[:, 1]
    depth = 2.0 + 8.0 * u[:, 2]
    sigma = 1.0 + 3.0 * u[:, 3]
    v = torch.rand(Nl + No, 5, generator=g, dtype=torch.float64).numpy()
    lpx, lpy = W * v[:, 0], H * v[:, 1]
    lsig = 35.0 + 165.0 * v[:, 3]
    side = np.arange(No) % 3                                                # 0 left, 1 right, 2 below
    out = slice(Nl, Nl + No)
    lpx[out] = np.where(side == 0, -0.15 * W - 50 - 150 * v[out, 4], np.where(side == 1, 1.15 * W + 50 + 150 * v[out, 4], lpx[out]))
    lpy[out] = np.where(side == 2, 1.15 * H + 50 + 150 * v[out, 4], lpy[out])
    lsig[out] = 160.0 + 40.0 * v[out, 3]
    px, py = np.concatenate([px, lpx]), np.concatenate([py, lpy])
    depth = np.concatenate([depth, 3.0 + 5.0 * v[:, 2]])
    sigma = np.concatenate([sigma, lsig])
    P = Ns + Nl + No
    aniso = 0.5 + torch.rand(P, 3, generator=g, dtype=torch.float64).numpy()
    logits = np.concatenate([2.0 * torch.randn(Ns, generator=g).numpy(), -2.0 + 3.0 * v[:, 4]])
    sh = torch.randn(P, 4, 3, generator=g).numpy()
    sh[:, 1:] *= 0.15
    scene = pixel_scene(cam, px, py, depth, sigma, logits, sh, g, aniso)
    return Case("large", scene, cam, torch.tensor([0.1, 0.1, 0.2]), synth.grad_image(W, H, 3001), large=np.arange(Ns, P))


def _saturation(aa=False):
    """Stacks of 40 Gaussians per tile, a third of them opaque (logit 8: alpha clamps at 0.99), so T < 1e-4 stops pixels partway
    down the list; DC colours down to -3 clamp some channels at 0.  With `aa` the splats are 8..16 px instead of 2..6 px: o^ =
    sigmoid * s exceeds 0.99 only where s > 0.9904, i.e. above 5.5 px."""
    W, H = 80, 48
    cam = synth.make_camera(W, H)
    g = torch.Generator().manual_seed(4000)
    tiles = np.repeat(np.arange(15), 40)
    P = tiles.size
    u = torch.rand(P, 5, generator=g, dtype=torch.float64).numpy()
    px = 16 * (tiles % 5) + 8 + 10 * (u[:, 0] - 0.5)
    py = 16 * (tiles // 5) + 8 + 10 * (u[:, 1] - 0.5)
    depth = 2.5 + 4.0 * u[:, 2]
    sigma = 8.0 + 8.0 * u[:, 3] if aa else 2.0 + 4.0 * u[:, 3]
    logits = np.where(u[:, 4] < 1.0 / 3.0, 8.0, torch.randn(P, generator=g, dtype=torch.float64).numpy())
    sh = 1.5 * torch.randn(P, 1, 3, generator=g).numpy() - 0.5
    scene = pixel_scene(cam, px, py, depth, sigma, logits, sh, g)
    return Case("saturation", scene, cam, torch.tensor([0.5, 0.2, 0.4]), synth.grad_image(W, H, 4001), lam=0.05)


def _aa_needles():
    """256x160, anti-aliased: 400 needles (scales (L, L t, L t), L 2..12 px, thinness t 1e-2..1e-4 log-uniform, random
    rotations), whose det0 = a c - b^2 cancels (a c / det0 up to ~1e8) and whose q = det0 / det1 spans the clamp at 2.5e-5; plus
    48 needles lying along the image's x or y axis (b ~ 0, no cancellation) whose width is bisected in fp32 until the forward's
    q_f lies within 1e-3 relative of the clamp, half on each side.  Sigmoid 0.05..0.999, 60 % of it above 0.9."""
    W, H = 256, 160
    cam = synth.make_camera(W, H)
    g = torch.Generator().manual_seed(6000)
    Nr, Nt = 400, 48
    P = Nr + Nt
    u = torch.rand(P, 6, generator=g, dtype=torch.float64).numpy()
    px, py = 8 + (W - 16) * u[:, 0], 8 + (H - 16) * u[:, 1]
    depth = 3.0 + 5.0 * u[:, 2]
    sigma = 2.0 + 10.0 * u[:, 3]
    t = 10.0 ** (-2.0 - 2.0 * u[:, 4])
    aniso = np.stack([np.ones(P), t, t], 1)
    p = np.where(u[:, 5] < 0.6, 0.9 + 0.099 * u[:, 5] / 0.6, 0.05 + 0.85 * (u[:, 5] - 0.6) / 0.4)
    logits = np.log(p / (1.0 - p))
    sh = torch.randn(P, 4, 3, generator=g).numpy()
    sh[:, 1:] *= 0.2
    q = torch.randn(P, 4, generator=g, dtype=torch.float64).numpy()
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    # the default camera looks along +z: a rotation about z by 0 or 90 degrees keeps the needle's long axis on an image axis
    half = np.where(np.arange(Nt) % 2 == 0, 0.0, 0.25 * math.pi)
    q[Nr:] = np.stack([np.cos(half), np.zeros(Nt), np.zeros(Nt), np.sin(half)], 1)
    sigma[Nr:] = 4.0 + 4.0 * u[Nr:, 3]
    # target q_f = 2.5e-5 (1 + d), d = +-(1e-5 .. 1e-3): bisect the width factor of each axis-aligned needle on the fp32 forward
    d = np.where(np.arange(Nt) % 4 < 2, 1.0, -1.0) * 10.0 ** (-5.0 + 2.0 * u[Nr:, 4])
    target = np.float64(AA_MIN_RATIO) * (1.0 + d)
    lo, hi = np.full(Nt, -5.0), np.full(Nt, -2.0)                     # log10 of the thinness
    kw = Case("", None, cam, None, None).cam_kw()
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        aniso[Nr:, 1] = aniso[Nr:, 2] = 10.0 ** mid
        sub = pixel_scene(cam, px[Nr:], py[Nr:], depth[Nr:], sigma[Nr:], logits[Nr:], sh[Nr:], g, aniso[Nr:], q[Nr:])
        o = gs_oracle.preprocess(sub.means3D, sub.scales, 1.0, sub.rotations, sub.opacity, sub.sh, sub.degrees, None, None,
                                 kw["viewmatrix"], kw["projmatrix"], kw["campos"], W, H, kw["tan_fovx"], kw["tan_fovy"],
                                 antialiasing=True)
        up = o["aa_q"].astype(np.float64) < target
        lo, hi = np.where(up, mid, lo), np.where(up, hi, mid)
    aniso[Nr:, 1] = aniso[Nr:, 2] = 10.0 ** lo
    up = np.arange(Nt) % 4 < 2
    aniso[Nr:][up, 1:] = 10.0 ** hi[up, None]                          # the side of the target each one is meant to be on
    scene = pixel_scene(cam, px, py, depth, sigma, logits, sh, g, aniso, q)
    return Case("aa_needles", scene, cam, torch.tensor([0.2, 0.3, 0.4]), synth.grad_image(W, H, 6001), lam=0.05,
                near=np.arange(Nr, P))


def _aa_subpixel():
    """192x128, anti-aliased: 600 splats of 0.05..0.5 px standard deviation (s = 0.008..0.45) with sigmoid 0.5..0.999, so that
    o^ = sigmoid * s reaches 1/255 near their centres, over 60 of 2..5 px that they are composited with."""
    W, H = 192, 128
    cam = synth.make_camera(W, H)
    g = torch.Generator().manual_seed(6100)
    Ns, Nb = 600, 60
    P = Ns + Nb
    u = torch.rand(P, 5, generator=g, dtype=torch.float64).numpy()
    px, py = W * u[:, 0], H * u[:, 1]
    depth = 2.5 + 4.0 * u[:, 2]
    sigma = np.concatenate([0.05 + 0.45 * u[:Ns, 3], 2.0 + 3.0 * u[Ns:, 3]])
    aniso = 0.6 + 0.8 * torch.rand(P, 3, generator=g, dtype=torch.float64).numpy()
    p = np.concatenate([0.5 + 0.499 * u[:Ns, 4], 0.1 + 0.5 * u[Ns:, 4]])
    logits = np.log(p / (1.0 - p))
    sh = torch.randn(P, 4, 3, generator=g).numpy()
    sh[:, 1:] *= 0.2
    scene = pixel_scene(cam, px, py, depth, sigma, logits, sh, g, aniso)
    return Case("aa_subpixel", scene, cam, torch.tensor([0.1, 0.2, 0.3]), synth.grad_image(W, H, 6101))


def dense_scene(kind, aa=False):
    """The sort-path scenes of test_gpu_parity.test_sort_paths_ties_and_dense_tiles -> (scene, cam, bg).  `dense_faint` is
    `dense_12k` with opacities around sigmoid(-5) = 0.0067: its pixels are not stopped by T, so the backward walks lists of
    more than 8 192 entries."""
    g = torch.Generator().manual_seed(7)
    if kind == "ties":
        P, W, H = 30_000, 128, 128
        xyz = torch.rand(P, 3, generator=g) * 2 - 1
        xyz[:, 2] = 0.0                                  # one plane facing the camera: identical view-space depth
        xyz[::3, 2] = 0.25                               # ... and a second plane
        scale = 0.02
    elif kind == "dense_ties":
        # tiles of 2049..8192 instances whose depths are all identical: the 8192-bin distribution sort of that class must hand
        # them to the radix fallback (a bin holds more than 32 entries), and ties must come out in ascending Gaussian id
        P, W, H = 8_000, 64, 48
        xyz = (torch.rand(P, 3, generator=g) * 2 - 1) * torch.tensor([0.5, 0.4, 1.0])
        xyz[:, 2] = 0.0
        scale = 0.01
    else:
        P = {"dense_4k": 12_000, "dense_12k": 40_000, "dense_faint": 40_000, "dense_40k": 120_000}[kind]
        W, H = 64, 48
        xyz = (torch.rand(P, 3, generator=g) * 2 - 1) * torch.tensor([0.5, 0.4, 1.0])
        scale = 0.01
    scales = torch.full((P, 3), scale) * (0.5 + torch.rand(P, 3, generator=g))
    q = torch.nn.functional.normalize(torch.randn(P, 4, generator=g))
    op = torch.randn(P, 1, generator=g) - 2.0
    if kind == "dense_faint":
        op = 0.3 * op - 4.4                              # 0.3 * (N(0,1) - 2) - 4.4 = N(-5, 0.3)
        if aa:
            op = op + 3.0                                # s ~ 0.05 for these 0.1 px splats: sigmoid ~ 0.12 keeps o^ ~ 0.006
    sh = torch.randn(P, 1, 3, generator=g)
    deg = torch.zeros(P, 1, dtype=torch.int32)
    scene = synth.Scene(xyz.contiguous(), op, scales.contiguous(), q.contiguous(), sh, deg)
    return scene, synth.make_camera(W, H), torch.zeros(3)


def build(name, aa=False):
    """The case `name`; `aa` builds the variant of a BE.CASES scene meant to be rendered with antialiasing=True (the AA_CASES
    always are)."""
    case = _build(name, aa)
    case.meta["aa"] = aa or name in AA_CASES
    return case


def _build(name, aa):
    if name == "aa_needles":
        return _aa_needles()
    if name == "aa_subpixel":
        return _aa_subpixel()
    if name.startswith("staircase"):
        return _staircase(name.endswith("ties"), aa)
    if name.startswith("odd_"):
        W, H = (int(v) for v in name[4:].split("x"))
        return _odd(W, H)
    if name == "large":
        return _large()
    if name == "saturation":
        return _saturation(aa)
    scene, cam, bg = dense_scene(name, aa)
    return Case(name, scene, cam, torch.tensor([0.2, 0.1, 0.3]), synth.grad_image(cam.image_width, cam.image_height, 5000))


# ---- the oracle's side -------------------------------------------------------------------------------------------------------

def oracle(case, dL=None, fwd=None, aa=False):
    """-> (forward state, fp64 backward, fp32 backward) of the oracle, anti-aliased with `aa`; `fwd` / `dL` override the state /
    dL/dpixel (near-misses)."""
    s = case.scene
    o = fwd if fwd is not None else gs_oracle.forward(s.means3D, s.opacity, s.scales, s.rotations, s.sh, s.degrees, bg=case.bg,
                                                      antialiasing=aa, **case.cam_kw())
    kw = dict(bg=case.bg, lambda_sh_sparsity=case.lam, antialiasing=aa, **case.cam_kw())
    dL = case.dL if dL is None else dL
    o64 = gs_oracle.backward(o, dL, s.means3D, s.scales, s.rotations, s.sh, s.degrees, f64=True, **kw)
    o32 = gs_oracle.backward(o, dL, s.means3D, s.scales, s.rotations, s.sh, s.degrees, f64=False, **kw)
    return o, o64, o32


def tile_of_instances(o, W):
    """Tile index of every entry of the sorted list."""
    return (o["keys"] >> np.uint64(32)).astype(np.int64)


def tile_hi(o, W, H):
    """Largest n_contrib of each tile (the backward's `hi`)."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    pad = np.zeros((gy * 16, gx * 16), np.int64)
    pad[:H, :W] = o["n_contrib"]
    return pad.reshape(gy, 16, gx, 16).max(axis=(1, 3)).reshape(-1)


def _pair_alpha(o, ids, px, py):
    """fp32 power and fp64 raw alpha (before the 0.99 clamp) of Gaussians `ids` at pixel (px, py)."""
    m = o["means2D"][ids].astype(np.float32)
    co = o["conic_opacity"][ids].astype(np.float32)
    dx, dy = m[:, 0] - np.float32(px), m[:, 1] - np.float32(py)
    power = (np.float32(-0.5) * (co[:, 0] * dx * dx + co[:, 2] * dy * dy) - co[:, 1] * dx * dy).astype(np.float64)
    return power, co[:, 3].astype(np.float64) * np.exp(power)


def excluded(case, o):
    """Gaussians whose gradient an ulp of the GPU's exponential may legitimately change.  At each borderline pixel (where some
    pair lies within a few ulp of a threshold the forward branches on) a Gaussian is excluded when
      - its own pair there is near a threshold (alpha 1/255 or 0.99, power 0) or next to the pixel's termination, or
      - it contributes there and has fewer than 2 000 contributing pixels: a flipped decision of another Gaussian changes one
        pixel term by at most a factor 1/(1 - alpha) ~ 1.004; over 2 000 or more terms that stays below the per-element bar.
    A power-0 flip (alpha = opacity) excludes every contributor of the pixel."""
    near, count, _ = borderline_pairs(o, case.W, case.H)
    touched = count > 0
    if not touched.any():
        return near
    stats = o if "touched_pixels" in o else gs_oracle.render_forward_stats(o, o, case.bg, case.W, case.H)
    return near | (touched & (stats["touched_pixels"] < 2000))


def borderline_pairs(o, W, H):
    """-> (near, count, behind): per Gaussian, whether its pair at some borderline pixel is near a threshold or next to that
    pixel's termination (a power-0 flip marks every pair of the pixel that passes), at how many borderline pixels its pair passes
    the alpha test, and at how many of those it lies behind a pair near a threshold (whose flip scales the pixel's T from there
    on by up to 1 / (1 - 1/255))."""
    P = o["radii"].shape[0]
    near = np.zeros(P, bool)
    count = np.zeros(P, np.int64)
    behind = np.zeros(P, np.int64)
    gx = (W + 15) // 16
    ys, xs = np.nonzero(o["borderline"])
    for y, x in zip(ys, xs):
        t = (y // 16) * gx + x // 16
        r0, r1 = (int(v) for v in o["ranges"][t])
        ids = o["point_list"][r0:r1].astype(np.int64)
        power, a = _pair_alpha(o, ids, x, y)
        passes = (power <= 1e-6) & (a >= (1.0 / 255.0) * (1 - 1e-5))
        thr = passes & ((np.abs(a * 255.0 - 1.0) < 1e-5) | (np.abs(a / 0.99 - 1.0) < 1e-5) | (np.abs(power) < 1e-6))
        if thr.any():
            behind[ids[passes & (np.arange(ids.size) > np.argmax(thr))]] += 1
        n = int(o["n_contrib"][y, x])
        after = np.nonzero(passes[n:])[0]
        if n > 0:
            thr[n - 1] = True
        if after.size:
            thr[n + after[0]] = True
        if (passes & (np.abs(power) < 1e-6)).any():
            thr |= passes
        near[ids[thr]] = True
        count[ids[passes]] += 1
    return near, count, behind


def compare(name, o, o64, o32, got, chk, glob=None, verbose=True, bar=(R_REL, A_ABS), arrays=ARRAYS):
    """The per-element check of `got` (a dict of arrays) against the oracle on the Gaussians of mask `chk` -> (ratios, failures).
    The yardsticks are taken per Gaussian (row) of each array: E32 = max over the row of |o32 - o64| and |o64|_row = max over
    the row of |o64|, because the elements of a row share their rounding (they are chained from the same per-Gaussian sums):
        e <= max(K * E32, R_REL * |o64|_row, A_ABS * max|o64|).
    `ratios[array]` = (largest e / max(E32, R_REL |o64|_row, A_ABS max|o64|), largest e / bar); `glob` = (mask, fraction) holds
    those Gaussians to fraction * max|o64| instead; `failures` lists what broke a bar."""
    vis = o["radii"] > 0
    P = vis.shape[0]
    chk = chk & vis
    r_rel, a_abs = bar
    ratios, failures = {}, []
    for n in arrays:
        a = np.asarray(o64[n], np.float64).reshape(P, -1)
        if a.size == 0:
            continue
        a32 = np.asarray(o32[n], np.float64).reshape(P, -1)
        b = np.asarray(got[n], np.float64).reshape(P, -1)
        scale = float(np.abs(a).max())
        e = np.abs(b - a)
        E32 = np.abs(a32 - a).max(axis=1, keepdims=True)
        Arow = np.abs(a).max(axis=1, keepdims=True)
        den = np.maximum(np.maximum(E32, R_REL * Arow), A_ABS * scale)
        bar_ = np.maximum(np.maximum(K * E32, r_rel * Arow), a_abs * scale)
        with np.errstate(divide="ignore", invalid="ignore"):
            rho = np.where(den > 0, e / den, np.where(e > 0, np.inf, 0.0))
            q = np.where(bar_ > 0, e / bar_, np.where(e > 0, np.inf, 0.0))
        ratios[n] = (float(rho[chk].max()), float(q[chk].max())) if chk.any() else (0.0, 0.0)
        bad = chk[:, None] & (e > bar_)
        if bad.any():
            failures.append((n, "per-element", np.unique(np.nonzero(bad)[0])))
        if glob is not None:
            gbad = (glob[0] & vis)[:, None] & (e > glob[1] * scale)
            if gbad.any():
                failures.append((n, "%g of scale (excluded Gaussians)" % glob[1], np.unique(np.nonzero(gbad)[0])))
        if (b[~vis] != 0).any():
            failures.append((n, "culled Gaussians must carry exactly zero", np.unique(np.nonzero((b != 0) & ~vis[:, None])[0])))
    if verbose:
        print("\n[%s] %d of %d visible Gaussians per element; max e / max(E32, %.0e|o64|_row, %.0e max|o64|) and max e / bar: %s" % (
            name, int(chk.sum()), int(vis.sum()), R_REL, A_ABS, ", ".join("%s %.3g %.3g" % (k, v[0], v[1]) for k, v in ratios.items())))
    return ratios, failures


def well_conditioned(case, o):
    """Visible Gaussians every gradient array of which compare_aa checks: on aa_needles those with a c / det0 < AA_WELL_CONDITIONED,
    elsewhere all."""
    vis = o["radii"] > 0
    return vis & (cancellation(case, o) < AA_WELL_CONDITIONED) if case.name == "aa_needles" else vis


def compare_aa(label, case, o, o64, o32, got, chk, glob=None, bar=(R_REL, A_ABS), arrays=ARRAYS):
    """compare() of an anti-aliased backward: every array on the well-conditioned Gaussians, all but ILL_CONDITIONED_ARRAYS on the
    others -> failures."""
    well = well_conditioned(case, o)
    _, failures = compare(label, o, o64, o32, got, chk & well, glob, bar=bar, arrays=arrays)
    if (chk & ~well & (o["radii"] > 0)).any():
        _, more = compare(label + ", a c / det0 >= %g" % AA_WELL_CONDITIONED, o, o64, o32, got, chk & ~well, bar=bar,
                          arrays=[n for n in arrays if n not in ILL_CONDITIONED_ARRAYS])
        failures = failures + more
    return failures


def describe(failures, o, o64, got, W, H, limit=5):
    """Where the failures are: array, Gaussians, the tiles listing them and those tiles' `hi`."""
    tiles, hi = tile_of_instances(o, W), tile_hi(o, W, H)
    pl = o["point_list"]
    P = o["radii"].shape[0]
    lines = []
    for n, what, rows in failures:
        lines.append("%s: %s: %d Gaussians" % (n, what, rows.size))
        a = np.asarray(o64[n], np.float64).reshape(P, -1)
        b = np.asarray(got[n], np.float64).reshape(P, -1)
        for g in rows[:limit]:
            t = np.unique(tiles[pl == g])
            lines.append("  id %d: o64 %s ours %s; tiles %s hi %s" % (g, a[g], b[g], t[:8].tolist(), hi[t[:8]].tolist()))
    return "\n".join(lines)


def clamp_branch(case, o):
    """Visible Gaussians whose |tx/tz| or |ty/tz| exceeds 1.3 tan(fov / 2) (fp32, as the preprocess computes it)."""
    v = case.cam.world_view_transform.numpy().astype(np.float32).reshape(-1)
    m = case.scene.means3D.numpy().astype(np.float32)
    tx = v[0] * m[:, 0] + v[4] * m[:, 1] + v[8] * m[:, 2] + v[12]
    ty = v[1] * m[:, 0] + v[5] * m[:, 1] + v[9] * m[:, 2] + v[13]
    tz = v[2] * m[:, 0] + v[6] * m[:, 1] + v[10] * m[:, 2] + v[14]
    kw = case.cam_kw()
    limx, limy = np.float32(1.3) * np.float32(kw["tan_fovx"]), np.float32(1.3) * np.float32(kw["tan_fovy"])
    return (o["radii"] > 0) & ((np.abs(tx / tz) > limx) | (np.abs(ty / tz) > limy))


def cancellation(case, o):
    """a c / det0 of the undilated screen covariance of every Gaussian, in float64 from the oracle's cov3D: how much of det0 =
    a c - b^2 the fp32 forward loses to cancellation."""
    kw = case.cam_kw()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64))
    _, _, a, b, c = R64.screen_cov(t(case.scene.means3D.numpy()), t(kw["viewmatrix"].numpy()), t(o["cov3D"]), case.W, case.H,
                                   kw["tan_fovx"], kw["tan_fovy"])
    a, b, c = a.numpy(), b.numpy(), c.numpy()
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.abs(a * c / (a * c - b * b))


AA_MIN_CHECKED = 20                          # per AA property below: at least this many Gaussians checked per element


def assert_reaches(case, o, excl):
    """What the case is built for, from the oracle's forward state (so a change to synth cannot quietly drop coverage)."""
    W, H = case.W, case.H
    vis = o["radii"] > 0
    hi = tile_hi(o, W, H)
    counts = (o["ranges"][:, 1] - o["ranges"][:, 0]).astype(np.int64)
    frac = excl[vis].mean() if vis.any() else 0.0
    limit = EXCLUDED_MAX.get(case.name, EXCLUDED_DEFAULT)
    if case.meta.get("aa"):
        limit = EXCLUDED_MAX_AA.get(case.name, limit)
    assert frac <= limit, (case.name, frac)
    if case.name.startswith("staircase"):
        k = case.meta["tile_k"]
        assert np.array_equal(o["tiles_touched"], np.ones_like(o["tiles_touched"])), "every Gaussian's rect is its tile alone"
        assert np.array_equal(counts, k) and np.array_equal(hi, k), (counts.tolist(), hi.tolist())
        d = o["depths"][o["point_list"]].view(np.uint32)
        tiles = tile_of_instances(o, W)
        if case.name.endswith("ties"):
            sel = tiles == TIE_TILE
            assert np.unique(d[sel]).size == 1, "the tie tile repeats one depth"
            assert np.all(np.diff(o["point_list"][sel].astype(np.int64)) > 0), "ties are listed by ascending id"
        else:
            assert all(np.unique(d[tiles == t]).size == k[t] for t in range(k.size)), "depths are distinct within a tile"
        assert o["final_T"].min() > 1e-4
    elif case.name.startswith("odd_"):
        assert vis.any() and hi.max() > 0
        assert not np.array_equal(case.bg.numpy(), np.zeros(3))
    elif case.name == "large":
        big = case.meta["large"]
        r = o["radii"][big]
        assert (r >= 100).sum() >= 30 and r.max() >= 500 and r.min() > 0, r.tolist()
        clamp = clamp_branch(case, o)
        assert clamp[big].sum() >= 8, "the frustum clamp fires for the Gaussians centred beyond 1.3 tan(fov / 2)"
        assert (clamp & ~excl).sum() >= 4, "some of them are checked per element"
    elif case.name == "aa_needles":
        chk = vis & ~excl
        qf = o["aa_q"]
        above, clamped = chk & (qf > AA_MIN_RATIO), chk & (qf <= AA_MIN_RATIO)
        rel = qf.astype(np.float64) / np.float64(AA_MIN_RATIO) - 1.0
        assert (above & (cancellation(case, o) > 1e3)).sum() >= AA_MIN_CHECKED, "needles above the clamp whose det0 cancels"
        assert clamped.sum() >= AA_MIN_CHECKED, "needles whose q_f is clamped (no gradient through q)"
        assert (above & (rel <= 1e-3)).sum() >= 8 and (clamped & (rel >= -1e-3)).sum() >= 8, "q_f within 1e-3 of the clamp"
        # ... and among the Gaussians whose every gradient array is checked (compare_aa), so the clamp decision and the gradient
        # through q reach dL_dcov3D / dL_dscales / dL_drotations / dL_dmeans3D of checked rows
        well = well_conditioned(case, o)
        assert (clamped & well).sum() >= AA_MIN_CHECKED, "clamped needles checked in every array"
        assert (above & well & (rel <= 1e-3)).sum() >= 8 and (clamped & well & (rel >= -1e-3)).sum() >= 8, "near the clamp, every array"
        assert (above & well & (rel > 1e-3)).sum() >= 8, "unclamped needles away from the clamp, every array"
        sig = o["aa_sigmoid"]
        assert (chk & (sig > 0.9)).sum() >= 100 and sig[chk].min() < 0.1 and sig[chk].max() > 0.99
    elif case.name == "aa_subpixel":
        assert ((vis & ~excl) & (o["aa_s"] < 0.1)).sum() >= AA_MIN_CHECKED, "sub-pixel splats: s < 0.1"
        assert np.abs(o["n_contrib"]).max() > 0
    elif case.name == "saturation":
        assert o["clamped"][vis].any(axis=1).sum() >= 20, "SH colours clamped at 0 in some channels"
        terminated = 0
        clamped_alpha = 0
        gx = (W + 15) // 16
        for y in range(H):
            for x in range(W):
                t = (y // 16) * gx + x // 16
                r0, r1 = (int(v) for v in o["ranges"][t])
                ids = o["point_list"][r0:r1].astype(np.int64)
                power, a = _pair_alpha(o, ids, x, y)
                passes = (power <= 0) & (a >= 1.0 / 255.0)
                clamped_alpha += int((passes & (a > 0.99)).sum())
                terminated += int(passes[int(o["n_contrib"][y, x]):].any())
        assert terminated >= W * H // 4, "T < 1e-4 stops many pixels before the end of their list"
        assert clamped_alpha >= 100, "alpha clamps at 0.99"
    else:
        if case.name == "dense_4k":
            assert counts.max() > 2048
        if case.name == "dense_12k":
            assert counts.max() > 8192
        if case.name == "dense_ties":
            assert ((counts > 2048) & (counts <= 8192)).any()
        if case.name == "dense_faint":
            assert hi.max() > 8192, hi.max()
