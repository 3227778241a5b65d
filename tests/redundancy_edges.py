"""The redundancy score of resolution-aware pruning on scenes built to reach its decision boundaries, and its oracle chain.

Shared by test_redundancy_edges_oracle.py (CPU: every scene reaches what it is built for, and the exact comparison rejects
near-misses made with the oracles themselves) and test_gpu_redundancy_edges.py (the kNN, pixel-size, sphere / ellipsoid,
minimum and fused kernels against the chain, bit for bit).

The chain is the "defined" semantics that gsb_redundancy_score documents, from the oracles alone:
  knn_oracle (brute force)  ->  gs_oracle.min_projected_pixel_size  ->  radius ((cube * ps) * fp32(sqrt 3)) / 2 in numpy fp32
  ->  gs_oracle.sphere_ellipsoid_intersection  ->  hits of missing neighbours (index -1) cleared, red = hits + 1
  ->  gs_oracle.min_redundancy_value over [self | neighbours].
A -1 slot is never handed to an oracle or to an unfused entry point (both index with it): it is replaced by the row's own index
(`nb`), and its mask bit cleared afterwards.

Every stage is exact: the kNN's distance and the pixel size are plain IEEE operations with explicit fmaf in the kernel's order.
The sphere test squares with powf(v, 2.0f), which on sm_90a is 1 ulp off v * v for 3.3 % of all floats but never where v * v
is exact (tools/probe_powf_square.py, gs_oracle.cpp square_is_exact); the oracle marks a row `borderline` when one of its pairs
is within 2^-20 of dot = 1 with an inexact square, and no row of these scenes is.

kNN cases (KNN_CASES; distIndex2 at each K, distCUDA2, and the distIndexQ case QUERY):
  p<P>          clustered_cloud at P = 31, 32, 33 (one leaf of 32), 1023..1025 (one level-1 box of 32 leaves), 4095..4097 (the
                onesweep tile), 32768, 32769 (level 2; the last query warp partial)
  lattice       the 32^3 integer lattice in index order, and `lattice_perm` in a seeded permutation: the K-th distance of K = 30
                (d^2 = 4) and K = 64 (d^2 = 6) is tied across leaves and boxes
  duplicates    5 000 copies of one point, 3 000 points within 1e-3 of it and 2 000 around: zero-distance ties over ~157 leaves
                and five level-1 boxes
  overflow      a 1e-3 cluster with outliers at +-1e6 (finite), +-1e20 (the square overflows), +-3e38 (the difference
                overflows) and (+-1.4e19, +-1.4e19, 0) (the sum of squares overflows): overflowed pairs are never neighbours
  denormal      a cluster whose squared distances are subnormal, and one whose coordinates are
  nonfinite     a cluster with rows holding NaN, +inf or -inf: never neighbours, their own rows (FLT_MAX, -1)
Redundancy scenes (SCENES; each runs the whole chain):
  planes        cameras W > H, W = H, W < H 1000 apart, centres bisected in fp32 against the oracle across each camera's planes
                qx = +-1, qy = +-1, qz = 0 and qz = 1; a fourth camera with integer matrix entries that puts centres at qz = 0
                exactly; centres where ph[3] + 1e-7 is 0 and +-2^-47 (the sum of two floats near 1e-7 cannot be subnormal)
  cams_1024     1 024 cameras (the kernel's limit) of many shapes, and centres no camera sees (10000)
  sphere_k<K>   K = 1, 30, 64, one camera, general and 90-degree-swap rotations; 48 planted pairs whose `dot` is exactly
                1 - 2^-24 (hit) or 1.0 (no hit), each with exact squares (see _planted); unseen centres (radius from 10000) that
                hit every neighbour, up to slot 63 at K = 64 (bit 63 of the fused mask); with the neighbour's rotation many
                decisions flip, the planted ones among them
  zero          pixel_scale 0 (radius 0), zero scales and exact duplicates: rcp(0) * 0 is NaN, no hit
  small_p<P>_k<K>  P <= K: missing slots
"""
import math

import numpy as np
import torch

import gs_oracle
import knn_cases as KC
import knn_oracle
from gs_b200 import synth

F32 = np.float32
FLT_MAX = np.finfo(F32).max
SQRT3 = np.sqrt(F32(3.0))                   # torch.sqrt(torch.tensor([3])) in fp32, and the fused kernel's __fsqrt_rn(3.0f)
ONE_BELOW = np.nextafter(F32(1.0), F32(0.0))
KMAX = 64
N_MIN = 8                                   # boundary pairs each scene must reach per plane / class

KNN_PS = (31, 32, 33, 1023, 1024, 1025, 4095, 4096, 4097, 32768, 32769)
KNN_KS = (1, 3, 30, 64)
KNN_CASES = {**{"p%d" % p: KNN_KS for p in KNN_PS}, "lattice": (30, 64), "lattice_perm": (30, 64), "duplicates": KNN_KS,
             "overflow": KNN_KS, "denormal": (3, 30), "nonfinite": (3, 30, 64)}
QUERY_KS = (1, 30, 64)
SCENES = ["planes", "cams_1024", "sphere_k1", "sphere_k30", "sphere_k64", "zero", "small_p1_k30", "small_p20_k30", "small_p30_k30",
          "small_p64_k64"]


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


# ---- kNN ---------------------------------------------------------------------------------------------------------------------

def knn_points(name):
    """float32 [P, 3] of kNN case `name`."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("p"):
        return KC.clustered_cloud(int(name[1:]), 100 + int(name[1:])).numpy()
    if name.startswith("lattice"):
        g = np.stack(np.meshgrid(np.arange(32), np.arange(32), np.arange(32), indexing="ij"), -1).reshape(-1, 3).astype(F32)
        return g[np.random.default_rng(17).permutation(g.shape[0])] if name == "lattice_perm" else g
    if name == "duplicates":
        c = np.array([0.25, -0.5, 0.75], F32)
        pts = np.concatenate([np.repeat(c[None], 5000, 0), c + rng.uniform(-1e-3, 1e-3, (3000, 3)), c + rng.normal(0, 0.3, (2000, 3))])
        return pts[rng.permutation(pts.shape[0])].astype(F32)
    if name == "overflow":
        out = []
        for v in (1e6, 1e20, 3e38):
            for a in range(3):
                for s in (1, -1):
                    p = np.zeros(3)
                    p[a] = s * v
                    out.append(p)
        out += [(x, y, 0.0) for x in (1.4e19, -1.4e19) for y in (1.4e19, -1.4e19)]
        pts = np.concatenate([rng.uniform(-1e-3, 1e-3, (2000, 3)), np.array(out)]).astype(F32)
        return pts[rng.permutation(pts.shape[0])]
    if name == "denormal":
        return np.concatenate([rng.uniform(-1e-19, 1e-19, (1000, 3)), rng.uniform(-1e-40, 1e-40, (500, 3))]).astype(F32)
    if name == "nonfinite":
        pts = rng.uniform(-1, 1, (1000, 3)).astype(F32)
        bad = rng.choice(1000, 30, replace=False)
        for j, r in enumerate(bad):
            pts[r, j % 3] = (np.nan, np.inf, -np.inf)[j % 3]
        return pts
    raise KeyError(name)


def knn_oracle_rows(pts, K=KMAX, q=None, n=None):
    """The oracle's rows at K = KMAX as [rows, KMAX] (dist, index): the rows at any K <= KMAX are their first K columns (a row
    is the K smallest (distance, index) keys, in order)."""
    d, i, _ = knn_oracle.knn(pts, K, q, n)
    return d.reshape(-1, K), i.reshape(-1, K)


def mean3(d):
    """distCUDA2 from the first three columns: ((d0 + d1) + d2) / 3 in fp32 (simple_knn.cu:184)."""
    with np.errstate(over="ignore"):
        return ((d[:, 0] + d[:, 1]) + d[:, 2]) / F32(3.0)


def query_case():
    """(points, q_indices, n_indices) of the distIndexQ case: repeated query ids, queries that are no candidates, repeated candidate
    ids, and a candidate list longer than P whose entries beyond the first P list ids that must not count."""
    pts = KC.clustered_cloud(5000, 77).numpy()
    rng = np.random.default_rng(78)
    P = pts.shape[0]
    even = np.arange(0, P, 2)
    q = np.concatenate([rng.choice(P, 600), np.repeat(rng.choice(P, 20), 5), np.arange(1, 200, 2)]).astype(np.int32)
    n = np.concatenate([rng.choice(even, P - 400), np.repeat(even[:100], 4), np.arange(1, P, 2)[:1500]]).astype(np.int32)
    return pts, q, n


def morton_rank(pts):
    """Sorted position of each point in the kNN's (90-bit Morton code, index) order (gsb_knn.cu knn_grid / knn_cell / knn_word):
    position // 32 is its leaf, position // 1024 its level-1 box.  Finite inputs only."""
    p = pts.astype(np.float64)
    lo, ext = p.min(0), p.max(0) - p.min(0)
    scale = np.where((ext > 0) & (ext <= 1e300), 1073741823.0 / np.where(ext > 0, ext, 1.0), 0.0)
    cell = np.fmin(np.fmax((p - lo) * scale, 0.0), 1073741823.0).astype(np.int64).tolist()
    keys = []
    for j, c in enumerate(cell):
        k = 0
        for b in range(29, -1, -1):
            k = (k << 3) | (((c[2] >> b) & 1) << 2) | (((c[1] >> b) & 1) << 1) | ((c[0] >> b) & 1)
        keys.append((k, j))
    rank = np.empty(pts.shape[0], np.int64)
    rank[[j for _, j in sorted(keys)]] = np.arange(pts.shape[0])
    return rank


def kth_ties(pts, K, d, i):
    """Rows whose K-th distance is shared by a candidate beyond slot K, with the tied candidates' indices: -> {row: ids}."""
    out = {}
    for r in np.nonzero((d[:, K - 1] == d[:, K]) & (d[:, K - 1] < FLT_MAX))[0]:
        t = d[r, K - 1]
        out[int(r)] = i[r][d[r] == t]
    return out


# ---- cameras and scenes --------------------------------------------------------------------------------------------------------

class Cam:
    """The camera attributes the redundancy score reads (the reference's Camera), with the inverse fixed on the host so that the
    kernels and the oracle get the same matrices."""

    def __init__(self, proj, W, H, inv=None):
        self.full_proj_transform = torch.as_tensor(proj, dtype=torch.float32).contiguous()
        self.inverse_full_proj_transform = (self.full_proj_transform.inverse() if inv is None else
                                            torch.as_tensor(inv, dtype=torch.float32)).contiguous()
        self.image_width, self.image_height = int(W), int(H)

    @staticmethod
    def synth(c):
        return Cam(c.full_proj_transform, c.image_width, c.image_height)

    def to(self, dev):
        return Cam(self.full_proj_transform.to(dev), self.image_width, self.image_height, self.inverse_full_proj_transform.to(dev))


class Scene:
    def __init__(self, name, xyz, scales, rots, cams, K, ps=1.0, meta=None):
        self.name, self.K, self.ps, self.meta = name, int(K), float(ps), meta or {}
        self.xyz, self.scales, self.rots = (np.ascontiguousarray(a, F32) for a in (xyz, scales, rots))
        self.cams = cams
        self.P = self.xyz.shape[0]

    def cam_arrays(self):
        return (np.stack([c.full_proj_transform.numpy() for c in self.cams]), np.stack([c.inverse_full_proj_transform.numpy() for c in self.cams]),
                np.array([c.image_height for c in self.cams], np.int32), np.array([c.image_width for c in self.cams], np.int32))

    def on(self, dev):
        """The scene as calculate_redundancy_metric reads it (the reference's Scene), on `dev`."""
        s = self

        class G:
            _xyz = torch.from_numpy(s.xyz).to(dev)
            get_scaling = torch.from_numpy(s.scales).to(dev)
            get_rotation = torch.from_numpy(s.rots).to(dev)

        class S:
            gaussians = G()
            cams = [c.to(dev) for c in s.cams]

            def getTrainCameras(self):
                return self.cams
        return S()


def radius(px, ps):
    """scene/__init__.py:156-157 in fp32: ((cube_size * pixel_scale) * sqrt(3)) / 2."""
    return ((np.asarray(px, F32) * F32(ps)) * SQRT3) / F32(2.0)


def pixel_size(xyz, cams):
    s = Scene("", np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 4)), cams, 1)
    projs, invs, H, W = s.cam_arrays()
    return gs_oracle.min_projected_pixel_size(projs, invs, np.ascontiguousarray(xyz, F32), H, W).reshape(-1)


def chain(s):
    """The oracle chain of scene `s` -> dict of every stage: dist, idx [P, K]; px [P, 1]; rad [P, 1]; nb [P, K] (missing slots ->
    own index); raw_red [P, 1], raw_mask [P, K] (the unfused sphere test on nb), dots, borderline; mask (missing cleared), red
    (hits + 1) [P, 1]; cat_idx, cat_mask [P, K + 1]; minimum [P, 1]."""
    P, K = s.P, s.K
    d, i = knn_oracle_rows(s.xyz, K)
    projs, invs, H, W = s.cam_arrays()
    px = gs_oracle.min_projected_pixel_size(projs, invs, s.xyz, H, W)
    rad = radius(px, s.ps)
    own = np.arange(P, dtype=np.int32)[:, None]
    valid = i >= 0
    nb = np.where(valid, i, own).astype(np.int32)
    raw_red, raw_mask, bl, dots = gs_oracle.sphere_ellipsoid_intersection(s.xyz, s.scales, s.rots, nb, rad, K, dots=True)
    mask = raw_mask & valid
    red = mask.sum(1, keepdims=True).astype(np.int32) + 1
    cat_idx = np.ascontiguousarray(np.concatenate([own, nb], 1), np.int32)
    cat_mask = np.concatenate([np.ones((P, 1), bool), mask], 1)
    minimum = gs_oracle.min_redundancy_value(red, cat_idx, cat_mask, K + 1)
    return dict(dist=d, idx=i, px=px, rad=rad, nb=nb, raw_red=raw_red, raw_mask=raw_mask, dots=dots, borderline=bl, mask=mask,
                red=red, cat_idx=cat_idx, cat_mask=cat_mask, minimum=minimum)


def pair_test(ci, ri, rad_i, cn, sn, rn=None):
    """The oracle's sphere test of M pairs (centre ci [M,3] with rotation ri [M,4] and radius rad_i [M] against the neighbour at cn
    with scales sn), rotation of the centre unless `rn` (the neighbour's) is given -> (hit [M], dot [M])."""
    M = ci.shape[0]
    rot = ri if rn is None else rn
    xyz = np.concatenate([ci, cn]).astype(F32)
    sc = np.concatenate([np.zeros_like(sn), sn]).astype(F32)
    rots = np.concatenate([rot, rot]).astype(F32)
    rad = np.concatenate([np.asarray(rad_i, F32).reshape(-1), np.zeros(M, F32)])
    nb = np.concatenate([np.arange(M, 2 * M), np.arange(M)]).astype(np.int32).reshape(-1, 1)
    _, mask, _, dots = gs_oracle.sphere_ellipsoid_intersection(xyz, sc, rots, nb, rad, 1, dots=True)
    return mask[:M, 0], dots[:M, 0]


def neighbour_rotation_mask(s, o):
    """The mask the sphere test gives with each neighbour's own rotation instead of the current Gaussian's (the reference's quirk
    undone) on o's neighbours."""
    P, K = s.P, s.K
    r = np.repeat(np.arange(P), K)
    n = o["nb"].reshape(-1)
    hit, _ = pair_test(s.xyz[r], s.rots[r], np.repeat(o["rad"].reshape(-1), K), s.xyz[n], s.scales[n], rn=s.rots[n])
    return hit.reshape(P, K) & (o["idx"] >= 0)


def _key(f):
    i = np.asarray(f, F32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7fffffff), i)


def _unkey(k):
    k = np.asarray(k, np.int64)
    return np.where(k < 0, (-k) | 0x80000000, k).astype(np.uint32).view(F32)


def bisect(lo, hi, pred):
    """Elementwise over fp32: pred(lo) true, pred(hi) false -> adjacent floats (a, b) with pred(a) true and pred(b) false."""
    a, b = _key(lo), _key(hi)
    while True:
        gap = np.abs(b - a) > 1
        if not gap.any():
            return _unkey(a), _unkey(b)
        m = np.where(gap, (a + b) // 2, a)
        p = pred(_unkey(m))
        a, b = np.where(gap & p, m, a), np.where(gap & ~p, m, b)


def _quats(rng, n):
    """Unit quaternions (r, x, y, z): half general, half 90-degree swaps about x, y or z (either sign) or the axis cycle."""
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    h = F32(math.sqrt(0.5))
    swaps = np.array([[h, h, 0, 0], [h, 0, h, 0], [h, 0, 0, h], [h, -h, 0, 0], [h, 0, -h, 0], [h, 0, 0, -h], [0.5, 0.5, 0.5, 0.5]], F32)
    sw = rng.random(n) < 0.5
    q[sw] = swaps[rng.integers(0, len(swaps), int(sw.sum()))]
    return q.astype(F32), sw


def _fill(rng, xyz, log_scale=math.log(0.01)):
    n = xyz.shape[0]
    q, _ = _quats(rng, n)
    return np.exp(log_scale + 0.5 * rng.normal(size=(n, 3))).astype(F32), q


# ---- planes --------------------------------------------------------------------------------------------------------------------
PLANES = ("qx=+1", "qx=-1", "qy=+1", "qy=-1", "qz=0", "qz=1")
PLANE_CAMS = ((64, 48), (40, 40), (36, 60))   # W > H, W = H, W < H, at x = 0, 1000, 2000 looking +z
N_LINES = 12
NICE_X = 3000.0


def nice_camera():
    """ph = (x - 3000, y, z - 1, z): integer entries, so qz = 0 exactly at z = 1."""
    m = np.zeros(16)
    m[0], m[12], m[5], m[10], m[14], m[11] = 1.0, -NICE_X, 1.0, 1.0, -1.0, 1.0
    M = torch.tensor(m.reshape(4, 4), dtype=torch.float64)
    return Cam(M.float(), 40, 40, M.inverse().float())


def ndc(xyz, cam):
    """(qx, qy, qz, ph3 + 1e-7) in float64 from the fp32 inputs (to name the plane a bisected pair straddles)."""
    m = cam.full_proj_transform.numpy().astype(np.float64).reshape(-1)
    p = np.asarray(xyz, np.float64)
    ph = [p[:, 0] * m[r] + p[:, 1] * m[4 + r] + p[:, 2] * m[8 + r] + m[12 + r] for r in range(4)]
    w = ph[3] + 1e-7
    with np.errstate(divide="ignore", invalid="ignore"):
        return ph[0] / w, ph[1] / w, ph[2] / w, w


def _planes():
    rng = np.random.default_rng(5)
    cams = [Cam.synth(synth.make_camera(W, H, np.eye(3), np.array([-1000.0 * c, 0.0, 0.0]))) for c, (W, H) in enumerate(PLANE_CAMS)]
    nice = nice_camera()
    pts, groups = [], {}

    def add(name, a):
        groups[name] = np.arange(sum(len(x) for x in pts), sum(len(x) for x in pts) + len(a))
        pts.append(np.asarray(a, F32))

    for c, cam in enumerate(cams):
        ox = F32(1000.0 * c)
        inside = lambda p, cam=cam: pixel_size(p, [cam]) < 10000  # noqa: E731
        n = N_LINES
        z0 = rng.uniform(0.5, 5.0, n)
        small = rng.uniform(-0.2, 0.2, n) * z0
        for plane in PLANES:
            base = np.zeros((n, 3))
            if plane.startswith("qx"):
                axis, sign = 0, float(plane[3] + "1")
                base[:, 1], base[:, 2] = small, z0
                lo, hi = np.full(n, ox, F32), (ox + sign * 10.0 * z0).astype(F32)
            elif plane.startswith("qy"):
                axis, sign = 1, float(plane[3] + "1")
                base[:, 0], base[:, 2] = ox + small, z0
                lo, hi = np.zeros(n, F32), (sign * 10.0 * z0).astype(F32)
            elif plane == "qz=0":
                axis = 2
                base[:, 0], base[:, 1] = ox + rng.uniform(-1e-3, 1e-3, n), rng.uniform(-1e-3, 1e-3, n)
                lo, hi = np.ones(n, F32), np.full(n, 1e-3, F32)
            else:
                axis = 2
                base[:, 0], base[:, 1] = ox + rng.uniform(-5, 5, n), rng.uniform(-5, 5, n)
                lo, hi = np.full(n, 50.0, F32), np.full(n, 200.0, F32)
            base = base.astype(F32)

            def pred(v, base=base, axis=axis, inside=inside):
                p = base.copy()
                p[:, axis] = v
                return inside(p)
            a, b = bisect(lo, hi, pred)
            pa, pb = base.copy(), base.copy()
            pa[:, axis], pb[:, axis] = a, b
            add("cam%d %s in" % (c, plane), pa)
            add("cam%d %s out" % (c, plane), pb)
    # qz = 0 exactly on the integer camera, and the float below z = 1 (qz < 0)
    n = 16
    xy = rng.uniform(-0.8, 0.8, (n, 2)).astype(F32)
    exact = np.stack([F32(NICE_X) + xy[:, 0], xy[:, 1], np.ones(n, F32)], 1)
    add("nice qz=0 exact", exact)
    below = exact.copy()
    below[:, 2] = ONE_BELOW
    add("nice qz<0", below)
    # ph[3] + 1e-7 == 0 and +-2^-47 on camera 0 (at the origin, R = I: ph[3] = z exactly)
    z = -F32(1e-7)
    xs = np.array([[0, 0], [0.5, 0], [0, -0.5], [1e-9, 1e-9]], F32)
    add("w+1e-7 == 0", np.concatenate([xs, np.full((4, 1), z, F32)], 1))
    add("w+1e-7 tiny", np.concatenate([np.concatenate([xs, xs]), np.concatenate([np.full((4, 1), np.nextafter(z, F32(-1))),
                                                                                 np.full((4, 1), np.nextafter(z, F32(1)))])], 1))
    xyz = np.concatenate(pts)
    sc, q = _fill(rng, xyz)
    return Scene("planes", xyz, sc, q, cams + [nice], 30, 1.0, dict(groups=groups, plane_cams=cams, nice=nice))


def _cams_1024():
    rng = np.random.default_rng(6)
    cams = []
    for k in range(1024):
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        C = d * rng.uniform(3.0, 8.0)
        zc = -d
        up = np.array([0.0, 1.0, 0.0]) if abs(zc[1]) < 0.9 else np.array([1.0, 0.0, 0.0])
        xc = np.cross(up, zc)
        xc /= np.linalg.norm(xc)
        R = np.stack([xc, np.cross(zc, xc), zc], 1)
        W, H = int(rng.integers(8, 200)), int(rng.integers(8, 200))
        cams.append(Cam.synth(synth.make_camera(W, H, R, -R.T @ C, fovy_deg=float(rng.uniform(20, 90)))))
    xyz = np.concatenate([rng.uniform(-2, 2, (3000, 3)), rng.uniform(-1, 1, (64, 3)) + np.array([500.0, 500.0, 500.0])]).astype(F32)
    sc, q = _fill(rng, xyz, math.log(0.02))
    return Scene("cams_1024", xyz, sc, q, cams, 30, 1.0, dict(unseen=np.arange(3000, 3064)))


# ---- sphere / ellipsoid --------------------------------------------------------------------------------------------------------
# The device's powf(v, 2.0f) is 1 ulp off v * v for 3.3 % of all floats, never where v * v is exact (gs_oracle.cpp,
# square_is_exact).  So the pairs planted at dot = 1 have exact squares: the centre on a 2^-14 grid with the identity rotation (its
# rotated offsets are the offsets themselves), the neighbour at an integer offset (a, b, c) * 2^-14 with a^2 + b^2 + c^2 within 2 of
# T^2, T < 2^12, and its three scales set so that scale + radius == T * 2^-14 in fp32.  Of those pairs, the ones whose dot rounds
# to 1 - 2^-24 (a hit) or to 1.0 (no hit) are kept.
N_PAIRS = 48
GRID = 2.0 ** -14


def _planted(rng, n, rad_of):
    """n isolated (centre, neighbour) pairs whose dot is 1 - 2^-24 or 1.0 -> (xyz [2m, 3], scales of the neighbours [m, 3], target [m])."""
    cands = []
    while len(cands) < 12 * n:
        T = int(rng.integers(1400, 4096))
        a, b = int(rng.integers(0, T)), int(rng.integers(0, T))
        r = T * T - a * a - b * b
        if r < 0:
            continue
        c = int(round(math.sqrt(r)))
        if abs(a * a + b * b + c * c - T * T) <= 2:
            cands.append((a * rng.choice((-1, 1)), b * rng.choice((-1, 1)), c * rng.choice((-1, 1)), T))
    cands = np.array(cands, np.int64)
    m = len(cands)
    # centres on a lattice 0.5 apart (a pair spans at most 0.25) in a slab 3 to 6 units beyond the origin, in view of the camera
    j = np.arange(m)
    ci = np.stack([-3.0 + 0.5 * (j % 12), -2.5 + 0.5 * ((j // 12) % 10), 3.0 + 0.5 * (j // 120)], 1).astype(F32)
    ci = (np.round(ci / GRID) * GRID).astype(F32)
    cn = (ci + cands[:, :3] * GRID).astype(F32)
    rad = rad_of(ci)
    Tf = (cands[:, 3] * GRID).astype(F32)
    s = (Tf - rad).astype(F32)
    for _ in range(4):                         # scale + radius == T * 2^-14 in fp32
        err = (s + rad).astype(F32) - Tf
        s = np.where(err > 0, np.nextafter(s, F32(-1)), np.where(err < 0, np.nextafter(s, F32(1)), s)).astype(F32)
    ok = ((s + rad).astype(F32) == Tf) & (s > 0)
    sn = np.repeat(s[:, None], 3, 1)
    ident = np.tile(np.array([1, 0, 0, 0], F32), (m, 1))
    _, dot = pair_test(ci, ident, rad, cn, sn)
    below, at = ok & (dot == ONE_BELOW), ok & (dot == F32(1.0))
    pick = np.concatenate([np.nonzero(below)[0][: n // 2], np.nonzero(at)[0][: n - n // 2]])
    return ci[pick], cn[pick], sn[pick], dot[pick]


def _sphere(K):
    rng = np.random.default_rng(10 + K)
    cam = Cam.synth(synth.make_camera(80, 60))
    nb_ = 12
    centres = rng.uniform(-1.2, 1.2, (nb_, 3))
    lab = rng.integers(0, nb_, 3000)
    seen = centres[lab] + rng.normal(size=(3000, 3)) * rng.uniform(0.05, 0.2, nb_)[lab, None]
    unseen = rng.normal(size=(100, 3)) * 0.1 + np.array([0.0, 0.0, -6.0])     # behind the camera (at z = -4)
    base = np.concatenate([seen, unseen]).astype(F32)
    sc, q = _fill(rng, base)
    ci, cn, sn, dot = _planted(rng, N_PAIRS, lambda c: radius(pixel_size(c, [cam]), 1.0).reshape(-1))
    m = ci.shape[0]
    P0 = base.shape[0]
    xyz = np.concatenate([base, ci, cn])
    q_c, _ = _quats(rng, m)
    rots = np.concatenate([q, np.tile(np.array([1, 0, 0, 0], F32), (m, 1)), q_c])
    scs = np.concatenate([sc, np.exp(math.log(0.01) + 0.5 * rng.normal(size=(m, 3))).astype(F32), sn])
    pairs = (P0 + np.arange(m), P0 + m + np.arange(m))
    return Scene("sphere_k%d" % K, xyz, scs, rots, [cam], K, 1.0, dict(pairs=pairs, dot=dot, unseen=np.arange(3000, P0)))


def _zero():
    rng = np.random.default_rng(20)
    cam = Cam.synth(synth.make_camera(80, 60))
    base = rng.normal(size=(400, 3)).astype(F32) * 0.05
    sc, q = _fill(rng, base, math.log(0.05))
    zero = rng.choice(400, 120, replace=False)
    sc[zero] = 0.0
    dup = zero[:100]
    xyz = np.concatenate([base, base[dup]])
    return Scene("zero", xyz, np.concatenate([sc, sc[dup]]), np.concatenate([q, q[dup]]), [cam], 30, 0.0,
                 dict(zero_scale=np.concatenate([zero, 400 + np.arange(100)]), dup=(dup, 400 + np.arange(100))))


def _small(P, K):
    rng = np.random.default_rng(30 + P)
    cam = Cam.synth(synth.make_camera(80, 60))
    xyz = (rng.normal(size=(P, 3)) * 0.05).astype(F32)
    sc, q = _fill(rng, xyz, math.log(0.03))
    return Scene("small_p%d_k%d" % (P, K), xyz, sc, q, [cam], K, 1.0)


def build(name):
    if name == "planes":
        return _planes()
    if name == "cams_1024":
        return _cams_1024()
    if name.startswith("sphere_k"):
        return _sphere(int(name[8:]))
    if name == "zero":
        return _zero()
    if name.startswith("small_p"):
        p, k = name[7:].split("_k")
        return _small(int(p), int(k))
    raise KeyError(name)


# ---- the comparison --------------------------------------------------------------------------------------------------------------

def compare(what, want, got, allow=None):
    """Exact comparison (floats by their bits) -> list of failure strings; `allow` [rows] masks rows the oracle marks borderline."""
    want, got = np.asarray(want), np.asarray(got)
    if want.shape != got.shape:
        return ["%s: shape %s, expected %s" % (what, got.shape, want.shape)]
    if want.dtype.kind == "f":
        bad = bits(want) != bits(got)
    else:
        bad = want != got
    bad = bad.reshape(bad.shape[0], -1).any(1)
    if allow is not None:
        bad &= ~np.asarray(allow).reshape(-1)
    if not bad.any():
        return []
    rows = np.nonzero(bad)[0]
    r = rows[0]
    return ["%s: %d rows differ, first %d: expected %s, got %s" % (what, rows.size, r, want[r].reshape(-1)[:8], got[r].reshape(-1)[:8])]
