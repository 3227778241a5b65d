"""Definitions of the kNN golden cases (the reference's simple_knn._C: distCUDA2, distIndex2, distIndexQ).  Inputs are regenerated
from seeds; only the reference's outputs are stored (tests/golden/make_golden_knn.py).

    kn1      ~8 k points of a clustered, multi-scale cloud (clustered_cloud): raw distCUDA2, distIndex2 at K = 1, 3, 30, and one
             distIndexQ with a query subset and a candidate list longer than P (only its first P entries count)
    kn_edge  P = 1..5 at K = 30; all points identical; all on one plane; all on one line
    kn_red   the redundancy score of scene/__init__.py:142-174 end to end (distIndex2 -> sphere_ellipsoid_intersection ->
             allocate_minimum_redundancy_value) on a t1-like scene of 20 k Gaussians
    kn_large compact records at 3 M points: the C3 positions and clustered_cloud at that size
"""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import cases  # noqa: E402

KNN_CASES = {
    "kn1": dict(P=8_192, seed=41, ks=(1, 3, 30), q_count=1_500, q_k=8, n_extra=1_000),
    "kn_red": dict(P=20_000, K=30),
    "kn_large": dict(P=3_000_000, seed=43, K=30, rows=2_048),
}
EDGE_K = 30


def clustered_cloud(P: int, seed: int) -> torch.Tensor:
    """float32 [P,3]: Gaussian blobs of sizes from 0.01 to 0.3, a sparse far shell (background, ~8 %), a few far outliers and ~2 %
    exact duplicates of other points (densification clones)."""
    rng = np.random.default_rng(seed)
    n_shell = int(P * 0.08)
    n_out = min(5, max(P // 1000, 1))
    n_blob = P - n_shell - n_out
    nb = 24
    centres = rng.uniform(-3.0, 3.0, (nb, 3))
    sig = np.exp(rng.uniform(math.log(0.01), math.log(0.3), nb))
    w = rng.uniform(0.2, 1.0, nb)
    lab = rng.choice(nb, n_blob, p=w / w.sum())
    blob = centres[lab] + rng.standard_normal((n_blob, 3)) * sig[lab, None]
    d = rng.standard_normal((n_shell, 3))
    shell = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(40.0, 60.0, (n_shell, 1))
    d = rng.standard_normal((n_out, 3))
    out = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(500.0, 2000.0, (n_out, 1))
    pts = np.concatenate([blob, shell, out]).astype(np.float32)
    pts = pts[rng.permutation(P)]
    n_dup = int(P * 0.02)
    dst = rng.choice(P, n_dup, replace=False)
    pts[dst] = pts[rng.choice(P, n_dup)]
    return torch.from_numpy(np.ascontiguousarray(pts))


def kn1_inputs():
    """(points, q_indices, n_indices) of kn1.  n_indices has P + n_extra entries: P drawn from the even ids, then odd ids that a
    correct implementation of the reference's quirk must ignore."""
    c = KNN_CASES["kn1"]
    pts = clustered_cloud(c["P"], c["seed"])
    rng = np.random.default_rng(c["seed"] + 1)
    q = rng.choice(c["P"], c["q_count"], replace=False).astype(np.int32)
    n = np.concatenate([rng.choice(np.arange(0, c["P"], 2), c["P"]), rng.choice(np.arange(1, c["P"], 2), c["n_extra"])]).astype(np.int32)
    return pts, torch.from_numpy(q), torch.from_numpy(n)


def edge_inputs():
    """{name: float32 [P,3]} of kn_edge."""
    rng = np.random.default_rng(42)
    out = {f"p{P}": torch.from_numpy(rng.uniform(-1.0, 1.0, (P, 3)).astype(np.float32)) for P in range(1, 6)}
    out["same"] = torch.tensor([[1.5, -2.0, 0.25]], dtype=torch.float32).repeat(100, 1).contiguous()
    pl = rng.uniform(-1.0, 1.0, (400, 3)).astype(np.float32)
    pl[:, 2] = 0.5
    out["plane"] = torch.from_numpy(pl)
    ln = np.zeros((300, 3), np.float32)
    ln[:, 0] = rng.uniform(-5.0, 5.0, 300)
    ln[:, 1], ln[:, 2] = -1.0, 2.0
    out["line"] = torch.from_numpy(ln)
    return out


def red_inputs():
    """(case, scene, cams) of kn_red: the t1 tools scene at 20 k Gaussians."""
    c, scene, cams, _ = cases.build_tools_inputs("t1", P=KNN_CASES["kn_red"]["P"])
    return c, scene, cams


def c3_positions(P: int) -> torch.Tensor:
    """The means3D of synth.config_scene("C3", P) without drawing the rest of the scene (make_scene's first draws: uniform positions
    in the box, then the near-plane fraction)."""
    g = torch.Generator().manual_seed(3)
    xyz = (torch.rand(P, 3, generator=g) * 2.0 - 1.0) * torch.tensor((3.6, 2.0, 1.0))
    n_near = int(round(P * 0.001))
    if n_near > 0:
        idx = torch.randperm(P, generator=g)[:n_near]
        xyz[idx, 2] = -4.5 + 0.7 * torch.rand(n_near, generator=g)
    return xyz.contiguous()


def large_inputs(P=None):
    """{name: float32 [P,3]} (default 3 M): the C3 positions and the kn1 distribution at that size."""
    P = P or KNN_CASES["kn_large"]["P"]
    return {"C3": c3_positions(P), "clustered": clustered_cloud(P, KNN_CASES["kn_large"]["seed"])}


def redundancy_pipeline(knn_mod, C_mod, scene, cams, pixel_scale, K=30, dev="cuda"):
    """Reference scene/__init__.py:142-174 calculate_redundancy_metric, with `knn_mod` in the place of simple_knn._C and `C_mod` in
    the place of diff_gaussian_rasterization._C.  -> (min_redundancy int32 [P,1], redundancy [P,1] (+1 applied), indices [P,K])."""
    ct = {k: v.to(dev) for k, v in cases.tools_camera_tensors(cams).items()}
    xyz, scaling, rotation = scene.means3D.to(dev), scene.scales.to(dev), scene.rotations.to(dev)
    opacity = scene.opacity.to(dev)
    P = xyz.shape[0]
    cube_size = C_mod.find_minimum_projected_pixel_size(ct["projs"], ct["inv_projs"], xyz, ct["H"], ct["W"])
    scaled_pixel_size = cube_size * pixel_scale
    half_diagonal = scaled_pixel_size * torch.sqrt(torch.tensor([3], device=dev)) / 2
    _, indices = knn_mod.distIndex2(xyz, K)
    indices = indices.view(-1, K)
    red, mask = C_mod.sphere_ellipsoid_intersection(xyz, scaling, rotation, indices, half_diagonal, K)
    red += 1
    idx = torch.cat((torch.arange(P, device=dev, dtype=torch.int).view(-1, 1), indices), dim=1)
    mk = torch.cat((torch.ones_like(opacity, device=dev, dtype=bool), mask), dim=1)
    min_red = C_mod.allocate_minimum_redundancy_value(red, idx, mk, K + 1)[0]
    return min_red, red, indices


def sorted_rows(d, i, K):
    """Rows of a flat (dists, indices) pair sorted by (distance, index), as numpy [rows, K] arrays."""
    d = np.asarray(d.cpu() if hasattr(d, "cpu") else d, np.float32).reshape(-1, K)
    i = np.asarray(i.cpu() if hasattr(i, "cpu") else i, np.int32).reshape(-1, K)
    key = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | i.view(np.uint32).astype(np.uint64)
    o = np.argsort(key, axis=1, kind="stable")
    return np.take_along_axis(d, o, 1), np.take_along_axis(i, o, 1)


def boundary_ties(d_k1, K):
    """Rows whose K-th and (K+1)-th smallest distances are equal, from the sorted distances of a K+1 search: there several
    candidates compete for the last slot, and which one is kept is not part of the contract."""
    d = np.sort(np.asarray(d_k1, np.float32).reshape(-1, K + 1), axis=1)
    return np.nonzero((d[:, K - 1] == d[:, K]) & (d[:, K - 1] < np.finfo(np.float32).max))[0].astype(np.int64)


def sorted_rows_t(d: torch.Tensor, i: torch.Tensor, K: int):
    """sorted_rows on the device (large cases): -> (dists [rows, K], indices [rows, K]) tensors."""
    key = (d.view(torch.int32).to(torch.int64) << 32) | (i.to(torch.int64) & 0xFFFFFFFF)
    key = key.view(-1, K).sort(dim=1).values
    return (key >> 32).to(torch.int32).view(torch.float32), (key & 0xFFFFFFFF).to(torch.int32)
