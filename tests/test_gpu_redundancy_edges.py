"""GPU: the redundancy score of resolution-aware pruning against the oracle chain of tests/redundancy_edges.py, exactly (floats by
their bits, integers and masks equal), on every kNN case and redundancy scene:
  - simple_knn._C distIndex2 at each K of a case, distCUDA2, and distIndexQ on the query case: distances as bits and indices;
  - _C.find_minimum_projected_pixel_size (pixel_size_kernel): bits;
  - _C.sphere_ellipsoid_intersection (sphere_ellipsoid_kernel) on the chain's neighbours (missing slots -> own index) and radii:
    the mask per pair and the counts;
  - _C.allocate_minimum_redundancy_value (min_redundancy_kernel) over [self | neighbours] with the chain's mask and counts;
  - gs_b200.densify.calculate_redundancy_metric (the kNN, pixel_size_kernel and redundancy_fused_kernel in one call):
    min_redundancy, and cube_size as bits.
Rows the oracle marks `borderline` (a pair within 2^-20 of dot = 1 with a square the device's powf may round 1 ulp away) would be
excused from the mask and count checks, and their neighbours from the minima; no pair of these scenes is one (checked on the CPU).
Observed on one H100 80GB HBM3: all 38 tests exact, in ~26 s.  Each of these one-line kernel edits fails the file there:
  - `dot < 1.0f` -> `<=` in sphere_hits: the planted dot = 1.0 pairs of sphere_k1 / k30 / k64, unfused and fused (6 tests);
  - `qz >= 0.0f` -> `>` in pixel_size_kernel: the centres at qz = 0 exactly in `planes`, unfused and fused (2);
  - the kNN's `need` test `<= thr` -> `< thr`: `lattice`, `lattice_perm` and `duplicates` (3);
  - the neighbour's rotation instead of the current Gaussian's, in both sphere kernels: every scene with hits (18).
"""
import numpy as np
import pytest
import torch

import redundancy_edges as RE
from gs_b200 import densify

pytestmark = pytest.mark.gpu
DEV = "cuda"
_cache = {}


def _knn_mod():
    from simple_knn import _C
    return _C


def _dgr():
    from diff_gaussian_rasterization import _C
    return _C


def _scene(name):
    key = "scene " + name
    if key not in _cache:
        s = RE.build(name)
        _cache[key] = s, RE.chain(s)
    return _cache[key]


def _fail(failures):
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("name", list(RE.KNN_CASES))
def test_knn_against_oracle(name):
    C = _knn_mod()
    pts = RE.knn_points(name)
    d, i = RE.knn_oracle_rows(pts)
    g = torch.from_numpy(pts).to(DEV)
    failures = RE.compare("distCUDA2", RE.mean3(d), C.distCUDA2(g).cpu().numpy())
    for K in RE.KNN_CASES[name]:
        gd, gi = C.distIndex2(g, K)
        failures += RE.compare("distIndex2 K=%d distances" % K, d[:, :K], gd.cpu().numpy().reshape(-1, K))
        failures += RE.compare("distIndex2 K=%d indices" % K, i[:, :K], gi.cpu().numpy().reshape(-1, K))
    _fail(failures)


def test_knn_query_against_oracle():
    C = _knn_mod()
    pts, q, n = RE.query_case()
    d, i = RE.knn_oracle_rows(pts, RE.KMAX, q, n)
    failures = []
    for K in RE.QUERY_KS:
        gd, gi = C.distIndexQ(torch.from_numpy(pts).to(DEV), torch.from_numpy(q).to(DEV), torch.from_numpy(n).to(DEV), K)
        failures += RE.compare("distIndexQ K=%d distances" % K, d[:, :K], gd.cpu().numpy().reshape(-1, K))
        failures += RE.compare("distIndexQ K=%d indices" % K, i[:, :K], gi.cpu().numpy().reshape(-1, K))
    _fail(failures)


@pytest.mark.parametrize("name", RE.SCENES)
def test_unfused_stages_against_oracle(name):
    s, o = _scene(name)
    C = _dgr()
    projs, invs, H, W = (torch.from_numpy(a).to(DEV) for a in s.cam_arrays())
    xyz, sc, rot = (torch.from_numpy(a).to(DEV) for a in (s.xyz, s.scales, s.rots))
    px = C.find_minimum_projected_pixel_size(projs, invs, xyz, H, W)
    failures = RE.compare("pixel size", o["px"], px.cpu().numpy())
    bl = o["borderline"]
    red, mask = C.sphere_ellipsoid_intersection(xyz, sc, rot, torch.from_numpy(o["nb"]).to(DEV), torch.from_numpy(o["rad"]).to(DEV), s.K)
    failures += RE.compare("intersection mask", o["raw_mask"], mask.cpu().numpy(), allow=bl)
    failures += RE.compare("redundancy", o["raw_red"], red.cpu().numpy(), allow=bl)
    mn = C.allocate_minimum_redundancy_value(torch.from_numpy(o["red"]).to(DEV), torch.from_numpy(o["cat_idx"]).to(DEV),
                                             torch.from_numpy(o["cat_mask"]).to(DEV), s.K + 1)[0]
    failures += RE.compare("minimum", o["minimum"], mn.cpu().numpy())
    _fail(failures)


@pytest.mark.parametrize("name", RE.SCENES)
def test_fused_against_oracle(name):
    s, o = _scene(name)
    d, i = _knn_mod().distIndex2(torch.from_numpy(s.xyz).to(DEV), s.K)
    failures = RE.compare("kNN distances", o["dist"], d.cpu().numpy().reshape(-1, s.K))
    failures += RE.compare("kNN indices", o["idx"], i.cpu().numpy().reshape(-1, s.K))
    m, cube = densify.calculate_redundancy_metric(s.on(DEV), pixel_scale=s.ps, num_neighbours=s.K)
    failures += RE.compare("cube_size", o["px"], cube.cpu().numpy())
    allow = np.zeros(s.P, bool)
    b = np.nonzero(o["borderline"])[0]
    allow[b] = True
    allow[o["nb"][b].reshape(-1)] = True
    failures += RE.compare("min_redundancy", o["minimum"], m.cpu().numpy(), allow=allow)
    _fail(failures)
