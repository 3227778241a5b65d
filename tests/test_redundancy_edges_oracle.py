"""CPU: the kNN cases and redundancy scenes of tests/redundancy_edges.py reach the boundaries they are built for, and the exact
comparison of test_gpu_redundancy_edges.py rejects near-misses made with the oracles themselves.  Only the oracles run here."""
import numpy as np
import pytest

import gs_oracle
import knn_oracle
import redundancy_edges as RE

_cache = {}


def _knn(name):
    if name not in _cache:
        pts = RE.knn_points(name)
        _cache[name] = pts, RE.knn_oracle_rows(pts, RE.KMAX + 1)
    return _cache[name]


def _scene(name):
    key = "scene " + name
    if key not in _cache:
        s = RE.build(name)
        _cache[key] = s, RE.chain(s)
    return _cache[key]


def _spans(rank, ids, size):
    return np.unique(rank[ids] // size).size > 1


def test_oracle_rows_at_smaller_k_are_prefixes():
    pts, (d, i) = _knn("p1025")
    for K in (1, 3, 30):
        dk, ik = knn_oracle.distIndex2(pts, K)
        assert np.array_equal(RE.bits(dk.reshape(-1, K)), RE.bits(d[:, :K])) and np.array_equal(ik.reshape(-1, K), i[:, :K])
    assert np.array_equal(RE.bits(knn_oracle.distCUDA2(pts)), RE.bits(RE.mean3(d)))


@pytest.mark.parametrize("name", list(RE.KNN_CASES))
def test_knn_case_reaches_its_boundary(name):
    pts, (d, i) = _knn(name)
    P = pts.shape[0]
    assert d.shape == (P, RE.KMAX + 1)
    if name.startswith("p"):
        assert P == int(name[1:])
    if name in ("lattice", "lattice_perm", "duplicates"):
        rank = RE.morton_rank(pts)
        for K in RE.KNN_CASES[name]:
            if K < 30:
                continue
            ties = RE.kth_ties(pts, K, d, i)
            cross = [r for r, ids in ties.items() if _spans(rank, np.append(ids, r), 32)]
            print("\n[%s K=%d] %d rows tied at the K-th distance, %d of them across leaves" % (name, K, len(ties), len(cross)))
            assert len(cross) >= RE.N_MIN
        if name == "duplicates":
            zero = np.nonzero((d[:, :64] == 0).all(1))[0]
            assert zero.size >= 4900 and _spans(rank, zero, 32 * 32)
    if name == "overflow":
        with np.errstate(over="ignore", invalid="ignore"):
            diff = pts[:, None, :] - pts[None, :, :]
            sq = diff * diff
            tot = (sq[..., 1] + sq[..., 0]) + sq[..., 2]
        sub = np.isinf(diff).any(-1)
        square = ~sub & np.isinf(sq).any(-1)
        summed = ~sub & ~square & np.isinf(tot)
        assert sub.any() and square.any() and summed.any()
        bad = sub | square | summed
        r, c = np.nonzero(bad)
        assert not (i[r] == c[:, None]).any(), "an overflowed pair is a neighbour"
        far = np.nonzero((np.abs(pts) == np.float32(1e6)).any(1))[0]
        assert (i[far, 0] >= 0).all(), "a finite far outlier still has neighbours"
        empty = np.nonzero(bad.sum(1) == P - 1)[0]
        assert empty.size >= 10 and (i[empty] == -1).all() and (d[empty] == RE.FLT_MAX).all()
    if name == "denormal":
        tiny = d[(d > 0) & (d < np.finfo(np.float32).tiny)]
        assert tiny.size > 1000 and (d[:, 0] == 0).any()
    if name == "nonfinite":
        bad = np.nonzero(~np.isfinite(pts).all(1))[0]
        assert bad.size == 30 and (i[bad] == -1).all() and (d[bad] == RE.FLT_MAX).all()
        assert not np.isin(i, bad).any()


def test_query_case_reaches_its_boundary():
    pts, q, n = RE.query_case()
    P = pts.shape[0]
    assert n.size > P and np.unique(q).size < q.size and np.unique(n[:P]).size < P
    listed = np.zeros(P, bool)
    listed[n[:P]] = True
    assert (~listed[q]).sum() >= RE.N_MIN and listed[n[P:]].sum() < n.size - P
    d, i = RE.knn_oracle_rows(pts, RE.KMAX, q, n)
    assert listed[i[i >= 0]].all() and not np.isin(i, np.nonzero(~listed)[0]).any()


@pytest.mark.parametrize("name", RE.SCENES)
def test_scene_reaches_its_boundary(name):
    s, o = _scene(name)
    P, K = s.P, s.K
    assert not o["borderline"].any(), "no pair may be within reach of the device powf's 1-ulp squares"
    assert o["idx"].shape == (P, K) and o["minimum"].shape == (P, 1)
    if name == "planes":
        g = s.meta["groups"]
        for c in range(len(RE.PLANE_CAMS)):
            cam = s.meta["plane_cams"][c]
            for plane in RE.PLANES:
                a, b = g["cam%d %s in" % (c, plane)], g["cam%d %s out" % (c, plane)]
                assert a.size >= RE.N_MIN
                assert (o["px"][a] < 10000).all() and (o["px"][b] == 10000).all()
                assert (np.abs(RE._key(s.xyz[a]) - RE._key(s.xyz[b])).sum(1) == 1).all(), "not adjacent floats"
                q = RE.ndc(np.concatenate([s.xyz[a], s.xyz[b]]), cam)
                k, v = "xyz".index(plane[1]), float(plane[3:])
                assert np.abs(q[k] - v).max() < 1e-3, (plane, np.abs(q[k] - v).max())    # fp32 rounding of the matrix terms
        W = [(c.image_width, c.image_height) for c in s.cams]
        assert any(w > h for w, h in W) and any(w == h for w, h in W) and any(w < h for w, h in W)
        ex, lo = g["nice qz=0 exact"], g["nice qz<0"]
        assert (RE.ndc(s.xyz[ex], s.meta["nice"])[2] == 0).all() and (o["px"][ex] < 10000).all() and (o["px"][lo] == 10000).all()
        z = s.xyz[g["w+1e-7 == 0"], 2]
        assert ((z + np.float32(1e-7)) == 0).all() and (o["px"][g["w+1e-7 == 0"]] == 10000).all()
        t = s.xyz[g["w+1e-7 tiny"], 2] + np.float32(1e-7)
        assert set(np.abs(t).tolist()) == {2.0 ** -47}
    if name == "cams_1024":
        assert len(s.cams) == 1024
        assert (o["px"][s.meta["unseen"]] == 10000).all() and (o["px"] < 10000).sum() >= 2000
    if name.startswith("sphere_k"):
        pi, pn = s.meta["pairs"]
        k = np.array([list(o["idx"][a]).index(b) for a, b in zip(pi, pn)])
        dot = o["dots"][pi, k]
        below, at = dot == RE.ONE_BELOW, dot == np.float32(1.0)
        assert below.sum() >= RE.N_MIN and at.sum() >= RE.N_MIN and (below | at).all()
        assert o["mask"][pi, k][below].all() and not o["mask"][pi, k][at].any()
        un = s.meta["unseen"]
        assert (o["px"][un] == 10000).all() and o["mask"][un].all()
        if K == 64:
            assert o["mask"][:, 63].sum() >= RE.N_MIN
        if K > 1:
            assert (o["minimum"] < o["red"]).sum() >= RE.N_MIN, "minima taken from a neighbour"
        swap = (np.abs(s.rots) == np.float32(np.sqrt(0.5))).sum(1) == 2
        assert swap.sum() >= 100 and (~swap).sum() >= 100
        flips = RE.neighbour_rotation_mask(s, o) != o["mask"]
        assert flips.sum() >= RE.N_MIN and flips[pi, k].sum() >= RE.N_MIN
    if name == "zero":
        assert (o["rad"] == 0).all()
        nan = np.isnan(o["dots"])
        assert nan.sum() >= 100 and not o["mask"][nan].any()
    if name.startswith("small_p"):
        assert P <= K and (o["idx"] < 0).sum() == P * K - P * (P - 1)


def _first_failure(s, o, **override):
    """The chain with one stage replaced -> the comparison's failures against the real chain."""
    fails = []
    for k, v in override.items():
        fails += RE.compare(k, o[k], v)
    return fails


def test_near_misses_are_rejected():
    # 1. the neighbour's rotation instead of the current Gaussian's
    s, o = _scene("sphere_k30")
    assert _first_failure(s, o, mask=RE.neighbour_rotation_mask(s, o))
    # 2. dot <= 1 instead of dot < 1
    assert _first_failure(s, o, mask=(o["dots"] <= 1) & (o["idx"] >= 0))
    # 3. the self "+1" dropped: the counts, and the minima built on them
    red = o["mask"].sum(1, keepdims=True).astype(np.int32)
    assert _first_failure(s, o, red=red)
    mn = gs_oracle.min_redundancy_value(red, o["cat_idx"], o["cat_mask"], s.K + 1)
    assert _first_failure(s, o, minimum=mn)
    # 4. a missing slot counted: the substituted own index hits itself (dot 0)
    s, o = _scene("small_p20_k30")
    red = o["raw_mask"].sum(1, keepdims=True).astype(np.int32) + 1
    assert (o["raw_mask"] & (o["idx"] < 0)).any() and _first_failure(s, o, red=red)
    # 5. qz > 0 instead of qz >= 0: the centres at qz = 0 exactly are seen by the integer camera only
    s, o = _scene("planes")
    px = RE.pixel_size(s.xyz, s.cams[:-1]).reshape(-1, 1)
    ex = s.meta["groups"]["nice qz=0 exact"]
    strict = o["px"].copy()
    strict[ex] = px[ex]
    assert (strict[ex] == 10000).all() and _first_failure(s, o, px=strict)
    # 6. the later index kept on a K-th-distance tie
    for name, K in (("lattice", 30), ("duplicates", 64)):
        pts, (d, i) = _knn(name)
        ties = RE.kth_ties(pts, K, d, i)
        later = i[:, :K].copy()
        for r in ties:
            later[r, K - 1] = i[r, K]
        assert ties and RE.compare("indices", i[:, :K], later)
