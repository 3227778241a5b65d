"""GPU: the drop-in simple_knn._C (distCUDA2, distIndex2, distIndexQ on gsb_knn) against (a) the reference's own outputs recorded in
tests/golden/kn*.npz (tests/golden/make_golden_knn.py) and (b) the brute-force CPU oracle (oracle/knn_oracle.cpp).

Contract (simple_knn/_C.py): distCUDA2 bit-identical; each row sorted by (distance, index), its distances bit-identical to the
reference's sorted row; its indices equal to the reference's except in rows with a tie at the K-th distance, where the reference
keeps the candidate it visited first and ours keeps the smallest index (the oracle's rows, exactly)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (os.path.join(HERE, "golden"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "reduced-3dgs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import knn_cases as KC  # noqa: E402
import refsummary as S  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(HERE, "golden")
FLT_MAX = np.finfo(np.float32).max


def _knn():
    from simple_knn import _C
    return _C


def _has(name):
    return os.path.isfile(os.path.join(GOLD, name + ".npz"))


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _check_rows(ours_d, ours_i, ref_d, ref_i, K, ties, oracle=None, what=""):
    """ours: flat rows as returned (must already be sorted); ref: flat rows in the reference's slot order."""
    od, oi = np.asarray(ours_d).reshape(-1, K), np.asarray(ours_i).reshape(-1, K)
    sd, si = KC.sorted_rows(od, oi, K)
    assert np.array_equal(_bits(sd), _bits(od)) and np.array_equal(si, oi), what + ": rows are not sorted by (distance, index)"
    rd, ri = KC.sorted_rows(ref_d, ref_i, K)
    assert np.array_equal(_bits(od), _bits(rd)), what + ": sorted distances differ from the reference"
    tie = np.zeros(od.shape[0], bool)
    tie[np.asarray(ties, np.int64)] = True
    assert np.array_equal(oi[~tie], ri[~tie]), what + ": indices differ outside boundary-tie rows"
    for r in np.nonzero(tie)[0]:
        t = od[r, K - 1]
        m = od[r] < t
        assert np.array_equal(oi[r][m], ri[r][m]), (what, r)
    if oracle is not None:
        assert np.array_equal(_bits(od), _bits(np.asarray(oracle[0]).reshape(-1, K))), what + ": distances differ from the oracle"
        assert np.array_equal(oi, np.asarray(oracle[1]).reshape(-1, K)), what + ": indices differ from the oracle"


@pytest.mark.skipif(not _has("kn1"), reason="tests/golden/kn1.npz missing")
def test_kn1_against_reference_goldens():
    import knn_oracle as O
    C = _knn()
    c = KC.KNN_CASES["kn1"]
    ref = S.load_parts("kn1")
    pts, q, n = KC.kn1_inputs()
    P = pts.shape[0]
    g = pts.cuda()
    d2 = C.distCUDA2(g)
    assert d2.dtype == torch.float32 and tuple(d2.shape) == (P,) and d2.device == g.device
    assert np.array_equal(_bits(d2.cpu().numpy()), _bits(ref["d2"])), "distCUDA2 is expected bit-identical"
    for K in c["ks"]:
        d, i = C.distIndex2(g, K)
        assert d.dtype == torch.float32 and i.dtype == torch.int32 and tuple(d.shape) == (P * K,) == tuple(i.shape)
        _check_rows(d.cpu().numpy(), i.cpu().numpy(), ref[f"k{K}_d"], ref[f"k{K}_i"], K, ref[f"k{K}_ties"], O.distIndex2(pts, K), f"K={K}")
    d, i = C.distIndexQ(g, q.cuda(), n.cuda(), c["q_k"])
    assert tuple(d.shape) == (q.shape[0] * c["q_k"],)
    _check_rows(d.cpu().numpy(), i.cpu().numpy(), ref["q_d"], ref["q_i"], c["q_k"], ref["q_ties"], O.distIndexQ(pts, q, n, c["q_k"]), "Q")
    assert set(i.cpu().numpy().tolist()) - {-1} <= set(n[:P].numpy().tolist()), "a candidate beyond the first P entries was used"


@pytest.mark.skipif(not _has("kn_edge"), reason="tests/golden/kn_edge.npz missing")
def test_kn_edge_against_reference_goldens():
    import knn_oracle as O
    C = _knn()
    ref = S.load_parts("kn_edge")
    K = KC.EDGE_K
    for name, pts in KC.edge_inputs().items():
        g = pts.cuda()
        d2 = C.distCUDA2(g).cpu().numpy()
        assert np.array_equal(_bits(d2), _bits(ref[name + "_d2"])), name + ": distCUDA2"
        d, i = C.distIndex2(g, K)
        _check_rows(d.cpu().numpy(), i.cpu().numpy(), ref[name + "_d"], ref[name + "_i"], K, ref[name + "_ties"], O.distIndex2(pts, K), name)
    P1 = C.distCUDA2(KC.edge_inputs()["p1"].cuda()).cpu().numpy()
    assert np.isinf(P1).all()


@pytest.mark.skipif(not _has("kn_red"), reason="tests/golden/kn_red.npz missing")
def test_redundancy_pipeline_through_the_drop_ins():
    """The reference's own calculate_redundancy_metric sequence (scene/__init__.py:142-174) with `simple_knn._C` and
    `diff_gaussian_rasterization._C` both resolving to this project."""
    from simple_knn._C import distIndex2  # noqa: F401  (the import the reference's scene/__init__.py does)
    from diff_gaussian_rasterization import _C as dgr
    ref = S.load_parts("kn_red")
    K = KC.KNN_CASES["kn_red"]["K"]
    c, scene, cams = KC.red_inputs()
    min_red, red, idx = KC.redundancy_pipeline(_knn(), dgr, scene, cams, c["radius_scale"], K)
    d, i = _knn().distIndex2(scene.means3D.cuda(), K)
    sd, _ = KC.sorted_rows_t(d, i, K)
    assert S.digest(sd) == str(ref["sorted_d"]), "sorted neighbour distances differ from the reference"
    assert np.array_equal(idx.view(-1).cpu().numpy(), i.cpu().numpy())
    if int(ref["n_ties"]) == 0:
        assert np.array_equal(red.cpu().numpy(), ref["redundancy"])
        assert np.array_equal(min_red.cpu().numpy(), ref["min_redundancy"]), "min_redundancy differs on a tie-free case"
    else:
        keep = np.ones(scene.P, bool)
        keep[ref["ties"]] = False
        assert np.array_equal(red.cpu().numpy()[keep], ref["redundancy"][keep])


@pytest.mark.skipif(not _has("kn_large"), reason="tests/golden/kn_large.npz missing")
@pytest.mark.parametrize("name", ["C3", "clustered"])
def test_kn_large_against_reference_record(name):
    C = _knn()
    c = KC.KNN_CASES["kn_large"]
    K = c["K"]
    ref = S.load_parts("kn_large")
    pts = KC.large_inputs()[name].cuda()
    P = pts.shape[0]
    assert S.digest(C.distCUDA2(pts)) == str(ref[name + "_d2"]), "distCUDA2 at 3 M points"
    d, i = C.distIndex2(pts, K)
    sd, si = KC.sorted_rows_t(d, i, K)
    assert torch.equal(sd.view(torch.int32), d.view(-1, K).view(torch.int32)), "rows are not sorted"
    assert S.digest(sd) == str(ref[name + "_sorted_d"]), "sorted distIndex2 distances at 3 M points"
    rows = S.sample_index(P, c["rows"])
    od, oi = sd[torch.as_tensor(rows, device=sd.device)].cpu().numpy(), si[torch.as_tensor(rows, device=sd.device)].cpu().numpy()
    tie = np.isin(rows, ref[name + "_ties"])
    assert np.array_equal(_bits(od), _bits(ref[name + "_rows_d"]))
    assert np.array_equal(oi[~tie], ref[name + "_rows_i"][~tie])


def test_against_oracle_50k():
    import knn_oracle as O
    C = _knn()
    pts = KC.clustered_cloud(50_000, 7)
    g = pts.cuda()
    assert np.array_equal(_bits(C.distCUDA2(g).cpu().numpy()), _bits(O.distCUDA2(pts)))
    d, i = C.distIndex2(g, 30)
    od, oi = O.distIndex2(pts, 30)
    assert np.array_equal(_bits(d.cpu().numpy()), _bits(od)) and np.array_equal(i.cpu().numpy(), oi), "rows differ from the oracle"
    rng = np.random.default_rng(8)
    q = torch.from_numpy(rng.choice(50_000, 3_000).astype(np.int32))
    n = torch.from_numpy(rng.choice(50_000, 20_000).astype(np.int32))
    d, i = C.distIndexQ(g, q.cuda(), n.cuda(), 17)
    od, oi = O.distIndexQ(pts, q, n, 17)
    assert np.array_equal(_bits(d.cpu().numpy()), _bits(od)) and np.array_equal(i.cpu().numpy(), oi)


def test_boundary_tie_smaller_index_wins():
    """Four candidates at exactly distance 1 from point 0 compete for the last of K = 2 slots: index 2 (the smallest) wins."""
    pts = torch.tensor([[0, 0, 0], [5, 5, 5], [0, 0, 1], [0, 1, 0], [1, 0, 0], [0, 0, 0.5], [-1, 0, 0], [7, 7, 7]], dtype=torch.float32)
    perm = [0, 6, 3, 1, 7, 5, 4, 2]                  # the same cloud with the tied points in another order
    for p in (pts, pts[perm]):
        d, i = _knn().distIndex2(p.cuda(), 2)
        tied = [j for j in range(8) if j and float(((p[j] - p[0]) ** 2).sum()) == 1.0]
        half = [j for j in range(8) if float(((p[j] - p[0]) ** 2).sum()) == 0.25]
        assert i.view(-1, 2)[0].tolist() == [half[0], min(tied)]
        assert d.view(-1, 2)[0].tolist() == [0.25, 1.0]


def test_k_above_p_minus_1_and_empty_inputs():
    C = _knn()
    pts = torch.rand(5, 3, generator=torch.Generator().manual_seed(3)).cuda()
    d, i = C.distIndex2(pts, 10)
    d, i = d.view(5, 10).cpu(), i.view(5, 10).cpu()
    assert (i[:, 4:] == -1).all() and (d[:, 4:] == float(FLT_MAX)).all()
    assert (i[:, :4] >= 0).all() and (d[:, :4] < float(FLT_MAX)).all()
    for r in range(5):
        assert sorted(i[r, :4].tolist()) == [j for j in range(5) if j != r]
    e = torch.empty(0, 3, device="cuda")
    assert C.distCUDA2(e).shape == (0,)
    assert [t.shape for t in C.distIndex2(e, 30)] == [(0,), (0,)]
    assert [t.shape for t in C.distIndex2(pts, 0)] == [(0,), (0,)]
    with pytest.raises(RuntimeError):
        C.distIndex2(pts, -1)
    with pytest.raises(RuntimeError, match="maximum"):
        C.distIndex2(pts, 65)
    d, i = C.distIndex2(pts, 64)
    assert d.shape == (5 * 64,)


def test_out_of_range_ids():
    """Query ids outside [0, P) give rows of (FLT_MAX, -1); candidate ids outside [0, P) are ignored."""
    import knn_oracle as O
    C = _knn()
    pts = KC.clustered_cloud(2_000, 9)
    q = torch.tensor([5, -1, 2_000, 17, 1 << 30], dtype=torch.int32)
    n = torch.tensor(list(range(0, 2_000, 3)) + [-7, 2_000, 99_999], dtype=torch.int32)
    d, i = C.distIndexQ(pts.cuda(), q.cuda(), n.cuda(), 6)
    d, i = d.view(5, 6).cpu().numpy(), i.view(5, 6).cpu().numpy()
    for r in (1, 2, 4):
        assert (i[r] == -1).all() and (d[r] == FLT_MAX).all()
    od, oi = O.distIndexQ(pts, q, n, 6)
    assert np.array_equal(_bits(d), _bits(od.reshape(5, 6))) and np.array_equal(i, oi.reshape(5, 6))
    d, i = C.distIndexQ(pts.cuda(), q.cuda(), torch.empty(0, dtype=torch.int32, device="cuda"), 6)
    assert (i == -1).all()


def test_two_runs_bit_identical():
    C = _knn()
    pts = KC.clustered_cloud(300_000, 11).cuda()
    a, b = C.distIndex2(pts, 30), C.distIndex2(pts, 30)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])
    assert torch.equal(C.distCUDA2(pts).view(torch.int32), C.distCUDA2(pts).view(torch.int32))


def test_non_default_stream():
    C = _knn()
    pts = KC.clustered_cloud(100_000, 12).cuda()
    base = C.distIndex2(pts, 30)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        other = C.distIndex2(pts, 30)
        m = C.distCUDA2(pts)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(base[0].view(torch.int32), other[0].view(torch.int32)) and torch.equal(base[1], other[1])
    assert torch.equal(m.view(torch.int32), C.distCUDA2(pts).view(torch.int32))


def test_second_device_in_the_same_process():
    """cuda:1 in the same process as cuda:0 (its own dynamic-shared-memory opt-in) gives identical rows.  Needs 2 visible GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs in one process")
    C = _knn()
    pts = KC.clustered_cloud(60_000, 13)
    a = C.distIndex2(pts.to("cuda:0"), 64)
    b = C.distIndex2(pts.to("cuda:1"), 64)
    assert b[0].device == torch.device("cuda:1")
    assert torch.equal(a[0].cpu().view(torch.int32), b[0].cpu().view(torch.int32)) and torch.equal(a[1].cpu(), b[1].cpu())
