"""CPU: the brute-force kNN oracle (oracle/knn_oracle.cpp) against the reference's own outputs (tests/golden/kn1*.npz, kn_edge*.npz,
written by tests/golden/make_golden_knn.py), the argument checks of gsb_knn, and the drop-in simple_knn._C refusing CPU tensors.

The oracle's rows follow the drop-in's contract (sorted by (distance, index), the smaller index winning a tie at the K-th distance),
so against the reference: distCUDA2 bit-identical, per-row-sorted distances bit-identical, indices equal outside boundary-tie rows."""
import ctypes as C
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
import knn_oracle as O  # noqa: E402
import refsummary as S  # noqa: E402

GOLD = os.path.join(HERE, "golden")


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _check(od, oi, rd, ri, K, ties, what):
    od, oi = np.asarray(od).reshape(-1, K), np.asarray(oi).reshape(-1, K)
    sd, si = KC.sorted_rows(od, oi, K)
    assert np.array_equal(_bits(sd), _bits(od)) and np.array_equal(si, oi), what + ": oracle rows not sorted"
    rd, ri = KC.sorted_rows(rd, ri, K)
    assert np.array_equal(_bits(od), _bits(rd)), what + ": sorted distances differ from the reference"
    tie = np.zeros(od.shape[0], bool)
    tie[np.asarray(ties, np.int64)] = True
    assert np.array_equal(oi[~tie], ri[~tie]), what + ": indices differ outside boundary-tie rows"
    for r in np.nonzero(tie)[0]:
        m = od[r] < od[r, K - 1]
        assert np.array_equal(oi[r][m], ri[r][m]), (what, r)
        assert np.array_equal(np.sort(oi[r][~m]), oi[r][~m])      # the tied slots hold the smallest tied indices, ascending


@pytest.mark.skipif(not os.path.isfile(os.path.join(GOLD, "kn1.npz")), reason="tests/golden/kn1.npz missing")
def test_oracle_against_kn1():
    ref = S.load_parts("kn1")
    c = KC.KNN_CASES["kn1"]
    pts, q, n = KC.kn1_inputs()
    assert np.array_equal(_bits(O.distCUDA2(pts)), _bits(ref["d2"])), "distCUDA2 is expected bit-identical"
    for K in c["ks"]:
        _check(*O.distIndex2(pts, K), ref[f"k{K}_d"], ref[f"k{K}_i"], K, ref[f"k{K}_ties"], f"K={K}")
    _check(*O.distIndexQ(pts, q, n, c["q_k"]), ref["q_d"], ref["q_i"], c["q_k"], ref["q_ties"], "distIndexQ")
    assert ref["k30_ties"].size < pts.shape[0] // 10


@pytest.mark.skipif(not os.path.isfile(os.path.join(GOLD, "kn_edge.npz")), reason="tests/golden/kn_edge.npz missing")
def test_oracle_against_kn_edge():
    ref = S.load_parts("kn_edge")
    K = KC.EDGE_K
    for name, pts in KC.edge_inputs().items():
        assert np.array_equal(_bits(O.distCUDA2(pts)), _bits(ref[name + "_d2"])), name
        _check(*O.distIndex2(pts, K), ref[name + "_d"], ref[name + "_i"], K, ref[name + "_ties"], name)
    d2 = {n: O.distCUDA2(p) for n, p in KC.edge_inputs().items()}
    assert np.isinf(d2["p1"]).all() and np.isinf(d2["p2"]).all()
    assert np.isfinite(d2["p3"]).all() and (d2["p3"] > 1e38).all()
    assert (d2["same"] == 0).all()


def test_oracle_contract_small():
    """Duplicates count at distance 0, self is excluded by index, unfilled slots are (FLT_MAX, -1), ties go to the smaller index."""
    pts = np.array([[0, 0, 0], [0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    d, i = O.distIndex2(pts, 4)
    d, i = d.reshape(4, 4), i.reshape(4, 4)
    assert i[0].tolist() == [1, 2, 3, -1] and d[0].tolist() == [0.0, 1.0, 1.0, float(np.finfo(np.float32).max)]
    d, i = O.distIndexQ(pts, np.array([0, 9, -1], np.int32), np.array([3, 2, 0, 2, 1], np.int32), 1)
    assert i.tolist() == [2, -1, -1]        # first min(N, P) = 4 entries count; out-of-range queries give empty rows


def test_gsb_knn_argument_validation_needs_no_gpu():
    """Every call below is rejected before the first CUDA call."""
    from gs_b200 import lib
    L = lib.lib()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    cases = [
        (dict(P=-1), "P < 0"),
        (dict(K=-1), "K < 0"),
        (dict(K=65), "maximum of 64"),
        (dict(K=4, mean3=p), "K == 3"),
        (dict(points=None), "NULL"),
        (dict(workspace=None), "NULL"),
        (dict(dists=None, indices=None), "no output"),
        (dict(n_queries=4), "query_ids is NULL"),
        (dict(n_candidates=4), "candidate_ids is NULL"),
    ]
    for over, msg in cases:
        a = dict(points=p, P=10, K=3, query_ids=None, n_queries=-1, candidate_ids=None, n_candidates=-1, mean3=None, dists=p, indices=p,
                 workspace=p)
        a.update(over)
        st = L.gsb_knn(a["points"], a["P"], a["K"], a["query_ids"], a["n_queries"], a["candidate_ids"], a["n_candidates"], a["mean3"],
                       a["dists"], a["indices"], a["workspace"], None)
        assert st == -1, over
        assert msg in L.gsb_last_error().decode(), (over, L.gsb_last_error())
    assert L.gsb_knn(None, 0, 30, None, -1, None, -1, None, None, None, None, None) == 0      # nothing to do
    assert L.gsb_knn_workspace_bytes(1000, -1) < L.gsb_knn_workspace_bytes(100000, -1) < L.gsb_knn_workspace_bytes(100000, 200000)
    assert L.gsb_knn(p, 10, 3, p, 1 << 30, None, -1, None, p, p, p, None) == -4          # GSB_ERANGE


def test_simple_knn_refuses_cpu_tensors():
    from simple_knn import _C
    pts = torch.rand(100, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.distCUDA2(pts)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.distIndex2(pts, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.distIndexQ(pts, torch.arange(3, dtype=torch.int32), torch.arange(3, dtype=torch.int32), 3)
