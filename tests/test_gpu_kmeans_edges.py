"""GPU: the codebook k-means (gsb_kmeans.cu, DESIGN.md §5j) on the cases of tests/kmeans_edges.py.
  1. centre sets: the ids at 0 iterations on both paths are the brute-force assignment (the reference's rule) and the centres come
     back unchanged; the deterministic centres after 1, 2 and 3 iterations are the restatement's bit for bit; the default path's
     centres after one iteration are the float64 means of the brute-force clusters within the float32 summation bound;
  2. value sets: the deterministic centres after 1, 2 and 3 iterations equal the restatement bit for bit, and the ids are the
     assignment of the returned centres; on the sets that converge in seconds also at convergence, with the same iteration
     count; the default path's first iteration within the summation bound, as in 1;
  3. exact sets (multiples of 2^-6, sum of |v| below 2^24 steps): after 3 iterations with tol = 0 the default path, the deterministic
     path, the restatement and gs_oracle.kmeans give the same centres bit for bit and the same ids, up to 9 M values at K = 1 024.
With the raw float_key order of the centres (before the canonical key) exactly the five sets of kmeans_edges.KEY_ORDER_BREAKS fail
1, each in the ids of both paths and in the deterministic centres (and, on zero_pm, in the default path's centres).  On an H100 80GB HBM3 the file takes about 66 s, most of it in the float32
restatement of the three 9 M-value cases."""
import time

import numpy as np
import pytest
import torch

import gs_oracle
import kmeans_edges as KE
from diff_gaussian_rasterization import _C

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32


@pytest.fixture(scope="module", autouse=True)
def _runtime():
    t = time.perf_counter()
    yield
    print(f"\ntest_gpu_kmeans_edges.py: {time.perf_counter() - t:.1f} s")


def _km(values, centres, iterations, det, tol=0.0):
    ids, c = _C.kmeans_cuda(torch.from_numpy(np.ascontiguousarray(values)).view(-1, 1).to(DEV), torch.from_numpy(centres).to(DEV),
                            tol, iterations, deterministic=det)
    return ids.cpu().numpy().reshape(-1), c.cpu().numpy()


def _same_bits(a, b):
    return KE.bits(a).tolist() == KE.bits(b).tolist()


def _within_sum_bound(values, ids, got):
    """Per cluster: |got - float64 mean| <= 2^-23 (sum |v| + |mean|), the bound of a float32 sum in any order and one division;
    an empty cluster gives 0.  Clusters holding non-finite values or sums near the float32 range are left out."""
    K = got.size
    v = values.astype(np.float64)
    fin = np.isfinite(v)
    bad = np.bincount(ids, weights=~fin, minlength=K) > 0
    v = np.where(fin, v, 0.0)
    size = np.bincount(ids, minlength=K)
    s, a = np.bincount(ids, weights=v, minlength=K), np.bincount(ids, weights=np.abs(v), minlength=K)
    mean = np.where(size > 0, s / np.maximum(size, 1), 0.0)
    ok = bad | (a > 1e37) | (np.abs(got - mean) <= 2.0 ** -23 * (a + np.abs(mean)) + 2.0 ** -149)
    return bool(np.all(ok)), np.flatnonzero(~ok)


# ---- 1. centre sets --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(KE.CENTRE_SETS))
def test_centre_set(name):
    c, v = KE.centre_set(name)
    want = KE.brute(v, c)
    failed = []                      # every check runs, so that a failure names each path and kernel it reaches
    for det in (False, True):
        ids, cc = _km(v, c, 0, det)
        if not np.array_equal(ids, want):
            failed.append(f"ids at 0 iterations, det={det}: values {np.flatnonzero(ids != want)[:8].tolist()}")
        if not _same_bits(cc, c):
            failed.append(f"centres at 0 iterations, det={det}")
    for it, r_c in enumerate(KE.restate(v, c, 3), 1):
        ids, cc = _km(v, c, it, True)
        if not _same_bits(cc, r_c):
            failed.append(f"deterministic centres after {it}")
        if not np.array_equal(ids, KE.brute(v, r_c)):
            failed.append(f"deterministic ids after {it}")
    ids, cc = _km(v, c, 1, False)
    ok, where = _within_sum_bound(v, want, cc)
    if not ok:
        failed.append(f"default centres after 1: clusters {where[:8].tolist()}")
    if not np.array_equal(ids, KE.brute(v, cc)):
        failed.append("default ids after 1")
    assert not failed, failed


# ---- 2. value sets ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(KE.VALUE_SETS))
def test_value_set_deterministic(name):
    v, c = KE.value_set(name)
    for it, r_c in enumerate(KE.restate(v, c, 3), 1):
        ids, cc = _km(v, c, it, True)
        assert _same_bits(cc, r_c), it
        assert np.array_equal(ids, KE.brute(v, r_c)), it
    ids, cc = _km(v, c, 1, False)
    ok, where = _within_sum_bound(v, KE.brute(v, c), cc)
    assert ok, where[:8]
    if name in KE.CONVERGED_VALUE_SETS:
        tol = 1e-4
        steps = KE.restate(v, c, 500, tol)
        ids, cc = _km(v, c, 500, True, tol)
        assert _same_bits(cc, steps[-1]) and np.array_equal(ids, KE.brute(v, cc))
        assert _same_bits(_km(v, c, len(steps), True, tol)[1], steps[-1])
        if len(steps) > 1:           # one iteration fewer gives the restatement's centres of that iteration
            assert _same_bits(_km(v, c, len(steps) - 1, True, tol)[1], steps[-2])
        print(f"{name}: {len(steps)} iterations to converge")


# ---- 3. exact sets ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(KE.EXACT_SETS))
def test_exact_set_both_paths(name, monkeypatch):
    v, c, _ = KE.exact_set(name)
    it = 3
    d_ids, d_c = _km(v, c, it, False)
    e_ids, e_c = _km(v, c, it, True)
    r_c = KE.restate(v, c, it)[-1]
    r_ids = KE.brute(v, r_c)
    per_value = gs_oracle.kmeans_update_ids

    def distinct_values_once(values, centers):
        u, inv = np.unique(values, return_inverse=True)
        return per_value(u, centers)[inv.reshape(-1)]

    # gs_oracle.kmeans with its assignment taken once per distinct value: the same function of the value, and far cheaper at 9 M values
    monkeypatch.setattr(gs_oracle, "kmeans_update_ids", distinct_values_once)
    o_ids, o_c, o_it = gs_oracle.kmeans(v, c, 0.0, it)
    assert o_it == it
    assert _same_bits(d_c, r_c) and _same_bits(e_c, r_c) and _same_bits(o_c, r_c)
    assert np.array_equal(d_ids, r_ids) and np.array_equal(e_ids, r_ids) and np.array_equal(o_ids.reshape(-1), r_ids)
    assert np.unique(r_ids).size > c.size // 4
