"""float32 restatement of the deterministic gsb_kmeans (DESIGN.md §5j): the assignment, the order in which each cluster's values are
added, the update and the stopping rule, in numpy.  The device path must reproduce its centres bit for bit, its iteration count and
its ids.  It is kept apart from gs_oracle so that the goldens made from gs_oracle keep measuring what they measure.

The summation order is a function of the sorted values and their ids alone.  Sorted position p lies in block b = p // 4096 and in
chunk t = (p % 4096) // 16 of that block.  -0.0, the exact identity of IEEE addition, stands for "no value":
    leaf(b, t, k) = (((-0 + v_p0) + v_p1) + ...) over the positions of chunk t with id k, ascending
    part(b, k)    = aligned pairwise tree over t = 0..255 of leaf(b, t, k)
    lane(l, k)    = (((-0 + part(l, k)) + part(l + 256, k)) + ...) over the blocks b = l (mod 256), ascending
    sum(k)        = (aligned pairwise tree over l = 0..255 of lane(l, k)) + 0.0
"""
from __future__ import annotations

import numpy as np

CHUNK = 16
CHUNKS_PER_BLOCK = 256
BLOCK = CHUNK * CHUNKS_PER_BLOCK
LANES = 256
F32 = np.float32


def float_key(v: np.ndarray) -> np.ndarray:
    """The order-preserving uint32 image of float32 values that the device sorts (-NaN < -inf < ... < -0 < +0 < ... < +inf < +NaN)."""
    u = np.ascontiguousarray(v, dtype=F32).view(np.uint32)
    return np.where(u >> 31 != 0, ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def key_float(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k, dtype=np.uint32)
    return np.where(k >> 31 != 0, k & np.uint32(0x7fffffff), ~k).astype(np.uint32).view(F32)


def sort_values(values: np.ndarray) -> np.ndarray:
    return key_float(np.sort(float_key(values)))


def assign(values: np.ndarray, centres: np.ndarray, block: int = 1 << 16) -> np.ndarray:
    """ids[i] = the smallest index among the centres at the smallest distance sqrt((c - v)^2) (float32), 0 when no distance is
    below +inf (NaN distances never win).  Brute force over the centres, in slices of `block` values."""
    v = np.asarray(values, dtype=F32).reshape(-1)
    c = np.asarray(centres, dtype=F32).reshape(-1)
    out = np.zeros(v.shape[0], dtype=np.int32)
    with np.errstate(all="ignore"):
        for s in range(0, v.shape[0], block):
            d = c[None, :] - v[s:s + block, None]
            d = np.sqrt(d * d)
            d = np.where(np.isnan(d), F32(np.inf), d)
            dmin = d.min(axis=1) if c.size else np.full(d.shape[0], np.inf, F32)
            ids = np.argmax(d == dmin[:, None], axis=1).astype(np.int32)
            out[s:s + block] = np.where(dmin < np.inf, ids, 0)
    return out


def _pairwise(x: np.ndarray) -> np.ndarray:
    """Aligned pairwise tree over the last axis (a power of two): (0+1), (2+3), ..., then (01+23), ..."""
    while x.shape[-1] > 1:
        x = x[..., 0::2] + x[..., 1::2]
    return x[..., 0]


def cluster_sums(sorted_values: np.ndarray, ids: np.ndarray, K: int) -> np.ndarray:
    """sum(k) for k = 0..K-1 in the order of the module docstring; sorted_values ascending by float_key, ids their clusters."""
    v = np.asarray(sorted_values, dtype=F32).reshape(-1)
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    n = v.shape[0]
    sums = np.zeros(K, dtype=F32)
    if n == 0:
        return sums
    n_blocks = (n + BLOCK - 1) // BLOCK
    pos = np.arange(n)
    block, chunk = pos // BLOCK, (pos % BLOCK) // CHUNK
    # leaves: one per (block, chunk, cluster) present, each a left fold from -0 over its positions in ascending order
    group = (block * CHUNKS_PER_BLOCK + chunk) * K + ids
    order = np.argsort(group, kind="stable")
    g_sorted, v_sorted = group[order], v[order]
    starts = np.flatnonzero(np.r_[True, g_sorted[1:] != g_sorted[:-1]])
    lengths = np.diff(np.r_[starts, n])
    leaf = np.full(starts.shape[0], -0.0, dtype=F32)
    with np.errstate(all="ignore"):
        for i in range(CHUNK):
            m = lengths > i
            leaf[m] = leaf[m] + v_sorted[starts[m] + i]
    g = g_sorted[starts]
    leaf_k, leaf_bc = g % K, g // K
    leaf_b, leaf_t = leaf_bc // CHUNKS_PER_BLOCK, leaf_bc % CHUNKS_PER_BLOCK
    # part(b, k): a dense row of 256 leaves per (block, cluster) present, -0 where the chunk has no value of the cluster
    bk = leaf_b * K + leaf_k
    pairs, row = np.unique(bk, return_inverse=True)
    dense = np.full((pairs.shape[0], CHUNKS_PER_BLOCK), -0.0, dtype=F32)
    dense[row, leaf_t] = leaf
    with np.errstate(all="ignore"):
        part = _pairwise(dense)
    part_b, part_k = pairs // K, pairs % K
    # lane(l, k) and sum(k)
    rows = (n_blocks + LANES - 1) // LANES
    lanes = np.full((K, rows * LANES), -0.0, dtype=F32)
    lanes[part_k, part_b] = part
    lanes = lanes.reshape(K, rows, LANES)
    acc = np.full((K, LANES), -0.0, dtype=F32)
    with np.errstate(all="ignore"):
        for r in range(rows):
            acc = acc + lanes[:, r, :]
        return _pairwise(acc) + F32(0.0)


def update(centres: np.ndarray, sums: np.ndarray, sizes: np.ndarray):
    """km_update_kernel: new = sums / sizes (NaN -> 0); shift = sum |old - new| as 256 thread partials (thread t: i = t, t + 256, ...)
    added by the halving tree s[t] += s[t + o], o = 128, 64, ..., 1.  -> (new centres, shift)."""
    K = centres.shape[0]
    with np.errstate(all="ignore"):
        new = sums.astype(F32) / sizes.astype(F32)
        new = np.where(np.isnan(new), F32(0.0), new).astype(F32)
        diff = np.abs(centres.astype(F32) - new)
        part = np.zeros(256, dtype=F32)
        for s in range(0, K, 256):
            d = diff[s:s + 256]
            part[:d.shape[0]] = part[:d.shape[0]] + d
        o = 128
        while o > 0:
            part[:o] = part[:o] + part[o:2 * o]
            o >>= 1
    return new, F32(part[0])


def kmeans(values: np.ndarray, centres: np.ndarray, tol: float, max_iterations: int):
    """-> (ids int32 [n] for the returned centres, centres float32 [K], Lloyd iterations run)."""
    values = np.asarray(values, dtype=F32).reshape(-1)
    c = np.asarray(centres, dtype=F32).reshape(-1).copy()
    K = c.shape[0]
    it = 0
    if values.shape[0] > 0 and max_iterations > 0:
        sv = sort_values(values)
        tol = F32(tol)
        while True:
            ids = assign(sv, c)
            sums = cluster_sums(sv, ids, K)
            sizes = np.bincount(ids, minlength=K)[:K]
            c, shift = update(c, sums, sizes)
            it += 1
            if shift < tol or it >= max_iterations:
                break
    return assign(values, c), c, it
