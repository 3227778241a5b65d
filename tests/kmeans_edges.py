"""Boundary cases of the codebook k-means (gsb_kmeans.cu, DESIGN.md §5j), shared by test_kmeans_edges_oracle.py (CPU) and
test_gpu_kmeans_edges.py.

* Centre sets: the assignment's edges.  Signed zeros in both orders and mixed, runs of equal centres up to all K = 1024 equal,
  exact midpoints, ties between centres that are not neighbours in sorted order (rounding makes |1e8 - c| equal for c = 1, 2, 3),
  ±inf and NaN centres of both signs, subnormal centres, and distances that overflow for some or for all centres.  Each set
  comes with probe values around its centres.
* Value sets: the sort and the two summation paths.  n below one chunk, n = 4096·m - 1, 4096·m, 4096·m + 1, more than 256
  deterministic blocks (1 048 577 and 1.2 M values), a 9 M zeros-heavy set shaped like a culled f_rest codebook, values that skip
  radix passes (final buffer 1 and 0, all four passes skipped), -NaN / ±inf values, and a block that holds all 1 024 clusters.
* Exact sets: multiples of 2^-6 whose sum of |v| is below 2^24 steps, so every partial sum is exact in any order and both paths
  and gs_oracle.kmeans must give the same centres bit for bit.
* Two emulations of km_assign over the sorted centres (the canonical key and the raw float_key it replaced), the brute-force
  assignment, reach predicates and the two planted summation-order near-misses.
"""
import functools

import numpy as np

import kmeans_det_order as KD

F32 = np.float32
BLOCK, LANES, K_MAX = KD.BLOCK, KD.LANES, 1024
STEP = F32(2.0 ** -6)                                  # the exact sets' unit


def bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.uint32)


def _f(x):
    return np.array(x, dtype=F32)


NAN_NEG = np.array([0xffc00000], np.uint32).view(F32)[0]
NAN_POS = np.array([0x7fc00000], np.uint32).view(F32)[0]


# ---------------------------------------------------------------------------------------------------------------- centre sets
def _zero_many(rng):
    c = rng.normal(size=K_MAX).astype(F32)
    z = rng.choice(np.arange(1, K_MAX), 300, replace=False)
    c[z] = np.where(rng.random(300) < 0.5, F32(-0.0), F32(0.0))
    c[0] = 0.0                                          # +0 at the lowest index, -0s both before and after it in key order
    return c


def _runs(rng):
    vals = rng.normal(size=60).astype(F32)
    mult = rng.integers(1, 40, size=60)
    c = np.repeat(vals, mult)[:K_MAX]
    c = np.concatenate([c, np.full(K_MAX - c.size, vals[0], F32)])
    return c[rng.permutation(K_MAX)]


CENTRE_SETS = {
    "zero_pm": lambda rng: _f([0.0, -0.0]),
    "zero_mp": lambda rng: _f([-0.0, 0.0]),
    "zero_mixed": lambda rng: _f([5.0, 0.0, 3.0, -0.0, -0.0, 0.0, -0.0, -4.0]),
    "zero_many": _zero_many,
    "runs": _runs,
    "all_equal": lambda rng: np.full(K_MAX, 0.25, F32),
    "midpoints": lambda rng: (2 * rng.permutation(np.arange(-256, 256))).astype(F32),
    "far_ties": lambda rng: _f([1e9, 1.0, 3.0, 2.0]),
    "inf": lambda rng: _f([2.0, np.inf, -np.inf, -5.0, np.inf, 7.0, -np.inf]),
    "nan_pos": lambda rng: np.array([NAN_POS, 2.0, -1.0, NAN_POS, 4.0], F32),
    "nan_neg": lambda rng: np.array([NAN_NEG, 2.0], F32),
    # no -inf centre: the lower-bound search would stop on it and never reach the NaNs before it in the raw key order
    "nan_mixed": lambda rng: np.array([NAN_POS, 2.0, np.inf, NAN_NEG, -3.0, NAN_NEG, 0.5], F32),
    "subnormal": lambda rng: _f([1e-45, -1e-45, 3e-45, 1.1754942e-38, 1.17549435e-38, -2e-39, 1e-30, 0.0]),
    "overflow_some": lambda rng: _f([-3e38, 1.0, 3e38, 2e19]),
    "overflow_all": lambda rng: _f([3e38, -3e38, 2e19]),
    "random1024": lambda rng: rng.normal(size=K_MAX).astype(F32),
    "k1": lambda rng: _f([0.25]),
}
# the sets on which the raw float_key order of the centres breaks the reference's rule
KEY_ORDER_BREAKS = {"zero_pm", "zero_mixed", "zero_many", "nan_neg", "nan_mixed"}

_SPECIAL = _f([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1e8, -1e8, 2e8, -2e8, 1e8 + 8, 1e19, -1e19, 3e38, -3e38, 3.4e38, 1.0,
               -1.0, 0.5, 0.25, -2.0, 2.5, 1e-38, -1e-38])


def probes(c, rng, n_random=2000):
    """Values around the centres: each finite centre, its neighbours in float32 and its zero-signed twin, the midpoints of
    neighbouring distinct centres and their neighbours, special values, NaNs of both signs, random values at the centres' scale."""
    f = np.unique(c[np.isfinite(c)])
    mid = ((f[:-1].astype(np.float64) + f[1:]) / 2).astype(F32)
    base = np.concatenate([f, mid, _SPECIAL])
    with np.errstate(all="ignore"):
        near = np.concatenate([np.nextafter(base, F32(np.inf)), np.nextafter(base, F32(-np.inf)), -base])
    big = float(np.abs(f).max(initial=0.0))
    rnd = (rng.normal(size=n_random) * (big if 1.0 < big < 1e30 else 1.0)).astype(F32)
    odd = np.arange(-513, 514, 2).astype(F32)           # the midpoints of the even-integer centres
    v = np.concatenate([base, near, rnd, odd, np.array([NAN_POS, NAN_NEG], F32)]).astype(F32)
    return v[rng.permutation(v.size)]


@functools.lru_cache(maxsize=None)
def centre_set(name):
    """-> (centres float32 [K], probe values float32 [n])."""
    rng = np.random.default_rng(sorted(CENTRE_SETS).index(name) + 100)
    c = CENTRE_SETS[name](rng)
    return c, probes(c, rng)


# ---------------------------------------------------------------------------------------------------------------- value sets
def _normal_with_zeros(rng, n, zero_share, scale=1.0):
    v = (scale * rng.normal(size=n)).astype(F32)
    v[rng.random(n) < zero_share] = 0.0
    return v


def _culled_f_rest(rng, rows=3_000_000, culled=0.95):
    """f_rest of one SH coefficient after band culling: [rows, 3], the culled rows all zero, the rest small normal values."""
    v = (0.05 * rng.normal(size=(rows, 3))).astype(F32)
    v[rng.random(rows) < culled] = 0.0
    return v.reshape(-1)


def _low_bits(rng, n, nbits):
    """Values whose float bits differ only in the low `nbits` bits: the other radix passes find one digit and are skipped."""
    return (np.uint32(0x3fc00000) | rng.integers(0, 1 << nbits, size=n).astype(np.uint32)).view(F32)


def _nonfinite(rng, n):
    v = rng.normal(size=n).astype(F32)
    for x, share in ((NAN_POS, 0.01), (NAN_NEG, 0.01), (np.inf, 0.005), (-np.inf, 0.005), (-0.0, 0.01)):
        v[rng.random(n) < share] = x
    return v


def _allk(rng):
    return np.repeat(np.arange(K_MAX, dtype=F32), 4)[rng.permutation(4 * K_MAX)]


# name -> (values(rng), K); the centres are K values drawn from the finite ones, as generate_codebook does
VALUE_SETS = {
    "n15": (lambda rng: rng.normal(size=15).astype(F32), 4),
    "m5_minus": (lambda rng: rng.normal(size=5 * BLOCK - 1).astype(F32), 64),
    "m5": (lambda rng: rng.normal(size=5 * BLOCK).astype(F32), 64),
    "m5_plus": (lambda rng: rng.normal(size=5 * BLOCK + 1).astype(F32), 64),
    "b257": (lambda rng: rng.normal(size=256 * BLOCK + 1).astype(F32), 1),
    "b293": (lambda rng: _normal_with_zeros(rng, 1_200_001, 0.95), 32),
    "culled9m": (lambda rng: _culled_f_rest(rng), 256),
    "radix_low8": (lambda rng: _low_bits(rng, 50_003, 8), 32),
    "radix_low16": (lambda rng: _low_bits(rng, 50_003, 16), 32),
    "radix_none": (lambda rng: np.full(2 * BLOCK + 3, 0.75, F32), 4),
    "nonfinite": (lambda rng: _nonfinite(rng, 40_000), 16),
    "allk": (_allk, K_MAX),
}
SMALL_VALUE_SETS = [k for k in VALUE_SETS if k not in ("b257", "b293", "culled9m")]
# the sets whose restatement converges in seconds (m5 and its neighbours take ~400 iterations; one of them is run)
CONVERGED_VALUE_SETS = ["n15", "m5_plus", "radix_low8", "radix_low16", "radix_none", "nonfinite", "allk"]


def _sample_centres(rng, v, K):
    f = v[np.isfinite(v)]
    return f[rng.integers(0, f.size, K)].copy()


@functools.lru_cache(maxsize=2)
def value_set(name):
    """-> (values float32 [n], initial centres float32 [K])."""
    rng = np.random.default_rng(sorted(VALUE_SETS).index(name) + 200)
    make, K = VALUE_SETS[name]
    v = make(rng)
    c = rng.permutation(np.arange(K_MAX, dtype=F32)) if name == "allk" else _sample_centres(rng, v, K)
    return v, c


# ---------------------------------------------------------------------------------------------------------------- exact sets
def _exact_ints(rng, n, zero_share):
    """Integers, mostly 0 and small, with 1 000 up to ±2000, so that there are about a thousand distinct values."""
    k = (1 + rng.geometric(0.35, size=n)).astype(np.int64) * rng.choice([-1, 1], size=n)
    k[rng.random(n) < zero_share] = 0
    tail = rng.choice(n, 1000, replace=False)
    k[tail] = rng.integers(-2000, 2001, size=1000)
    return k


# name -> (n, zero share, K)
EXACT_SETS = {
    "exact_allk": (4 * K_MAX, None, K_MAX),
    "exact_m5_plus": (5 * BLOCK + 1, 0.3, 64),
    "exact_b293": (1_200_001, 0.5, 256),
    "exact9m_k256": (9_000_000, 0.8, 256),
    "exact9m_k1024": (9_000_000, 0.8, K_MAX),
}


@functools.lru_cache(maxsize=1)
def exact_set(name):
    """-> (values float32 [n], initial centres float32 [K], integer images int64 [n]): values = ints · 2^-6."""
    rng = np.random.default_rng(sorted(EXACT_SETS).index(name) + 300)
    n, zero_share, K = EXACT_SETS[name]
    if zero_share is None:
        k = np.repeat(np.arange(K_MAX, dtype=np.int64), 4)[rng.permutation(n)]
    else:
        k = _exact_ints(rng, n, zero_share)
    v = (k * np.float64(STEP)).astype(F32)
    u = np.unique(v)                                     # centres drawn from the distinct values, so that most clusters are used
    return v, rng.choice(u, K, replace=K > u.size).astype(F32), k


# ---------------------------------------------------------------------------------------------------------------- assignment
def brute(values, centres):
    """The reference's rule (the restatement's brute-force assign), computed once per distinct value."""
    v = np.asarray(values, F32).reshape(-1)
    u, inv = np.unique(v, return_inverse=True)           # -0 / +0 and all NaNs merge: their distances are the same
    return KD.assign(u, centres)[inv.reshape(-1)]


def _dist(v, c):
    with np.errstate(all="ignore"):
        d = (c - v).astype(F32)
        return np.sqrt(d * d).astype(F32)


def centre_key(c, canonical=True):
    """The sort key of km_load_sorted_centres: canonical (-0 -> +0, every NaN -> the +NaN key 0xffffffff) or the raw float_key."""
    c = np.asarray(c, F32)
    if not canonical:
        return KD.float_key(c)
    k = KD.float_key(np.where(c == 0, F32(0.0), c))
    return np.where(np.isnan(c), np.uint32(0xffffffff), k).astype(np.uint32)


def emulate(values, centres, canonical=True):
    """km_load_sorted_centres + km_assign, vectorised over the values: sort by (key, index), runs of == centres, the lower-bound
    binary search on `c < v`, then the tie walks outwards from it."""
    v = np.asarray(values, F32).reshape(-1)
    c = np.asarray(centres, F32).reshape(-1)
    K = c.size
    key = centre_key(c, canonical)
    order = np.lexsort((np.arange(K), key))
    S_c, S_idx = KD.key_float(key[order]), order.astype(np.int64)
    run_start, run_end = np.arange(K), np.arange(1, K + 1)
    for i in range(K):
        a = i
        while a > 0 and S_c[a - 1] == S_c[i]:
            a -= 1
        b = i + 1
        while b < K and S_c[b] == S_c[i]:
            b += 1
        run_start[i], run_end[i] = a, b
    lo, hi = np.zeros(v.size, np.int64), np.full(v.size, K, np.int64)
    with np.errstate(invalid="ignore"):
        while np.any(lo < hi):
            act = lo < hi
            mid = (lo + hi) >> 1
            below = S_c[np.minimum(mid, K - 1)] < v
            lo = np.where(act & below, mid + 1, lo)
            hi = np.where(act & ~below, mid, hi)
    j = lo
    inf = F32(np.inf)
    dl = np.where(j > 0, _dist(v, S_c[np.maximum(j - 1, 0)]), inf)
    dr = np.where(j < K, _dist(v, S_c[np.minimum(j, K - 1)]), inf)
    dmin = np.fmin(dl, dr)
    best = np.full(v.size, np.iinfo(np.int64).max)
    p = j - 1
    live = p >= 0
    while np.any(live):
        q = np.maximum(p, 0)
        live &= _dist(v, S_c[q]) == dmin
        best = np.where(live, np.minimum(best, S_idx[run_start[q]]), best)
        p = np.where(live, run_start[q] - 1, p)
        live &= p >= 0
    p = j.copy()
    live = p < K
    while np.any(live):
        q = np.minimum(p, K - 1)
        live &= _dist(v, S_c[q]) == dmin
        best = np.where(live, np.minimum(best, S_idx[q]), best)
        p = np.where(live, run_end[q], p)
        live &= p < K
    with np.errstate(invalid="ignore"):
        return np.where(dmin < inf, best, 0).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------- restatement
def restate(values, centres, iterations, tol=0.0):
    """kmeans_det_order.kmeans with the assignment through `brute` -> the centres after each iteration run (the last one is where
    the shift fell below tol or `iterations` was reached)."""
    v = np.asarray(values, F32).reshape(-1)
    c = np.asarray(centres, F32).copy()
    sv = KD.sort_values(v)
    out = []
    for _ in range(iterations):
        ids = brute(sv, c)
        c, shift = KD.update(c, KD.cluster_sums(sv, ids, c.size), np.bincount(ids, minlength=c.size)[:c.size])
        out.append(c)
        if shift < F32(tol):
            break
    return out


def spans(ids, K):
    """(lo, hi) block of each cluster in the sorted order; lo > hi for an empty cluster."""
    b = np.arange(ids.size) // BLOCK
    lo, hi = np.full(K, np.iinfo(np.int64).max), np.full(K, -1)
    np.minimum.at(lo, ids, b)
    np.maximum.at(hi, ids, b)
    return lo, hi


def planted_sums(sorted_values, ids, K, mutation):
    """cluster_sums with a planted error in the lane stage of km_det_cluster_kernel:
    'lane_is_block'  lane l = b instead of b % 256 (a pairwise tree over all blocks);
    'lane_from_lo'   the span's first block is lane 0 (l = (b - lo) % 256)."""
    part_b, part_k, part = KD.block_parts(sorted_values, ids, K)
    if mutation == "lane_from_lo":
        lo, _ = spans(ids, K)
        return KD.lane_sums(part_b - lo[part_k], part_k, part, K)
    assert mutation == "lane_is_block"
    width = LANES
    while width <= part_b.max(initial=0):
        width *= 2
    lanes = np.full((K, width), -0.0, F32)
    lanes[part_k, part_b] = part
    with np.errstate(all="ignore"):
        return KD._pairwise(lanes) + F32(0.0)


# ---------------------------------------------------------------------------------------------------------------- reach
def final_buffer(values):
    """km_sort_plan_kernel: a pass is skipped when every key has the same digit; the sorted keys end in buffer (#passes run) % 2.
    -> (final buffer, passes skipped)."""
    k = KD.float_key(np.asarray(values, F32))
    skipped = sum(int(np.all(((k >> np.uint32(8 * p)) & 0xff) == ((k[0] >> np.uint32(8 * p)) & 0xff))) for p in range(4))
    return (4 - skipped) % 2, skipped


def value_reach(sorted_ids, K):
    """What the deterministic path meets on a sorted assignment: blocks, clusters per block, the longest span and parts per lane,
    whether a cluster spanning more than one lane row starts off lane 0, and whether a lane adds two parts."""
    n = sorted_ids.size
    n_blocks = (n + BLOCK - 1) // BLOCK
    lo, hi = spans(sorted_ids, K)
    used = lo <= hi
    per_block = max(np.unique(sorted_ids[b * BLOCK:(b + 1) * BLOCK]).size for b in range(n_blocks)) if n else 0
    width = np.where(used, hi - lo + 1, 0)
    return dict(blocks=n_blocks, clusters_per_block=per_block, longest_span=int(width.max(initial=0)),
                parts_per_lane=int(((width + LANES - 1) // LANES).max(initial=0)),
                off_lane0_long=bool(np.any(used & (width > LANES) & (lo % LANES != 0))),
                lane_adds=bool(np.any(width > LANES)),
                off_lane0=bool(np.any(used & (width >= 3) & (lo % LANES != 0))))


def centre_reach(c, v):
    """The assignment edges a centre set and its probes meet."""
    c, v = np.asarray(c, F32), np.asarray(v, F32)
    out = set()
    sb = bits(c) >> 31
    zeros = np.flatnonzero(c == 0)
    if zeros.size and np.any(sb[zeros] == 1) and np.any(sb[zeros] == 0):
        out.add("signed_zeros")
        if sb[zeros[0]] == 0:
            out.add("pos_zero_first")
    if np.any(np.isnan(c) & (sb == 1)):
        out.add("nan_neg")
    if np.any(np.isnan(c) & (sb == 0)):
        out.add("nan_pos")
    if np.any(c == np.inf) and np.any(c == -np.inf):
        out.add("inf")
    if np.any((c != 0) & (np.abs(c) < np.finfo(F32).tiny)):
        out.add("subnormal")
    fin = c[~np.isnan(c)]
    _, counts = np.unique(fin, return_counts=True)
    if counts.size and counts.max() >= 8:
        out.add("runs")
    if c.size == K_MAX and np.all(c == c[0]):
        out.add("all_equal")
    vv = v[np.isfinite(v)][:, None]
    d = _dist(vv, c[None, :])
    d = np.where(np.isnan(d), F32(np.inf), d)
    dmin = d.min(axis=1)
    finite = dmin < np.inf
    at_min = (d == dmin[:, None]) & finite[:, None]
    distinct = np.array([np.unique(c[r]).size for r in at_min])
    if np.any(distinct == 2):
        out.add("midpoint")
    if np.any(distinct >= 3):
        out.add("far_tie")
    if np.any(finite & np.any(np.isinf(d) & ~np.isnan(c)[None, :], axis=1)):
        out.add("overflow_some")
    if np.any(~finite & np.all(np.isinf(_dist(vv, c[None, :])), axis=1)):
        out.add("overflow_all")
    return out


CENTRE_REACH = {
    "zero_pm": {"signed_zeros", "pos_zero_first"},
    "zero_mp": {"signed_zeros"},
    "zero_mixed": {"signed_zeros", "pos_zero_first", "midpoint"},
    "zero_many": {"signed_zeros", "pos_zero_first", "runs", "midpoint"},
    "runs": {"runs", "midpoint"},
    "all_equal": {"runs", "all_equal"},
    "midpoints": {"midpoint"},
    "far_ties": {"far_tie"},
    "inf": {"inf", "midpoint"},
    "nan_pos": {"nan_pos", "midpoint"},
    "nan_neg": {"nan_neg"},
    "nan_mixed": {"nan_pos", "nan_neg"},
    "subnormal": {"subnormal", "far_tie"},
    "overflow_some": {"overflow_some"},
    "overflow_all": {"overflow_all"},
    "random1024": {"midpoint"},
    "k1": set(),
}
