"""CPU: the k-means cases of tests/kmeans_edges.py reach the boundaries they are built for; the brute-force assignment of the
restatement (kmeans_det_order.assign) is gs_oracle's; an emulation of km_assign over canonically keyed sorted centres is the
reference's rule on every centre set, while the raw float_key order it replaced breaks it on exactly the signed-zero and -NaN sets;
and the bit-for-bit comparison of test_gpu_kmeans_edges.py rejects two planted summation-order near-misses."""
import numpy as np
import pytest

import gs_oracle
import kmeans_det_order as KD
import kmeans_edges as KE


@pytest.mark.parametrize("name", list(KE.CENTRE_SETS))
def test_centre_set_reaches_its_boundary(name):
    c, v = KE.centre_set(name)
    assert KE.CENTRE_REACH[name] <= KE.centre_reach(c, v)
    assert np.isnan(v).sum() >= 2 and np.isinf(v).sum() >= 2


def test_centre_sets_cover_every_edge():
    assert set().union(*KE.CENTRE_REACH.values()) == {"signed_zeros", "pos_zero_first", "runs", "all_equal", "midpoint", "far_tie",
                                                      "inf", "nan_pos", "nan_neg", "subnormal", "overflow_some", "overflow_all"}
    # ±0 in both orders, and 1024 centres of which ~300 are zeros of either sign with +0 at index 0
    assert KE.bits(KE.centre_set("zero_pm")[0]).tolist() == [0, 0x80000000]
    assert KE.bits(KE.centre_set("zero_mp")[0]).tolist() == [0x80000000, 0]
    c = KE.centre_set("zero_many")[0]
    assert KE.bits(c[0]) == 0 and (KE.bits(c) == 0x80000000).sum() > 100 and (KE.bits(c) == 0).sum() > 100
    # 1e8 is at distance 1e8 from 1, 2 and 3 after rounding: a three-way tie across two neighbours, won by index 1
    assert KE.brute(np.array([1e8, -1e8], KE.F32), KE.centre_set("far_ties")[0]).tolist() == [1, 1]


@pytest.mark.parametrize("name", list(KE.CENTRE_SETS))
def test_restatement_assign_is_the_oracle(name):
    c, v = KE.centre_set(name)
    with np.errstate(all="ignore"):
        want = gs_oracle.kmeans_update_ids(v, c)
    assert np.array_equal(KD.assign(v, c), want)
    assert np.array_equal(KE.brute(v, c), want)


@pytest.mark.parametrize("name", list(KE.CENTRE_SETS))
def test_sorted_centre_assignment_emulations(name):
    c, v = KE.centre_set(name)
    want = KE.brute(v, c)
    assert np.array_equal(KE.emulate(v, c, canonical=True), want)
    assert np.array_equal(KE.emulate(v, c, canonical=False), want) == (name not in KE.KEY_ORDER_BREAKS)


def test_the_raw_key_order_breaks_the_documented_examples():
    f = KE.F32
    # [+0, -0]: the run's first sorted element is the -0 at index 1
    assert KE.emulate(f([0.5, -0.0]), f([0.0, -0.0]), canonical=False).tolist() == [1, 1]
    assert KE.emulate(f([0.5, -0.0]), f([0.0, -0.0])).tolist() == [0, 0]
    # [5, +0, 3, -0]
    v, c = f([-2.0, 1.0, 0.5]), f([5.0, 0.0, 3.0, -0.0])
    assert KE.emulate(v, c, canonical=False).tolist() == [3, 3, 3] and KE.emulate(v, c).tolist() == [1, 1, 1]
    # [-NaN, 2]: the binary search stops on the NaN
    c = np.array([KE.NAN_NEG, 2.0], KE.F32)
    assert KE.emulate(f([1.0]), c, canonical=False).tolist() == [0] and KE.emulate(f([1.0]), c).tolist() == [1]
    assert KE.brute(f([1.0, -0.0]), c).tolist() == [1, 1]


_EXPECT = {            # name -> (n, blocks, final buffer, passes skipped)
    "n15": (15, 1, 0, 0),
    "m5_minus": (5 * 4096 - 1, 5, 0, 0),
    "m5": (5 * 4096, 5, 0, 0),
    "m5_plus": (5 * 4096 + 1, 6, 0, 0),
    "b257": (1_048_577, 257, 0, 0),
    "b293": (1_200_001, 293, 0, 0),
    "culled9m": (9_000_000, 2198, 0, 0),
    "radix_low8": (50_003, 13, 1, 3),
    "radix_low16": (50_003, 13, 0, 2),
    "radix_none": (8195, 3, 0, 4),
    "nonfinite": (40_000, 10, 0, 0),
    "allk": (4096, 1, 1, 1),
}


@pytest.mark.parametrize("name", list(KE.VALUE_SETS))
def test_value_set_reaches_its_boundary(name):
    v, c = KE.value_set(name)
    sv = KD.sort_values(v)
    ids = KE.brute(sv, c)
    r = KE.value_reach(ids, c.size)
    n, blocks, buf, skipped = _EXPECT[name]
    assert v.size == n and r["blocks"] == blocks and KE.final_buffer(v) == (buf, skipped)
    assert np.all(np.isfinite(c))
    if name == "n15":
        assert n < KD.CHUNK
    if name == "b257":                      # lane 0 adds blocks 0 and 256, the last block holds one value
        assert r["lane_adds"] and r["longest_span"] == 257
    if name == "b293":                      # more than 256 blocks, a cluster that starts off lane 0
        assert r["lane_adds"] and r["off_lane0"]
    if name == "culled9m":                  # 3 M rows x 3, >= 95 % zeros; a lane folds 9 parts; a long span starts off lane 0
        assert (v == 0).mean() > 0.94 and r["parts_per_lane"] == 9 and r["off_lane0_long"]
    if name == "allk":                      # one block holds all 1 024 clusters
        assert r["clusters_per_block"] == KE.K_MAX
    if name == "nonfinite":
        b = KE.bits(v)
        assert {0x7fc00000, 0xffc00000, 0x7f800000, 0xff800000, 0x80000000} <= set(b.tolist())
    # the restatement's assignment is the oracle's here as well (both are per-value functions: compared on the distinct values)
    u = np.unique(v)
    with np.errstate(all="ignore"):
        assert np.array_equal(KD.assign(u, c), gs_oracle.kmeans_update_ids(u, c))


def test_parity_of_the_final_buffer_is_reached_both_ways():
    assert {KE.final_buffer(KE.value_set(n)[0])[0] for n in KE.SMALL_VALUE_SETS} == {0, 1}


@pytest.mark.parametrize("name", list(KE.EXACT_SETS))
def test_exact_set_sums_exactly(name):
    v, c, k = KE.exact_set(name)
    n, _, K = KE.EXACT_SETS[name]
    assert v.size == n and c.size == K and np.all(np.isfinite(c))
    assert np.array_equal(v.astype(np.float64), k * np.float64(KE.STEP))
    assert int(np.abs(k).sum()) < 2 ** 24                  # every partial sum, in any order, is an exact float32
    if n >= 1_000_000:
        assert np.unique(k).size > 500 and (n + KE.BLOCK - 1) // KE.BLOCK > 256
    # the fp32 sums of any order are the float64 sums, so the restatement's sums are exact
    sv = KD.sort_values(v)
    ids = KE.brute(sv, c)
    got = KD.cluster_sums(sv, ids, K)
    assert np.array_equal(got.astype(np.float64), np.bincount(ids, weights=sv.astype(np.float64), minlength=K))


@pytest.mark.parametrize("mutation", ["lane_is_block", "lane_from_lo"])
def test_planted_near_misses_are_caught(mutation):
    caught = []
    for name in ("b257", "b293") + tuple(KE.SMALL_VALUE_SETS):
        v, c = KE.value_set(name)
        sv = KD.sort_values(v)
        ids = KE.brute(sv, c)
        good = KD.cluster_sums(sv, ids, c.size)
        bad = KE.planted_sums(sv, ids, c.size, mutation)
        if not np.array_equal(KE.bits(good), KE.bits(bad)):
            caught.append(name)
    print(mutation, "caught by", caught)
    # both only change the lane stage, so only sets with more than 256 blocks or spans off lane 0 can tell
    assert caught and set(caught) <= {"b257", "b293"}
