# coding=utf-8
"""The statistics of tests/sampling_stats.py have power at the sample sizes the GPU tests use: each accepts exact
samples from numpy.random.Generator (independent of Philox) and rejects a planted defect, a few lines of numpy each.
tests/test_gpu_sampling_stats.py names, for each of its checks, the test here that shows its statistic's power."""
import math

import numpy as np
import pytest

import sampling_stats as st


def _rng(tag):
    return np.random.default_rng(20261018 + tag)


def _reservoir(n, d, k, rng, lo=1):
    """n rows of Algorithm R over [0, d): slot j starts at j; for i >= k draw j in [0, i + lo) and keep i if j < k.
    lo = 1 is the algorithm; lo = 0 draws j from [0, i), the off-by-one."""
    res = np.tile(np.arange(k), (n, 1))
    rows = np.arange(n)
    for i in range(k, d):
        j = rng.integers(0, i + lo, size=n)
        hit = j < k
        res[rows[hit], j[hit]] = i
    return res


def _exact_subsets(n, d, k, rng):
    """n independent uniform k-subsets of [0, d), from random keys (an algorithm unlike the kernels')."""
    return np.argsort(rng.random((n, d)), axis=1)[:, :k]


def _rejects(fn, *args):
    """True when the require_* check fails."""
    try:
        fn(*args)
    except AssertionError:
        return True
    return False


# ---- fan-out without replacement --------------------------------------------------------------------------------

@pytest.mark.parametrize("d,k", [(5, 2), (7, 3), (10, 3)])
def test_inclusion_and_subsets_accept_exact_and_reject_algorithm_r_off_by_one(d, k):
    """test_gpu_sampling_stats thread-tier, ratio (d 10, k 3) and exclusion checks: per-position inclusion and whole-
    subset uniformity at ROWS rows."""
    for sample in (_exact_subsets(st.ROWS, d, k, _rng(1)), _reservoir(st.ROWS, d, k, _rng(2))):
        st.check_subsets(sample, d)
        st.require(st.inclusion_p(sample, d), "inclusion")
        if math.comb(d, k) <= 120:
            st.require(st.subset_p(sample, d), "subsets")
    bad = _reservoir(st.ROWS, d, k, _rng(3), lo=0)
    assert st.inclusion_p(bad, d) < st.P_FLOOR
    if math.comb(d, k) <= 120:
        assert st.subset_p(bad, d) < st.P_FLOOR


@pytest.mark.parametrize("d", [127, 128, 129, 1000])
def test_wide_rows_inclusion_and_pairs(d):
    """test_gpu_sampling_stats K13 checks across the thread-row limit: ROWS_WIDE rows with k = d // 2; per-position
    inclusion and the pairs (0, 1), (0, d - 1), (d - 2, d - 1).  Planted: a reservoir that skips the last entry
    (pairs with d - 1) and one whose slot 0 is never replaced (pairs with 0).  (Algorithm R's off-by-one moves a
    position's inclusion by about 1/k, too little to see here; the small rows above catch it.)"""
    k = d // 2
    pairs = ((0, 1), (0, d - 1), (d - 2, d - 1))
    good = _reservoir(st.ROWS_WIDE, d, k, _rng(4))
    st.require(st.inclusion_p(good, d), "inclusion")
    for a, b in pairs:
        st.require(st.pair_p(good, d, a, b), "pair")
    no_last = _reservoir(st.ROWS_WIDE, d - 1, k, _rng(6))
    assert st.pair_p(no_last, d, d - 2, d - 1) < st.P_FLOOR and st.pair_p(no_last, d, 0, d - 1) < st.P_FLOOR
    stuck0 = np.concatenate([np.zeros((st.ROWS_WIDE, 1), np.int64), 1 + _reservoir(st.ROWS_WIDE, d - 1, k - 1, _rng(7))],
                            axis=1)
    assert st.pair_p(stuck0, d, 0, 1) < st.P_FLOOR and st.pair_p(stuck0, d, 0, d - 1) < st.P_FLOOR


def _hub_tally(sampler):
    t = st.HubTally(st.HUB_DEGREE)
    for key in range(st.HUB_KEYS):
        t.add(sampler(_rng(100 + key)))
    return t.ps()


def _hub_rows(rng, d, skip_last=False, stuck0=False):
    n = st.HUB_ROWS
    if stuck0:
        return np.concatenate([np.zeros((n, 1), np.int64),
                               1 + np.stack([rng.choice(d - 1, st.HUB_K - 1, replace=False) for _ in range(n)])], axis=1)
    return np.stack([rng.choice(d - 1 if skip_last else d, st.HUB_K, replace=False) for _ in range(n)])


def test_hub_tally_accepts_exact_and_rejects_edge_defects():
    """test_gpu_sampling_stats hub checks (the CTA path): HUB_ROWS x HUB_KEYS samples of k = d / 2 from d = 60 000,
    position buckets and the three pairs.  Planted: the last entry never drawn; slot 0 never replaced."""
    d = st.HUB_DEGREE
    good = _hub_tally(lambda rng: _hub_rows(rng, d))
    for name, p in good.items():
        st.require(p, "hub {}".format(name))
    last = _hub_tally(lambda rng: _hub_rows(rng, d, skip_last=True))
    assert last[(d - 2, d - 1)] < st.P_FLOOR and last[(0, d - 1)] < st.P_FLOOR
    zero = _hub_tally(lambda rng: _hub_rows(rng, d, stuck0=True))
    assert zero[(0, 1)] < st.P_FLOOR and zero[(0, d - 1)] < st.P_FLOOR


# ---- replacement ------------------------------------------------------------------------------------------------

def test_replacement_accepts_iid_and_rejects_a_missing_last_neighbour():
    """test_gpu_sampling_stats padding checks: ROWS rows of 8 draws over 5 neighbours."""
    d, k = 5, 8
    p_pos, p_pair = st.replacement_p(_rng(8).integers(0, d, size=(st.ROWS, k)), d)
    st.require(p_pos, "positions")
    st.require(p_pair, "ordered pairs")
    p_pos, p_pair = st.replacement_p(_rng(9).integers(0, d - 1, size=(st.ROWS, k)), d)
    assert p_pos < st.P_FLOOR and p_pair < st.P_FLOOR
    # the same draw repeated across a row: uniform positions, but the ordered pairs are not
    same = np.repeat(_rng(10).integers(0, d, size=(st.ROWS, 1)), k, axis=1)
    assert st.replacement_p(same, d)[1] < st.P_FLOOR


# ---- means ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d,k", [(10, 5), (300, 150)])
def test_mean_variance_separates_without_from_with_replacement(d, k):
    """test_gpu_sampling_stats estimator checks: EST_SAMPLES means of k of d values.  Planted: with replacement."""
    v = _rng(11).standard_normal(d)
    sub = _exact_subsets(st.EST_SAMPLES, d, k, _rng(12))
    st.require_mean(v[sub].mean(axis=1), v, k, "without replacement")
    rep = _rng(13).integers(0, d, size=(st.EST_SAMPLES, k))
    assert _rejects(st.require_mean, v[rep].mean(axis=1), v, k, "with replacement")


# ---- independence -----------------------------------------------------------------------------------------------

def test_independence_accepts_independent_rows_and_rejects_copies():
    """test_gpu_sampling_stats independence checks: ROWS / 2 row pairs of 2-subsets of 5 (two rows of one call, hop 0
    against hop 1, consecutive unseeded calls).  Planted: one row's draws copied to every row; the same key at both
    hops (the two samples of a row equal)."""
    a = st.subset_codes(_exact_subsets(st.ROWS, 5, 2, _rng(14)))
    st.require(st.independence_p(a[0::2], a[1::2]), "two rows")
    b = st.subset_codes(_exact_subsets(st.ROWS, 5, 2, _rng(15)))
    st.require(st.independence_p(a, b), "two hops")
    copied = np.tile(a[:1], st.ROWS)
    assert st.independence_p(copied[0::2], copied[1::2]) < st.P_FLOOR
    assert st.independence_p(a, a) < st.P_FLOOR                     # hop 1 keyed like hop 0
    # half the rows copied is enough
    half = a.copy()
    half[1::4] = half[0::4]
    assert st.independence_p(half[0::2], half[1::2]) < st.P_FLOOR


def test_negative_batches_independence():
    """test_gpu_sampling_stats negative_sampling batch checks: NODE_DRAWS // 8 pairs of ids over 7 nodes."""
    n = st.NODE_DRAWS // 8
    a, b = _rng(17).integers(0, 7, n), _rng(18).integers(0, 7, n)
    st.require(st.independence_p(a, b), "batches")
    assert st.independence_p(a, a) < st.P_FLOOR


def test_negative_inclusion_without_replacement():
    """test_gpu_sampling_stats negative_sampling without replacement: NEG_BATCHES batches of S of C = 65 candidates,
    shuffle (S = 40) and redraw (S = 20) sizes.  Planted: draws that never reach the last candidate."""
    C = 65
    for S in (40, 20):
        good = _exact_subsets(st.NEG_BATCHES, C, S, _rng(19))
        st.require(st.inclusion_p(good, C), "inclusion")
        for a, b in ((0, 1), (0, C - 1)):
            st.require(st.pair_p(good, C, a, b), "pair")
        short = _exact_subsets(st.NEG_BATCHES, C - 1, S, _rng(20))
        assert st.inclusion_p(short, C) < st.P_FLOOR and st.pair_p(short, C, 0, C - 1) < st.P_FLOOR


# ---- Bernoulli --------------------------------------------------------------------------------------------------

def test_keep_probabilities():
    assert st.dropout_keep(0.0) == 1.0 and st.dropout_keep(1.0) == 0.0
    assert st.dropout_keep(0.5) == 0.5
    assert st.bernoulli_keep(1.0) == 1.0 and st.bernoulli_keep(0.0) == 1 / (1 << 24)
    assert st.bernoulli_keep(0.5) == 0.5 + 1 / (1 << 24)
    # 0.1 is not a float32: the threshold is its float32 rounding
    assert st.dropout_keep(0.1) == 1.0 - math.ceil(float(np.float32(0.1)) * (1 << 24)) / (1 << 24)


@pytest.mark.parametrize("rate", [0.1, 0.5, 0.9])
def test_keep_rate_and_adjacency_have_power(rate):
    """test_gpu_sampling_stats Bernoulli checks: BERNOULLI_N trials.  Planted: a keep rate off by 0.003; dropout lanes
    that share one 32-bit word (elements 2m and 2m + 1 read the same u)."""
    p_keep = st.dropout_keep(rate)
    u = (_rng(21).integers(0, 1 << 32, st.BERNOULLI_N, dtype=np.uint64) >> np.uint64(8)).astype(np.float64) / (1 << 24)
    keep = u >= np.float32(rate)
    st.require(st.keep_rate_p(keep.sum(), keep.size, p_keep), "keep rate")
    st.require(st.adjacent_p(keep), "adjacent elements")
    assert st.keep_rate_p(keep.sum(), keep.size, p_keep + 0.003) < st.P_FLOOR
    shared = np.repeat(u[::2], 2)[:st.BERNOULLI_N] >= np.float32(rate)
    st.require(st.keep_rate_p(shared.sum(), shared.size, p_keep), "shared-word keep rate")
    assert st.adjacent_p(shared) < st.P_FLOOR


# ---- node ids ---------------------------------------------------------------------------------------------------

NODE_NS = [7, 1000, 111059956, 244160499, 1600000000, (1 << 31) - 1]


@pytest.mark.parametrize("N", NODE_NS)
def test_node_ids_accept_uniform_draws(N):
    """test_gpu_sampling_stats node-id checks: NODE_DRAWS ids, uniform on [0, N)."""
    st.require_node_ids(_rng(22).integers(0, N, st.NODE_DRAWS), N, "uniform")


def _u32(tag):
    return _rng(tag).integers(0, 1 << 32, st.NODE_DRAWS, dtype=np.uint64)


@pytest.mark.parametrize("N", [111059956, 244160499, 1600000000])
def test_heavy_share_rejects_32_bit_multiply_shift(N):
    """32-bit multiply-shift, (u * N) >> 32: the heavy ids take more than their share."""
    v = ((_u32(23) * np.uint64(N)) >> np.uint64(32)).astype(np.int64)
    share, want, p = st.heavy_p(v, N)
    assert share > want and p < st.P_FLOOR, (share, want, p)


def test_heavy_ids_count_the_preimages():
    """2^32 mod N ids of [0, N) have ceil(2^32 / N) multiply-shift preimages, the rest one fewer."""
    for N in (7, 1000, 3001, 1 << 20):
        assert st.heavy_ids(np.arange(N), N).sum() == ((1 << 32) % N or N)


def test_range_and_low_bit_statistics_have_power():
    """Range buckets reject u mod N (low ids over-weighted); low bits reject ids drawn as twice a draw below N / 2
    (even ids only)."""
    N = 1600000000
    assert st.range_p((_u32(24) % np.uint64(N)).astype(np.int64), N) < st.P_FLOOR
    even = ((_u32(25) * np.uint64(N // 2)) >> np.uint64(32)).astype(np.int64) * 2
    assert st.low_bits_p(even, N) < st.P_FLOOR
