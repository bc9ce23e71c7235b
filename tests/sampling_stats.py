# coding=utf-8
"""Exact distributions of the samplers' draws and the statistics that test them.

The probabilities here are written from the operators' contracts, not from their code: a fan-out of k from a row of
degree d without replacement keeps every k-subset with probability 1 / C(d, k); with replacement it makes k independent
uniform draws; node ids are uniform on [0, N); a Bernoulli keep rule keeps with the probability its float32 threshold
gives.  Nothing here restates Philox or any kernel, so a defect shared by a kernel and its bit-exact restatement (an
off-by-one in Algorithm R, a reused key, a biased integer draw) still fails these checks.

Every check compares a p-value with one floor, P_FLOOR, and every caller draws with fixed keys, so a check is
deterministic.  The sample sizes are constants here because tests/test_sampling_stats_host.py shows, at exactly these
sizes, that each statistic accepts exact samples and rejects the defects it is meant to catch; the GPU tests
(tests/test_gpu_sampling_stats.py) use the same constants.
TEST INFRASTRUCTURE ONLY: nothing under tf_geometric_b200/ imports it."""
import math

import numpy as np
from scipy import stats

P_FLOOR = 1e-6

# sample sizes shared by the host power tests and the GPU tests
ROWS = 20000              # rows of each tested degree in one call (thread tier, ratio, padding, independence)
ROWS_WIDE = 2000          # rows of degree 127 ... 1000 in one call (K13 on both sides of its thread-row limit)
HUB_DEGREE = 60000        # a CTA-path row far past the thread-row limit
HUB_ROWS = 64             # hub rows per call
HUB_KEYS = 16             # calls over the hub rows: HUB_ROWS * HUB_KEYS independent hub samples
HUB_K = HUB_DEGREE // 2   # the hub's fan-out: pair inclusion near 1/4
HUB_BUCKETS = 600         # per-position inclusion of a hub row over equal position ranges
NODE_DRAWS = 400000       # node ids per N
NEG_BATCHES = 3000        # negative_sampling batches for per-candidate and pair inclusion
EST_SAMPLES = 2048        # mean-aggregation samples per estimator check
BERNOULLI_N = 1 << 20     # elements or edges per keep-rate check
BUCKETS = 1024            # range buckets and low-bit classes of the node-id statistics


def require(p, what):
    """Fail with the statistic's p-value when it is below the floor."""
    assert p > P_FLOOR, "{}: p = {:.3g} <= {:g}".format(what, p, P_FLOOR)


def _chi2_counts(observed, expected, dof=None):
    """Pearson's chi-square p-value of counts against expected counts (classes with zero expectation must be empty)."""
    observed = np.asarray(observed, np.float64).ravel()
    expected = np.asarray(expected, np.float64).ravel()
    zero = expected == 0
    if observed[zero].any():
        return 0.0
    o, e = observed[~zero], expected[~zero]
    t = float(((o - e) ** 2 / e).sum())
    return float(stats.chi2.sf(t, len(o) - 1 if dof is None else dof))


# ---- fan-out without replacement --------------------------------------------------------------------------------

def check_subsets(pos, d):
    """pos int [n, k]: every row holds k distinct positions in [0, d) (exact, not statistical)."""
    pos = np.asarray(pos)
    assert pos.min() >= 0 and pos.max() < d, (pos.min(), pos.max(), d)
    s = np.sort(pos, axis=1)
    assert (s[:, 1:] != s[:, :-1]).all(), "a position drawn twice where the sample is without replacement"


def inclusion_p(pos, d):
    """Per-position inclusion of n independent k-subsets of [0, d): P(p kept) = k / d.
    The counts' covariance is c d / (d - 1) (I - 11'/d) n with c = (k/d)(1 - k/d), so
    sum (O - E)^2 (d - 1) / (n c d) is chi-square with d - 1 degrees of freedom."""
    pos = np.asarray(pos)
    n, k = pos.shape
    cnt = np.bincount(pos.ravel(), minlength=d).astype(np.float64)
    p = k / d
    c = p * (1.0 - p)
    t = float(((cnt - n * p) ** 2).sum()) * (d - 1) / (n * c * d)
    return float(stats.chi2.sf(t, d - 1))


class HubTally(object):
    """Per-position inclusion of large rows over HUB_BUCKETS equal ranges and the pair inclusion of (0, 1), (0, d - 1)
    and (d - 2, d - 1), accumulated chunk by chunk so that no [n, k] array of a hub's samples is kept."""

    def __init__(self, d):
        self.d, self.n, self.k = d, 0, None
        self.buckets = np.zeros(HUB_BUCKETS, np.int64)
        self.pairs = {(0, 1): 0, (0, d - 1): 0, (d - 2, d - 1): 0}

    def add(self, pos):
        pos = np.asarray(pos)
        check_subsets(pos, self.d)
        self.n += pos.shape[0]
        self.k = pos.shape[1]
        self.buckets += np.bincount(pos.ravel().astype(np.int64) * HUB_BUCKETS // self.d, minlength=HUB_BUCKETS)
        kept = {p: (pos == p).any(axis=1) for p in (0, 1, self.d - 2, self.d - 1)}
        for a, b in self.pairs:
            self.pairs[(a, b)] += int((kept[a] & kept[b]).sum())

    def ps(self):
        """{"buckets": p, (a, b): p for each pair}"""
        d, k = self.d, self.k
        size = np.diff(np.ceil(np.arange(HUB_BUCKETS + 1) * d / HUB_BUCKETS)).astype(np.float64)
        out = {"buckets": _chi2_counts(self.buckets, self.n * k * size / d)}
        for ab, both in self.pairs.items():
            out[ab] = float(stats.binomtest(both, self.n, k * (k - 1) / (d * (d - 1))).pvalue)
        return out


def subset_p(pos, d):
    """Whole-subset uniformity: every one of the C(d, k) subsets has probability 1 / C(d, k)."""
    pos = np.asarray(pos)
    k = pos.shape[1]
    code = (np.int64(1) << pos.astype(np.int64)).sum(axis=1)
    _, cnt = np.unique(code, return_counts=True)
    m = math.comb(d, k)
    obs = np.concatenate([cnt, np.zeros(m - len(cnt))])
    return _chi2_counts(obs, np.full(m, len(pos) / m))


def subset_codes(pos):
    """Each row's subset as one integer (rows of one degree), for contingency tests."""
    return (np.int64(1) << np.asarray(pos).astype(np.int64)).sum(axis=1)


def pair_p(pos, d, a, b):
    """Pair inclusion: P(a and b both kept) = k (k - 1) / (d (d - 1)), rows independent (exact binomial test)."""
    pos = np.asarray(pos)
    n, k = pos.shape
    both = int(((pos == a).any(axis=1) & (pos == b).any(axis=1)).sum())
    return float(stats.binomtest(both, n, k * (k - 1) / (d * (d - 1))).pvalue)


# ---- fan-out with replacement -----------------------------------------------------------------------------------

def replacement_p(draws, d):
    """k independent uniform draws over [0, d) per row: (position counts over all draws, the ordered pair (draw 0,
    draw 1) over d^2 classes) p-values."""
    draws = np.asarray(draws)
    n, k = draws.shape
    p_pos = _chi2_counts(np.bincount(draws.ravel(), minlength=d), np.full(d, n * k / d))
    pair = draws[:, 0].astype(np.int64) * d + draws[:, 1]
    p_pair = _chi2_counts(np.bincount(pair, minlength=d * d), np.full(d * d, n / (d * d)))
    return p_pos, p_pair


# ---- sample means -----------------------------------------------------------------------------------------------

def mean_check(means, v, k):
    """Sample means over rows of values v (k drawn without replacement): the mean is near mean(v); the variance is consistent with sigma^2 / k (d - k) / (d - 1), and inconsistent with the with-replacement
    sigma^2 / k.  Returns (z of the mean, z of the variance against the finite-population value, z against the
    with-replacement value); the variance's standard error comes from the sample's fourth moment."""
    means = np.asarray(means, np.float64)
    v = np.asarray(v, np.float64)
    n, d = len(means), len(v)
    sigma2 = v.var()
    v_fpc = sigma2 / k * (d - k) / (d - 1)
    v_rep = sigma2 / k
    z_mean = (means.mean() - v.mean()) / math.sqrt(v_fpc / n)
    dev = means - means.mean()
    s2 = (dev ** 2).sum() / (n - 1)
    se = math.sqrt(max(((dev ** 4).mean() - s2 ** 2) / n, 1e-300))
    return z_mean, (s2 - v_fpc) / se, (s2 - v_rep) / se


def require_mean(means, v, k, what):
    zm, zf, zr = mean_check(means, v, k)
    zf_max = stats.norm.isf(P_FLOOR / 2)
    assert abs(zm) < 4.0, "{}: sample mean {:.2f} standard errors from the population mean".format(what, zm)
    assert abs(zf) < zf_max, "{}: variance {:.2f} se from the finite-population value".format(what, zf)
    assert zr < -zf_max, "{}: variance only {:.2f} se below the with-replacement value".format(what, zr)


# ---- Bernoulli rules --------------------------------------------------------------------------------------------

def dropout_keep(rate):
    """Keep probability of u >= rate, u uniform on the 2^24 values i / 2^24 (dropout, drop_edge)."""
    rate = float(np.float32(rate))
    return 1.0 - min(math.ceil(rate * (1 << 24)), 1 << 24) / (1 << 24)


def bernoulli_keep(prob):
    """Keep probability of u <= prob with prob rounded to float32 (UniformNeighborSampler)."""
    prob = float(np.float32(prob))
    return min(math.floor(prob * (1 << 24)) + 1, 1 << 24) / (1 << 24) if prob >= 0 else 0.0


def keep_rate_p(kept, n, p_keep):
    """Exact binomial test of kept out of n independent trials."""
    return float(stats.binomtest(int(kept), int(n), p_keep).pvalue)


def independence_p(a, b):
    """Contingency test of paired categorical outcomes (a[i], b[i]); empty classes are dropped."""
    _, ia = np.unique(np.asarray(a), return_inverse=True)
    _, ib = np.unique(np.asarray(b), return_inverse=True)
    table = np.zeros((ia.max() + 1, ib.max() + 1))
    np.add.at(table, (ia, ib), 1)
    if table.shape[0] < 2 or table.shape[1] < 2:
        return 0.0 if len(a) > 1 else 1.0
    return float(stats.chi2_contingency(table, correction=False)[1])


def adjacent_p(flags):
    """Independence of flag[i] and flag[i + 1] for each lane i & 3 (lane 3's neighbour is in the next Philox block):
    the smallest of the four p-values, each over disjoint pairs."""
    f = np.asarray(flags).astype(np.int64)
    n4 = (len(f) - 1) // 4 * 4
    ps = [independence_p(f[lane:n4:4], f[lane + 1:n4 + 1:4]) for lane in range(4)]
    return min(ps)


# ---- node ids uniform on [0, N) ---------------------------------------------------------------------------------

def _ceil_div(a, n):
    return (a + np.uint64(n - 1)) // np.uint64(n)


def heavy_ids(v, N):
    """True where id v has ceil(2^32 / N) preimages under 32-bit multiply-shift (u * N) >> 32."""
    v = np.asarray(v, np.uint64)
    pre = _ceil_div((v + np.uint64(1)) << np.uint64(32), N) - _ceil_div(v << np.uint64(32), N)
    return pre == np.uint64(-(-(1 << 32) // N))


def heavy_share(N):
    """Share of [0, N) that multiply-shift over-weights: 2^32 mod N ids (none when N divides 2^32)."""
    return ((1 << 32) % N) / N


def heavy_p(v, N):
    """(observed heavy share, expected share, p-value): draws landing on the heavy ids against their share of [0, N)."""
    share = heavy_share(N)
    if share == 0.0:                    # N divides 2^32: every id has the same number of preimages
        return 0.0, 0.0, 1.0
    h = int(heavy_ids(v, N).sum())
    return h / len(v), share, float(stats.binomtest(h, len(v), share).pvalue)


def range_p(v, N, buckets=BUCKETS):
    """Chi-square of the ids over `buckets` equal ranges of [0, N) (the exact number of ids in each range)."""
    v = np.asarray(v, np.int64)
    b = v * buckets // N
    edges = -(-np.arange(buckets + 1, dtype=np.int64) * N // buckets)
    return _chi2_counts(np.bincount(b, minlength=buckets), len(v) * np.diff(edges) / N)


def low_bits_p(v, N, buckets=BUCKETS):
    """Chi-square of v mod `buckets` against the exact number of ids of [0, N) in each class."""
    v = np.asarray(v, np.int64)
    size = np.full(buckets, N // buckets, np.float64) + (np.arange(buckets) < N % buckets)
    return _chi2_counts(np.bincount(v % buckets, minlength=buckets), len(v) * size / N)


def node_id_ps(v, N):
    """The three node-id statistics: {"heavy": (share, expected, p), "range": p, "low": p}; ids outside [0, N) fail."""
    v = np.asarray(v, np.int64)
    assert v.min() >= 0 and v.max() < N, (v.min(), v.max(), N)
    return {"heavy": heavy_p(v, N), "range": range_p(v, N), "low": low_bits_p(v, N)}


def require_node_ids(v, N, what):
    ps = node_id_ps(v, N)
    share, want, p = ps["heavy"]
    require(p, "{} N={}: heavy-id share {:.4f}, {:.4f} under uniform draws".format(what, N, share, want))
    require(ps["range"], "{} N={}: range buckets".format(what, N))
    require(ps["low"], "{} N={}: low bits".format(what, N))
