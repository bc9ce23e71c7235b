# coding=utf-8
"""Exact distributions of layer-neighbour (LABOR-0) draws and the statistics that test them, written from the rule's
properties (include/tfgk.h, "LABOR block sampler"), not from its code: each candidate of a row is kept with probability
pi(k, d); given the count m, the kept set is uniform over the m-subsets of the row's distinct columns; two rows holding
one column both keep it with probability min(pi_1, pi_2) (under one key); a column is reached with probability the max
of pi over the rows holding it, independently of other columns.  One p-value floor and fixed keys, as
tests/sampling_stats.py.  TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np
from scipy import stats

from sampling_stats import P_FLOOR, require, _chi2_counts  # noqa: F401  (require is re-exported for the tests)


def inclusion_p(kept, p):
    """kept bool [n, d]: n independent rows of d distinct columns, each kept with probability p independently of the
    other columns' (distinct columns have independent variates).  Chi-square over the d columns' counts, d dof."""
    kept = np.asarray(kept, bool)
    n = kept.shape[0]
    cnt = kept.sum(axis=0).astype(np.float64)
    t = float(((cnt - n * p) ** 2).sum() / (n * p * (1.0 - p)))
    return float(stats.chi2.sf(t, kept.shape[1]))


def subset_given_count_p(kept):
    """kept bool [n, d] (d <= 20): given its count m, each row's kept set is uniform over the C(d, m) m-subsets.  The
    per-count chi-squares are summed, with their degrees of freedom."""
    kept = np.asarray(kept, bool)
    d = kept.shape[1]
    code = (kept.astype(np.int64) << np.arange(d, dtype=np.int64)).sum(axis=1)
    m = kept.sum(axis=1)
    t, dof = 0.0, 0
    for c in np.unique(m):
        sub = code[m == c]
        size = math.comb(d, int(c))
        if size < 2:
            continue
        _, cnt = np.unique(sub, return_counts=True)
        obs = np.concatenate([cnt, np.zeros(size - len(cnt))]).astype(np.float64)
        e = len(sub) / size
        t += float(((obs - e) ** 2 / e).sum())
        dof += size - 1
    return float(stats.chi2.sf(t, dof)) if dof else 1.0


def empty_p(kept, p):
    """Rows that keep nothing: probability (1 - p)^d over d distinct columns (exact binomial test)."""
    kept = np.asarray(kept, bool)
    n, d = kept.shape
    return float(stats.binomtest(int((~kept.any(axis=1)).sum()), n, (1.0 - p) ** d).pvalue)


def pair_p(both, n, p):
    """Exact binomial test of `both` joint keeps out of n independent trials of joint probability p."""
    return float(stats.binomtest(int(both), int(n), p).pvalue)


def total_p(total, mean, var):
    """A sum of many independent Bernoulli reaches against its mean and variance (normal, two-sided)."""
    return float(2.0 * stats.norm.sf(abs(total - mean) / math.sqrt(var)))
