# coding=utf-8
"""Exact distributions of the weighted fan-outs, written from the draw rule's contract (successive sampling without
replacement, independent draws P = w / W with replacement), not from the kernels: nothing here restates Philox or the
key.  The floor, the verdict and the chi-square statistic are tests/sampling_stats.py's.  The sample sizes are constants
because tests/test_weighted_sampling_host.py shows, at exactly these sizes, that each statistic accepts exact samples and
rejects planted defects; tests/test_gpu_weighted_sampling.py uses the same constants.
TEST INFRASTRUCTURE ONLY: nothing under tf_geometric_b200/ imports it."""
import itertools

import numpy as np

from sampling_stats import P_FLOOR, require, _chi2_counts  # noqa: F401  (re-exported for the GPU tests)

SUBSET_ROWS = 20000         # rows of one weight vector per subset check
REPLACE_ROWS = 20000        # rows per with-replacement check
HUB_ROWS = 64               # CTA-path rows per call
HUB_KEYS = 16               # calls over them


def subset_probs(w, k):
    """{sorted tuple of entries: probability} of successive sampling of k entries by weight (entries of weight 0 are
    never drawn); enumerated over ordered draws."""
    w = np.asarray(w, np.float64)
    cand = [i for i in range(len(w)) if w[i] > 0]
    k = min(k, len(cand))
    out = {}
    for seq in itertools.permutations(cand, k):
        p, rest = 1.0, w[cand].sum()
        for i in seq:
            p *= w[i] / rest
            rest -= w[i]
        key = tuple(sorted(seq))
        out[key] = out.get(key, 0.0) + p
    return out


def subset_p(pos, w, k):
    """Chi-square p-value of the drawn subsets (pos int [n, k'], each row's entries) against subset_probs."""
    probs = subset_probs(w, k)
    keys = sorted(probs)
    index = {s: i for i, s in enumerate(keys)}
    counts = np.zeros(len(keys) + 1)
    for row in np.asarray(pos):
        counts[index.get(tuple(sorted(int(x) for x in row)), len(keys))] += 1
    expected = np.array([probs[s] for s in keys] + [0.0]) * len(pos)
    return _chi2_counts(counts, expected)


def inclusion_probs(w, k):
    """Per-entry inclusion of successive sampling for k in {1, 2}: w_i / W, and w_i / W + sum_j (w_j / W) w_i / (W - w_j)."""
    w = np.asarray(w, np.float64)
    W = w.sum()
    p1 = w / W
    if k == 1:
        return p1
    assert k == 2
    second = np.array([sum(w[j] / W * w[i] / (W - w[j]) for j in range(len(w)) if j != i and w[j] > 0)
                       for i in range(len(w))])
    return p1 + second


def inclusion_p(pos, w, k):
    """Bonferroni p-value of per-entry inclusion counts (n rows, k draws each) against inclusion_probs: every entry's
    count is Binomial(n, pi_i), tested two-sided by its normal z-score."""
    from scipy import stats
    pos = np.asarray(pos)
    n = pos.shape[0]
    pi = inclusion_probs(w, k)
    counts = np.bincount(pos.ravel(), minlength=len(w)).astype(np.float64)
    live = pi > 0
    if counts[~live].any():
        return 0.0
    z = np.abs(counts[live] - n * pi[live]) / np.sqrt(n * pi[live] * (1 - pi[live]) + 1e-300)
    return float(min(1.0, 2 * stats.norm.sf(z.max()) * live.sum()))


def replacement_p(draws, w):
    """Chi-square p-value of every with-replacement draw (int [n, k]) against P = w / W, per draw column and over the
    pair (draw 0, draw 1) for independence; the smallest of the p-values."""
    draws = np.asarray(draws)
    w = np.asarray(w, np.float64)
    p = w / w.sum()
    d = len(w)
    ps = [_chi2_counts(np.bincount(draws[:, j], minlength=d), p * len(draws)) for j in range(draws.shape[1])]
    if draws.shape[1] > 1:
        pair = np.bincount(draws[:, 0] * d + draws[:, 1], minlength=d * d)
        ps.append(_chi2_counts(pair, np.outer(p, p).ravel() * len(draws)))
    return min(ps)


def independence_p(a, b, d):
    """Chi-square p-value of the joint counts of first entries a, b (ints in [0, d)) of two independent samples against
    the product of their margins."""
    a, b = np.asarray(a), np.asarray(b)
    joint = np.bincount(a * d + b, minlength=d * d).reshape(d, d).astype(np.float64)
    expected = np.outer(joint.sum(1), joint.sum(0)) / len(a)
    keep = expected.ravel() > 0
    dof = (np.count_nonzero(joint.sum(1)) - 1) * (np.count_nonzero(joint.sum(0)) - 1)
    return _chi2_counts(joint.ravel()[keep], expected.ravel()[keep], dof=max(dof, 1))
