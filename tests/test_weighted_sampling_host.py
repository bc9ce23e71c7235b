# coding=utf-8
"""CPU checks of weighted neighbour sampling: the ln routine of the key against math.log, the numpy restatement of the
draw rule against its own contract, the statistics of tests/weighted_stats.py (each accepts exact samples and rejects a
planted defect at the sample sizes the GPU tests use), and the refusals that need no device.

The draw rule (include/tfgk.h, "weighted block sampler"): a row's candidates are its kept entries of weight > 0; entry v of
row r gets E = -ln(u) / w, u from 53 bits of Philox counter (v, r, 3, j); without replacement the min(k, d+) candidates of
smallest (E, v) with j = 0, in CSR order; with padding and k >= d+, draw j is the smallest (E, v) with counter j + 1."""
import math

import numpy as np
import pytest
import torch

import weighted_ref as wr
import weighted_stats as ws

SEED = 0x5EED


# ---- ln ------------------------------------------------------------------------------------------------------------

def test_log_within_two_ulp_over_the_full_range_of_u():
    rs = np.random.RandomState(1)
    u = np.concatenate([np.ldexp(rs.randint(1, 2 ** 53, 100000, dtype=np.int64).astype(np.float64), -53),
                        np.ldexp(np.arange(1, 4097, dtype=np.float64), -53),          # the smallest u
                        1.0 - np.ldexp(np.arange(0, 4096, dtype=np.float64), -53),    # u near and at 1
                        2.0 ** -np.arange(0, 54, dtype=np.float64),                    # every exponent
                        np.sqrt(0.5) * (1 + np.ldexp(np.arange(-64, 64, dtype=np.float64), -52))])  # the halving edge
    got = wr.log_rn(u)
    assert got[u == 1.0].tolist() == [0.0] * int((u == 1.0).sum())
    worst = max(wr.ulp_error(g, x) for g, x in zip(got.tolist(), u.tolist()) if x != 1.0)
    assert worst <= 2.0, worst


def test_keys_order_as_their_doubles():
    v = np.arange(64, dtype=np.uint32)
    w = np.linspace(0.01, 5.0, 64).astype(np.float32)
    k = wr.keys(SEED, wr.RNG_STREAM_WEIGHTED, v, 7, 0, w)
    e = -wr.log_rn(wr.uniform(SEED, wr.RNG_STREAM_WEIGHTED, v, 7, 0)) / w.astype(np.float64)
    assert np.array_equal(np.argsort(k, kind="stable"), np.argsort(e, kind="stable"))
    assert (k >> np.uint64(63)).max() == 0


# ---- the rule -------------------------------------------------------------------------------------------------------

def test_draw_row_rule():
    w = np.array([0.5, 0.0, 2.0, 1.0, 0.0, 3.0], np.float32)
    assert wr.draw_row(w, 3, 10, False, SEED).tolist() == [0, 2, 3, 5]          # k >= d+: every positive entry
    assert wr.draw_row(np.zeros(5, np.float32), 3, 4, True, SEED).size == 0      # d+ = 0
    assert wr.draw_row(w, 3, 0, True, SEED).size == 0
    two = wr.draw_row(w, 3, 2, False, SEED)
    assert two.size == 2 and np.all(np.diff(two) > 0) and np.all(w[two] > 0)
    rep = wr.draw_row(w, 3, 9, True, SEED)                                       # k >= d+: with replacement
    assert rep.size == 9 and np.all(w[rep] > 0)
    assert wr.draw_row(w, 3, 3, True, SEED).size == 3 and len(set(wr.draw_row(w, 3, 3, True, SEED))) == 3


def test_row_positions_skip_excluded_entries():
    rowptr = np.array([0, 6], np.int64)
    w = np.array([1, 2, 3, 4, 5, 6], np.float32)
    got = wr.row_positions(rowptr, w, 0, 2, False, SEED, excluded=[1, 4])
    assert set(got.tolist()) <= {0, 2, 3, 5}
    assert wr.row_positions(rowptr, w, 0, None, False, SEED, excluded=[1]).tolist() == [0, 2, 3, 4, 5]


# ---- statistical power ----------------------------------------------------------------------------------------------

W8 = np.array([0.2, 1.0, 3.0, 0.0, 0.7, 2.5, 1.3, 0.05], np.float32)


def _draws(w, k, n, seed, key_w=None, scale=False, j=0):
    """n rows' draws of successive sampling by the exact keys (rows r = 0..n-1), or with a planted defect: key_w the
    weights the keys use, scale: E = -ln(u) * w."""
    w = np.asarray(w, np.float32)
    kw = w if key_w is None else np.asarray(key_w, np.float32)
    cand = np.flatnonzero(w > 0)
    r = np.repeat(np.arange(n, dtype=np.uint32), cand.size).reshape(n, cand.size)
    v = np.broadcast_to(cand.astype(np.uint32), (n, cand.size))
    u = wr.uniform(seed, wr.RNG_STREAM_WEIGHTED, v, r, j)
    e = -wr.log_rn(u) * kw[cand] if scale else -wr.log_rn(u) / kw[cand].astype(np.float64)
    order = np.argsort(e, axis=1, kind="stable")
    return cand[order[:, :k]]


@pytest.mark.parametrize("k", [1, 2, 3])
def test_subset_statistic_accepts_exact_and_rejects_defects(k):
    n = ws.SUBSET_ROWS
    ws.require(ws.subset_p(_draws(W8, k, n, SEED), W8, k), "exact")
    assert ws.subset_p(_draws(W8, k, n, SEED, key_w=np.where(W8 > 0, 1.0, 0.0)), W8, k) <= ws.P_FLOOR   # weight ignored
    assert ws.subset_p(_draws(W8, k, n, SEED, scale=True), W8, k) <= ws.P_FLOOR                         # -ln(u) * w
    # each key taking its neighbour's weight.  (A counter whose virtual position is off by one under exclusion keeps
    # every key's own weight, so its subsets stay exactly distributed; only the bit-for-bit exclusion tests of
    # tests/test_gpu_weighted_sampling.py catch it.  Nor can any feasible sample see u taking 0 or 1 with a wrong mass
    # of order 2^-53: the bit-for-bit tests pin u.)
    shifted = np.roll(W8, 1)
    assert ws.subset_p(_draws(W8, k, n, SEED, key_w=np.where(W8 > 0, np.where(shifted > 0, shifted, 1.0), 0.0)),
                       W8, k) <= ws.P_FLOOR


@pytest.mark.parametrize("k", [1, 2])
def test_inclusion_statistic_accepts_exact_and_rejects_weight_ignored(k):
    w = np.random.RandomState(5).rand(300).astype(np.float32) + 0.01
    w[::7] *= 20
    n = ws.HUB_ROWS * ws.HUB_KEYS * 40
    ws.require(ws.inclusion_p(_draws(w, k, n, SEED), w, k), "exact")
    assert ws.inclusion_p(_draws(w, k, n, SEED, key_w=np.ones_like(w)), w, k) <= ws.P_FLOOR


def test_replacement_statistic_accepts_exact_and_rejects_reused_draw_index():
    w = np.array([0.3, 2.0, 0.0, 1.0, 0.7], np.float32)
    n = ws.REPLACE_ROWS
    exact = np.stack([_draws(w, 1, n, SEED, j=j + 1)[:, 0] for j in range(3)], axis=1)
    ws.require(ws.replacement_p(exact, w), "exact")
    reused = np.stack([_draws(w, 1, n, SEED, j=1)[:, 0]] * 3, axis=1)            # the counter ignores the draw index
    assert ws.replacement_p(reused, w) <= ws.P_FLOOR
    assert ws.replacement_p(np.stack([_draws(w, 1, n, SEED, j=j + 1, key_w=np.where(w > 0, 1.0, 0.0))[:, 0]
                                      for j in range(3)], axis=1), w) <= ws.P_FLOOR


def test_independence_statistic_rejects_a_key_that_ignores_the_hop():
    n = ws.SUBSET_ROWS
    a = _draws(W8, 1, n, wr.hop_seed(SEED, 0))[:, 0]
    ws.require(ws.independence_p(a, _draws(W8, 1, n, wr.hop_seed(SEED, 1))[:, 0], len(W8)), "exact")
    assert ws.independence_p(a, _draws(W8, 1, n, wr.hop_seed(SEED, 0))[:, 0], len(W8)) <= ws.P_FLOOR


# ---- refusals without a device ---------------------------------------------------------------------------------------

def test_head_rule_is_refused_before_any_device_work():
    from tf_geometric_b200.utils import sampling
    with pytest.raises(ValueError, match="head"):
        sampling._check_weighted_padding(True, "head")
    sampling._check_weighted_padding(False, "head")
    sampling._check_weighted_padding(True, True)


def test_weighted_block_refuses_gcn_norm():
    from tf_geometric_b200.utils.sampling import Block
    e = torch.zeros((2, 0), dtype=torch.int32)
    blk = Block(1, 1, e, torch.zeros(0), e[0], None, fanout=3, dst_ids=e[0], degrees=lambda: None, weighted=True)
    with pytest.raises(NotImplementedError, match="inclusion probabilities"):
        blk.with_gcn_norm()
    assert Block(1, 1, e, torch.zeros(0), e[0], None, fanout=3).weighted is False


def test_invalid_weights_are_refused():
    from tf_geometric_b200.utils import sampling
    with pytest.raises(ValueError, match="3 negative, NaN or infinite"):
        sampling._check_weights(3)
    sampling._check_weights(0)


def test_weighted_stream_id():
    from tf_geometric_b200 import ops
    assert ops.RNG_STREAM_WEIGHTED == wr.RNG_STREAM_WEIGHTED == 3
    assert len({ops.RNG_STREAM_DROPOUT, ops.RNG_STREAM_SAMPLER, ops.RNG_STREAM_LINK, ops.RNG_STREAM_WEIGHTED}) == 4
    assert math.isclose(ws.P_FLOOR, 1e-6)
