# coding=utf-8
"""CPU checks of layer-neighbour (LABOR-0) sampling: the entry declarations and argument checks, the refusals (before
any device work, so the relabelling map stays clean), Block.labor and the work-plan rule of LABOR blocks, the unchanged
call of labor=False, and the power of tests/labor_stats.py: each statistic accepts exact samples of tests/labor_ref.py
and rejects a planted defect at the sample sizes the GPU tests use.

The rule (include/tfgk.h, "LABOR block sampler"): u_c = lane 0 of Philox counter (c, 0, 4, 0) under the hop key; a row
of d > k candidates keeps (row, c) iff u_c * d < k 2^32, a row of d <= k keeps every candidate."""
import ctypes

import numpy as np
import pytest
import torch

import labor_ref as lr
import labor_stats as ls
from weighted_ref import hop_seed

SEED = 0x1AB0
ENTRIES = {"tfgk_block_sample_count_labor": 15, "tfgk_block_sample_count_labor_excl": 18,
           "tfgk_block_sample_count_labor_mapped_excl": 18, "tfgk_block_sample_fill_labor": 23,
           "tfgk_block_sample_fill_labor_excl": 26, "tfgk_block_sample_fill_labor_mapped": 23,
           "tfgk_block_sample_fill_labor_mapped_excl": 26}
# the GPU tests' statistics graph (tests/test_gpu_labor_sampling.py)
COPIES, KEYS, DA, DB = 4000, 8, 6, 10


# ---- declarations, argument checks, refusals --------------------------------------------------------------------------

def test_entries_are_declared_and_refuse_capture():
    from tf_geometric_b200 import _ffi, ops
    for name, n in ENTRIES.items():
        assert len(_ffi.SIGNATURES[name]) == n, name
        assert name in _ffi.NOT_CAPTURABLE and "host-side key" in _ffi.NOT_CAPTURABLE[name][1], name
    assert ops.RNG_STREAM_LABOR == lr.RNG_STREAM_LABOR == 4
    assert len({ops.RNG_STREAM_DROPOUT, ops.RNG_STREAM_SAMPLER, ops.RNG_STREAM_LINK, ops.RNG_STREAM_WEIGHTED,
                ops.RNG_STREAM_LABOR}) == 5


def test_entries_refuse_fan_out_none_without_a_device():
    from tf_geometric_b200 import _ffi
    fake = ctypes.c_void_p(256)                       # never dereferenced: the checks come first
    need = ctypes.c_size_t()
    _ffi.call("tfgk_block_sample_workspace_bytes", 8, 0, ctypes.byref(need))
    ws = ctypes.create_string_buffer(need.value)
    cases = [
        ("tfgk_block_sample_count_labor", (fake, 4, None, fake, fake, 0, 2, 8, -1, 1, 4, fake, ws, need.value, None),
         "null columns"),
        ("tfgk_block_sample_count_labor", (fake, 4, fake, fake, fake, 0, 2, 8, -1, 1, 4, fake, ws, need.value, None),
         "LABOR"),
        ("tfgk_block_sample_count_labor_excl", (fake, 4, fake, fake, fake, 0, 2, 8, 3, 1, 4, None, None, 0, fake, ws,
                                                need.value, None), "exclusion"),
        ("tfgk_block_sample_fill_labor", (fake, 4, fake, fake, 4, fake, fake, fake, 0, 2, 8, 16, -1, 1, 4, fake, fake,
                                          fake, fake, fake, ws, need.value, None), "LABOR"),
        ("tfgk_block_sample_fill_labor_mapped_excl", (fake, 4, fake, fake, 4, fake, fake, fake, 0, 2, 8, 16, 3, 1, 4,
                                                      fake, fake, fake, fake, fake, None, None, 0, ws, need.value,
                                                      None), "exclusion"),
    ]
    for name, args, words in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(name, *args)
        assert err.value.code == _ffi.ERR_INVALID_ARGUMENT, name
        assert words in str(err.value), (name, str(err.value))


class _NoDevice(object):
    """A stand-in sampler whose structures must not be touched: the refusals come first."""
    _has_weights = True
    _closed = False

    def _check_open(self):
        pass

    def __getattr__(self, name):
        raise AssertionError("{} touched before the refusal".format(name))


@pytest.mark.parametrize("kw,err,words", [(dict(labor=True, padding=True), ValueError, "no padding"),
                                          (dict(labor=True, padding="head"), ValueError, "no padding"),
                                          (dict(layer_dependency=True), ValueError, "needs labor=True"),
                                          (dict(labor=True, weighted=True), NotImplementedError, "weighted LABOR")])
def test_refusals_come_before_any_device_work(kw, err, words):
    from tf_geometric_b200.utils import sampling
    for cls in (sampling.RandomNeighborSampler, sampling.HostNeighborSampler):
        with pytest.raises(err, match=words):
            cls.sample_blocks(_NoDevice(), np.arange(4, dtype=np.int32), [3], seed=1, **kw)
        with pytest.raises(err, match=words):
            cls.sample_link_blocks(_NoDevice(), np.array([[0], [1]], np.int32), [3], seed=1, **kw)


def test_ops_refuse_labor_with_padding_or_weights():
    from tf_geometric_b200 import ops
    with pytest.raises(ValueError, match="no padding"):
        ops._check_block_fanouts([3], True, None, True)
    with pytest.raises(NotImplementedError):
        ops._check_block_fanouts([3], False, torch.zeros(4, dtype=torch.int32), True)
    assert ops._check_block_fanouts([3, None], False, None, True) == 0


def test_block_labor_slot_and_work_plans(monkeypatch):
    from tf_geometric_b200 import ops
    from tf_geometric_b200.utils import sampling
    e = torch.zeros((2, 0), dtype=torch.int32)
    assert sampling.Block(1, 1, e, torch.zeros(0), e[0], None, fanout=3).labor is False
    assert sampling.Block(1, 1, e, torch.zeros(0), e[0], None, fanout=3, labor=True).labor is True
    planned = []
    monkeypatch.setattr(ops, "build_plan", lambda csr: planned.append(csr.n_rows))
    rp = torch.tensor([0, 2, 3], dtype=torch.int64)
    hop = (rp, torch.tensor([0, 0, 1], dtype=torch.int32), torch.tensor([2, 3, 4], dtype=torch.int32),
           torch.tensor([7, 8, 9], dtype=torch.int32), torch.ones(3))
    node_index = torch.arange(5, dtype=torch.int32)
    blocks = sampling._blocks_of("cpu", node_index, [2, 5], [hop], [5], None)
    assert planned == [] and not blocks[0].labor                 # k = 5 bounds a uniform block's rows
    blocks = sampling._blocks_of("cpu", node_index, [2, 5], [hop], [5], None, labor=True)
    assert planned == [2] and blocks[0].labor and blocks[0].fanout == 5      # not a LABOR block's
    blocks = sampling._blocks_of("cpu", node_index, [2, 5], [hop], [None], None, labor=True)
    assert planned == [2, 2] and not blocks[0].labor                         # fan-out None takes every neighbour


def test_hop_keys_with_layer_dependency():
    from tf_geometric_b200.utils import sampling
    fan, keys = sampling._hop_keys([15, 10, 5], SEED)
    assert fan == [5, 10, 15] and keys == [hop_seed(SEED, h) for h in range(3)] == lr.hop_keys(SEED, 3)
    assert sampling._hop_keys([15, 10, 5], SEED, True)[1] == [hop_seed(SEED, 0)] * 3 == lr.hop_keys(SEED, 3, True)


def test_labor_false_calls_the_block_sampler_as_before(monkeypatch):
    import block_fake_backend as fake_blocks
    from conftest import random_graph
    fake_blocks.install(monkeypatch)
    import tf_geometric_b200 as tfg
    monkeypatch.setattr(tfg.ops, "build_plan", lambda csr: None)
    seen = []
    real = tfg.ops.block_sample

    def spy(*args, **kw):
        seen.append(sorted(kw))
        return real(*args, **kw)
    monkeypatch.setattr(tfg.ops, "block_sample", spy)
    ei = random_graph(200, 1200, seed=3)
    s = tfg.utils.RandomNeighborSampler(ei)
    a = s.sample_blocks(np.arange(8, dtype=np.int32), [4, 3], seed=5)
    b = s.sample_blocks(np.arange(8, dtype=np.int32), [4, 3], seed=5, labor=False, layer_dependency=False)
    assert seen == [["padding"], ["padding"]]
    assert torch.equal(a.node_index, b.node_index) and not any(blk.labor for blk in b.blocks)


# ---- the rule ---------------------------------------------------------------------------------------------------------

def test_rule_edges():
    u = lr.variates(np.arange(10), SEED)
    assert lr.keep_mask(u, 10, 0).sum() == 0                     # k = 0
    assert lr.keep_mask(u[:5], 5, 5).all() and lr.keep_mask(u[:1], 1, 5).all()     # d <= k: every candidate
    assert lr.pi(5, 6) == float(-(-(5 << 32) // 6)) / 2 ** 32 and lr.pi(5, 5) == 1.0 and lr.pi(0, 3) == 0.0
    # the test is exact: u * d < k 2^32 at the boundary u = ceil(k 2^32 / d) - 1
    d, k = 7, 3
    edge = -(-(k << 32) // d)
    assert lr.keep_mask(np.array([edge - 1, edge], np.uint32), d, k).tolist() == [True, False]


def test_variates_depend_on_the_column_and_key_only():
    rowptr = np.array([0, 4, 8], np.int64)
    col = np.array([5, 6, 7, 8, 8, 7, 6, 5], np.int32)
    a = lr.row_positions(rowptr, col, 0, 2, SEED)
    b = lr.row_positions(rowptr, col, 1, 2, SEED)
    assert set(col[a].tolist()) == set(col[b].tolist())          # same columns, same d: the same kept set
    assert lr.row_positions(rowptr, col, 0, None, SEED, excluded=[1]).tolist() == [0, 2, 3]


# ---- statistical power ------------------------------------------------------------------------------------------------
# Sample generators over the GPU tests' copies: copy i's row A holds t_i and DA - 1 fillers, row B holds DB - 1 fillers
# and t_i, every id distinct; column ids below are those of tests/test_gpu_labor_sampling.py's layout.

def _cols():
    t = np.arange(COPIES)
    fa = COPIES + np.arange(COPIES * (DA - 1)).reshape(COPIES, DA - 1)
    fb = fa.max() + 1 + np.arange(COPIES * (DB - 1)).reshape(COPIES, DB - 1)
    return np.concatenate([t[:, None], fa], 1), np.concatenate([fb, t[:, None]], 1)


def _keep(cols, key, d, k=2, row_salt=None, positions=False, threshold_d=None):
    """kept bool [COPIES, d] of one hop under `key`; planted defects: row_salt (variates keyed by (row, t)), positions
    (keyed by CSR position), threshold_d (the d in the test)"""
    ids = cols
    if positions:
        ids = np.broadcast_to(np.arange(cols.shape[1]), cols.shape) + (0 if row_salt is None else row_salt)
    elif row_salt is not None:
        ids = cols * 7919 + row_salt
    u = lr.variates(ids, key)
    dd = d if threshold_d is None else threshold_d
    return u.astype(np.uint64) * np.uint64(dd) < np.uint64(k) << np.uint64(32)


def test_inclusion_and_subsets_accept_exact_and_reject_defects():
    ca, _ = _cols()
    exact = np.concatenate([_keep(ca, hop_seed(SEED, s), DA) for s in range(KEYS)])
    ls.require(ls.inclusion_p(exact, lr.pi(2, DA)), "exact inclusion")
    ls.require(ls.subset_given_count_p(exact), "exact subsets")
    ls.require(ls.empty_p(exact, lr.pi(2, DA)), "exact empty rows")
    minus_one = np.concatenate([_keep(ca, hop_seed(SEED, s), DA, threshold_d=DA - 1) for s in range(KEYS)])
    assert ls.inclusion_p(minus_one, lr.pi(2, DA)) <= ls.P_FLOOR                 # the threshold k / (d - 1)
    with_excluded = np.concatenate([_keep(ca, hop_seed(SEED, s), DA, threshold_d=DA + 1) for s in range(KEYS)])
    assert ls.inclusion_p(with_excluded, lr.pi(2, DA)) <= ls.P_FLOOR             # one excluded entry counted in d
    # kept sets that are not uniform given their count: the first column's variate is used for the first two columns
    skew = exact.copy()
    skew[:, 1] = skew[:, 0]
    assert ls.subset_given_count_p(skew) <= ls.P_FLOOR


def test_coupling_within_a_hop_rejects_row_or_position_keyed_variates():
    ca, cb = _cols()
    n = COPIES * KEYS
    want = min(lr.pi(2, DA), lr.pi(2, DB))

    def both(**kw):
        out = 0
        for s in range(KEYS):
            key = hop_seed(SEED, s)
            a = _keep(ca, key, DA, **({} if not kw else dict(kw, row_salt=kw.get("row_salt", 0) + 1)))
            b = _keep(cb, key, DB, **({} if not kw else dict(kw, row_salt=kw.get("row_salt", 0) + 2)))
            out += int((a[:, 0] & b[:, -1]).sum())
        return out
    ls.require(ls.pair_p(both(), n, want), "exact")
    assert ls.pair_p(both(row_salt=0), n, want) <= ls.P_FLOOR                   # keyed by (row, t)
    assert ls.pair_p(both(positions=True, row_salt=1000), n, want) <= ls.P_FLOOR    # keyed by CSR position


@pytest.mark.parametrize("layer_dependency", [False, True])
def test_coupling_across_hops_rejects_layer_dependency_ignored_or_misapplied(layer_dependency):
    ca, cb = _cols()
    n = COPIES * KEYS
    pa, pb = lr.pi(2, DA), lr.pi(2, DB)
    want = min(pa, pb) if layer_dependency else pa * pb

    def both(ld):
        out = 0
        for s in range(KEYS):
            keys = lr.hop_keys(1000 + s, 2, ld)
            out += int((_keep(ca, keys[0], DA)[:, 0] & _keep(cb, keys[1], DB)[:, -1]).sum())
        return out
    ls.require(ls.pair_p(both(layer_dependency), n, want), "exact")
    assert ls.pair_p(both(not layer_dependency), n, want) <= ls.P_FLOOR


def test_independence_across_batches_rejects_a_reused_key():
    ca, _ = _cols()
    pa = lr.pi(2, DA)
    a = _keep(ca, hop_seed(1000, 0), DA)[:, 0]
    ls.require(ls.pair_p(int((a & _keep(ca, hop_seed(1001, 0), DA)[:, 0]).sum()), COPIES, pa * pa), "exact")
    assert ls.pair_p(int((a & _keep(ca, hop_seed(1000, 0), DA)[:, 0]).sum()), COPIES, pa * pa) <= ls.P_FLOOR


def test_distinct_sources_total_rejects_independent_rows():
    ca, cb = _cols()
    pa, pb = lr.pi(2, DA), lr.pi(2, DB)
    reach = [max(pa, pb)] + [pa] * (DA - 1) + [pb] * (DB - 1)
    mean, var = KEYS * COPIES * sum(reach), KEYS * COPIES * sum(p * (1 - p) for p in reach)

    def total(**kw):
        out = 0
        for s in range(KEYS):
            key = hop_seed(SEED, s)
            a = _keep(ca, key, DA)
            b = _keep(cb, key, DB, **kw)
            out += int(a[:, 1:].sum() + b[:, :-1].sum() + (a[:, 0] | b[:, -1]).sum())
        return out
    ls.require(ls.total_p(total(), mean, var), "exact")
    assert ls.total_p(total(row_salt=3), mean, var) <= ls.P_FLOOR               # rows drawing independently
