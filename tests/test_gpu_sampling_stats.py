# coding=utf-8
"""The samplers' draws against their exact distributions (tests/sampling_stats.py), on the device.

The bit-exact tests elsewhere compare each kernel with a restatement of the same algorithm; these compare the draws
with what they are supposed to mean, so a defect that a kernel and its restatement share still fails.  Draws are keyed by
(key, row id), so the rows of one degree in one call are independent samples: every graph here is a set of rows that
share one list of leaf neighbours per degree, and a sampled leaf's id minus the list's first id is its CSR position.
Repeated rows of one K13 list draw the same positions by design, and no list here repeats a row.

Every check names, in its docstring, the host test in tests/test_sampling_stats_host.py that shows its statistic
rejects the corresponding defect at the same sample size."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from tf_geometric_b200.utils import sampling
import link_oracle as lo
import sampling_stats as st

pytestmark = pytest.mark.gpu

RNS = tfg.utils.RandomNeighborSampler
HNS = tfg.utils.HostNeighborSampler
NODE_NS = [7, 1000, 111059956, 244160499, 1600000000, (1 << 31) - 1]


def fan_graph(groups):
    """groups [(rows, d)] -> (edge_index int32 [2, E], [(first row, first leaf)]): every row of group g has the d
    leaves of g as neighbours, in ascending order; leaves come after all rows and have no neighbours."""
    n_rows = sum(r for r, _ in groups)
    src, dst, where = [], [], []
    r0, leaf = 0, n_rows
    for rows, d in groups:
        src.append(np.repeat(np.arange(r0, r0 + rows), d))
        dst.append(np.tile(np.arange(leaf, leaf + d), rows))
        where.append((r0, leaf))
        r0, leaf = r0 + rows, leaf + d
    return np.stack([np.concatenate(src), np.concatenate(dst)]).astype(np.int32), where


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _host(t):
    return t.cpu().numpy()


def _host_sampler(ei):
    """HostNeighborSampler whose build cuts the CSR into at least three ranges (int64 positions over the host link)."""
    E, N = ei.shape[1], int(ei.max()) + 1
    eb = sampling.HOST_CSR_EDGE_BYTES_UNWEIGHTED
    budget = eb * (E // 4 + 1) + sampling.HOST_CSR_ROW_BYTES * N
    rp = np.concatenate([[0], np.cumsum(np.bincount(ei[0], minlength=N))])
    assert len(sampling._row_ranges(rp, budget, eb)) >= 3
    return HNS(ei, device_bytes=budget + 8 * (N + 1) + 8 * (E // 1024 + 1) + sampling.HOST_CSR_FIXED_BYTES)


class Paths(object):
    """Fan-out positions [n, k] of the rows [r0, r0 + n) of a fan graph by each sampling path."""

    def __init__(self, ei):
        self.ei = ei
        self.rns = RNS(_dev(ei))
        self.csr, _, self.rowptr, _ = self.rns._neighborhood_structure()
        self.hns = None

    def host_sampler(self):
        if self.hns is None:
            self.hns = _host_sampler(self.ei)
        return self.hns

    def positions(self, path, r0, n, leaf, k=None, ratio=None, padding=False, seed=1):
        """(positions int64 [n, num] or a list of rows when the counts differ) of rows r0 .. r0 + n - 1."""
        if path == "neighbor_sample":
            row, pos, orp = ops.neighbor_sample(self.csr, k=k, ratio=ratio, padding=padding, seed=seed)
            orp = _host(orp)
            pos = _host(pos)[orp[r0]:orp[r0 + n]].astype(np.int64)
            start = np.repeat(_host(self.rowptr)[r0:r0 + n], np.diff(orp[r0:r0 + n + 1]))
            return self._rows(pos - start, np.diff(orp[r0:r0 + n + 1]))
        if path == "rows":
            rows = torch.arange(r0, r0 + n, dtype=torch.int32, device="cuda")
            _, pos, orp = ops.neighbor_sample_rows(self.rowptr, rows, k=k, ratio=ratio, padding=padding, seed=seed)
            cnt = np.diff(_host(orp))
            start = np.repeat(_host(self.rowptr)[r0:r0 + n], cnt)
            return self._rows(_host(pos).astype(np.int64) - start, cnt)
        sampler = self.rns if path == "blocks" else self.host_sampler()
        sb = sampler.sample_blocks(np.arange(r0, r0 + n), [k], padding=padding, seed=seed)
        return block_positions(sb.blocks[-1], sb.node_index, n, leaf)

    @staticmethod
    def _rows(flat, cnt):
        if len(cnt) and (cnt == cnt[0]).all():
            return flat.reshape(len(cnt), int(cnt[0]))
        return np.split(flat, np.cumsum(cnt)[:-1])


def block_positions(block, node_index, n, leaf):
    """Positions [n, k] of the first n output rows of a block (every row with k edges), from the edges' global ids."""
    dst = _host(block.edge_index[0])
    gcol = _host(block.global_col).astype(np.int64)
    sel = dst < n
    dst, gcol = dst[sel], gcol[sel]
    cnt = np.bincount(dst, minlength=n)
    assert (cnt == cnt[0]).all() and (np.diff(dst) >= 0).all()
    return (gcol - leaf).reshape(n, int(cnt[0]))


# ---- fan-out without replacement, thread tier ------------------------------------------------------------------

THREAD_GROUPS = [(st.ROWS, 5), (st.ROWS, 7), (st.ROWS, 10)]


@pytest.fixture(scope="module")
def thread_paths():
    ei, where = fan_graph(THREAD_GROUPS)
    return Paths(ei), where


@pytest.mark.parametrize("path", ["neighbor_sample", "rows", "blocks", "host_blocks"])
def test_thread_tier_subsets(thread_paths, path):
    """Per-position inclusion and whole-subset uniformity of k = 2 and 3 over rows of degree 5, 7 and 10, and two
    rows of one call independent.  Power: test_inclusion_and_subsets_accept_exact_and_reject_algorithm_r_off_by_one,
    test_independence_accepts_independent_rows_and_rejects_copies."""
    paths, where = thread_paths
    for k, seed in ((2, 11), (3, 12)):
        for (rows, d), (r0, leaf) in zip(THREAD_GROUPS, where):
            pos = paths.positions(path, r0, rows, leaf, k=k, seed=seed)
            what = "{} k={} d={}".format(path, k, d)
            assert pos.shape == (rows, k), (what, pos.shape)
            st.check_subsets(pos, d)
            st.require(st.inclusion_p(pos, d), what + " inclusion")
            st.require(st.subset_p(pos, d), what + " subsets")
            code = st.subset_codes(pos)
            st.require(st.independence_p(code[0::2], code[1::2]), what + " two rows")


@pytest.mark.parametrize("path", ["neighbor_sample", "rows", "blocks", "host_blocks"])
def test_deterministic_rules_and_padding(thread_paths, path):
    """k >= d without padding and the head rule keep the first entries in order; padding draws k independent uniform
    positions.  Power of the padding check: test_replacement_accepts_iid_and_rejects_a_missing_last_neighbour."""
    paths, where = thread_paths
    (rows, d), (r0, leaf) = THREAD_GROUPS[0], where[0]
    every = paths.positions(path, r0, rows, leaf, k=d + 3, seed=3)
    assert np.array_equal(every, np.tile(np.arange(d), (rows, 1)))
    head = paths.positions(path, r0, rows, leaf, k=3, padding="head", seed=4)
    assert np.array_equal(head, np.tile(np.arange(3), (rows, 1)))
    draws = paths.positions(path, r0, rows, leaf, k=8, padding=True, seed=5)
    assert draws.shape == (rows, 8)
    p_pos, p_pair = st.replacement_p(draws, d)
    st.require(p_pos, path + " padding positions")
    st.require(p_pair, path + " padding ordered pairs")


@pytest.mark.parametrize("path", ["neighbor_sample", "rows"])
def test_ratio_mode(thread_paths, path):
    """ratio 0.25 keeps ceil(0.25 d) = 3 of 10 without replacement.  Power:
    test_inclusion_and_subsets_accept_exact_and_reject_algorithm_r_off_by_one[10-3]."""
    paths, where = thread_paths
    (rows, d), (r0, leaf) = THREAD_GROUPS[2], where[2]
    pos = paths.positions(path, r0, rows, leaf, ratio=0.25, seed=6)
    assert pos.shape == (rows, 3)
    st.check_subsets(pos, d)
    st.require(st.inclusion_p(pos, d), path + " ratio inclusion")
    st.require(st.subset_p(pos, d), path + " ratio subsets")
    head = paths.positions(path, r0, rows, leaf, ratio=0.25, padding="head", seed=6)
    assert np.array_equal(head, np.tile(np.arange(3), (rows, 1)))


# ---- K13 across its thread-row limit, and the CTA path ----------------------------------------------------------

WIDE = [127, 128, 129, 1000]


@pytest.fixture(scope="module")
def wide_paths():
    ei, where = fan_graph([(st.ROWS_WIDE, d) for d in WIDE])
    return Paths(ei), where


@pytest.mark.parametrize("path", ["rows", "blocks"])
def test_rows_across_thread_row_limit(wide_paths, path):
    """K13 at degrees 127, 128 (one thread per row) and 129, 1000 (the CTA's atomicMax reservoir), k = d // 2:
    per-position inclusion and the pairs (0, 1), (0, d - 1), (d - 2, d - 1).  Power:
    test_wide_rows_inclusion_and_pairs."""
    paths, where = wide_paths
    for d, (r0, leaf) in zip(WIDE, where):
        pos = paths.positions(path, r0, st.ROWS_WIDE, leaf, k=d // 2, seed=20 + d)
        what = "{} d={}".format(path, d)
        st.check_subsets(pos, d)
        st.require(st.inclusion_p(pos, d), what + " inclusion")
        for a, b in ((0, 1), (0, d - 1), (d - 2, d - 1)):
            st.require(st.pair_p(pos, d, a, b), "{} pair ({}, {})".format(what, a, b))


def test_hub_rows():
    """HUB_ROWS rows of 60 000 edges, HUB_KEYS keys, k = 30 000 (the CTA path): position buckets and the pairs
    (0, 1), (0, d - 1), (d - 2, d - 1).  Power: test_hub_tally_accepts_exact_and_rejects_edge_defects."""
    d = st.HUB_DEGREE
    ei, ((r0, leaf),) = fan_graph([(st.HUB_ROWS, d)])
    paths = Paths(ei)
    tally = st.HubTally(d)
    for key in range(st.HUB_KEYS):
        tally.add(paths.positions("rows", r0, st.HUB_ROWS, leaf, k=st.HUB_K, seed=1000 + key))
    for name, p in tally.ps().items():
        st.require(p, "hub {}".format(name))


# ---- exclusion --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("exclude", ["self", "reverse"])
def test_link_blocks_exclusion(exclude):
    """sample_link_blocks: rows of degree 130 with 1, 2 or 3 target edges, so the kept degree is 129 (CTA), 128 or 127
    (thread); k = 60.  Excluded entries never appear; the kept ones follow per-position inclusion and pair inclusion
    over the kept degree.  Power: test_wide_rows_inclusion_and_pairs."""
    d, k, per = 130, 60, st.ROWS_WIDE
    ei, ((r0, leaf),) = fan_graph([(3 * per, d)])
    cut = {1: [129], 2: [0, 129], 3: [0, 64, 129]}
    src, dst = [], []
    for g, x in enumerate((1, 2, 3)):
        rows = np.arange(r0 + g * per, r0 + (g + 1) * per)
        src.append(np.repeat(rows, x))
        dst.append(np.tile(leaf + np.array(cut[x]), per))
    pairs = np.stack([np.concatenate(src), np.concatenate(dst)]).astype(np.int32)
    lb = RNS(_dev(ei)).sample_link_blocks(pairs, [k], num_negatives=0, exclude=exclude, seed=77)
    block, nodes = lb.blocks[-1], _host(lb.node_index)
    dst_t = _host(block.edge_index[0])
    gid = nodes[dst_t]
    gcol = _host(block.global_col).astype(np.int64) - leaf
    sel = gid < r0 + 3 * per
    order = np.argsort(gid[sel], kind="stable")
    rows_of, pos = gid[sel][order], gcol[sel][order]
    assert np.array_equal(np.unique(rows_of), np.arange(r0, r0 + 3 * per))
    pos = pos.reshape(3 * per, k)
    for g, x in enumerate((1, 2, 3)):
        p = pos[g * per:(g + 1) * per]
        assert not np.isin(p, cut[x]).any(), "an excluded entry was sampled"
        keep = np.setdiff1d(np.arange(d), cut[x])
        virt = np.searchsorted(keep, p)
        dk = d - x
        what = "exclude={} kept degree {}".format(exclude, dk)
        st.check_subsets(virt, dk)
        st.require(st.inclusion_p(virt, dk), what + " inclusion")
        for a, b in ((0, 1), (0, dk - 1), (dk - 2, dk - 1)):
            st.require(st.pair_p(virt, dk, a, b), "{} pair ({}, {})".format(what, a, b))


# ---- independence -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("sampler", ["device", "host"])
def test_hop_and_call_independence(thread_paths, sampler):
    """A seed row's 2-subsets of 5 at hop 0 and hop 1 of one sample_blocks batch (the hop keys differ), and in two
    consecutive calls without a seed.  Power: test_independence_accepts_independent_rows_and_rejects_copies."""
    paths, where = thread_paths
    (rows, d), (r0, leaf) = THREAD_GROUPS[0], where[0]
    s = paths.rns if sampler == "device" else paths.host_sampler()
    seeds = np.arange(r0, r0 + rows)
    sb = s.sample_blocks(seeds, [2, 2], seed=31)
    hop0 = block_positions(sb.blocks[-1], sb.node_index, rows, leaf)
    hop1 = block_positions(sb.blocks[0], sb.node_index, rows, leaf)
    assert np.array_equal(_host(sb.node_index[:rows]), seeds)
    st.require(st.independence_p(st.subset_codes(hop0), st.subset_codes(hop1)), sampler + " hop 0 / hop 1")
    a, b = [block_positions(c.blocks[-1], c.node_index, rows, leaf)
            for c in (s.sample_blocks(seeds, [2]), s.sample_blocks(seeds, [2]))]
    st.require(st.independence_p(st.subset_codes(a), st.subset_codes(b)), sampler + " consecutive seed=None calls")


def test_negative_sampling_batches_independent():
    """Sample s of batch 0 against sample s of batch 1 of negative_sampling(batch_size=2) over 7 nodes.  Power:
    test_negative_batches_independence."""
    n = st.NODE_DRAWS // 8
    b0, b1 = tfg.utils.negative_sampling(n, 7, batch_size=2, seed=41)
    b0, b1 = _host(b0), _host(b1)
    for r in (0, 1):
        st.require(st.independence_p(b0[r], b1[r]), "negative_sampling batches, row {}".format(r))
    st.require(st.independence_p(b0[0], b0[1]), "negative_sampling pair ends")


# ---- estimators -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("sampler", ["device", "host"])
@pytest.mark.parametrize("d,k", [(10, 5), (300, 150)])
def test_block_mean_aggregation(sampler, d, k):
    """Mean aggregation of a block (the spmm mean-GraphSAGE runs) over EST_SAMPLES rows, 16 keys of 128 seeds, at a
    thread-tier row (d 10) and a CTA-tier row (d 300): the mean within 4 standard errors of the float64 mean over all
    neighbours, the variance consistent with sigma^2 / k (d - k) / (d - 1) and not with sigma^2 / k.  Power:
    test_mean_variance_separates_without_from_with_replacement."""
    per_key = 128
    ei, ((r0, leaf),) = fan_graph([(per_key, d)])
    N = per_key + d
    v = np.random.default_rng(50 + d).standard_normal((d, 4)).astype(np.float32)
    x = np.zeros((N, 4), np.float32)
    x[leaf:leaf + d] = v
    xd = _dev(x)
    s = RNS(_dev(ei)) if sampler == "device" else _host_sampler(ei)
    means = []
    for key in range(st.EST_SAMPLES // per_key):
        sb = s.sample_blocks(np.arange(r0, r0 + per_key), [k], seed=500 + key)
        blk = sb.blocks[-1]
        x_src = xd[sb.node_index[:blk.num_src].long()]
        agg = ops.spmm(blk.csr, blk.edge_weight, x_src, reduce="mean")
        means.append(_host(agg[:per_key]))
    means = np.concatenate(means).astype(np.float64)
    for c in range(4):
        st.require_mean(means[:, c], v[:, c].astype(np.float64), k, "{} d={} column {}".format(sampler, d, c))


# ---- Bernoulli operators ----------------------------------------------------------------------------------------

RATES = [0.0, 0.1, 0.5, 0.9, 1.0]


def _require_keep(flags, p_keep, what):
    flags = np.asarray(flags, bool)
    if p_keep in (0.0, 1.0):
        assert flags.all() if p_keep == 1.0 else not flags.any(), what
        return
    st.require(st.keep_rate_p(flags.sum(), flags.size, p_keep), what + " keep rate")
    st.require(st.adjacent_p(flags), what + " adjacent elements")


@pytest.mark.parametrize("rate", RATES)
def test_dropout_keep_rate(rate):
    """ops.dropout and GCN's edge dropout (SparseMatrix.dropout): keep rate 1 - ceil(rate 2^24) / 2^24, everything
    kept at 0, rate 1 refused, and adjacent elements independent across Philox lanes and blocks.  Power:
    test_keep_rate_and_adjacency_have_power."""
    n = st.BERNOULLI_N
    if rate == 1.0:
        with pytest.raises(_ffi.TfgkError, match="outside"):
            ops.dropout(torch.ones(n, device="cuda"), rate, 61)
        return
    out = ops.dropout(torch.ones(n, device="cuda"), rate, 61)
    _require_keep(_host(out) != 0, st.dropout_keep(rate), "dropout {}".format(rate))
    idx = torch.stack([torch.arange(n, dtype=torch.int32), torch.arange(n, dtype=torch.int32)]).cuda()
    a = tfg.SparseMatrix(idx, torch.ones(n, device="cuda"), [n, n]).dropout(rate, training=True, seed=62)
    _require_keep(_host(a.value) != 0, st.dropout_keep(rate), "edge dropout {}".format(rate))


@pytest.mark.parametrize("force_undirected", [False, True])
@pytest.mark.parametrize("rate", RATES)
def test_drop_edge_keep_rate(rate, force_undirected):
    """drop_edge over BERNOULLI_N upper edges (edge e = (e, n + e)): keep rate and adjacent edges.  Power:
    test_keep_rate_and_adjacency_have_power."""
    n = st.BERNOULLI_N
    e = np.arange(n, dtype=np.int32)
    ei = _dev(np.stack([e, e + n]))
    kept = _host(tfg.nn.drop_edge([ei], rate=rate, force_undirected=force_undirected, training=True, seed=63)[0])
    if force_undirected:
        h = kept.shape[1] // 2
        assert np.array_equal(kept[:, h:], kept[::-1, :h])
        kept = kept[:, :h]
    flags = np.zeros(n, bool)
    flags[kept[0]] = True
    assert len(np.unique(kept[0])) == kept.shape[1]
    _require_keep(flags, st.dropout_keep(rate), "drop_edge {} undirected={}".format(rate, force_undirected))


@pytest.mark.parametrize("prob", [0.1, 0.5, 0.9, 1.0])
def test_uniform_neighbor_sampler_keep_rate(prob):
    """UniformNeighborSampler keeps an edge with probability (floor(prob 2^24) + 1) / 2^24 (u <= prob).  Power:
    test_keep_rate_and_adjacency_have_power."""
    n = st.BERNOULLI_N
    e = np.arange(n, dtype=np.int32)
    kept, _ = tfg.utils.UniformNeighborSampler(_dev(np.stack([e, e + n]))).sample(prob, seed=64)
    flags = np.zeros(n, bool)
    flags[_host(kept)[0]] = True
    _require_keep(flags, st.bernoulli_keep(prob), "UniformNeighborSampler {}".format(prob))


# ---- node ids ---------------------------------------------------------------------------------------------------

def _node_ids(entry, N):
    n = st.NODE_DRAWS
    if entry == "link_tail_negatives":
        q = 8
        src = torch.zeros(n // q, dtype=torch.int32, device="cuda")
        row = torch.empty(n, dtype=torch.int32, device="cuda")
        col = torch.empty(n, dtype=torch.int32, device="cuda")
        ops.link_tail_negatives(src, q, N, 71, row, col)
        return _host(col)
    if entry == "negative_sampling":
        return _host(tfg.utils.negative_sampling(n // 2, N, seed=72)).ravel()
    start = torch.zeros(n, dtype=torch.int32, device="cuda")
    return _host(tfg.utils.negative_sampling_with_start_node(start, N, None, seed=73)[1])


@pytest.mark.parametrize("N", NODE_NS)
@pytest.mark.parametrize("entry", ["link_tail_negatives", "negative_sampling", "negative_sampling_with_start_node"])
def test_node_ids_uniform(entry, N):
    """NODE_DRAWS node ids uniform on [0, N): the multiply-shift heavy ids' share, 1024 range buckets and v mod 1024.
    N is only a number here: nothing N-sized is allocated.  Power: test_heavy_share_rejects_32_bit_multiply_shift,
    test_range_and_low_bit_statistics_have_power (acceptance: test_node_ids_accept_uniform_draws)."""
    v = _node_ids(entry, N).astype(np.int64)
    share, want, p = st.heavy_p(np.clip(v, 0, N - 1), N)
    print("{} N={}: heavy-id share {:.5f}, {:.5f} under uniform draws (p = {:.3g})".format(entry, N, share, want, p))
    st.require_node_ids(v, N, entry)


# ---- negative_sampling without replacement ----------------------------------------------------------------------

@pytest.mark.parametrize("S", [40, 20])
def test_negative_sampling_without_replacement(S):
    """NEG_BATCHES batches of S distinct pairs over 12 nodes with the edge (0, 1): C = 65 candidates, the shuffle path
    (2 S > C) and the duplicate-redraw path.  Per-candidate inclusion S / C and pair inclusion.  Power:
    test_negative_inclusion_without_replacement."""
    N = 12
    ei = np.array([[0], [1]], np.int32)
    cand = lo.negative_candidates(ei, N)
    C = cand.shape[1]
    index = {(int(a), int(b)): i for i, (a, b) in enumerate(cand.T)}
    batches = tfg.utils.negative_sampling(S, N, edge_index=_dev(ei), replace=False, batch_size=st.NEG_BATCHES, seed=81)
    k = np.array([[index[(int(a), int(b))] for a, b in _host(bt).T] for bt in batches])
    st.check_subsets(k, C)
    st.require(st.inclusion_p(k, C), "S={} inclusion".format(S))
    for a, b in ((0, 1), (0, C - 1)):
        st.require(st.pair_p(k, C, a, b), "S={} pair ({}, {})".format(S, a, b))
