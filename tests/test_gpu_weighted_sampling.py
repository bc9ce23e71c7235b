# coding=utf-8
"""Weighted neighbour sampling on the device (sample_blocks / sample_neighborhood / sample_link_blocks with
weighted=True), on RandomNeighborSampler and on HostNeighborSampler with its host CSR cut into about ten ranges.

The rule (include/tfgk.h, "weighted block sampler"): a row's candidates are its kept entries of weight > 0, numbered by
virtual position v; E = -ln(u) / w with u from 53 bits of Philox counter (v, r, 3, j); without replacement the min(k, d+)
candidates of smallest (E, v), j = 0, in CSR order; with padding and k >= d+, draw j is the smallest (E, v) with counter
j + 1; fan-out None takes every kept entry.  Checked bit for bit against tests/weighted_ref.py, then against the exact
distributions of tests/weighted_stats.py."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from tf_geometric_b200.utils import sampling
import weighted_ref as wr
import weighted_stats as ws
from link_blocks_fake_backend import pair_begin_np

pytestmark = pytest.mark.gpu

HUB, HUB_DEGREE = 9, 60000
N = 3000


def host(t):
    return t.detach().cpu().numpy()


# rows whose entries are exactly the listed ones (the random rows avoid the ids 9 ... 15), and their d+
SPECIAL = {HUB: None, 11: None, 12: 1, 13: 6, 14: 0, 15: 1}


def _graph():
    rs = np.random.RandomState(41)
    rnd = rs.randint(0, N - 7, 400000)
    rnd = rnd + 7 * (rnd >= HUB)                             # no random entry in rows 9 ... 15
    row = np.concatenate([rnd, np.full(HUB_DEGREE, HUB), np.full(400, 11), np.full(140, 12), np.full(6, 13),
                          np.full(5, 14), np.full(20, 15)])
    col = rs.randint(0, N, row.size)
    col[row == 13] = 17                                      # row 13: one column six times (duplicate edges)
    w = (rs.rand(row.size) * 3).astype(np.float32)
    w[rs.rand(row.size) < 0.2] = 0.0                         # zero-weight entries everywhere
    w[row == 13] = 0.5 + np.arange(6, dtype=np.float32)      # d+ = 6: fewer than the fan-outs above 6
    w[row == 14] = 0.0                                       # d+ = 0
    for r, at in ((12, 70), (15, 3)):                        # d+ = 1 past the warp limit, and within it
        w[row == r] = 0.0
        w[np.flatnonzero(row == r)[at]] = 1.5
    p = rs.permutation(row.size)
    return np.stack([row[p], col[p]]).astype(np.int32), w[p]


@pytest.fixture(scope="module")
def graph():
    ei, w = _graph()
    dev = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    csr, w_csr, rowptr, _ = dev._neighborhood_structure()
    ref = (host(rowptr), host(csr.col), host(w_csr))
    pos_deg = host(dev._positive_degrees())
    degree = np.diff(ref[0])
    assert degree[12] > 128 and 20 == degree[15] and degree[13] == 6 and degree[HUB] == HUB_DEGREE
    for r, d in SPECIAL.items():
        assert d is None or pos_deg[r] == d, (r, pos_deg[r], d)
    c = np.concatenate([[0], np.cumsum(ref[2] > 0)])
    assert np.array_equal(pos_deg, c[ref[0][1:]] - c[ref[0][:-1]])
    from test_gpu_host_sampler import _device_bytes
    hs = sampling.HostNeighborSampler(ei, w, device_bytes=_device_bytes(ei, 2200000))    # the hub's range fits
    assert 5 <= len(hs._ranges) <= 20, len(hs._ranges)
    yield dev, hs, ref, ei, w
    hs.close()


def _seeds(n):
    s = np.random.RandomState(43).permutation(N)[:n].astype(np.int32)
    first = list(SPECIAL)
    s = s[~np.isin(s, first)]
    return np.concatenate([first, s])[:n].astype(np.int32)


def _assert_batch(b, want, what):
    nodes, edges, weights, sizes = want
    assert np.array_equal(host(b.node_index), nodes), what
    assert list(b.hop_sizes) == list(sizes), what
    L = len(b.blocks)
    for i, blk in enumerate(b.blocks):
        assert np.array_equal(host(blk.edge_index), edges[i]), (what, i)
        assert np.array_equal(host(blk.edge_weight), weights[i]), (what, i)
        assert np.array_equal(host(blk.global_col), nodes[edges[i][1]]), (what, i)
        rp = np.concatenate([[0], np.cumsum(np.bincount(edges[i][0], minlength=sizes[L - 1 - i]))])
        assert np.array_equal(host(blk.csr.rowptr), rp), (what, i)
        assert blk.weighted


CASES = [([15, 10, 5], False, 48), ([4, 25], True, 48), ([None, 4], False, 24), ([200], False, 64),
         ([3000], True, 5), ([30000], False, 2)]


@pytest.mark.parametrize("fanouts,padding,n_seeds", CASES)
def test_bit_for_bit_against_the_restatement(graph, fanouts, padding, n_seeds):
    dev, hs, (rowptr, col, w_csr), _, _ = graph
    seeds = _seeds(n_seeds)
    want = wr.neighborhood(rowptr, col, w_csr, seeds, fanouts, padding=padding, seed=77)
    for name, s in (("device", dev), ("host", hs)):
        for _ in range(2):                               # every result twice
            _assert_batch(s.sample_blocks(seeds, fanouts, padding=padding, seed=77, weighted=True), want, name)
    nb = dev.sample_neighborhood(seeds, fanouts, padding=padding, seed=77, weighted=True)
    assert np.array_equal(host(nb.node_index), want[0])
    for i in range(len(fanouts)):
        assert np.array_equal(host(nb.edge_index_list[i]), want[1][i])
        assert np.array_equal(host(nb.edge_weight_list[i]), want[2][i])


def test_unweighted_keyword_changes_nothing(graph):
    dev, hs, _, _, _ = graph
    seeds = _seeds(48)
    for s in (dev, hs):
        a = s.sample_blocks(seeds, [6, 3], seed=5)
        b = s.sample_blocks(seeds, [6, 3], seed=5, weighted=False)
        assert torch.equal(a.node_index, b.node_index)
        for x, y in zip(a.blocks, b.blocks):
            assert torch.equal(x.edge_index, y.edge_index) and torch.equal(x.edge_weight, y.edge_weight)
            assert not y.weighted


@pytest.mark.parametrize("exclude", ["self", "reverse"])
def test_exclusion_equals_the_graph_without_those_entries(graph, exclude):
    dev, hs, (rowptr, col, w_csr), _, _ = graph
    rs = np.random.RandomState(45)
    hub_pos = np.arange(rowptr[HUB], rowptr[HUB + 1])
    pick = rs.choice(hub_pos, 40, replace=False)
    others = rs.randint(0, N, 30)
    pairs = np.concatenate([np.stack([np.full(40, HUB), col[pick]]), np.stack([others, rs.randint(0, N, 30)])],
                           axis=1).astype(np.int32)
    seeds, _, _ = pair_begin_np(pairs, N)
    where = {int(v): t for t, v in enumerate(seeds)}
    targets = {}
    for u, v in pairs.T.tolist():
        targets.setdefault(where[u], set()).add(v)
        if exclude == "reverse":
            targets.setdefault(where[v], set()).add(u)
    excluded = {}
    for t, dests in targets.items():
        r = int(seeds[t])
        excluded[t] = [p for p in range(rowptr[r], rowptr[r + 1]) if int(col[p]) in dests]
    for fanouts, padding in (([10, 5], False), ([4, 3], True), ([30000], False)):
        want = wr.neighborhood(rowptr, col, w_csr, seeds, fanouts, padding=padding, seed=9, excluded=excluded)
        for name, s in (("device", dev), ("host", hs)):
            b = s.sample_link_blocks(pairs, fanouts, num_negatives=0, exclude=exclude, padding=padding, seed=9,
                                     weighted=True)
            _assert_batch(b, want, (name, exclude, fanouts))


def test_refusals_leave_the_map_clean(graph):
    dev, hs, _, ei, _ = graph
    plain = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32))
    with pytest.raises(ValueError, match="without one"):
        plain.sample_blocks(_seeds(8), [3], weighted=True)
    for s in (dev, hs):
        with pytest.raises(ValueError, match="head"):
            s.sample_blocks(_seeds(8), [3], padding="head", weighted=True)
        with pytest.raises(NotImplementedError):
            s.sample_blocks(_seeds(8), [3], seed=1, weighted=True).blocks[0].with_gcn_norm()
        assert int((s._node_map if s is hs else s._neighborhood_structure()[3]).max()) == -1
    bad = np.ones(ei.shape[1], np.float32)
    bad[5], bad[7] = -1.0, np.nan
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(bad))
    with pytest.raises(ValueError, match="2 negative, NaN or infinite"):
        s.sample_blocks(_seeds(8), [3], weighted=True)
    with sampling.HostNeighborSampler(ei, bad) as h:
        with pytest.raises(ValueError, match="2 negative, NaN or infinite"):
            h.sample_blocks(_seeds(8), [3], weighted=True)
        assert int(h._node_map.max()) == -1


def test_one_read_back_per_batch(graph):
    """Under torch.cuda.set_sync_debug_mode("error") a weighted batch makes no synchronisation torch can see, and the
    library reads back once per batch (tfgk_block_sample_end) plus once per hop of fan-out None.  The first weighted
    call on a sampler makes one more, the invalid-weight count read after the positive degrees (a torch .item(), seen in
    "warn" mode)."""
    import warnings
    _, _, _, ei, w = graph
    host_entries = ("tfgk_block_sample_read_total", "tfgk_block_sample_end")
    for make in (lambda: tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w)),
                 lambda: sampling.HostNeighborSampler(ei, w)):
        s = make()
        seeds = ops.as_device(_seeds(64), torch.int32)
        s.sample_blocks(seeds, [5, 3], seed=1)                     # build the structures
        torch.cuda.synchronize()
        trace = _ffi.CallTrace()
        prev = _ffi.set_trace(trace)
        with warnings.catch_warnings(record=True) as seen:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                s.sample_blocks(seeds, [5, 3], seed=1, weighted=True)      # the first weighted call
            finally:
                torch.cuda.set_sync_debug_mode(0)
                _ffi.set_trace(prev)
        syncs = [x for x in seen if "called a synchronizing" in str(x.message)]
        assert len(syncs) == 1, [str(x.message) for x in seen]
        assert sum(trace.counts.get(n, 0) for n in host_entries) == 1
        assert trace.counts.get("tfgk_csr_positive_degree_f32", 0) >= 1
        for fanouts, reads in (([5, 3], 1), ([None, 3], 2)):
            trace = _ffi.CallTrace()
            prev = _ffi.set_trace(trace)
            torch.cuda.set_sync_debug_mode("error")
            try:
                s.sample_blocks(seeds, fanouts, seed=2, weighted=True)
            finally:
                torch.cuda.set_sync_debug_mode(0)
                _ffi.set_trace(prev)
            assert sum(trace.counts.get(n, 0) for n in host_entries) == reads, (fanouts, trace.counts)
            assert "tfgk_csr_positive_degree_f32" not in trace.counts


# ---- exact distributions --------------------------------------------------------------------------------------------

def _star_rows(w, n_rows):
    """n_rows rows, each with the same len(w) entries: row r's entry i has column n_rows + i and weight w[i]."""
    d = len(w)
    row = np.repeat(np.arange(n_rows), d)
    col = n_rows + np.tile(np.arange(d), n_rows)
    return np.stack([row, col]).astype(np.int32), np.tile(np.asarray(w, np.float32), n_rows)


def _draws(s, n_rows, k, padding=False, seed=3):
    b = s.sample_blocks(np.arange(n_rows, dtype=np.int32), [k], padding=padding, seed=seed, weighted=True)
    blk = b.blocks[0]
    rp = host(blk.csr.rowptr)
    gcol = host(blk.global_col) - n_rows
    return gcol, rp


@pytest.mark.parametrize("k", [1, 2, 3])
def test_subsets_of_successive_sampling(k):
    W8 = np.array([0.2, 1.0, 3.0, 0.0, 0.7, 2.5, 1.3, 0.05], np.float32)
    n = ws.SUBSET_ROWS
    ei, w = _star_rows(W8, n)
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    gcol, rp = _draws(s, n, k)
    assert np.all(np.diff(rp) == k)
    assert not np.isin(gcol, np.flatnonzero(W8 == 0)).any()            # zero weights are never drawn
    ws.require(ws.subset_p(gcol.reshape(n, k), W8, k), "subsets k={}".format(k))


@pytest.mark.parametrize("k", [1, 2])
def test_inclusion_on_cta_rows(k):
    w = np.random.RandomState(5).rand(300).astype(np.float32) + 0.01
    w[::7] *= 20
    n = ws.HUB_ROWS
    ei, ww = _star_rows(w, n)
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(ww))
    draws = [_draws(s, n, k, seed=100 + key)[0].reshape(n, k) for key in range(ws.HUB_KEYS * 40)]
    ws.require(ws.inclusion_p(np.concatenate(draws), w, k), "inclusion k={}".format(k))


def test_with_replacement_draws_are_independent_multinomials():
    w = np.array([0.3, 2.0, 0.0, 1.0, 0.7], np.float32)
    n = ws.REPLACE_ROWS
    ei, ww = _star_rows(w, n)
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(ww))
    gcol, rp = _draws(s, n, 4, padding=True)          # k = 4 >= d+ = 4: with replacement
    assert np.all(np.diff(rp) == 4)
    ws.require(ws.replacement_p(gcol.reshape(n, 4), w), "with replacement")


def test_hops_and_batches_are_independent():
    W8 = np.array([0.2, 1.0, 3.0, 0.0, 0.7, 2.5, 1.3, 0.05], np.float32)
    n = ws.SUBSET_ROWS
    ei, w = _star_rows(W8, n)
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    a = _draws(s, n, 1, seed=11)[0]
    b = _draws(s, n, 1, seed=12)[0]
    ws.require(ws.independence_p(a, b, len(W8)), "batches")
    c = _draws(s, n, 1, seed=(11 + 0x9E3779B97F4A7C15) & ((1 << 64) - 1))[0]     # batch 11's second hop key
    ws.require(ws.independence_p(a, c, len(W8)), "hops")


# ---- the estimator --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("sampler", ["device", "host"])
@pytest.mark.parametrize("d,k", [(10, 12), (300, 300)])
def test_neighbour_sum_over_k_estimates_the_weighted_mean(sampler, d, k):
    """padding=True on rows with d+ <= k, so every draw is with replacement: the layer-0 neighbour sum (ops.spmm, SUM,
    unit values) over k, over EST_SAMPLES = 2 048 rows (128 seeds, 16 keys), has mean sum_i (w_i / W) x_i, computed in
    float64; the sample mean is within 4 standard errors of it.  d = 10: warp rows; d = 300: CTA rows."""
    per_key, n_keys = 128, 16
    rs = np.random.RandomState(60 + d)
    w = (rs.rand(d) * 2).astype(np.float32)
    w[rs.rand(d) < 0.2] = 0.0
    ei, ww = _star_rows(w, per_key)
    v = rs.randn(d, 4).astype(np.float32)
    x = np.zeros((per_key + d, 4), np.float32)
    x[per_key:] = v
    xd = ops.as_device(x)
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(ww)) if sampler == "device" \
        else sampling.HostNeighborSampler(ei, ww)
    est = []
    for key in range(n_keys):
        b = s.sample_blocks(np.arange(per_key, dtype=np.int32), [k], padding=True, seed=700 + key, weighted=True)
        blk = b.blocks[-1]
        assert np.all(np.diff(host(blk.csr.rowptr)) == k)
        x_src = xd[b.node_index[:blk.num_src].long()]
        agg = ops.spmm(blk.csr, torch.ones_like(blk.edge_weight), x_src, reduce="sum")
        est.append(host(agg[:per_key]).astype(np.float64) / k)
    est = np.concatenate(est)
    assert est.shape[0] == 2048
    want = (w.astype(np.float64) / w.astype(np.float64).sum()) @ v.astype(np.float64)
    se = est.std(axis=0, ddof=1) / np.sqrt(est.shape[0])
    assert np.all(np.abs(est.mean(axis=0) - want) <= 4 * se), (est.mean(axis=0), want, se)
    if sampler == "host":
        s.close()


# ---- training on weighted blocks ------------------------------------------------------------------------------------

def _weighted_ring_sampler():
    from test_gpu_blocks import _ring_graph
    ei, _ = _ring_graph()
    w = np.random.RandomState(72).rand(ei.shape[1]).astype(np.float32) * 2
    w[np.random.RandomState(73).rand(ei.shape[1]) < 0.15] = 0.0
    return tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))


@pytest.mark.parametrize("fanouts,padding", [([6, 4], False), ([5, 4], True)])
def test_mean_graphsage_on_weighted_blocks_against_float64(fanouts, padding):
    """2-layer mean GraphSAGE on weighted blocks: gradients within train_bound's per-entry bound of float64 autograd
    (tests/test_gpu_blocks.py's reference of the same block computation), and the same bits twice."""
    import train_bound as tb
    from test_gpu_blocks import _layer, _reference
    s = _weighted_ring_sampler()
    n, F, U = 2000, 20, 16
    b = s.sample_blocks(np.random.RandomState(5).permutation(n)[:200].astype(np.int32), fanouts, padding=padding,
                        seed=6, weighted=True)
    assert all(blk.weighted for blk in b.blocks)
    L = len(fanouts)
    layers = [_layer("mean", U if i < L - 1 else 8, seed=10 + i, concat=True,
                     activation=tfg.nn.relu if i < L - 1 else None) for i in range(L)]
    x = ops.as_device(np.random.RandomState(7).randn(b.hop_sizes[-1], F).astype(np.float32)).requires_grad_()

    def run():
        for layer in layers:
            layer.zero_grad(set_to_none=True)
        x.grad = None
        h, masks = x, []
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, blk], training=True)
            masks.append((None, torch.as_tensor((host(h) > 0).astype(np.float64)) if layer.activation else None))
        g = torch.randn(h.shape, generator=torch.Generator().manual_seed(9)).to(h.device)
        (h * g).sum().backward()
        return [{k: host(v.grad) for k, v in layer.named_parameters()} for layer in layers], host(x.grad), masks, g

    grads, dx, masks, g = run()
    shares = [None] * L
    want, want_dx = _reference("mean", layers, b.blocks, x, g, False, masks, shares, True)
    mag, mag_dx = _reference("mean", layers, b.blocks, x, g, True, masks, shares, True)
    n_max = max(b.hop_sizes)
    out_deg = max(int(np.bincount(host(blk.edge_index[1]), minlength=blk.num_src).max()) for blk in b.blocks)
    e = tb.eps(L * (max(fanouts) + out_deg + n_max + 16), *([4 * U] * (3 * L)))
    for got, ref, m in zip(grads, want, mag):
        for name in got:
            assert tb.ratio(got[name], ref[name], m[name], e) <= 1.0, name
    assert tb.ratio(dx, want_dx, mag_dx, e) <= 1.0
    grads2, dx2, _, _ = run()
    np.testing.assert_array_equal(dx2, dx)


def test_gat_on_weighted_blocks_against_float64():
    """2-layer GAT on self-looped weighted blocks: forward and gradients against float64 autograd of the same block
    computation (tests/test_gpu_block_gat.py's reference and tolerance), and the same bits twice."""
    from conftest import assert_close
    from test_gpu_block_gat import _gat64, _params
    s = _weighted_ring_sampler()
    H, L, split = 4, 2, True
    b = s.sample_blocks(np.random.RandomState(8).permutation(2000)[:128].astype(np.int32), [10, 5], seed=21,
                        weighted=True)
    looped = [blk.with_self_loops() for blk in b.blocks]
    rs = np.random.RandomState(H + L)
    params = [_params(rs, [32, 64][i], 64, 64, H, split) for i in range(L)]
    x = rs.randn(b.hop_sizes[-1], 32).astype(np.float32)
    gout = rs.randn(b.hop_sizes[0], 64)

    def run():
        tp = [[ops.as_device(t.astype(np.float32)).requires_grad_(True) for t in p] for p in params]
        xd = ops.as_device(x).requires_grad_(True)
        h = xd
        for i, lb in enumerate(looped):
            h = tfg.nn.gat(h, lb, tp[i][0], tp[i][1], tfg.nn.relu, tp[i][2], tp[i][3], tfg.nn.relu, tp[i][4], tp[i][5],
                           tfg.nn.relu if i < L - 1 else None, num_heads=H, split_value_heads=split, training=True,
                           seed=1234 + i)
        (h * ops.as_device(gout.astype(np.float32))).sum().backward()
        return [h.detach()] + [t.grad for p in tp for t in p] + [xd.grad]

    got = run()
    assert all(torch.equal(u, v) for u, v in zip(got, run()))
    tp64 = [[torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in p] for p in params]
    x64 = torch.tensor(x.astype(np.float64), requires_grad=True)
    h = x64
    for i, lb in enumerate(looped):
        h = _gat64(h, lb, tp64[i], H, split, i < L - 1, None)
    (h * torch.from_numpy(gout)).sum().backward()
    want = [h.detach().numpy()] + [t.grad.numpy() for p in tp64 for t in p] + [x64.grad.numpy()]
    assert_close(host(got[0]), want[0], what="forward")
    for j, (g, w) in enumerate(zip(got[1:], want[1:])):
        assert_close(host(g), w, rtol=1e-3, atol_scale=2e-4, what="gradient {}".format(j))


def test_weighted_sampling_learns_a_planted_partition():
    """Mean GraphSAGE with fan-outs [3, 3] on a planted partition whose inter-community edges carry weight 0.05 (about
    half of a node's edges leave its community): the weighted sampler draws mostly within it and reaches held-out
    accuracy >= 0.8.  The uniform sampler's accuracy on the same graph and schedule is printed, not asserted (0.887
    against the weighted 0.988 on an H100)."""
    rs = np.random.RandomState(62)
    n, classes, f = 20000, 4, 32
    labels = rs.randint(0, classes, n)
    src = rs.randint(0, n, 200000)
    by_label = np.argsort(labels, kind="stable")
    count = np.bincount(labels, minlength=classes)
    first = np.concatenate([[0], np.cumsum(count)[:-1]])
    same_class = by_label[first[labels[src]] + (rs.rand(src.size) * count[labels[src]]).astype(np.int64)]
    dst = np.where(rs.rand(src.size) < 0.3, same_class, rs.randint(0, n, src.size))
    ei = np.stack([np.concatenate([src, dst]), np.concatenate([dst, src])]).astype(np.int32)
    w = np.where(labels[ei[0]] == labels[ei[1]], 1.0, 0.05).astype(np.float32)
    centers = rs.randn(classes, f).astype(np.float32)
    x = (centers[labels] * 0.2 + rs.randn(n, f)).astype(np.float32)
    perm = rs.permutation(n)
    train, test = perm[:15000], perm[15000:]
    xd, yd = ops.as_device(x), ops.as_device(labels.astype(np.int64))
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))

    def accuracy(weighted):
        l1 = tfg.layers.MeanGraphSage(64, seed=1, trainable=True)
        l2 = tfg.layers.MeanGraphSage(classes, seed=2, trainable=True, activation=None, concat=False)
        with torch.no_grad():
            b = s.sample_blocks(train[:8].astype(np.int32), [3, 3], seed=0, weighted=weighted)
            l2([l1([b.source_rows(xd), b.blocks[0]]), b.blocks[1]])
        opt = torch.optim.Adam(list(l1.parameters()) + list(l2.parameters()), lr=0.01)
        order_rs, step = np.random.RandomState(63), 0
        for epoch in range(3):
            order = order_rs.permutation(train)
            for i in range(0, len(order), 512):
                seeds = order[i:i + 512].astype(np.int32)
                b = s.sample_blocks(seeds, [3, 3], seed=step, weighted=weighted)
                step += 1
                h = l2([l1([b.source_rows(xd), b.blocks[0]], training=True), b.blocks[1]], training=True)
                loss = torch.nn.functional.cross_entropy(h, yd[torch.from_numpy(seeds).long().to(xd.device)])
                opt.zero_grad()
                loss.backward()
                opt.step()
        with torch.no_grad():
            b = s.sample_blocks(test.astype(np.int32), [3, 3], seed=12345, weighted=weighted)
            h = l2([l1([b.source_rows(xd), b.blocks[0]]), b.blocks[1]])
            return float((h.argmax(1).cpu().numpy() == labels[test]).mean())

    acc_w, acc_u = accuracy(True), accuracy(False)
    print("planted partition, fan-outs [3, 3]: weighted {:.3f}, uniform {:.3f}".format(acc_w, acc_u))
    assert acc_w >= 0.8, "weighted {:.3f} (uniform {:.3f})".format(acc_w, acc_u)
