# coding=utf-8
"""Layer-neighbour (LABOR-0) sampling on the device (sample_blocks / sample_link_blocks with labor=True), on
RandomNeighborSampler and on HostNeighborSampler with its host CSR in one range and cut into several.

The rule (include/tfgk.h, "LABOR block sampler"): column c gets u_c from Philox counter (c, 0, 4, 0) under the hop key
(hop 0's at every hop with layer_dependency); a row of d > k candidates keeps (row, c) iff u_c * d < k 2^32, a row of
d <= k keeps every candidate.  Checked bit for bit against tests/labor_ref.py, then against the closed forms of
tests/labor_stats.py on graphs of independent copies (columns never shared between copies, so one batch holds many
independent samples)."""
import math

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from tf_geometric_b200.utils import sampling
import labor_ref as lr
import labor_stats as ls
from link_blocks_fake_backend import pair_begin_np

pytestmark = pytest.mark.gpu

N = 3000
HUB, HUB_DEGREE = 9, 60000
# rows whose entries are exactly the listed ones (the random rows avoid the ids 9 ... 16): the hub, d = 0, 1, k, k + 1
# for k = 5 (row 13 holds one column three times), and 127, 128, 129 entries on both sides of the warp / CTA split
SPECIAL = {HUB: HUB_DEGREE, 10: 0, 11: 1, 12: 5, 13: 6, 14: 127, 15: 128, 16: 129}


def host(t):
    return t.detach().cpu().numpy()


def _graph():
    rs = np.random.RandomState(81)
    rnd = rs.randint(0, N - 8, 200000)
    rnd = rnd + 8 * (rnd >= HUB)                             # no random entry in rows 9 ... 16
    row = np.concatenate([rnd] + [np.full(d, r) for r, d in SPECIAL.items()])
    col = rs.randint(0, N, row.size)
    col[np.flatnonzero(row == 13)[:3]] = 17                  # row 13: one column three times (duplicate edges)
    w = (rs.rand(row.size) * 3).astype(np.float32)
    p = rs.permutation(row.size)
    return np.stack([row[p], col[p]]).astype(np.int32), w[p]


@pytest.fixture(scope="module")
def graph():
    from test_gpu_host_sampler import _device_bytes
    ei, w = _graph()
    dev = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    csr, w_csr, rowptr, _ = dev._neighborhood_structure()
    ref = (host(rowptr), host(csr.col), host(w_csr))
    degree = np.diff(ref[0])
    for r, d in SPECIAL.items():
        assert degree[r] == d, (r, degree[r], d)
    one = sampling.HostNeighborSampler(ei, w)
    several = sampling.HostNeighborSampler(ei, w, device_bytes=_device_bytes(ei, 2200000))   # the hub's range fits
    assert len(one._ranges) == 1 and len(several._ranges) >= 3, (len(one._ranges), len(several._ranges))
    yield dev, (one, several), ref, ei, w
    one.close()
    several.close()


def _seeds(n):
    s = np.random.RandomState(83).permutation(N)[:n].astype(np.int32)
    first = list(SPECIAL)
    s = s[~np.isin(s, first)]
    return np.concatenate([first, s])[:n].astype(np.int32)


def _assert_batch(b, want, what):
    nodes, edges, weights, gcols, sizes = want
    assert np.array_equal(host(b.node_index), nodes), what
    assert list(b.hop_sizes) == list(sizes), what
    L = len(b.blocks)
    for i, blk in enumerate(b.blocks):
        assert np.array_equal(host(blk.edge_index), edges[i]), (what, i)
        assert np.array_equal(host(blk.edge_weight), weights[i]), (what, i)
        assert np.array_equal(host(blk.global_col), gcols[i]), (what, i)
        rp = np.concatenate([[0], np.cumsum(np.bincount(edges[i][0], minlength=sizes[L - 1 - i]))])
        assert np.array_equal(host(blk.csr.rowptr), rp), (what, i)
        assert blk.labor == (blk.fanout is not None), (what, i)


CASES = [([15, 10, 5], False, 40), ([15, 10, 5], True, 40), ([5, 5], False, 64), ([None, 5], False, 24),
         ([5, 0], False, 16), ([0, None, 5], True, 16), ([5], False, 300), ([30000], False, 3), ([30000, 5], True, 2)]


@pytest.mark.parametrize("fanouts,layer_dependency,n_seeds", CASES)
def test_bit_for_bit_against_the_restatement(graph, fanouts, layer_dependency, n_seeds):
    dev, hosts, (rowptr, col, w_csr), _, _ = graph
    seeds = _seeds(n_seeds)
    want = lr.neighborhood(rowptr, col, w_csr, seeds, fanouts, seed=77, layer_dependency=layer_dependency)
    for name, s in (("device", dev), ("host, one range", hosts[0]), ("host, several", hosts[1])):
        for _ in range(2):                               # every result twice
            _assert_batch(s.sample_blocks(seeds, fanouts, seed=77, labor=True, layer_dependency=layer_dependency),
                          want, (name, fanouts, layer_dependency))


def test_hub_with_k_5_and_30000_keeps_pi_of_its_entries(graph):
    dev, _, (rowptr, col, w_csr), _, _ = graph
    for k in (5, 30000):
        b = dev.sample_blocks(np.array([HUB], np.int32), [k], seed=3, labor=True)
        kept = int(host(b.blocks[0].csr.rowptr)[1])
        want = HUB_DEGREE * lr.pi(k, HUB_DEGREE)
        assert abs(kept - want) < 5 * math.sqrt(want) + 1, (k, kept, want)


def test_labor_false_changes_nothing(graph):
    dev, hosts, _, _, _ = graph
    seeds = _seeds(48)
    for s in (dev,) + hosts:
        a = s.sample_blocks(seeds, [6, 3], seed=5)
        b = s.sample_blocks(seeds, [6, 3], seed=5, labor=False, layer_dependency=False)
        assert torch.equal(a.node_index, b.node_index)
        for x, y in zip(a.blocks, b.blocks):
            assert torch.equal(x.edge_index, y.edge_index) and torch.equal(x.edge_weight, y.edge_weight)
            assert not y.labor


@pytest.mark.parametrize("exclude", ["self", "reverse"])
def test_link_batches_exclude_before_the_rule(graph, exclude):
    dev, hosts, (rowptr, col, w_csr), _, _ = graph
    rs = np.random.RandomState(85)
    hub_pos = np.arange(rowptr[HUB], rowptr[HUB + 1])
    pick = rs.choice(hub_pos, 40, replace=False)
    others = rs.randint(0, N, 30)
    pairs = np.concatenate([np.stack([np.full(40, HUB), col[pick]]), np.stack([others, rs.randint(0, N, 30)]),
                            np.array([[13, 12], [17, 15]])], axis=1).astype(np.int32)
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
    for fanouts, ld in (([10, 5], False), ([4, 3], True), ([30000], False)):
        want = lr.neighborhood(rowptr, col, w_csr, seeds, fanouts, seed=9, layer_dependency=ld, excluded=excluded)
        for name, s in (("device", dev), ("host", hosts[1])):
            b = s.sample_link_blocks(pairs, fanouts, num_negatives=0, exclude=exclude, seed=9, labor=True,
                                     layer_dependency=ld)
            _assert_batch(b, want, (name, exclude, fanouts))


def test_refusals_leave_the_map_clean(graph):
    dev, hosts, _, _, _ = graph
    for s in (dev,) + hosts:
        for kw, err in ((dict(padding=True, labor=True), ValueError), (dict(padding="head", labor=True), ValueError),
                        (dict(layer_dependency=True), ValueError), (dict(weighted=True, labor=True),
                                                                     NotImplementedError)):
            with pytest.raises(err):
                s.sample_blocks(_seeds(8), [3], seed=1, **kw)
            with pytest.raises(err):
                s.sample_link_blocks(np.array([[1], [2]], np.int32), [3], seed=1, **kw)
        assert int((s._node_map if s in hosts else s._neighborhood_structure()[3]).max()) == -1


def test_read_backs_per_batch(graph):
    """A LABOR batch of L integer hops reads back 1 + 2 L times: its end, each hop's edge total and each block's work
    plan (a LABOR block is planned as a fan-out None block); under set_sync_debug_mode("error") torch sees none."""
    dev, hosts, _, _, _ = graph
    seeds = ops.as_device(_seeds(64), torch.int32)
    for s in (dev, hosts[1]):
        s.sample_blocks(seeds, [5, 3], seed=1, labor=True)
        torch.cuda.synchronize()
        trace = _ffi.CallTrace()
        prev = _ffi.set_trace(trace)
        torch.cuda.set_sync_debug_mode("error")
        try:
            s.sample_blocks(seeds, [5, 3], seed=2, labor=True)
        finally:
            torch.cuda.set_sync_debug_mode(0)
            _ffi.set_trace(prev)
        returning = {k: v for k, v in trace.counts.items() if k in _ffi.NOT_CAPTURABLE and
                     "returns" in _ffi.NOT_CAPTURABLE[k][1]}
        assert returning == {"tfgk_block_sample_end": 1, "tfgk_block_sample_read_total": 2, "tfgk_plan_build": 2}, \
            returning


# ---- exact distributions --------------------------------------------------------------------------------------------
# Copy i of the statistics graph: rows A_i (d = 6: t_i and 5 fillers) and B_i (d = 10: t_i and 9 fillers), every column
# its own node, and one CTA row H_i (1 000 fillers) for the first HUB_COPIES copies.  Seeds: every A_i, B_i and H_i.

COPIES, HUB_COPIES, KEYS = 4000, 48, 8
DA, DB, DH = 6, 10, 1000


def _stats_graph():
    a = np.arange(COPIES) * 2
    b = a + 1
    nxt = 2 * COPIES
    hubs = nxt + np.arange(HUB_COPIES)
    nxt += HUB_COPIES
    t = nxt + np.arange(COPIES)
    nxt += COPIES
    fa = nxt + np.arange(COPIES * (DA - 1)).reshape(COPIES, DA - 1)
    nxt += fa.size
    fb = nxt + np.arange(COPIES * (DB - 1)).reshape(COPIES, DB - 1)
    nxt += fb.size
    fh = nxt + np.arange(HUB_COPIES * DH).reshape(HUB_COPIES, DH)
    cols_a = np.concatenate([t[:, None], fa], axis=1)         # t_i first in A_i's row, last in B_i's
    cols_b = np.concatenate([fb, t[:, None]], axis=1)
    row = np.concatenate([np.repeat(a, DA), np.repeat(b, DB), np.repeat(hubs, DH)])
    col = np.concatenate([cols_a.ravel(), cols_b.ravel(), fh.ravel()])
    seeds = np.concatenate([np.stack([a, b], 1).ravel(), hubs]).astype(np.int32)
    return np.stack([row, col]).astype(np.int32), seeds, cols_a, cols_b, fh


@pytest.fixture(scope="module")
def stats_graph():
    ei, seeds, cols_a, cols_b, fh = _stats_graph()
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32))
    return s, seeds, cols_a, cols_b, fh


def _kept(b, block, rows, cols):
    """bool [len(rows), cols.shape[1]]: whether list row rows[i] of `block` kept column cols[i, j]"""
    blk = b.blocks[block]
    r, g = host(blk.edge_index[0]).astype(np.int64), host(blk.global_col).astype(np.int64)
    edge = set(zip(r.tolist(), g.tolist()))
    return np.array([[(int(x), int(c)) in edge for c in cc] for x, cc in zip(rows, cols)], bool)


def _batches(stats_graph, layer_dependency, base):
    s, seeds, cols_a, cols_b, fh = stats_graph
    out = []
    for key in range(KEYS):
        b = s.sample_blocks(seeds, [2, 2], seed=base + key, labor=True, layer_dependency=layer_dependency)
        assert np.array_equal(host(b.node_index)[:seeds.size], seeds)
        pos_a, pos_b = 2 * np.arange(COPIES), 2 * np.arange(COPIES) + 1
        pos_h = 2 * COPIES + np.arange(HUB_COPIES)
        out.append(dict(
            a0=_kept(b, 1, pos_a, cols_a), b0=_kept(b, 1, pos_b, cols_b), h0=_kept(b, 1, pos_h, fh),
            a1=_kept(b, 0, pos_a, cols_a), b1=_kept(b, 0, pos_b, cols_b), new0=b.hop_sizes[1] - b.hop_sizes[0]))
    return out


@pytest.fixture(scope="module")
def draws(stats_graph):
    return {ld: _batches(stats_graph, ld, 1000) for ld in (False, True)}


def test_inclusion_and_subsets_given_the_count(draws):
    a = np.concatenate([d["a0"] for d in draws[False]])
    bb = np.concatenate([d["b0"] for d in draws[False]])
    h = np.concatenate([d["h0"] for d in draws[False]])
    ls.require(ls.inclusion_p(a, lr.pi(2, DA)), "A rows, inclusion")
    ls.require(ls.inclusion_p(bb, lr.pi(2, DB)), "B rows, inclusion")
    ls.require(ls.inclusion_p(h, lr.pi(2, DH)), "CTA rows, inclusion")
    ls.require(ls.subset_given_count_p(a), "A rows, subsets given the count")
    ls.require(ls.subset_given_count_p(bb), "B rows, subsets given the count")
    ls.require(ls.empty_p(a, lr.pi(2, DA)), "A rows, empty rows")


def test_rows_sharing_a_neighbour_keep_it_together(draws):
    both = sum(int((d["a0"][:, 0] & d["b0"][:, -1]).sum()) for d in draws[False])
    ls.require(ls.pair_p(both, COPIES * KEYS, min(lr.pi(2, DA), lr.pi(2, DB))), "within a hop")


@pytest.mark.parametrize("layer_dependency", [False, True])
def test_coupling_across_hops(draws, layer_dependency):
    both = sum(int((d["a0"][:, 0] & d["b1"][:, -1]).sum()) for d in draws[layer_dependency])
    pa, pb = lr.pi(2, DA), lr.pi(2, DB)
    ls.require(ls.pair_p(both, COPIES * KEYS, min(pa, pb) if layer_dependency else pa * pb), "across hops")


def test_batches_and_unseeded_calls_are_independent(stats_graph, draws):
    s, seeds = stats_graph[0], stats_graph[1]
    first, second = draws[False][0], draws[False][1]
    pa = lr.pi(2, DA)
    both = int((first["a0"][:, 0] & second["a0"][:, 0]).sum())
    ls.require(ls.pair_p(both, COPIES, pa * pa), "batches 1000 and 1001")
    u = [s.sample_blocks(seeds, [2], labor=True) for _ in range(2)]
    k = [_kept(b, 0, 2 * np.arange(COPIES), stats_graph[2])[:, 0] for b in u]
    ls.require(ls.pair_p(int((k[0] & k[1]).sum()), COPIES, pa * pa), "unseeded calls")


def test_distinct_sources_are_the_sum_of_max_pi(draws):
    pa, pb, ph = lr.pi(2, DA), lr.pi(2, DB), lr.pi(2, DH)
    reach = [max(pa, pb)] + [pa] * (DA - 1) + [pb] * (DB - 1)
    mean = COPIES * sum(reach) + HUB_COPIES * DH * ph
    var = COPIES * sum(p * (1 - p) for p in reach) + HUB_COPIES * DH * ph * (1 - ph)
    total = sum(d["new0"] for d in draws[False])
    ls.require(ls.total_p(total, KEYS * mean, KEYS * var), "distinct layer-0 sources")


# ---- estimators and layers ------------------------------------------------------------------------------------------

def test_mean_and_gcn_sum_estimate_the_full_graph():
    """Block mean aggregation and the GcnBlock neighbour sum of one row of 400 neighbours (k = 8), over many keys and
    conditional on k_r >= 1, within 4 standard errors of the float64 full-graph values."""
    rs = np.random.RandomState(91)
    d, F = 400, 4
    ei = np.stack([np.zeros(d, np.int64), 1 + np.arange(d)]).astype(np.int32)
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32))
    x = rs.randn(d + 1, F)
    xd = ops.as_device(x.astype(np.float32))
    means, sums = [], []
    for key in range(600):
        b = s.sample_blocks(np.array([0], np.int32), [8], seed=key, labor=True)
        blk = b.blocks[0]
        if blk.edge_index.shape[1] == 0:
            continue
        src = xd[b.node_index.long()].contiguous()
        means.append(host(src[blk.edge_index[1].long()].mean(0)).astype(np.float64))
        A = blk.with_gcn_norm().normalized(norm="left", add_self_loop=False)     # D^-1 A: the row's mean, rescaled
        sums.append(host(ops.spmm(A.csr, A.value_csr, src))[0].astype(np.float64))
    means, sums = np.array(means), np.array(sums)
    assert len(means) > 500
    for got, what in ((means, "mean"), (sums, "gcn neighbour sum")):
        want = x[1:].mean(0)
        z = (got.mean(0) - want) / (got.std(0, ddof=1) / math.sqrt(len(got)))
        assert np.all(np.abs(z) < 4.0), (what, z)


def _hub_sampler():
    """a ring-like random graph of 2 000 nodes and node 0 with 5 000 in-neighbours: a LABOR block with k = 3 000 holds
    a row longer than HUB_THRESHOLD"""
    from test_gpu_blocks import _ring_graph
    ei, w = _ring_graph()
    rs = np.random.RandomState(92)
    hub = np.stack([np.zeros(5000, np.int64), rs.randint(1, 2000, 5000)]).astype(np.int32)
    ei = np.concatenate([ei, hub], axis=1)
    w = np.concatenate([w, rs.rand(5000).astype(np.float32) + 0.5])
    return tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))


def _hub_batch(s, seed):
    seeds = np.concatenate([[0], np.random.RandomState(93).permutation(np.arange(1, 2000))[:150]]).astype(np.int32)
    b = s.sample_blocks(seeds, [6, 3000], seed=seed, labor=True)
    top = b.blocks[1]
    assert int(np.diff(host(top.csr.rowptr)).max()) > ops.HUB_THRESHOLD
    assert top.csr.plan is not None and top.csr.plan.n_hubs > 0
    return b


def test_mean_graphsage_on_labor_blocks_against_float64():
    import train_bound as tb
    from test_gpu_blocks import _layer, _reference
    s = _hub_sampler()
    b = _hub_batch(s, 6)
    L, F, U = 2, 20, 16
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
    row_max = max(int(np.diff(host(blk.csr.rowptr)).max()) for blk in b.blocks)
    out_deg = max(int(np.bincount(host(blk.edge_index[1]), minlength=blk.num_src).max()) for blk in b.blocks)
    e = tb.eps(L * (row_max + out_deg + n_max + 16), *([4 * U] * (3 * L)))
    for got, ref, m in zip(grads, want, mag):
        for name in got:
            assert tb.ratio(got[name], ref[name], m[name], e) <= 1.0, name
    assert tb.ratio(dx, want_dx, mag_dx, e) <= 1.0
    _, dx2, _, _ = run()
    np.testing.assert_array_equal(dx2, dx)


def test_gat_on_labor_blocks_against_float64():
    from conftest import assert_close
    from test_gpu_block_gat import _gat64, _params
    s = _hub_sampler()
    b = _hub_batch(s, 21)
    looped = [blk.with_self_loops() for blk in b.blocks]
    assert looped[1].csr.plan is not None and looped[1].csr.plan.n_hubs > 0
    H, L, split = 4, 2, True
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


def test_gcn_on_labor_blocks_against_float64():
    """2-layer GCN (with_gcn_norm, norm="both" with self loops) on LABOR blocks: forward and gradients of x against
    float64 autograd of the same normalised block matrices."""
    from conftest import assert_close
    s = _hub_sampler()
    b = _hub_batch(s, 33)
    rs = np.random.RandomState(94)
    F, U = 24, 16
    ws = [rs.randn(F, U).astype(np.float32) * 0.2, rs.randn(U, 8).astype(np.float32) * 0.2]
    x = rs.randn(b.hop_sizes[-1], F).astype(np.float32)
    mats = [blk.with_gcn_norm().normalized() for blk in b.blocks]
    xd = ops.as_device(x).requires_grad_(True)
    h = xd
    for i, (blk, W) in enumerate(zip(b.blocks, ws)):
        h = tfg.nn.gcn(h, blk.with_gcn_norm(), ops.as_device(W), None, tfg.nn.relu if i == 0 else None, training=True)
    g = rs.randn(*h.shape)
    (h * ops.as_device(g.astype(np.float32))).sum().backward()
    x64 = torch.tensor(x.astype(np.float64), requires_grad=True)
    h64 = x64
    for i, (A, W) in enumerate(zip(mats, ws)):
        idx = host(A.index).astype(np.int64)
        dense = torch.zeros(A.shape, dtype=torch.float64)
        dense.index_put_((torch.from_numpy(idx[0]), torch.from_numpy(idx[1])),
                         torch.from_numpy(host(A.value).astype(np.float64)), accumulate=True)
        h64 = dense @ (h64 @ torch.from_numpy(W.astype(np.float64)))
        if i == 0:
            h64 = torch.relu(h64)
    (h64 * torch.from_numpy(g)).sum().backward()
    assert_close(host(h), h64.detach().numpy(), what="forward")
    assert_close(host(xd.grad), x64.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what="dx")


# ---- learning -------------------------------------------------------------------------------------------------------

def test_labor_learns_a_planted_partition_as_uniform_does():
    """Mean GraphSAGE with fan-outs [5, 5] on a planted partition (30 % of edges within the community): LABOR blocks
    reach held-out accuracy within 0.05 of uniform blocks on the same graph and schedule (0.689 against 0.700 on an
    H100), and at least 0.6 (chance is 0.25)."""
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
    centers = rs.randn(classes, f).astype(np.float32)
    x = (centers[labels] * 0.2 + rs.randn(n, f)).astype(np.float32)
    perm = rs.permutation(n)
    train, test = perm[:15000], perm[15000:]
    xd, yd = ops.as_device(x), ops.as_device(labels.astype(np.int64))
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32))

    def accuracy(labor):
        l1 = tfg.layers.MeanGraphSage(64, seed=1, trainable=True)
        l2 = tfg.layers.MeanGraphSage(classes, seed=2, trainable=True, activation=None, concat=False)
        with torch.no_grad():
            b = s.sample_blocks(train[:8].astype(np.int32), [5, 5], seed=0, labor=labor)
            l2([l1([b.source_rows(xd), b.blocks[0]]), b.blocks[1]])
        opt = torch.optim.Adam(list(l1.parameters()) + list(l2.parameters()), lr=0.01)
        order_rs, step = np.random.RandomState(63), 0
        for epoch in range(3):
            order = order_rs.permutation(train)
            for i in range(0, len(order), 512):
                seeds = order[i:i + 512].astype(np.int32)
                b = s.sample_blocks(seeds, [5, 5], seed=step, labor=labor)
                step += 1
                h = l2([l1([b.source_rows(xd), b.blocks[0]], training=True), b.blocks[1]], training=True)
                loss = torch.nn.functional.cross_entropy(h, yd[torch.from_numpy(seeds).long().to(xd.device)])
                opt.zero_grad()
                loss.backward()
                opt.step()
        with torch.no_grad():
            b = s.sample_blocks(test.astype(np.int32), [5, 5], seed=12345, labor=labor)
            h = l2([l1([b.source_rows(xd), b.blocks[0]]), b.blocks[1]])
            return float((h.argmax(1).cpu().numpy() == labels[test]).mean())

    acc_l, acc_u = accuracy(True), accuracy(False)
    print("planted partition, fan-outs [5, 5]: LABOR {:.3f}, uniform {:.3f}".format(acc_l, acc_u))
    assert acc_l >= 0.6 and acc_l >= acc_u - 0.05, (acc_l, acc_u)
