# coding=utf-8
"""Bipartite blocks on the device: RandomNeighborSampler.sample_blocks bit for bit against sample_neighborhood, the block
structures against csr_build, one host synchronisation per batch, the four GraphSAGE aggregators over blocks forward
(against the single index space) and backward (against float64 autograd of the same block computation), training on a
planted partition, and the refusals."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
import train_bound as tb
from conftest import random_graph

pytestmark = pytest.mark.gpu

HOST_ENTRIES = {"tfgk_block_sample_read_total", "tfgk_block_sample_end"}


def host(t):
    return t.detach().cpu().numpy()


def _sampler_graph():
    ei = random_graph(3000, 30000, seed=31, isolated=30, hub=(9, 5000))
    ei = np.concatenate([ei, ei[:, :500], [[3], [3100]]], axis=1).astype(np.int32)
    w = np.random.RandomState(32).rand(ei.shape[1]).astype(np.float32)
    return ei, w


@pytest.fixture(scope="module")
def sampler():
    ei, w = _sampler_graph()
    return tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))


def _seeds(n, first=(9, 0, 3)):
    seeds = np.random.RandomState(33).permutation(3000)[:n].astype(np.int32)
    seeds[:min(n, len(first))] = first[:n]
    return seeds


def _assert_same_sample(b, nb):
    assert torch.equal(b.node_index, nb.node_index)
    assert b.hop_sizes == nb.hop_sizes
    L = len(b.blocks)
    for i, blk in enumerate(b.blocks):
        assert torch.equal(blk.edge_index, nb.edge_index_list[i]), i
        assert torch.equal(blk.edge_weight, nb.edge_weight_list[i]), i
        assert (blk.num_src, blk.num_dst) == (b.hop_sizes[L - i], b.hop_sizes[L - 1 - i])
        assert torch.equal(blk.global_col, b.node_index[blk.edge_index[1].long()])


@pytest.mark.parametrize("fanouts,padding,n_seeds", [([15, 10, 5], False, 256), ([4, 25], True, 256), ([6], "head", 256),
                                                     ([3, None], False, 64), ([None, 2], True, 64), ([5, 4], False, 0),
                                                     ([5, 4], False, 1)])
def test_sample_blocks_matches_sample_neighborhood(sampler, fanouts, padding, n_seeds):
    seeds = _seeds(n_seeds)
    b = sampler.sample_blocks(seeds, fanouts, padding=padding, seed=17)
    nb = sampler.sample_neighborhood(seeds, fanouts, padding=padding, seed=17)
    _assert_same_sample(b, nb)
    again = sampler.sample_blocks(ops.as_device(seeds, torch.int32), fanouts, padding=padding, seed=17)
    _assert_same_sample(again, nb)


def test_capacity_past_int32_takes_the_fallback(sampler):
    seeds = _seeds(300)
    fanouts = [3, 2 ** 23]                   # 300 * 2^23 edges of capacity at the first hop: read back, then the CSR rows
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    try:
        b = sampler.sample_blocks(seeds, fanouts, seed=4)
    finally:
        _ffi.set_trace(prev)
    assert trace.counts.get("tfgk_block_sample_read_total") == 1
    _assert_same_sample(b, sampler.sample_neighborhood(seeds, fanouts, seed=4))


def test_block_structures(sampler):
    seeds = _seeds(256)
    # a None fan-out takes every neighbour of the hub row 9 (in-degree 5 000): that block has a hub-row plan
    for fanouts in ([15, 10, 5], [None, 4], [200, 3]):
        b = sampler.sample_blocks(seeds, fanouts, seed=23)
        for i, blk in enumerate(b.blocks):
            row, col = blk.edge_index[0].contiguous(), blk.edge_index[1].contiguous()
            want = ops.csr_build(row, col, blk.num_dst, blk.num_src)
            for name in ("rowptr", "col", "perm"):
                assert torch.equal(getattr(blk.csr, name), getattr(want, name)), (fanouts, i, name)
            assert (blk.csr.n_rows, blk.csr.n_cols) == (blk.num_dst, blk.num_src)
            assert (blk.csr.plan is None) == (ops.build_plan(want) is None), (fanouts, i)
            csr_t, _ = blk.transposed()
            want_t = ops.csr_build(col, row, blk.num_src, blk.num_dst)
            for name in ("rowptr", "col", "perm"):
                assert torch.equal(getattr(csr_t, name), getattr(want_t, name)), (fanouts, i, name)
            assert (csr_t.plan is None) == (want_t.plan is None)


def test_transposed_plan_for_a_popular_source():
    """a source node reached from more than HUB_THRESHOLD destination rows: every node points at node 0"""
    n = 6000
    rs = np.random.RandomState(3)
    ei = np.concatenate([np.stack([np.arange(n), np.zeros(n, np.int64)]), rs.randint(0, n, (2, 20000))], axis=1)
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei.astype(np.int32), torch.int32))
    b = s.sample_blocks(rs.permutation(n)[:4000].astype(np.int32), [8], seed=1)
    blk = b.blocks[0]
    csr_t, _ = blk.transposed()
    row, col = blk.edge_index[0].contiguous(), blk.edge_index[1].contiguous()
    want_t = ops.csr_build(col, row, blk.num_src, blk.num_dst)
    assert int(host(want_t.degree_i64()).max()) > ops.HUB_THRESHOLD and want_t.plan is not None
    for name in ("rowptr", "col", "perm"):
        assert torch.equal(getattr(csr_t, name), getattr(want_t, name))
    assert csr_t.plan is not None and csr_t.plan.n_hubs == want_t.plan.n_hubs


def test_one_synchronisation_per_batch(sampler):
    seeds = ops.as_device(_seeds(512), torch.int32)
    sampler.sample_blocks(seeds, [15, 10, 5], seed=1)             # warm: the cached CSR is built once per sampler
    torch.cuda.synchronize()
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    torch.cuda.set_sync_debug_mode("error")
    try:
        sampler.sample_blocks(seeds, [15, 10, 5], seed=2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        _ffi.set_trace(prev)
    assert sum(trace.counts.get(n, 0) for n in HOST_ENTRIES) == 1
    assert trace.counts.get("tfgk_block_sample_end") == 1
    for name in ("tfgk_csr_build", "tfgk_plan_build", "tfgk_frontier_i32", "tfgk_neighbor_sample_rows_count"):
        assert name not in trace.counts, name


def test_errors_leave_no_state_behind(sampler):
    ei, w = _sampler_graph()
    for bad in (np.array([5, 6, 5], np.int32), np.array([5, 3101], np.int32), np.array([-1, 2], np.int32)):
        with pytest.raises(ValueError):
            sampler.sample_blocks(bad, [4, 3], seed=17)
    assert bool((sampler._node_map == -1).all())
    fresh = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    seeds = _seeds(128)
    a = sampler.sample_blocks(seeds, [4, 3], seed=17)
    b = fresh.sample_blocks(seeds, [4, 3], seed=17)
    assert torch.equal(a.node_index, b.node_index)
    for x, y in zip(a.blocks, b.blocks):
        assert torch.equal(x.edge_index, y.edge_index) and torch.equal(x.edge_weight, y.edge_weight)


def test_failed_batches_leave_no_state_behind(sampler, monkeypatch):
    """a refused fan-out, and a failure after the seeds are in the map, leave the map clean for the next call"""
    ei, w = _sampler_graph()
    seeds = _seeds(128)
    with pytest.raises(ValueError, match="head"):
        sampler.sample_blocks(seeds, [None], padding="head", seed=17)
    assert bool((sampler._node_map == -1).all())
    plain = ops._block_workspace

    def failing(cap_list, cap_edges, device):
        if cap_list > len(seeds):                       # the second hop's allocation, after begin and one hop
            raise RuntimeError("allocation failed")
        return plain(cap_list, cap_edges, device)
    monkeypatch.setattr(ops, "_block_workspace", failing)
    with pytest.raises(RuntimeError, match="allocation"):
        sampler.sample_blocks(seeds, [4, 3], seed=17)
    monkeypatch.setattr(ops, "_block_workspace", plain)
    assert bool((sampler._node_map == -1).all())
    fresh = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    for fanouts in ([4, 3], [5]):
        a = sampler.sample_blocks(seeds, fanouts, seed=17)
        b = fresh.sample_blocks(seeds, fanouts, seed=17)
        assert torch.equal(a.node_index, b.node_index) and a.hop_sizes == b.hop_sizes
        for x, y in zip(a.blocks, b.blocks):
            assert torch.equal(x.edge_index, y.edge_index) and torch.equal(x.edge_weight, y.edge_weight)


# ---- layers ------------------------------------------------------------------------------------------------------

def _layer(kind, units, seed, **kw):
    cls = {"mean": tfg.layers.MeanGraphSage, "sum": tfg.layers.SumGraphSage, "mean_pool": tfg.layers.MeanPoolGraphSage,
           "max_pool": tfg.layers.MaxPoolGraphSage}[kind]
    return cls(units, seed=seed, trainable=True, **kw)


@pytest.fixture(scope="module")
def features():
    return ops.as_device(np.random.RandomState(34).randn(3101, 24).astype(np.float32))


@pytest.mark.parametrize("kind", ["mean", "sum", "mean_pool", "max_pool"])
@pytest.mark.parametrize("concat,activation,normalize", [(True, tfg.nn.relu, False), (False, None, True),
                                                         (True, None, False), (False, tfg.nn.relu, True)])
def test_forward_matches_the_single_index_space(sampler, features, kind, concat, activation, normalize):
    seeds = _seeds(256)
    b = sampler.sample_blocks(seeds, [7, 5], seed=8)
    nb = sampler.sample_neighborhood(seeds, [7, 5], seed=8)
    x_all = features[nb.node_index.long()].contiguous()
    blk = b.blocks[0]
    # aggregates: bit for bit the single space's first num_dst rows
    if kind in ("mean", "sum"):
        csr = ops.csr_build(nb.edge_index_list[0][0].contiguous(), nb.edge_index_list[0][1].contiguous(),
                            x_all.shape[0], x_all.shape[0])
        want = ops.spmm(csr, ops.permute(nb.edge_weight_list[0], csr.perm), x_all, reduce=kind)[:blk.num_dst]
        got = ops.spmm(blk.csr, blk.edge_weight, x_all, reduce=kind)
        got_global = ops.spmm(blk.csr, blk.edge_weight, features, reduce=kind, col=blk.global_col)
        assert torch.equal(got, want) and torch.equal(got_global, want)
    layer = _layer(kind, 16, seed=3, concat=concat, activation=activation, normalize=normalize)
    with torch.no_grad():
        single = layer([x_all, nb.edge_index_list[0], nb.edge_weight_list[0]])
        out = layer([x_all, blk])
        out_src = layer([b.source_rows(features), blk])
    assert out.shape[0] == blk.num_dst
    np.testing.assert_array_equal(host(out_src), host(out))        # max-pool rows without in-edges overflow alike
    np.testing.assert_allclose(host(out), host(single)[:blk.num_dst], rtol=1e-5, atol=1e-5)


# ---- backward against float64 ------------------------------------------------------------------------------------

def _ring_graph():
    """every node has in-edges (max-pool rows are finite), duplicate edges (exact ties)"""
    n = 2000
    rs = np.random.RandomState(71)
    ei = rs.randint(0, n, (2, 12000))
    ring = np.stack([np.arange(n), (np.arange(n) + 1) % n])
    ei = np.concatenate([ei, ring, ei[:, :2000]], axis=1).astype(np.int32)
    return ei, rs.rand(ei.shape[1]).astype(np.float32) + 0.5


def _agg64(kind, h, row, col, w, n_dst, share):
    if kind == "max_pool":
        val = share
    elif kind == "mean_pool":
        val = torch.ones_like(w)
    else:
        val = w
    s = torch.zeros((n_dst, h.shape[1]), dtype=torch.float64)
    if kind == "max_pool":       # the tie shares are per (edge, column): the selection the float32 kernel made
        return s.index_add(0, row, share * h[col])
    s = s.index_add(0, row, val.unsqueeze(1) * h[col])
    if kind in ("mean", "mean_pool"):
        cnt = torch.zeros(n_dst, dtype=torch.float64).index_add(0, row, torch.ones_like(w))
        s = s / cnt.clamp(min=1).unsqueeze(1)
    return s


def _reference(kind, layers, blocks, x, g, magnitude, masks, shares, concat):
    """float64 forward + backward of the block model; returns {name: grad} per layer and dx"""
    R = tb.Replay(magnitude)
    xs = R.leaf(host(x))
    h = xs
    params = []
    for li, (layer, blk) in enumerate(zip(layers, blocks)):
        p = {k: R.leaf(host(v)) for k, v in layer.named_parameters()}
        params.append(p)
        row, col = (torch.as_tensor(host(blk.edge_index[i]).astype(np.int64)) for i in (0, 1))
        w = R.const(host(blk.edge_weight))
        n_dst = blk.num_dst
        if kind in ("mean_pool", "max_pool"):
            mk, mb, nk = layer._names
            hn = h @ p[mk] + p[mb]
            hn = R.relu(hn, masks[li][0]) if masks[li][0] is not None else hn
            agg = _agg64(kind, hn, row, col, w, n_dst, shares[li])
        else:
            nk = "neighbor_kernel"
            agg = _agg64(kind, h, row, col, w, n_dst, None)
        u = p["self_kernel"].shape[1]
        if concat:
            out = torch.cat([h[:n_dst] @ p["self_kernel"] + p["bias"][:u], agg @ p[nk] + p["bias"][u:]], dim=1)
        else:
            out = h[:n_dst] @ p["self_kernel"] + agg @ p[nk] + p["bias"]
        h = R.relu(out, masks[li][1]) if masks[li][1] is not None else out
    (h * R.upstream(host(g))).sum().backward()
    return [{k: v.grad.numpy() for k, v in p.items()} for p in params], xs.grad.numpy()


@pytest.mark.parametrize("kind", ["mean", "sum", "mean_pool", "max_pool"])
@pytest.mark.parametrize("fanouts", [[6, 4], [5, 4, 3]])
def test_backward_against_float64(kind, fanouts):
    ei, w = _ring_graph()
    n, F, U = 2000, 20, 16
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    b = s.sample_blocks(np.random.RandomState(5).permutation(n)[:200].astype(np.int32), fanouts,
                        padding=kind == "max_pool", seed=6)
    L = len(fanouts)
    concat = kind != "sum"
    layers = [_layer(kind, U if i < L - 1 else 8, seed=10 + i, concat=concat,
                     activation=tfg.nn.relu if i < L - 1 else None) for i in range(L)]
    x = ops.as_device(np.random.RandomState(7).randn(b.hop_sizes[-1], F).astype(np.float32)).requires_grad_()

    def run():
        for layer in layers:
            layer.zero_grad(set_to_none=True)
        x.grad = None
        h, masks, shares = x, [], []
        for layer, blk in zip(layers, b.blocks):
            prev = h.detach()
            h = layer([h, blk], training=True)
            hn_mask = share = None
            if kind in ("mean_pool", "max_pool"):       # the neighbour MLP's ReLU mask and max selection, as computed
                mk, mb, _ = layer._names
                act = ops.ACT_RELU if layer.activation else ops.ACT_NONE
                hn = host(ops.gemm(prev, getattr(layer, mk).detach(), bias=getattr(layer, mb).detach(), act=act))
                hn_mask = torch.as_tensor((hn > 0).astype(np.float64)) if layer.activation else None
                if kind == "max_pool":
                    row, col = host(blk.edge_index[0]), host(blk.edge_index[1])
                    mx = np.full((blk.num_dst, hn.shape[1]), -np.inf, np.float32)
                    np.maximum.at(mx, row, hn[col])
                    sel = (hn[col] == mx[row]).astype(np.float64)
                    cnt = np.zeros(mx.shape, np.float64)
                    np.add.at(cnt, row, sel)
                    share = torch.as_tensor(sel / cnt[row])
            masks.append((hn_mask, torch.as_tensor((host(h) > 0).astype(np.float64)) if layer.activation else None))
            shares.append(share)
        g = torch.randn(h.shape, generator=torch.Generator().manual_seed(9)).to(h.device)
        (h * g).sum().backward()
        grads = [{k: host(v.grad) for k, v in layer.named_parameters()} for layer in layers]
        return grads, host(x.grad), masks, shares, g

    grads, dx, masks, shares, g = run()
    want, want_dx = _reference(kind, layers, b.blocks, x, g, False, masks, shares, concat)
    mag, mag_dx = _reference(kind, layers, b.blocks, x, g, True, masks, shares, concat)
    n_max = max(b.hop_sizes)
    out_deg = max(int(np.bincount(host(blk.edge_index[1]), minlength=blk.num_src).max()) for blk in b.blocks)
    # every stage's longest chain, summed over the layers: aggregation (fan-out), transposed (out-degree), the
    # split-K weight gradients and column sums (rows), and K4 products of depth <= 4 U
    e = tb.eps(L * (max(fanouts) + out_deg + n_max + 16), *([4 * U] * (3 * L)))
    for got, ref, m in zip(grads, want, mag):
        for name in got:
            r = tb.ratio(got[name], ref[name], m[name], e)
            assert r <= 1.0, (kind, name, r, tb.worst_entry(got[name], ref[name], m[name], e))
    assert tb.ratio(dx, want_dx, mag_dx, e) <= 1.0
    grads2, dx2, _, _, _ = run()
    np.testing.assert_array_equal(dx2, dx)
    for a, c in zip(grads, grads2):
        for name in a:
            np.testing.assert_array_equal(a[name], c[name])


def test_source_rows_route_trains_the_weights_only(sampler, features):
    b = sampler.sample_blocks(_seeds(128), [5, 4], seed=2)
    l1, l2 = _layer("mean", 16, 1), _layer("mean", 8, 2, activation=None)
    h = l2([l1([b.source_rows(features), b.blocks[0]], training=True), b.blocks[1]], training=True)
    h.sum().backward()
    l1b, l2b = _layer("mean", 16, 1), _layer("mean", 8, 2, activation=None)
    xs = features[b.node_index.long()].contiguous()
    h2 = l2b([l1b([xs, b.blocks[0]], training=True), b.blocks[1]], training=True)
    h2.sum().backward()
    assert torch.equal(h, h2)
    for (n1, p1), (_, p2) in zip(list(l1.named_parameters()) + list(l2.named_parameters()),
                                 list(l1b.named_parameters()) + list(l2b.named_parameters())):
        assert torch.equal(p1.grad, p2.grad), n1


# ---- training ------------------------------------------------------------------------------------------------------

def test_block_training_on_planted_partition():
    rs = np.random.RandomState(61)
    n, classes, f = 20000, 4, 32
    labels = rs.randint(0, classes, n)
    src = rs.randint(0, n, 200000)
    by_label = np.argsort(labels, kind="stable")
    count = np.bincount(labels, minlength=classes)
    first = np.concatenate([[0], np.cumsum(count)[:-1]])
    same_class = by_label[first[labels[src]] + (rs.rand(src.size) * count[labels[src]]).astype(np.int64)]
    dst = np.where(rs.rand(src.size) < 0.8, same_class, rs.randint(0, n, src.size))
    ei = np.stack([np.concatenate([src, dst]), np.concatenate([dst, src])]).astype(np.int32)
    centers = rs.randn(classes, f).astype(np.float32)
    x = (centers[labels] * 0.35 + rs.randn(n, f)).astype(np.float32)
    perm = rs.permutation(n)
    train, test = perm[:15000], perm[15000:]
    xd, yd = ops.as_device(x), ops.as_device(labels.astype(np.int64))
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32))
    l1 = tfg.layers.MeanGraphSage(64, seed=1, trainable=True)
    l2 = tfg.layers.MeanGraphSage(classes, seed=2, trainable=True, activation=None, concat=False)
    with torch.no_grad():
        b = s.sample_blocks(train[:8].astype(np.int32), [10, 10], seed=0)
        l2([l1([b.source_rows(xd), b.blocks[0]]), b.blocks[1]])
    opt = torch.optim.Adam(list(l1.parameters()) + list(l2.parameters()), lr=0.01)
    step = 0
    for epoch in range(3):
        order = rs.permutation(train)
        for i in range(0, len(order), 512):
            seeds = order[i:i + 512].astype(np.int32)
            b = s.sample_blocks(seeds, [10, 10], seed=step)
            step += 1
            h = l2([l1([b.source_rows(xd), b.blocks[0]], training=True), b.blocks[1]], training=True)
            loss = torch.nn.functional.cross_entropy(h, yd[torch.from_numpy(seeds).long().to(xd.device)])
            opt.zero_grad()
            loss.backward()
            opt.step()
    with torch.no_grad():
        b = s.sample_blocks(test.astype(np.int32), [10, 10], seed=12345)
        h = l2([l1([b.source_rows(xd), b.blocks[0]]), b.blocks[1]])
        acc = float((h.argmax(1).cpu().numpy() == labels[test]).mean())
    assert acc >= 0.8, acc


# ---- refusals ------------------------------------------------------------------------------------------------------

def test_refusals(sampler, features):
    b = sampler.sample_blocks(_seeds(64), [4, 3], seed=1)
    blk = b.blocks[0]
    x = features[b.node_index.long()].contiguous()
    for kind in ("mean", "sum", "mean_pool", "max_pool"):
        layer = _layer(kind, 8, 1)
        with pytest.raises(ValueError, match="rows"):
            layer([x[:-1], blk])
        with pytest.raises(ValueError):
            layer([b.source_rows(features), b.blocks[1]])
        w = torch.ones(blk.edge_index.shape[1], device=x.device, requires_grad=True)
        with pytest.raises(NotImplementedError):
            layer([x, blk, w])
        bf = _layer(kind, 8, 1, message_dtype=torch.bfloat16)
        with pytest.raises(NotImplementedError):
            bf([x, blk])
    for layer in (tfg.layers.GCN(8), tfg.layers.GAT(8), tfg.layers.GCNGraphSage(8), tfg.layers.LSTMGraphSage(8)):
        with pytest.raises(TypeError, match="block"):
            layer([x, blk])
    with pytest.raises(TypeError):
        tfg.layers.GCN(8)([b.source_rows(features), torch.zeros((2, 1), dtype=torch.int32, device=x.device)])
