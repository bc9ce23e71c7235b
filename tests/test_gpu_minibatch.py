# coding=utf-8
"""Mini-batch sampling on the device: K13 bit for bit against the full-graph sampler on every listed row, the relabelled
neighbourhood against the dict-based restatement, mini-batch GraphSAGE against the full graph when nothing is dropped,
the sampled-subgraph helpers against the reference restated, and mini-batch training on a planted partition."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _structure, _ffi
from tf_geometric_b200.utils import graph_utils as gu
import minibatch_ref as ref
from conftest import random_graph
from oracle import c_oracle

pytestmark = pytest.mark.gpu

HUB = 60000


def host(t):
    return t.detach().cpu().numpy()


def _hub_graph():
    """isolated rows 0..49, a hub (row 77) of in-degree HUB, a row of degree 700 (the CTA tier), duplicate edges"""
    ei = random_graph(5000, 40000, seed=21, isolated=50, hub=(77, HUB))
    extra = np.stack([np.full(700, 1234), np.random.RandomState(22).randint(0, 5000, 700)])
    ei = np.concatenate([ei, ei[:, :3000], extra], axis=1).astype(np.int32)
    return ei


@pytest.fixture(scope="module")
def hub_csr():
    ei = _hub_graph()
    eid = ops.as_device(ei, torch.int32)
    return ops.csr_build(eid[0].contiguous(), eid[1].contiguous(), 5000, 5000)


def _expected_rows(csr, rows, **kw):
    _, pos, rp = ops.neighbor_sample(csr, seed=99, **kw)
    pos, rp = host(pos), host(rp)
    return [pos[rp[r]:rp[r + 1]] for r in rows]


@pytest.mark.parametrize("k", [1, 5, 25, HUB - 1, HUB, HUB + 1])
@pytest.mark.parametrize("padding", [False, True, "head"])
def test_k13_matches_full_graph_sampler(hub_csr, k, padding):
    rs = np.random.RandomState(k % 1000 + 3)
    n_list = 3000 if k < 1000 else 400                                  # padding=True draws k per row
    rows = rs.randint(0, 5000, n_list).astype(np.int32)
    rows[rs.randint(0, n_list, 40)] = 77
    rows[rs.randint(0, n_list, 40)] = 1234
    rows[:20] = rs.randint(0, 50, 20)                                    # isolated rows
    rows[20:30] = rows[30:40]                                           # repeats
    t, pos, rp = ops.neighbor_sample_rows(hub_csr.rowptr, ops.as_device(rows, torch.int32), k=k, padding=padding, seed=99)
    want = _expected_rows(hub_csr, rows, k=k, padding=padding)
    t, pos, rp = host(t), host(pos), host(rp)
    assert rp[-1] == sum(len(w) for w in want)
    for i, w in enumerate(want):
        np.testing.assert_array_equal(pos[rp[i]:rp[i + 1]], w)
        assert np.all(t[rp[i]:rp[i + 1]] == i)


@pytest.mark.parametrize("ratio", [0.001, 0.3, 1.0])
def test_k13_ratio_mode(hub_csr, ratio):
    rows = np.random.RandomState(5).permutation(5000).astype(np.int32)
    _, pos, rp = ops.neighbor_sample_rows(hub_csr.rowptr, ops.as_device(rows, torch.int32), ratio=ratio, seed=99)
    want = _expected_rows(hub_csr, rows, ratio=ratio)
    pos, rp = host(pos), host(rp)
    for i, w in enumerate(want):
        np.testing.assert_array_equal(pos[rp[i]:rp[i + 1]], w)


def test_k13_rejects_rows_outside_the_csr(hub_csr):
    with pytest.raises(_ffi.TfgkError, match="outside"):
        ops.neighbor_sample_rows(hub_csr.rowptr, ops.as_device(np.array([3, 5000], np.int32), torch.int32), k=3)


def _sampler_graph():
    ei = random_graph(3000, 30000, seed=31, isolated=30, hub=(9, 5000))
    ei = np.concatenate([ei, ei[:, :500], [[3], [3100]]], axis=1).astype(np.int32)
    w = np.random.RandomState(32).rand(ei.shape[1]).astype(np.float32)
    return ei, w


@pytest.mark.parametrize("fanouts,padding", [([15, 10, 5], False), ([4, 25], True), ([6], "head")])
def test_sample_neighborhood_matches_restatement(fanouts, padding):
    ei, w = _sampler_graph()
    sampler = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    seeds = np.random.RandomState(33).permutation(3000)[:256].astype(np.int32)
    seeds[:3] = [9, 0, 3]
    b = sampler.sample_neighborhood(seeds, fanouts, padding=padding, seed=17)
    rowptr, col, perm = c_oracle.csr_build(ei[0], ei[1], int(ei[0].max()) + 1)
    nodes, edges, weights, sizes = ref.neighborhood(rowptr, col, w[perm], seeds, fanouts, padding, 17)
    np.testing.assert_array_equal(host(b.node_index), nodes)
    np.testing.assert_array_equal(host(b.node_index)[:256], seeds)
    assert b.hop_sizes == sizes
    for i, (got, want, gw, ww) in enumerate(zip(b.edge_index_list, edges, b.edge_weight_list, weights)):
        np.testing.assert_array_equal(host(got), want)
        np.testing.assert_array_equal(host(gw), ww)
        assert host(got)[0].max(initial=-1) < sizes[-2 - i]
    again = sampler.sample_neighborhood(ops.as_device(seeds, torch.int32), fanouts, padding=padding, seed=17)
    assert torch.equal(again.node_index, b.node_index)
    for x, y in zip(b.edge_index_list + b.edge_weight_list, again.edge_index_list + again.edge_weight_list):
        assert torch.equal(x, y)
    with pytest.raises(ValueError, match="duplicate"):
        sampler.sample_neighborhood(np.array([5, 6, 5], np.int32), fanouts, seed=17)


def _sage_pair(f, u):
    torch.manual_seed(0)
    l1 = tfg.layers.MeanGraphSage(u, seed=1, trainable=True)
    l2 = tfg.layers.MeanGraphSage(u, seed=2, trainable=True, activation=None)
    return l1, l2


def test_minibatch_equals_full_graph_without_drops():
    """fan-out >= the largest in-degree keeps every edge in CSR order: the seed rows' mean aggregates are bit for bit the
    full graph's.  The layer outputs go through the dense projection with a different row count, so they are compared to
    the full graph within a float32 GEMM bound; the weight gradients are checked against float64 autograd of the same
    subgraph computation."""
    rs = np.random.RandomState(41)
    n, f, u = 4000, 32, 16
    ei = random_graph(n, 24000, seed=42, isolated=40)
    w = rs.rand(ei.shape[1]).astype(np.float32)
    x = rs.randn(n, f).astype(np.float32)
    max_deg = int(np.bincount(ei[0], minlength=n).max())
    eid, wd, xd = ops.as_device(ei, torch.int32), ops.as_device(w), ops.as_device(x)
    sampler = tfg.utils.RandomNeighborSampler(eid, wd)
    seeds = rs.permutation(n)[:300].astype(np.int32)
    b = sampler.sample_neighborhood(seeds, [max_deg, max_deg + 3], seed=5)
    R = len(seeds)
    xs = xd[b.node_index.long()]

    def aggregate(e, weight, h):
        csr, _ = _structure.csr_for_edge_index(e, h.shape[0])
        return ops.spmm(csr, _structure.weights_in_csr_order(weight, csr), h, reduce="mean")

    full_agg = host(aggregate(eid, wd, xd))
    sub_agg = host(aggregate(b.edge_index_list[1], b.edge_weight_list[1], xs))
    np.testing.assert_array_equal(sub_agg[:R], full_agg[seeds])

    l1, l2 = _sage_pair(f, u)
    with torch.no_grad():
        full = host(l2([l1([xd, eid, wd]), eid, wd]))
        h1 = l1([xs, b.edge_index_list[0], b.edge_weight_list[0]])
        hop1 = b.hop_sizes[1]
        full1 = host(l1([xd, eid, wd]))
        np.testing.assert_allclose(host(h1)[:hop1], full1[host(b.node_index)[:hop1]], rtol=1e-5, atol=1e-5)
        mini = host(l2([h1, b.edge_index_list[1], b.edge_weight_list[1]]))
    np.testing.assert_allclose(mini[:R], full[seeds], rtol=1e-5, atol=1e-5)

    # weight gradients against float64 autograd of the same subgraph computation
    g = torch.randn(R, u, device=xd.device)
    out = l2([l1([xs, b.edge_index_list[0], b.edge_weight_list[0]], training=True), b.edge_index_list[1],
              b.edge_weight_list[1]], training=True)
    (out[:R] * g).sum().backward()

    def mean_agg64(e, weight, h):
        r, c = e[0].long(), e[1].long()
        s = torch.zeros_like(h).index_add_(0, r, h[c] * weight[:, None])
        cnt = torch.zeros(h.shape[0], dtype=h.dtype, device=h.device).index_add_(0, r, torch.ones_like(weight))
        return s / cnt.clamp(min=1)[:, None]

    params64 = [{k: v.detach().double().requires_grad_() for k, v in l.named_parameters()} for l in (l1, l2)]
    h = xs.double()
    for i, (p, act) in enumerate(zip(params64, (torch.relu, None))):
        agg = mean_agg64(b.edge_index_list[i], b.edge_weight_list[i].double(), h)
        h = torch.cat([h @ p["self_kernel"], agg @ p["neighbor_kernel"]], dim=1) + p["bias"]
        h = act(h) if act else h
    (h[:R] * g.double()).sum().backward()
    for l, p in zip((l1, l2), params64):
        for name, got in l.named_parameters():
            want = p[name].grad
            scale = float(want.abs().max())
            assert float((got.grad.double() - want).abs().max()) <= 1e-4 * scale + 1e-6, name


def test_parity_helpers_on_device():
    rs = np.random.RandomState(51)
    ei = rs.randint(0, 400, (2, 5000)).astype(np.int32)
    ei = np.concatenate([ei, ei[::-1, :300], ei[:, 100:400]], axis=1)
    w = rs.rand(ei.shape[1]).astype(np.float32)
    nodes = rs.permutation(450)[:200].astype(np.int32)
    eid, wd, nd = ops.as_device(ei, torch.int32), ops.as_device(w), ops.as_device(nodes, torch.int32)
    out = gu.reindex_sampled_edge_index(eid, nd)
    assert out.is_cuda
    np.testing.assert_array_equal(host(out), ref.reindex_sampled_edge_index(ei, nodes))
    with pytest.raises(ValueError, match="duplicate"):
        gu.reindex_sampled_edge_index(eid, ops.as_device(np.concatenate([nodes, nodes[:1]]), torch.int32))
    mask = gu.compute_edge_mask_by_node_index(eid, nd)
    assert mask.is_cuda and mask.dtype == torch.bool
    np.testing.assert_array_equal(host(mask), ref.compute_edge_mask_by_node_index(ei, nodes))
    for mode in ("undirected", "directed"):
        got_i, got_w = gu.extract_unique_edge(eid, wd, mode=mode)
        want_i, want_w = ref.extract_unique_edge(ei, w, mode)
        assert got_i.is_cuda and got_w.is_cuda
        np.testing.assert_array_equal(host(got_i), want_i)
        np.testing.assert_array_equal(host(got_w), want_w)


def test_minibatch_training_on_planted_partition():
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
    x = (centers[labels] * 0.35 + rs.randn(n, f)).astype(np.float32)   # features alone separate the classes poorly
    perm = rs.permutation(n)
    train, test = perm[:15000], perm[15000:]
    xd, eid, yd = ops.as_device(x), ops.as_device(ei, torch.int32), ops.as_device(labels.astype(np.int64))
    sampler = tfg.utils.RandomNeighborSampler(eid)
    l1 = tfg.layers.MeanGraphSage(64, seed=1, trainable=True)
    l2 = tfg.layers.MeanGraphSage(classes, seed=2, trainable=True, activation=None, concat=False)
    with torch.no_grad():                                               # build the layers
        b = sampler.sample_neighborhood(train[:8].astype(np.int32), [10, 10], seed=0)
        l2([l1([xd[b.node_index.long()], b.edge_index_list[0], b.edge_weight_list[0]]), b.edge_index_list[1],
            b.edge_weight_list[1]])
    opt = torch.optim.Adam(list(l1.parameters()) + list(l2.parameters()), lr=0.01)
    step = 0
    for epoch in range(3):
        order = rs.permutation(train)
        for i in range(0, len(order), 512):
            seeds = order[i:i + 512].astype(np.int32)
            b = sampler.sample_neighborhood(seeds, [10, 10], seed=step)
            step += 1
            h = xd[b.node_index.long()]
            for layer, e, w in zip((l1, l2), b.edge_index_list, b.edge_weight_list):
                h = layer([h, e, w], training=True)
            loss = torch.nn.functional.cross_entropy(h[:len(seeds)], yd[torch.from_numpy(seeds).long().to(xd.device)])
            opt.zero_grad()
            loss.backward()
            opt.step()
    with torch.no_grad():
        b = sampler.sample_neighborhood(test.astype(np.int32), [10, 10], seed=12345)
        h = xd[b.node_index.long()]
        for layer, e, w in zip((l1, l2), b.edge_index_list, b.edge_weight_list):
            h = layer([h, e, w])
        acc = float((h[:len(test)].argmax(1).cpu().numpy() == labels[test]).mean())
    assert acc >= 0.8, acc
