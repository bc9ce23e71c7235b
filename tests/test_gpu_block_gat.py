# coding=utf-8
"""GAT on sampled blocks on the device: tfgk_block_self_loops_i32 against a numpy restatement and the looped CSR against
csr_build, with no synchronisation below the plan threshold; the fused attention over a looped block bit for bit against
the single index space and (every neighbour) the full graph, dense, streaming and packed-key routes; the GAT layer
forward against the single index space; the backward against float64 autograd of a bipartite restatement on the
recompute and coefficient-table routes; host-memory graphs and features bit for bit; learning; the refusals."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi, _structure
from oracle import tfg_oracle as o
from conftest import random_graph, assert_close

pytestmark = pytest.mark.gpu


def host(t):
    return t.detach().cpu().numpy()


def _graph():
    ei = random_graph(3000, 30000, seed=31, isolated=30, hub=(9, 5000))
    return np.concatenate([ei, ei[:, :500], [[3], [3100]]], axis=1).astype(np.int32)


@pytest.fixture(scope="module")
def sampler():
    return tfg.utils.RandomNeighborSampler(ops.as_device(_graph(), torch.int32))


def _seeds(n, first=(9, 0, 3)):
    seeds = np.random.RandomState(33).permutation(3000)[:n].astype(np.int32)
    seeds[:min(n, len(first))] = first[:n]
    return seeds


def _looped_restatement(e, n_dst):
    """Row by row: the sampled edges of row r in order, then (r, r)."""
    rows, cols, rowptr = [], [], [0]
    order = np.argsort(e[0], kind="stable")
    starts = np.searchsorted(e[0][order], np.arange(n_dst + 1))
    for r in range(n_dst):
        sel = order[starts[r]:starts[r + 1]]
        rows += [r] * (sel.size + 1)
        cols += e[1][sel].tolist() + [r]
        rowptr.append(len(rows))
    return np.array(rowptr, np.int64), np.array([rows, cols], np.int64).reshape(2, -1)


BATCHES = [([15, 10, 5], False, None), ([4, 25], True, None), ([6], "head", None), ([None, 4], False, None),
           ([5, 3], False, np.arange(30, dtype=np.int32))]                   # seeds without neighbours


@pytest.mark.parametrize("fanouts,padding,seeds", BATCHES)
def test_kernel_and_looped_csr(sampler, fanouts, padding, seeds):
    b = sampler.sample_blocks(_seeds(256) if seeds is None else seeds, fanouts, padding=padding, seed=17)
    hubs = 0
    for i, blk in enumerate(b.blocks):
        lb = blk.with_self_loops()
        rowptr, e = _looped_restatement(host(blk.edge_index), blk.num_dst)
        np.testing.assert_array_equal(host(lb.csr.rowptr), rowptr)
        np.testing.assert_array_equal(host(lb.edge_index), e)
        want = ops.csr_build(lb.edge_index[0].contiguous(), lb.edge_index[1].contiguous(), blk.num_dst, blk.num_src)
        for name in ("rowptr", "col", "perm"):
            assert torch.equal(getattr(lb.csr, name), getattr(want, name)), (fanouts, i, name)
        assert (lb.csr.plan is None) == (want.plan is None), (fanouts, i)
        if want.plan is not None:
            assert (lb.csr.plan.n_tasks, lb.csr.plan.n_hubs) == (want.plan.n_tasks, want.plan.n_hubs)
            hubs += want.plan.n_hubs
        csr_t = lb.transposed()
        want_t = ops.csr_build(lb.edge_index[1].contiguous(), lb.edge_index[0].contiguous(), blk.num_src, blk.num_dst)
        for name in ("rowptr", "col", "perm"):
            assert torch.equal(getattr(csr_t, name), getattr(want_t, name)), (fanouts, i, name)
    assert (hubs > 0) == (fanouts == [None, 4])         # the hub row 9 (in-degree 5 000) is cut by the plan


def test_no_synchronisation_below_the_plan_threshold(sampler):
    b = sampler.sample_blocks(_seeds(512), [15, 10, 5], seed=2)
    torch.cuda.synchronize()
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    torch.cuda.set_sync_debug_mode("error")
    try:
        looped = [blk.with_self_loops() for blk in b.blocks]
    finally:
        torch.cuda.set_sync_debug_mode(0)
        _ffi.set_trace(prev)
    assert trace.counts == {"tfgk_block_self_loops_i32": 3}
    assert all(lb.csr.plan is None for lb in looped)
    assert [blk.with_self_loops() for blk in b.blocks] == looped          # memoised


def _qkv(n, A, seed):
    rs = np.random.RandomState(seed)
    Q = ops.as_device(rs.randn(n, A).astype(np.float32))
    kv = ops.as_device(rs.randn(n, 2 * A).astype(np.float32))
    return Q, kv


def _attention_routes(csr, Q, kv, H):
    A = Q.shape[1]
    K, V = kv[:, :A], kv[:, A:]
    outs = [ops.gat_fused(csr, Q, K, V, H), ops.gat_fused(csr, Q, K.contiguous(), V.contiguous(), H)]
    stats = ops.gat_fused_stats(csr, Q, K, V, H)
    if stats is not None:
        outs += list(stats)
    Kr = torch.relu(K).contiguous()
    table, sizes = ops.packed_key_table(K.shape[0], A, Q.device)
    table[:, :A].copy_(V)
    ops.gat_pack_keys(Kr, table, sizes)
    outs += [ops.gat_fused_packed(csr, Q, table, sizes, H), ops.gat_fused(csr, Q, Kr, V.contiguous(), H)]
    return outs


@pytest.mark.parametrize("fanouts", [[15, 10, 5], [None, 4]])
@pytest.mark.parametrize("H", [1, 8])
def test_attention_bit_for_bit_against_the_single_space(sampler, fanouts, H):
    seeds = _seeds(256)
    b = sampler.sample_blocks(seeds, fanouts, seed=17)
    nb = sampler.sample_neighborhood(seeds, fanouts, seed=17)
    n = nb.hop_sizes[-1]
    Q, kv = _qkv(n, 64, 5)
    for i, blk in enumerate(b.blocks):
        csr, _ = _structure.csr_for_edge_index(nb.edge_index_list[i], n, add_self_loop=True)
        want = _attention_routes(csr, Q, kv, H)
        got = _attention_routes(blk.with_self_loops().csr, Q[:blk.num_dst], kv[:blk.num_src], H)
        assert len(got) == len(want)
        for j, (g, w) in enumerate(zip(got, want)):
            assert torch.equal(g, w[:blk.num_dst]), (i, j)


@pytest.mark.parametrize("H", [1, 8])
def test_attention_bit_for_bit_against_the_full_graph(sampler, H):
    ei = _graph()
    N = int(ei.max()) + 1
    seeds = _seeds(256)
    b = sampler.sample_blocks(seeds, [None], seed=3)
    lb = b.blocks[0].with_self_loops()
    assert lb.csr.plan is not None and lb.csr.plan.n_hubs > 0          # seed 9's row is cut into slices
    csr, _ = _structure.csr_for_edge_index(ops.as_device(ei, torch.int32), N, add_self_loop=True)
    Q, kv = _qkv(N, 64, 7)
    idx = b.node_index.long()
    want = _attention_routes(csr, Q, kv, H)
    got = _attention_routes(lb.csr, Q[idx[:lb.num_dst]].contiguous(), kv[idx].contiguous(), H)
    for j, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w[idx[:lb.num_dst]]), j


def _single_positions(blk):
    """For every looped-block position, the position of the same edge in the single index space's edge list with self
    loops (its E sampled edges, then one self loop per node)."""
    e = host(blk.edge_index)
    rowptr = host(blk.csr.rowptr)
    E, n = e.shape[1], blk.num_dst
    pos = np.empty(E + n, np.int64)
    pos[np.arange(E) + e[0]] = np.arange(E)
    pos[rowptr[1:n + 1] + np.arange(n)] = E + np.arange(n)
    return pos


@pytest.fixture(scope="module")
def features():
    return ops.as_device(np.random.RandomState(34).randn(3101, 32).astype(np.float32))


@pytest.mark.parametrize("H,split,act", [(1, True, None), (4, True, "relu"), (8, True, "relu"), (4, False, "relu"),
                                         (8, False, None)])
def test_layer_forward_matches_the_single_space(sampler, features, H, split, act):
    seeds = _seeds(256)
    b = sampler.sample_blocks(seeds, [10, 5], seed=9)
    nb = sampler.sample_neighborhood(seeds, [10, 5], seed=9)
    xs = features[nb.node_index.long()]
    layer = tfg.layers.GAT(64, num_heads=H, split_value_heads=split, activation=tfg.nn.relu if act else None, seed=3)
    with torch.no_grad():
        single = layer([xs, nb.edge_index_list[0]])
        blk = b.blocks[0]
        lb = blk.with_self_loops()
        out = layer([xs, lb])
        src = layer([b.source_rows(features), lb])
        assert out.shape == (blk.num_dst, 64)
        np.testing.assert_allclose(host(out), host(single)[:blk.num_dst], rtol=1e-5, atol=1e-5)
        assert torch.equal(src, out)
        p = {k: v.detach() for k, v in layer.named_parameters()}
        args = (p["query_kernel"], p["query_bias"], tfg.nn.relu, p["key_kernel"], p["key_bias"], tfg.nn.relu, p["kernel"],
                p["bias"])
        _, att = tfg.nn.gat(xs, lb, *args, num_heads=H, split_value_heads=split, return_attention=True)
        _, att_s = tfg.nn.gat(xs, nb.edge_index_list[0], *args, num_heads=H, split_value_heads=split,
                              return_attention=True)
    assert att.shape == (lb.edge_index.shape[1], H)
    np.testing.assert_allclose(host(att), host(att_s)[_single_positions(blk)], rtol=1e-5, atol=1e-6)


# ---- backward against float64 -------------------------------------------------------------------------------------

def _gat64(x, lb, p, H, split, relu, mult):
    """float64 bipartite GAT over a looped block: queries from x[:num_dst], keys and values from x, softmax per
    destination row, coefficients times `mult` ([nnz, H], the dropout multipliers at looped-CSR positions)."""
    e = torch.from_numpy(host(lb.edge_index).astype(np.int64))
    row, col = e[0], e[1]
    nd, E = lb.num_dst, e.shape[1]
    wq, bq, wk, bk, wv, b = p
    Q = torch.relu(x[:nd] @ wq + bq)
    K = torch.relu(x @ wk + bk)
    V = x @ wv
    A = Q.shape[1]
    d = A // H
    s = (Q[row].view(E, H, d) * K[col].view(E, H, d)).sum(-1) / np.sqrt(np.float32(d))
    m = torch.full((nd, H), -np.inf, dtype=torch.float64).index_reduce(0, row, s.detach(), "amax")
    ex = torch.exp(s - m[row])
    a = ex / (torch.zeros((nd, H), dtype=torch.float64).index_add(0, row, ex)[row] + 1e-8)
    if mult is not None:
        a = a * torch.from_numpy(mult.astype(np.float64))
    dv = V.shape[1] // H
    msg = a.unsqueeze(-1) * V[col].view(E, H, dv)
    out = torch.zeros((nd, H, dv), dtype=torch.float64).index_add(0, row, msg)
    out = out.reshape(nd, H * dv) if split else out.mean(1)
    out = out + b
    return torch.relu(out) if relu else out


def _params(rs, f, a, u, H, split):
    g = lambda i, j: (rs.rand(i, j) * 2 - 1) * np.sqrt(6.0 / (i + j))       # noqa: E731
    return [g(f, a), rs.randn(a) * .1, g(f, a), rs.randn(a) * .1, g(f, u if split else u * H), rs.randn(u) * .1]


# path: "recompute" = stats forward + tfgk_gat_bwd_*; "table" = coefficient table + tfgk_gat_softmax_bwd_f32
@pytest.mark.parametrize("fanouts,H,split,rate,path", [
    ([10, 5], 4, True, 0.0, "recompute"),
    ([6, 4, 3], 8, True, 0.0, "recompute"),
    ([10, 5], 4, False, 0.0, "table"),              # averaged heads
    ([6, 4, 3], 4, True, 0.3, "table"),             # attention dropout
    ([None, 3], 4, True, 0.0, "table"),             # a hub row: the looped CSR has a hub plan
    ([10, 5], 16, True, 0.0, "table")])             # more heads than the recompute backward packs
def test_backward_against_float64(sampler, features, fanouts, H, split, rate, path):
    L = len(fanouts)
    seeds = _seeds(128)
    b = sampler.sample_blocks(seeds, fanouts, seed=21)
    looped = [blk.with_self_loops() for blk in b.blocks]
    if fanouts[0] is None:
        assert looped[0].csr.plan is not None and looped[0].csr.plan.n_hubs > 0
    rs = np.random.RandomState(H + L)
    widths = [32] + [64] * L
    params = [_params(rs, widths[i], 64, 64, H, split) for i in range(L)]
    x = host(features[b.node_index.long()])
    gout = rs.randn(b.hop_sizes[0], 64)
    key = 1234

    def run():
        tp = [[ops.as_device(t.astype(np.float32)).requires_grad_(True) for t in p] for p in params]
        xd = ops.as_device(x).requires_grad_(True)
        h = xd
        for i, lb in enumerate(looped):
            h = tfg.nn.gat(h, lb, tp[i][0], tp[i][1], tfg.nn.relu, tp[i][2], tp[i][3], tfg.nn.relu, tp[i][4], tp[i][5],
                           tfg.nn.relu if i < L - 1 else None, num_heads=H, split_value_heads=split,
                           edge_drop_rate=rate, training=True, seed=key + i)
        (h * ops.as_device(gout.astype(np.float32))).sum().backward()
        return [h.detach()] + [t.grad for p in tp for t in p] + [xd.grad]

    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    try:
        got = run()
    finally:
        _ffi.set_trace(prev)
    recompute, table = trace.counts.get("tfgk_gat_bwd_dst_f32", 0), trace.counts.get("tfgk_gat_softmax_bwd_f32", 0)
    if path == "recompute":
        assert recompute == L and table == 0, trace.counts
    else:
        assert table >= 1, trace.counts
    again = run()
    assert all(torch.equal(u, v) for u, v in zip(got, again))          # deterministic: the same bits twice

    tp64 = [[torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in p] for p in params]
    x64 = torch.tensor(x.astype(np.float64), requires_grad=True)
    h = x64
    for i, lb in enumerate(looped):
        mult = None
        if rate > 0.0:
            mult = o.dropout_scale(lb.csr.nnz * H, rate, key + i).reshape(-1, H)
        h = _gat64(h, lb, tp64[i], H, split, i < L - 1, mult)
    (h * torch.from_numpy(gout)).sum().backward()
    want = [h.detach().numpy()] + [t.grad.numpy() for p in tp64 for t in p] + [x64.grad.numpy()]
    assert_close(host(got[0]), want[0], what="forward")
    for j, (g, w) in enumerate(zip(got[1:], want[1:])):
        assert_close(host(g), w, rtol=1e-3, atol_scale=2e-4, what="gradient {}".format(j))


# ---- host memory, learning, refusals -----------------------------------------------------------------------------

def test_host_graph_and_host_features_bit_for_bit():
    ei = random_graph(3000, 30000, seed=41, hub=(9, 3000)).astype(np.int32)
    x = torch.from_numpy(np.random.RandomState(15).randn(3000, 100).astype(np.float32))
    layers = [tfg.layers.GAT(64, num_heads=4, activation=tfg.nn.relu, seed=1, trainable=True),
              tfg.layers.GAT(16, num_heads=1, seed=2, trainable=True)]
    seeds = np.random.RandomState(16).permutation(3000)[:200].astype(np.int32)

    def run(b, x0):
        h = x0
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, blk.with_self_loops()], training=True)
        (h * h).sum().backward()
        grads = [p.grad.clone() for layer in layers for p in layer.parameters()]
        for layer in layers:
            layer.zero_grad()
        return [h.detach()] + grads

    b =tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32)).sample_blocks(seeds, [10, 5], seed=5)
    want = run(b, b.source_rows(x.cuda()))
    with tfg.utils.HostNeighborSampler(ei) as s, tfg.utils.HostFeatureTable(x) as t:
        hb = s.sample_blocks(seeds, [10, 5], seed=5)
        got = run(hb, hb.source_rows(t))
    assert all(torch.equal(u.view(torch.int32), v.view(torch.int32)) for u, v in zip(got, want))


def test_block_gat_learns_a_planted_partition():
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
    l1 = tfg.layers.GAT(64, num_heads=4, activation=tfg.nn.relu, seed=1, trainable=True)
    l2 = tfg.layers.GAT(classes, num_heads=1, seed=2, trainable=True)

    def forward(b, training):
        h = l1([b.source_rows(xd), b.blocks[0].with_self_loops()], training=training)
        return l2([h, b.blocks[1].with_self_loops()], training=training)
    with torch.no_grad():
        forward(s.sample_blocks(train[:8].astype(np.int32), [10, 10], seed=0), False)
    opt = torch.optim.Adam(list(l1.parameters()) + list(l2.parameters()), lr=0.01)
    step = 0
    for epoch in range(3):
        order = rs.permutation(train)
        for i in range(0, len(order), 512):
            seeds = order[i:i + 512].astype(np.int32)
            b = s.sample_blocks(seeds, [10, 10], seed=step)
            step += 1
            loss = torch.nn.functional.cross_entropy(forward(b, True), yd[torch.from_numpy(seeds).long().to(xd.device)])
            opt.zero_grad()
            loss.backward()
            opt.step()
    with torch.no_grad():
        h = forward(s.sample_blocks(test.astype(np.int32), [10, 10], seed=12345), False)
        acc = float((h.argmax(1).cpu().numpy() == labels[test]).mean())
    assert acc >= 0.8, acc


def test_refusals(sampler, features):
    b = sampler.sample_blocks(_seeds(64), [4, 3], seed=1)
    blk, lb = b.blocks[0], b.blocks[0].with_self_loops()
    xs = features[b.node_index.long()]
    for dt in (torch.bfloat16, torch.float8_e4m3fn):
        with pytest.raises(NotImplementedError, match="fp32"):
            tfg.layers.GAT(8, seed=1, message_dtype=dt)([xs, lb])
    with pytest.raises(ValueError, match="rows"):
        tfg.layers.GAT(8, seed=1)([xs[:-1], lb])
    with pytest.raises(ValueError, match="rows"):
        tfg.layers.GAT(8, seed=1)([b.source_rows(features), b.blocks[1].with_self_loops()])
    for fn in (lambda: tfg.layers.GAT(8)([xs, blk]), lambda: tfg.layers.GCN(8)([xs, lb]),
               lambda: tfg.layers.MeanGraphSage(8)([xs, lb]), lambda: tfg.layers.MeanPoolGraphSage(8)([xs, lb])):
        with pytest.raises(TypeError, match="block"):
            fn()
