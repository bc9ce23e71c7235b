# coding=utf-8
"""GCN on sampled blocks on the device: tfgk_block_gcn_values_f32 bit for bit against a numpy restatement for every
normalisation, with no synchronisation; with every neighbour, the block values, the aggregation (a hub row cut by the
plan included) and the layers against the full graph; the estimator's mean over fixed keys against the full graph's
aggregate; the backward against float64 autograd of a bipartite restatement within tests/train_bound.py's bound; the
host-memory routes bit for bit; learning evaluated on the full graph; the refusals."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi, _rng
from tf_geometric_b200.utils import sampling
from conftest import random_graph
import index_ref
import train_bound

pytestmark = pytest.mark.gpu

CONFIGS = [dict(), dict(improved=True), dict(renorm=False), dict(add_self_loop=False), dict(norm="left"),
           dict(norm="left", add_self_loop=False), dict(norm="right"), dict(norm="right", add_self_loop=False),
           dict(renorm=False, improved=True)]
N_NODES = 3101


def host(t):
    return t.detach().cpu().numpy()


def _graph():
    ei = random_graph(3000, 30000, seed=31, isolated=30, hub=(9, 5000))
    return np.concatenate([ei, ei[:, :500], [[3], [3100]]], axis=1).astype(np.int32)


def _weights(ei):
    return np.random.RandomState(32).rand(ei.shape[1]).astype(np.float32) + 0.05


@pytest.fixture(scope="module", params=[True, False], ids=["weighted", "unweighted"])
def graph(request):
    ei = _graph()
    w = _weights(ei) if request.param else None
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), None if w is None else ops.as_device(w))
    return s, ei, w


def _seeds(n, first=(9, 0, 3)):
    seeds = np.random.RandomState(33).permutation(3000)[:n].astype(np.int32)
    seeds[:min(n, len(first))] = first[:n]
    return seeds


def _codes(cfg):
    norm = cfg.get("norm", "both")
    loops, renorm = cfg.get("add_self_loop", True), cfg.get("renorm", True)
    fill = np.float32(2.0 if cfg.get("improved", False) else 1.0)
    deg_fill = fill if loops and (norm != "both" or renorm) else np.float32(0)
    return norm, loops, renorm, fill, deg_fill


def _restatement(blk, g_rowptr, rowsum, cfg):
    """The definition in numpy float32 (every operation correctly rounded, as the kernel's): the values of every slot of
    the block, in its looped layout with self loops."""
    norm, loops, renorm, fill, deg_fill = _codes(cfg)
    d = (rowsum + deg_fill).astype(np.float32)
    f = index_ref.deg_inv_exact(d, ops.POW_INV_SQRT if norm == "both" else ops.POW_INV)
    rp, gcol, w, dst = (host(t).astype(np.int64) if t.dtype != torch.float32 else host(t)
                        for t in (blk.csr.rowptr, blk.global_col, blk.edge_weight, blk.dst_ids))
    k = np.diff(rp[:blk.num_dst + 1])
    row = np.repeat(np.arange(blk.num_dst), k)
    g = dst[row]
    v = w.astype(np.float32)
    if norm != "right":
        v = f[g] * v
    if norm != "left":
        v = v * f[gcol]
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.diff(g_rowptr)[g].astype(np.float32) / k[row].astype(np.float32)
    v = (s * v).astype(np.float32)
    if not loops:
        return v
    out = np.empty(v.size + blk.num_dst, np.float32)
    out[np.arange(v.size) + row] = v
    fl = np.full(blk.num_dst, fill, np.float32)
    if norm != "both" or renorm:
        if norm != "right":
            fl = f[dst] * fl
        if norm != "left":
            fl = fl * f[dst]
    out[rp[1:blk.num_dst + 1] + np.arange(blk.num_dst)] = fl
    return out


BATCHES = [([15, 10, 5], False, None), ([4, 25], True, None), ([6], "head", None),
           ([None, 4], False, np.concatenate([[9], np.delete(np.arange(30), 9), [3100]]).astype(np.int32))]  # a hub,
# seeds with no in-edges, and 3100, an id with no row


@pytest.mark.parametrize("fanouts,padding,seeds", BATCHES)
def test_kernel_against_the_restatement(graph, fanouts, padding, seeds):
    s, ei, w = graph
    g_rowptr, rowsum = s._gcn_degrees()
    csr, w_csr = s._structure()
    want_rowsum = index_ref.rowsum_seq(host(csr.rowptr), host(w_csr))
    np.testing.assert_array_equal(host(rowsum)[:csr.n_rows], want_rowsum)
    assert not host(rowsum)[csr.n_rows:].any() and g_rowptr.numel() == N_NODES + 1
    b = s.sample_blocks(_seeds(256) if seeds is None else seeds, fanouts, padding=padding, seed=17)
    rp, rs = host(g_rowptr), host(rowsum)
    for blk in b.blocks:
        gb = blk.with_gcn_norm()
        for cfg in CONFIGS:
            got = host(gb.normalized(**cfg).value)
            want = _restatement(blk, rp, rs, cfg)
            assert np.array_equal(got.view(np.int32), want.view(np.int32)), (fanouts, cfg)


def test_no_synchronisation(graph):
    s, _, _ = graph
    s._gcn_degrees()
    b = s.sample_blocks(_seeds(512), [15, 10, 5], seed=3)
    x = torch.randn(b.hop_sizes[-1], 32, device="cuda")
    layers = [tfg.layers.GCN(16, seed=i) for i in range(3)]
    warm = s.sample_blocks(_seeds(64), [15, 10, 5], seed=4)            # builds the layers' weights
    with torch.no_grad():
        h = x[:warm.hop_sizes[-1]]
        for layer, blk in zip(layers, warm.blocks):
            h = layer([h, blk.with_gcn_norm()])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for blk in b.blocks:
            for cfg in CONFIGS:
                blk.with_gcn_norm().normalized(**cfg)
        with torch.no_grad():
            h = x
            for layer, blk in zip(layers, b.blocks):
                h = layer([h, blk.with_gcn_norm()])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert h.shape == (512, 16)


# ---- every neighbour: the full graph ---------------------------------------------------------------------------

def _full_adj(ei, w):
    return tfg.SparseMatrix(ops.as_device(ei, torch.int32), None if w is None else ops.as_device(w), [N_NODES, N_NODES])


def test_every_neighbour_gives_the_full_graph_bit_for_bit(graph):
    s, ei, w = graph
    seeds = np.concatenate([[9], _seeds(200)[1:]]).astype(np.int32)          # 9: a 5 000-edge hub row
    b = s.sample_blocks(seeds, [None, None], seed=4)
    h_full = torch.randn(N_NODES, 64, device="cuda")
    hubs = 0
    for cfg in CONFIGS:
        full = tfg.nn.gcn_norm_adj(_full_adj(ei, w), **cfg)
        frp, fval = host(full.csr.rowptr), host(full.value_csr)
        want_h = host(ops.spmm(full.csr, full.value_csr, h_full))
        for blk in b.blocks:
            normed = blk.with_gcn_norm().normalized(**cfg)
            dst = host(blk.dst_ids).astype(np.int64)
            want = np.concatenate([fval[frp[g]:frp[g + 1]] for g in dst])
            assert np.array_equal(host(normed.value).view(np.int32), want.view(np.int32)), cfg
            h_src = h_full[b.node_index[:blk.num_src].long()].contiguous()
            got_h = host(ops.spmm(normed.csr, normed.value_csr, h_src))
            assert np.array_equal(got_h.view(np.int32), want_h[dst].view(np.int32)), cfg
            plan = normed.csr.plan
            hubs += 0 if plan is None else plan.n_hubs
    assert hubs > 0                                      # the hub row was cut by the plan


@pytest.mark.parametrize("L", [2, 3])
@pytest.mark.parametrize("cfg", [dict(), dict(norm="left"), dict(add_self_loop=False), dict(renorm=False)],
                         ids=["default", "left", "no_loops", "no_renorm"])
def test_layers_match_the_full_graph(graph, L, cfg):
    s, ei, w = graph
    x = torch.from_numpy(np.random.RandomState(5).randn(N_NODES, 48).astype(np.float32)).cuda()
    layers = [tfg.layers.GCN(u, activation=tfg.nn.relu if i < L - 1 else None, seed=1 + i, **cfg)
              for i, u in enumerate([64, 100, 16][-L:])]
    b = s.sample_blocks(_seeds(300), [None] * L, seed=6)
    adj = _full_adj(ei, w)
    with torch.no_grad():
        h = x
        for layer in layers:
            h = layer([h, adj], cache={})
        full = host(h)[host(b.node_index[:b.hop_sizes[0]]).astype(np.int64)]
        h = b.source_rows(x)
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, blk.with_gcn_norm()])
    np.testing.assert_allclose(host(h), full, rtol=1e-5, atol=1e-5 * np.abs(full).max())


# ---- the estimator ---------------------------------------------------------------------------------------------

def test_estimator_is_unbiased_over_fixed_keys():
    rs = np.random.RandomState(71)
    n = 600
    src, dst = rs.randint(0, n, 120000), rs.randint(0, n, 120000)           # degrees near 200, fan-out 8
    ei = np.stack([src, dst]).astype(np.int32)
    w = (rs.rand(ei.shape[1]) + 0.5).astype(np.float32)
    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    seeds = np.array([0, 17, 300, 599], np.int32)
    x = torch.from_numpy(rs.randn(n, 16).astype(np.float32)).cuda()
    full = tfg.nn.gcn_norm_adj(tfg.SparseMatrix(ops.as_device(ei, torch.int32), ops.as_device(w), [n, n]),
                               add_self_loop=False)
    want = host(ops.spmm(full.csr, full.value_csr, x))[seeds].astype(np.float64)
    keys = 4096
    acc = np.zeros((seeds.size, 16))
    acc2 = np.zeros((seeds.size, 16))
    for key in range(keys):
        b = s.sample_blocks(seeds, [8], seed=key)
        blk = b.blocks[0]
        normed = blk.with_gcn_norm().normalized(add_self_loop=False)
        agg = host(ops.spmm(normed.csr, normed.value_csr, x[b.node_index.long()].contiguous())).astype(np.float64)
        acc += agg
        acc2 += agg * agg
    mean = acc / keys
    se = np.sqrt(np.maximum(acc2 / keys - mean * mean, 0.0) / keys)
    assert (se > 0).all()
    assert np.all(np.abs(mean - want) <= 4.0 * se), np.abs(mean - want).max() / se.max()


# ---- backward against float64 ----------------------------------------------------------------------------------

def _gcn64(x, adjs, params, masks, magnitude):
    """float64 bipartite GCN: act(A_i (h W_i) + b_i) over each block's values (their absolute values and the operands'
    for the magnitude run), ReLU as the fixed masks of the float32 path."""
    h = x.abs() if magnitude else x
    for i, ((row, col, val, nd), (W, b)) in enumerate(zip(adjs, params)):
        if magnitude:
            W, b, val = W.abs(), b.abs(), val.abs()
        p = h @ W
        h = torch.zeros((nd, p.shape[1]), dtype=torch.float64).index_add(0, row, val.unsqueeze(1) * p[col]) + b
        if masks[i] is not None:
            h = h * masks[i]
    return h


@pytest.mark.parametrize("fanouts,rate", [([10, 5], 0.0), ([6, 4, 3], 0.0), ([6, 4, 3], 0.3), ([None, 3], 0.0)],
                         ids=["two", "three", "dropout", "hub"])
def test_backward_against_float64(graph, monkeypatch, fanouts, rate):
    s, _, _ = graph
    L = len(fanouts)
    b = s.sample_blocks(_seeds(128), fanouts, seed=21)
    gbs = [blk.with_gcn_norm() for blk in b.blocks]
    if fanouts[0] is None:
        plan = gbs[0].normalized().csr.plan
        assert plan is not None and plan.n_hubs > 0
    rs = np.random.RandomState(L + int(rate * 10))
    widths = [32] + [64] * L
    params = [((rs.rand(widths[i], widths[i + 1]) * 2 - 1) * np.sqrt(6.0 / (widths[i] + widths[i + 1])),
               rs.randn(widths[i + 1]) * .1) for i in range(L)]
    x = rs.randn(b.hop_sizes[-1], 32)
    gout = rs.randn(b.hop_sizes[0], 64)
    dropped = []
    plain_dropout = ops.dropout

    def recording_dropout(value, *args, **kwargs):
        out = plain_dropout(value, *args, **kwargs)
        dropped.append(out)
        return out
    monkeypatch.setattr(ops, "dropout", recording_dropout)

    def run():
        del dropped[:]
        _rng.set_seed(77)                                   # the same dropout keys on both runs
        tp = [[ops.as_device(t.astype(np.float32)).requires_grad_(True) for t in p] for p in params]
        xd = ops.as_device(x.astype(np.float32)).requires_grad_(True)
        h, hs = xd, []
        for i, gb in enumerate(gbs):
            h = tfg.nn.gcn(h, gb, tp[i][0], tp[i][1], tfg.nn.relu if i < L - 1 else None, edge_drop_rate=rate,
                           training=True)
            hs.append(h.detach())
        (h * ops.as_device(gout.astype(np.float32))).sum().backward()
        return [h.detach()] + [t.grad for p in tp for t in p] + [xd.grad], hs, list(dropped)

    for gb in gbs:
        gb.normalized()
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    try:
        got, hs, values = run()
    finally:
        _ffi.set_trace(prev)
    assert trace.counts.get("tfgk_block_gcn_values_f32", 0) == 0          # made once, before: kept on the GcnBlock
    if rate == 0.0:
        values = [gb.normalized().value for gb in gbs]
    else:
        assert len(values) == L
    again, _, _ = run()
    assert all(torch.equal(u, v) for u, v in zip(got, again))           # deterministic: the same bits twice

    adjs = []
    for gb, val in zip(gbs, values):
        e = host(gb.normalized().index).astype(np.int64)
        adjs.append((torch.from_numpy(e[0]), torch.from_numpy(e[1]), torch.from_numpy(host(val).astype(np.float64)),
                     gb.num_dst))
    masks = [torch.from_numpy((host(h) > 0).astype(np.float64)) for h in hs[:-1]] + [None]
    results = []
    for magnitude in (False, True):
        tp64 = [[torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in p] for p in params]
        x64 = torch.tensor(x, dtype=torch.float64, requires_grad=True)
        h = _gcn64(x64, adjs, tp64, masks, magnitude)
        g = torch.from_numpy(np.abs(gout) if magnitude else gout)
        (h * g).sum().backward()
        results.append([h.detach().numpy()] + [t.grad.numpy() for p in tp64 for t in p] + [x64.grad.numpy()])
    want, S = results[0], [np.abs(m) for m in results[1]]          # |d/dt| of |t|: the sign of t drops out
    # longest chains: every stage's reduction (the block's longest row forward, its longest column backward, the
    # column sums over the rows) plus one K4 product per layer forward and two backward
    c = 0
    for gb in gbs:
        normed = gb.normalized()
        c += int(host(normed.csr.degree_i64()).max()) + int(host(normed._transposed_csr().degree_i64()).max()) + \
            gb.num_src + 4
    e = train_bound.eps(c, *([max(widths)] * (3 * L)))
    for j, (gt, w64, s64) in enumerate(zip(got, want, S)):
        r = train_bound.ratio(host(gt), w64, s64, e)
        assert r <= 1.0, ("output" if j == 0 else "gradient {}".format(j), r,
                          train_bound.worst_entry(host(gt), w64, s64, e))


# ---- host memory, learning, refusals -----------------------------------------------------------------------------

def test_host_sampler_degrees_and_routes_bit_for_bit():
    from test_gpu_host_sampler import _device_bytes
    # the hub graph in one range, and a graph without a hub cut into about ten ranges
    for ei, ranged in ((_graph(), False), (random_graph(3000, 30000, seed=35).astype(np.int32), True)):
        w = _weights(ei)
        for weighted in (True, False):
            dev = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w) if weighted else None)
            want_rp, want_rs = dev._gcn_degrees()
            device_bytes = None
            if ranged:
                edge_bytes = sampling.HOST_CSR_EDGE_BYTES if weighted else sampling.HOST_CSR_EDGE_BYTES_UNWEIGHTED
                n = int(ei.max()) + 1
                device_bytes = _device_bytes(ei, (edge_bytes * ei.shape[1] + sampling.HOST_CSR_ROW_BYTES * (n + 1)) // 10
                                             + 1000)
            with tfg.utils.HostNeighborSampler(ei, w if weighted else None, device_bytes=device_bytes) as hs:
                assert 9 <= len(hs._ranges) <= 12 if ranged else len(hs._ranges) == 1, len(hs._ranges)
                assert torch.equal(hs.rowptr, want_rp)
                assert torch.equal(hs.rowsum.view(torch.int32), want_rs.view(torch.int32))
    ei = _graph()
    w = _weights(ei)
    x = torch.from_numpy(np.random.RandomState(15).randn(N_NODES, 100).astype(np.float32))
    layers = [tfg.layers.GCN(64, activation=tfg.nn.relu, seed=1, trainable=True),
              tfg.layers.GCN(16, seed=2, trainable=True)]
    seeds = np.random.RandomState(16).permutation(3000)[:200].astype(np.int32)
    seeds[0] = 9

    def run(b, x0):
        h = x0
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, blk.with_gcn_norm()], training=True)
        (h * h).sum().backward()
        grads = [p.grad.clone() for layer in layers for p in layer.parameters()]
        for layer in layers:
            layer.zero_grad()
        return [h.detach()] + grads

    s = tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32), ops.as_device(w))
    b = s.sample_blocks(seeds, [10, 5], seed=5)
    want = run(b, b.source_rows(x.cuda()))
    with tfg.utils.HostNeighborSampler(ei, w) as hs, tfg.utils.HostFeatureTable(x) as t:
        hb = hs.sample_blocks(seeds, [10, 5], seed=5)
        got = run(hb, hb.source_rows(t))
    assert all(torch.equal(u.view(torch.int32), v.view(torch.int32)) for u, v in zip(got, want))


def test_block_gcn_learns_a_planted_partition_evaluated_on_the_full_graph():
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
    eid = ops.as_device(ei, torch.int32)
    s = tfg.utils.RandomNeighborSampler(eid)
    l1 = tfg.layers.GCN(64, activation=tfg.nn.relu, seed=1, trainable=True)
    l2 = tfg.layers.GCN(classes, seed=2, trainable=True)

    def forward(b, training):
        h = l1([b.source_rows(xd), b.blocks[0].with_gcn_norm()], training=training)
        return l2([h, b.blocks[1].with_gcn_norm()], training=training)
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
    with torch.no_grad():                                  # the same weights on the full graph
        cache = {}
        h = l2([l1([xd, eid], cache=cache), eid], cache=cache)
        acc = float((h.argmax(1).cpu().numpy()[test] == labels[test]).mean())
    assert acc >= 0.8, acc


def test_refusals(graph):
    s, _, _ = graph
    x_all = torch.randn(N_NODES, 12, device="cuda")
    b = s.sample_blocks(_seeds(64), [4, 3], seed=1)
    blk = b.blocks[0]
    gb, gb1 = blk.with_gcn_norm(), b.blocks[1].with_gcn_norm()
    xs = x_all[b.node_index.long()].contiguous()
    lb = blk.with_self_loops()
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    try:
        for dt in (torch.bfloat16, torch.float8_e4m3fn):
            with pytest.raises(NotImplementedError, match="fp32"):
                tfg.layers.GCN(8, seed=1, message_dtype=dt)([xs, gb])
        with pytest.raises(NotImplementedError):
            tfg.nn.gcn(xs.to_sparse(), gb, torch.ones(12, 4, device="cuda"))
        with pytest.raises(NotImplementedError, match="sym"):
            tfg.layers.GCN(8, seed=1, sym=False)([xs, gb])
        with pytest.raises(ValueError, match="rows"):
            tfg.layers.GCN(8, seed=1)([xs[:-1], gb])
        with pytest.raises(ValueError, match="rows"):
            tfg.layers.GCN(8, seed=1)([b.source_rows(x_all), gb1])
        with pytest.raises(ValueError, match="carries"):
            tfg.layers.GCN(8, seed=1)([xs, gb, torch.ones(blk.edge_index.shape[1], device="cuda")])
        with pytest.raises(NotImplementedError, match="edge-weight"):
            tfg.layers.GCN(8, seed=1)([xs, gb, torch.ones(blk.edge_index.shape[1], device="cuda", requires_grad=True)])
        for fn in (lambda: tfg.layers.GCN(8)([xs, blk]), lambda: tfg.layers.GCN(8)([xs, lb]),
                   lambda: tfg.layers.GAT(8)([xs, gb]), lambda: tfg.layers.MeanGraphSage(8)([xs, gb]),
                   lambda: tfg.layers.SGC(8)([xs, gb])):
            with pytest.raises(TypeError, match="with_gcn_norm"):
                fn()
    finally:
        _ffi.set_trace(prev)
    assert not trace.counts, trace.counts                # no device work before any refusal
