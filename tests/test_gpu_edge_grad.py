# coding=utf-8
"""Gradients with respect to edge weights on the H100: K7 (tfgk_sddmm_csr_f32) against float64, bit-stability of K7
across runs, task splits and output orders; edge-weight gradients of NeighborAggregate, SparseMatmul and gcn_norm_adj
(every normalisation, with edge dropout) and of every convolution that takes edge weights, against float64 torch autograd
over the reference's op sequence; caching, in-place optimizer steps, and an edge mask learned end to end."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, autograd, _structure
from tf_geometric_b200.sparse import SparseMatrix
from tf_geometric_b200.nn.conv import graph_sage as gs
from conftest import random_graph, assert_close, glorot
import edge_grad_ref as ref

pytestmark = pytest.mark.gpu


def dev(a, dtype=None):
    return ops.as_device(a, dtype)


def host(t):
    return t.detach().cpu().numpy()


def _i64(a):
    return torch.tensor(np.asarray(a), dtype=torch.int64)


def _bits(t):
    return host(t).view(np.uint32)


# ---- K7 ---------------------------------------------------------------------------------------------------------------

def _k7_graph(n, seed, hub_degree=0):
    """Random edges with empty rows, self loops, duplicate edges and optionally one hub row."""
    ei = random_graph(n, 8 * n, seed=seed, isolated=3, hub=(n // 2, hub_degree) if hub_degree else None)
    extra = np.array([[7, 7, 9, 9, 9], [7, 7, 1, 1, 9]], np.int32)                   # loops and duplicates
    return np.concatenate([ei, extra, ei[:, :11]], axis=1).astype(np.int32)


def _k7_ref(ei, csr_perm, G, X, scale, alpha):
    """float64 out[e] for every edge e of the list (edge order)."""
    row, col = ei[0].astype(np.int64), ei[1].astype(np.int64)
    s = (G[row].astype(np.float64) * X[col].astype(np.float64)).sum(-1) * alpha
    return s * (1.0 if scale is None else scale[row].astype(np.float64))


@pytest.mark.parametrize("D", [1, 3, 16, 64, 100, 128, 256, 600])
@pytest.mark.parametrize("layout", ["plain", "slice"])
def test_k7_matches_float64(D, layout):
    rs = np.random.RandomState(D)
    n = 3000
    ei = _k7_graph(n, seed=D)
    eid = dev(ei)
    csr, _ = _structure.csr_for_edge_index(eid, n)
    if layout == "plain":
        Gb, Xb = rs.randn(n, D).astype(np.float32), rs.randn(n, D).astype(np.float32)
        Gd, Xd = dev(Gb), dev(Xb)
        G, X = Gb, Xb
    else:                                    # column slices of wider tensors: odd leading dimensions, unaligned starts
        Gb, Xb = rs.randn(n, D + 7).astype(np.float32), rs.randn(n, D + 5).astype(np.float32)
        Gd, Xd = dev(Gb)[:, 3:3 + D], dev(Xb)[:, 1:1 + D]
        G, X = Gb[:, 3:3 + D], Xb[:, 1:1 + D]
    cnt = np.bincount(ei[0], minlength=n)
    scale = (1.0 / np.maximum(cnt, 1)).astype(np.float32)
    for row_scale, alpha in ((None, 1.0), (scale, -0.75)):
        want = _k7_ref(ei, None, G, X, row_scale, alpha)
        got = ops.sddmm_csr(csr, Gd, Xd, row_scale=None if row_scale is None else dev(row_scale), alpha=alpha)
        assert_close(host(got), want, what="K7 D={} {} edge order".format(D, layout))
        got_csr = ops.sddmm_csr(csr, Gd, Xd, row_scale=None if row_scale is None else dev(row_scale), alpha=alpha,
                                edge_order=False)
        # CSR order permuted afterwards gives the same bits as perm written directly
        np.testing.assert_array_equal(_bits(ops.permute(got_csr, csr.perm, inverse=True)), _bits(got))


@pytest.mark.parametrize("D", [16, 100, 128])
def test_k7_bits_do_not_depend_on_the_split(D, monkeypatch):
    rs = np.random.RandomState(5)
    n = 4000
    ei = _k7_graph(n, seed=1, hub_degree=50000)
    eid = dev(ei)
    csr, _ = _structure.csr_for_edge_index(eid, n)
    G, X = dev(rs.randn(n, D).astype(np.float32)), dev(rs.randn(n, D).astype(np.float32))
    scale = dev(rs.rand(n).astype(np.float32))
    first = ops.sddmm_csr(csr, G, X, row_scale=scale)
    again = ops.sddmm_csr(csr, G, X, row_scale=scale)
    np.testing.assert_array_equal(_bits(first), _bits(again))
    assert_close(host(first), _k7_ref(ei, None, host(G), host(X), host(scale), 1.0), what="K7 with a 50 000-edge hub")
    for task_edges in ("1073741824", "33", "4096"):            # one task (no row split), tiny tasks, hub-sized tasks
        monkeypatch.setenv("TFGK_SDDMM_TASK_EDGES", task_edges)
        np.testing.assert_array_equal(_bits(ops.sddmm_csr(csr, G, X, row_scale=scale)), _bits(first))


# ---- building blocks ----------------------------------------------------------------------------------------------

def _graph(n, seed, e=None):
    rs = np.random.RandomState(seed)
    ei = random_graph(n, e or 8 * n, seed=seed, symmetric=True, isolated=2)
    ei = np.concatenate([ei, [[5, 5, 7], [5, 5, 7]], ei[:, :3]], axis=1).astype(np.int32)
    w = (rs.rand(ei.shape[1]) + 0.2).astype(np.float32)
    return rs, ei, w


@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_neighbor_aggregate_edge_gradient(reduce):
    rs, ei, w = _graph(2000, 1)
    n, d = 2000, 48
    x = rs.randn(n, d).astype(np.float32)
    g = rs.randn(n, d)
    wt, xt = dev(w).requires_grad_(True), dev(x).requires_grad_(True)
    y = autograd.NeighborAggregate.apply(xt, dev(ei), wt, reduce, n)
    (y * dev(g.astype(np.float32))).sum().backward()
    w64, x64 = ref.t64(w, True), ref.t64(x, True)
    (ref.aggregate(_i64(ei[0]), _i64(ei[1]), w64, x64, n, reduce) * torch.tensor(g)).sum().backward()
    assert_close(host(wt.grad), w64.grad.numpy(), what="d w " + reduce)
    assert_close(host(xt.grad), x64.grad.numpy(), what="d x " + reduce)


def test_sparse_matmul_value_gradient_with_relu_and_bias():
    rs, ei, w = _graph(1500, 2)
    n, d = 1500, 32
    h, b = rs.randn(n, d).astype(np.float32), rs.randn(d).astype(np.float32)
    wt, ht, bt = (dev(a).requires_grad_(True) for a in (w, h, b))
    y = SparseMatrix(dev(ei), wt, [n, n]).matmul(ht, bias=bt, act=ops.ACT_RELU)
    g = rs.randn(n, d)
    (y * dev(g.astype(np.float32))).sum().backward()
    w64, h64, b64 = ref.t64(w, True), ref.t64(h, True), ref.t64(b, True)
    (torch.relu(ref.spmm(_i64(ei[0]), _i64(ei[1]), w64, h64, n) + b64) * torch.tensor(g)).sum().backward()
    for name, mine, want in (("value", wt, w64), ("h", ht, h64), ("bias", bt, b64)):
        assert_close(host(mine.grad), want.grad.numpy(), what="A @ h: d " + name)
    # A @ h with only A's values trainable
    w2 = dev(w).requires_grad_(True)
    (SparseMatrix(dev(ei), w2, [n, n]) @ dev(h)).sum().backward()
    w64b = ref.t64(w, True)
    ref.spmm(_i64(ei[0]), _i64(ei[1]), w64b, ref.t64(h), n).sum().backward()
    assert_close(host(w2.grad), w64b.grad.numpy(), what="A @ h: d value only")


def _dropout_multiplier(nnz, rate, seed):
    """The kept / dropped pattern of tfgk_dropout_f32 for (seed, entry), times 1 / (1 - rate), in float64."""
    kept = host(ops.dropout(torch.ones(nnz, dtype=torch.float32, device="cuda"), rate, seed)) != 0
    return torch.tensor(kept.astype(np.float64) / (1.0 - rate))


@pytest.mark.parametrize("combo", ref.NORM_COMBOS, ids=lambda c: "-".join(map(str, c)))
def test_gcn_norm_adj_edge_gradient_with_edge_dropout(combo):
    norm, loop, sym, renorm, improved = combo
    rs, ei, w = _graph(1200, 3)
    n = 1200
    wt = dev(w).requires_grad_(True)
    normed = tfg.nn.gcn_norm_adj(SparseMatrix(dev(ei), wt, [n, n]), norm, loop, sym, renorm, improved)
    plain = tfg.nn.gcn_norm_adj(SparseMatrix(dev(ei), dev(w), [n, n]), norm, loop, sym, renorm, improved)
    np.testing.assert_array_equal(_bits(normed.value), _bits(plain.value))            # requires_grad changes no bit
    dropped = normed.dropout(0.3, training=True, seed=77)
    np.testing.assert_array_equal(_bits(dropped.value), _bits(plain.dropout(0.3, training=True, seed=77).value))
    x = rs.randn(n, 8).astype(np.float32)
    g = rs.randn(n, 8)
    (dropped.matmul(dev(x)) * dev(g.astype(np.float32))).sum().backward()
    w64 = ref.t64(w, True)
    r, c, v = ref.gcn_norm(_i64(ei[0]), _i64(ei[1]), w64, [n, n], norm, loop, sym, renorm, improved)
    v = v * _dropout_multiplier(v.shape[0], 0.3, 77)
    (ref.spmm(r, c, v, ref.t64(x), n) * torch.tensor(g)).sum().backward()
    assert np.all(np.isfinite(host(wt.grad)))
    assert_close(host(wt.grad), w64.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what="d w {}".format(combo))


# ---- convolutions and layers ----------------------------------------------------------------------------------------

N, F, U = 700, 12, 8


def _conv(name, rs, ei):
    """(mine(x, edge_index, w, params), ref64(x, w, params), params) for one convolution, functional or layer."""
    r, c = _i64(ei[0]), _i64(ei[1])
    n = N

    def norm64(w, renorm=True):
        return ref.gcn_norm(r, c, w, [n, n], renorm=renorm)

    if name in ("gcn", "gcn_sparse_x", "GCN"):
        P = dict(k=glorot(rs, F, U), b=rs.randn(U).astype(np.float32))

        def want(x, w, p):
            nr, nc, nv = norm64(w)
            return torch.relu(ref.spmm(nr, nc, nv, x @ p["k"], n) + p["b"])
        if name == "gcn":
            mine = lambda x, e, w, p: tfg.nn.gcn(x, SparseMatrix(e, w, [n, n]), p["k"], p["b"], tfg.nn.relu)  # noqa: E731
        elif name == "gcn_sparse_x":
            def mine(x, e, w, p):
                xs = SparseMatrix(torch.nonzero(x).t().to(torch.int32).contiguous(), x[x != 0], list(x.shape))
                return tfg.nn.gcn(xs, SparseMatrix(e, w, [n, n]), p["k"], p["b"], tfg.nn.relu)
        else:
            mine = ("layer", lambda: tfg.layers.GCN(U, activation=tfg.nn.relu, trainable=True), {"kernel": "k", "bias": "b"})
    elif name in ("appnp", "APPNP"):
        P = dict(k0=glorot(rs, F, 16), b0=rs.randn(16).astype(np.float32), k1=glorot(rs, 16, U),
                 b1=rs.randn(U).astype(np.float32))

        def want(x, w, p):
            nr, nc, nv = norm64(w)
            h = torch.relu(x @ p["k0"] + p["b0"]) @ p["k1"] + p["b1"]
            out = h
            for _ in range(3):
                out = ref.spmm(nr, nc, nv, out, n) * (1.0 - 0.2) + h * 0.2
            return out
        if name == "appnp":
            mine = lambda x, e, w, p: tfg.nn.appnp(x, e, w, [p["k0"], p["k1"]], [p["b0"], p["b1"]], k=3, alpha=0.2)  # noqa
        else:
            mine = ("layer", lambda: tfg.layers.APPNP([16, U], k=3, alpha=0.2, trainable=True),
                    {"kernel_0": "k0", "bias_0": "b0", "kernel_1": "k1", "bias_1": "b1"})
    elif name in ("sgc", "SGC"):
        P = dict(k=glorot(rs, F, U), b=rs.randn(U).astype(np.float32))

        def want(x, w, p):
            nr, nc, nv = norm64(w)
            return ref.spmm(nr, nc, nv, ref.spmm(nr, nc, nv, x @ p["k"], n), n) + p["b"]
        mine = (lambda x, e, w, p: tfg.nn.sgc(x, e, w, 2, p["k"], p["b"])) if name == "sgc" else \
            ("layer", lambda: tfg.layers.SGC(U, k=2, trainable=True), {"kernel": "k", "bias": "b"})
    elif name in ("ssgc", "SSGC"):
        P = dict(k0=glorot(rs, F, U), b0=rs.randn(U).astype(np.float32))

        def want(x, w, p):
            nr, nc, nv = norm64(w)
            h = x @ p["k0"] + p["b0"]
            out = h * 0.2
            for _ in range(3):
                h = ref.spmm(nr, nc, nv, h, n)
                out = out + (1 - 0.2) * h / 3
            return out
        mine = (lambda x, e, w, p: tfg.nn.ssgc(x, e, w, [p["k0"]], [p["b0"]], k=3, alpha=0.2)) if name == "ssgc" else \
            ("layer", lambda: tfg.layers.SSGC([U], k=3, alpha=0.2, trainable=True), {"kernel_0": "k0", "bias_0": "b0"})
    elif name in ("tagcn", "TAGCN"):
        P = dict(k=glorot(rs, 3 * F, U), b=rs.randn(U).astype(np.float32))

        def want(x, w, p):
            nr, nc, nv = norm64(w, renorm=False)
            a1 = ref.spmm(nr, nc, nv, x, n)
            return torch.cat([x, a1, ref.spmm(nr, nc, nv, a1, n)], 1) @ p["k"] + p["b"]
        mine = (lambda x, e, w, p: tfg.nn.tagcn(x, e, w, 2, p["k"], p["b"])) if name == "tagcn" else \
            ("layer", lambda: tfg.layers.TAGCN(U, k=2, trainable=True), {"kernel": "k", "bias": "b"})
    elif name in ("le_conv", "LEConv"):
        P = {k: glorot(rs, F, U) for k in ("ws", "wa", "wn")}
        P.update(bs=rs.randn(U).astype(np.float32), ba=rs.randn(U).astype(np.float32))

        def want(x, w, p):
            return torch.relu(ref.spmm(r, c, w, (x @ p["wa"] + p["ba"]) - x @ p["wn"], n) + x @ p["ws"] + p["bs"])
        mine = (lambda x, e, w, p: tfg.nn.le_conv(x, e, w, p["ws"], p["bs"], p["wa"], p["ba"], p["wn"], None,
                                                  tfg.nn.relu)) if name == "le_conv" else \
            ("layer", lambda: tfg.layers.LEConv(U, activation=tfg.nn.relu, trainable=True),
             {"self_kernel": "ws", "self_bias": "bs", "aggr_self_kernel": "wa", "aggr_self_bias": "ba",
              "aggr_neighbor_kernel": "wn"})
    else:
        reduce = "mean" if name in ("mean_graph_sage", "MeanGraphSage") else "sum"
        P = dict(ws=glorot(rs, F, U // 2), wn=glorot(rs, F, U // 2), b=rs.randn(U).astype(np.float32))

        def want(x, w, p):
            return torch.relu(torch.cat([x @ p["ws"], ref.aggregate(r, c, w, x, n, reduce) @ p["wn"]], 1) + p["b"])
        if name.endswith("_graph_sage"):
            fn = getattr(tfg.nn, name)
            mine = lambda x, e, w, p: fn(x, e, w, p["ws"], p["wn"], p["b"], tfg.nn.relu)    # noqa: E731
        else:
            cls = getattr(tfg.layers, name)
            mine = ("layer", lambda: cls(U, trainable=True), {"self_kernel": "ws", "neighbor_kernel": "wn", "bias": "b"})
    return mine, want, P


CONVS = ["gcn", "gcn_sparse_x", "appnp", "sgc", "ssgc", "tagcn", "le_conv", "mean_graph_sage", "sum_graph_sage",
         "GCN", "APPNP", "SGC", "SSGC", "TAGCN", "LEConv", "MeanGraphSage", "SumGraphSage"]


@pytest.mark.parametrize("name", CONVS)
def test_convolution_edge_gradient_and_unchanged_bits(name):
    rs, ei, w = _graph(N, sum(map(ord, name)))
    x = rs.randn(N, F).astype(np.float32)
    if name == "gcn_sparse_x":
        x[rs.rand(N, F) < 0.6] = 0.0
    mine, want, P = _conv(name, rs, ei)
    eid = dev(ei)
    is_layer = isinstance(mine, tuple)

    def run(w_grad):
        tp = {k: dev(v) for k, v in P.items()}
        xd = dev(x)
        if not is_layer:
            for t in tp.values():
                t.requires_grad_(True)
            if name != "gcn_sparse_x":
                xd.requires_grad_(True)
        wd = dev(w).requires_grad_(w_grad)
        if is_layer:
            _, make, names = mine
            layer = make()
            layer([xd, eid, wd])                                              # builds the weights
            with torch.no_grad():
                for pname, key in names.items():
                    getattr(layer, pname).copy_(tp[key])
            y = layer([xd, eid, wd], training=True)
            params = {names[k]: v for k, v in layer.named_parameters() if k in names}
        else:
            y = mine(xd, eid, wd, tp)
            params = tp
        return y, xd, wd, params

    y0, x0, w0, p0 = run(False)
    y1, x1, w1, p1 = run(True)
    g = rs.randn(*y1.shape).astype(np.float32)
    (y0 * dev(g)).sum().backward()
    (y1 * dev(g)).sum().backward()
    # the forward and every other gradient are the bits of the same call without a trainable edge weight ...
    if name.lower().endswith("graphsage") or name.endswith("_graph_sage"):
        # ... of the route the SAGE variants take when the edge weights require grad (NeighborAggregate + Dense),
        # which is what they computed before this change
        reduce = "mean" if "mean" in name.lower() else "sum"
        tp = {k: dev(v).requires_grad_(True) for k, v in P.items()}
        xr = dev(x).requires_grad_(True)
        agg = autograd.NeighborAggregate.apply(xr, eid, dev(w), reduce, N)
        y0 = gs._project_pair_autograd(xr, agg, tp["ws"], tp["wn"], tp["b"], tfg.nn.relu, True, False)
        (y0 * dev(g)).sum().backward()
        x0, p0 = xr, tp
    np.testing.assert_array_equal(_bits(y1), _bits(y0))
    if x1.requires_grad:
        np.testing.assert_array_equal(_bits(x1.grad), _bits(x0.grad))
    for k in p1:
        np.testing.assert_array_equal(_bits(p1[k].grad), _bits(p0[k].grad), err_msg=k)
    assert w0.grad is None
    # ... and d edge_weight matches float64 autograd over the reference's op sequence
    w64 = ref.t64(w, True)
    y64 = want(ref.t64(x), w64, {k: ref.t64(v) for k, v in P.items()})
    assert_close(host(y1), y64.detach().numpy(), what=name + " forward")
    (y64 * torch.tensor(g.astype(np.float64))).sum().backward()
    assert_close(host(w1.grad), w64.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what=name + " d edge_weight")


@pytest.mark.parametrize("name", ["gcn", "mean_graph_sage", "appnp"])
def test_edge_gradients_are_deterministic(name):
    rs = np.random.RandomState(2)
    n = 6000
    ei = random_graph(n, 60000, seed=4, symmetric=True, hub=(17, 9000))
    ei = np.concatenate([ei, ei[::-1]], axis=1).astype(np.int32)
    w = (rs.rand(ei.shape[1]) + 0.1).astype(np.float32)
    x = dev(rs.randn(n, 64).astype(np.float32))
    k = dev(glorot(rs, 64, 32))
    eid = dev(ei)
    grads = []
    for _ in range(2):
        wd = dev(w).requires_grad_(True)
        if name == "gcn":
            y = tfg.nn.gcn(x, SparseMatrix(eid, wd, [n, n]), k, None, tfg.nn.relu)
        elif name == "appnp":
            y = tfg.nn.appnp(x, eid, wd, [k], [None], k=4)
        else:
            y = tfg.nn.mean_graph_sage(x, eid, wd, k, k, None, tfg.nn.relu)
        (y * y).sum().backward()
        grads.append(_bits(wd.grad))
    np.testing.assert_array_equal(grads[0], grads[1])


def test_warm_cache_gives_no_edge_gradient():
    rs, ei, w = _graph(N, 5)
    graph = tfg.Graph(rs.randn(N, F).astype(np.float32), ei, w).to_device()
    layer = tfg.layers.GCN(U, activation=tfg.nn.relu, trainable=True, seed=3)
    layer.build_cache_for_graph(graph)
    wd = dev(w).requires_grad_(True)
    y = layer([graph.x, graph.edge_index, wd], cache=graph.cache, training=True)
    y.sum().backward()
    assert wd.grad is None                         # the reference's cached normalisation is a constant too
    assert layer.kernel.grad is not None
    cold = dev(w).requires_grad_(True)
    layer([graph.x, graph.edge_index, cold], training=True).sum().backward()
    assert cold.grad is not None and torch.isfinite(cold.grad).all()


@pytest.mark.parametrize("name", ["gcn", "mean_graph_sage", "le_conv"])
def test_optimizer_steps_reach_the_next_forward(name):
    rs, ei, w = _graph(N, 8)
    x = dev(rs.randn(N, F).astype(np.float32))
    eid = dev(ei)
    ws, wn = dev(glorot(rs, F, U)), dev(glorot(rs, F, U))
    wd = dev(w).requires_grad_(True)
    kd = dev(glorot(rs, F, U)).requires_grad_(True)
    opt = torch.optim.SGD([wd, kd], lr=0.5)

    def forward(weights):
        if name == "gcn":
            return tfg.nn.gcn(x, SparseMatrix(eid, weights, [N, N]), kd, None, tfg.nn.relu)
        if name == "le_conv":
            return tfg.nn.le_conv(x, eid, weights, kd, None, ws, None, wn, None, tfg.nn.relu)
        return tfg.nn.mean_graph_sage(x, eid, weights, kd, wn, None, tfg.nn.relu)

    for _ in range(2):
        opt.zero_grad()
        y = forward(wd)
        (y * y).mean().backward()
        opt.step()                                              # in place: bumps the weight tensor's version
    with torch.no_grad():
        after = forward(wd)
        fresh = forward(wd.detach().clone())                    # a new tensor: nothing memoised for it
    np.testing.assert_array_equal(_bits(after), _bits(fresh))
    with torch.no_grad():
        stale = forward(dev(w))
    assert not np.array_equal(_bits(after), _bits(stale))


# ---- end to end: an edge mask learned with a GCN ------------------------------------------------------------------

def _auc(score, label):
    order = np.argsort(score, kind="stable")
    ranks = np.empty(len(score))
    ranks[order] = np.arange(1, len(score) + 1)
    pos = label.sum()
    neg = len(label) - pos
    return (ranks[label].sum() - pos * (pos + 1) / 2) / (pos * neg)


def learn_edge_mask(steps=150, seed=0):
    """Planted partition (2000 nodes, 4 communities, ~8 intra and ~4 inter edges per node), noisy features, a 2-layer GCN
    trained jointly with one logit per undirected pair; returns the ROC-AUC of the learned weights, intra vs inter."""
    rs = np.random.RandomState(seed)
    n, k, f, hidden = 2000, 4, 16, 32
    y = rs.randint(0, k, n)
    u, v = rs.randint(0, n, 4 * 8000), rs.randint(0, n, 4 * 8000)
    keep = (y[u] == y[v]) & (u < v)
    u, v = u[keep][:8000], v[keep][:8000]
    a, b = rs.randint(0, n, 4 * 4000), rs.randint(0, n, 4 * 4000)
    keep = (y[a] != y[b]) & (a < b)
    a, b = a[keep][:4000], b[keep][:4000]
    src, dst = np.concatenate([u, a]), np.concatenate([v, b])
    intra = np.concatenate([np.ones(len(u), bool), np.zeros(len(a), bool)])
    pairs = len(src)
    ei = dev(np.stack([np.concatenate([src, dst]), np.concatenate([dst, src])]).astype(np.int32))
    pair_of_edge = dev(np.concatenate([np.arange(pairs), np.arange(pairs)]), torch.int64)
    x = rs.randn(n, f).astype(np.float32)
    x[np.arange(n), y] += 1.0
    x, labels = dev(x), dev(y, torch.int64)
    theta = torch.zeros(pairs, dtype=torch.float32, device="cuda", requires_grad=True)
    w1 = dev(rs.randn(f, hidden).astype(np.float32) * 0.3).requires_grad_(True)
    w2 = dev(rs.randn(hidden, k).astype(np.float32) * 0.3).requires_grad_(True)
    opt = torch.optim.Adam([{"params": [theta], "lr": 0.1}, {"params": [w1, w2], "lr": 0.01, "weight_decay": 0.05}])
    for _ in range(steps):
        w = torch.sigmoid(theta)[pair_of_edge]
        adj = SparseMatrix(ei, w, [n, n])
        h = tfg.nn.gcn(x, adj, w1, None, tfg.nn.relu)
        out = tfg.nn.gcn(h, adj, w2, None)
        loss = torch.nn.functional.cross_entropy(out, labels)
        opt.zero_grad()
        loss.backward()
        opt.step()
    return _auc(host(theta).astype(np.float64), intra)


def test_learned_edge_mask_separates_communities():
    auc = learn_edge_mask()
    print("edge-mask ROC-AUC after 150 steps: {:.4f}".format(auc))
    assert auc > 0.85
