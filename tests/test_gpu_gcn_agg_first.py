# coding=utf-8
"""Aggregate, then project (tfgk_spmm_proj_f32) on the H100: every aggregate bit-identical to tfgk_spmm_f32's, every
output within ((deg_r + F + 1) 2^-24 + tiny) S_rj of float64, where S_rj = sum_k sum_e |w_e| |x[col_e, k]| |W_kj| + |b_j|,
and the GCN inference layers that take the route."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from conftest import random_graph, assert_close

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24


def _csr(ei, n):
    ei = torch.as_tensor(ei, device="cuda")
    return ops.csr_build(ei[0].contiguous(), ei[1].contiguous(), n)


def _host_csr(csr):
    return csr.rowptr.cpu().numpy(), csr.col.cpu().numpy()


def _within_bound(got, csr, w_csr, x, W, b, rows=None, act_relu=False):
    """got (pre- or post-relu) against float64, rows = None for all rows."""
    rowptr, col = _host_csr(csr)
    w = np.ones(len(col)) if w_csr is None else w_csr.cpu().numpy().astype(np.float64)
    xh, Wh = x.cpu().numpy().astype(np.float64), W.cpu().numpy().astype(np.float64)
    bh = np.zeros(W.shape[1]) if b is None else b.cpu().numpy().astype(np.float64)
    rows = np.arange(len(rowptr) - 1) if rows is None else rows
    got = got.cpu().numpy()[rows].astype(np.float64)
    for i, r in enumerate(rows):
        e0, e1 = rowptr[r], rowptr[r + 1]
        agg = (w[e0:e1, None] * xh[col[e0:e1]]).sum(0)
        agg_abs = (np.abs(w[e0:e1, None]) * np.abs(xh[col[e0:e1]])).sum(0)
        want = agg @ Wh + bh
        if act_relu:
            want = np.maximum(want, 0.0)
        S = agg_abs @ np.abs(Wh) + np.abs(bh)
        bound = ((e1 - e0 + x.shape[1] + 1) * U24) * S + 1e-30
        err = np.abs(got[i] - want)
        assert np.all(err <= bound), "row {} (deg {}): err {} > bound {}".format(r, e1 - e0, err.max(),
                                                                             bound[np.argmax(err - bound)])


def _case(n=3000, e=45000, seed=5, hub=(42, 1900), F=100, U=128, weighted=True, isolated=7):
    ei = random_graph(n, e, seed, isolated=isolated, hub=hub)
    csr = _csr(ei, n)
    rs = np.random.RandomState(seed)
    w = torch.tensor(rs.rand(csr.nnz).astype(np.float32) + 0.1, device="cuda") if weighted else None
    x = torch.tensor(rs.randn(n, F).astype(np.float32), device="cuda")
    W = torch.tensor((rs.randn(F, U) / np.sqrt(F)).astype(np.float32), device="cuda")
    b = torch.tensor(rs.randn(U).astype(np.float32), device="cuda")
    return csr, w, x, W, b


def _traced(fn):
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    try:
        out = fn()
    finally:
        _ffi.set_trace(prev)
    return out, trace


def _bits(a):
    return a.contiguous().view(torch.int32)


@pytest.mark.parametrize("F", [4, 32, 100, 124])
@pytest.mark.parametrize("hub", [(42, 1900), (42, 60000)], ids=["no_plan", "hub_plan"])
def test_aggregate_bit_identical_to_spmm(F, hub):
    """W = [I | 0] and x >= 0: the first F outputs are the aggregates, exactly (hub rows through the plan for F >= 32)."""
    csr, w, x, _, _ = _case(n=4000, e=60000, hub=hub, F=F, U=F + 4)
    x = x.abs()
    W = torch.zeros((F, F + 4), device="cuda")
    W[:, :F] = torch.eye(F, device="cuda")
    got = ops.spmm_proj(csr, w, x, W)
    want = ops.spmm(csr, w, x)
    assert torch.equal(_bits(got[:, :F]), _bits(want))
    assert torch.equal(got[:, F:], torch.zeros_like(got[:, F:]))


@pytest.mark.parametrize("F", [4, 12, 64, 100, 124])
@pytest.mark.parametrize("u_plus", [4, None], ids=["U=F+4", "U=128"])
@pytest.mark.parametrize("bias,relu", [(False, False), (True, False), (True, True)], ids=["plain", "bias", "bias_relu"])
def test_outputs_within_bound_of_float64(F, u_plus, bias, relu):
    U = 128 if u_plus is None else F + u_plus
    csr, w, x, W, b = _case(n=1500, e=20000, F=F, U=U, seed=F + U)
    b = b if bias else None
    act = ops.ACT_RELU if relu else ops.ACT_NONE
    got = ops.spmm_proj(csr, w, x, W, bias=b, act=act)
    _within_bound(got, csr, w, x, W, b, act_relu=relu)


def test_unweighted_empty_rows_odd_ldx_and_ldo_view():
    """ldx = 108 (odd multiple of 4 floats: x is a column view of a wider table), 7 empty rows, an out view with ldo > U."""
    csr, _, _, W, b = _case(n=2000, e=25000, F=100, U=120, weighted=False, isolated=7)
    rs = np.random.RandomState(3)
    wide = torch.tensor(rs.randn(2000, 108).astype(np.float32), device="cuda")
    x = wide[:, 4:104]
    assert x.stride(0) == 108 and x.data_ptr() % 16 == 0
    big = torch.full((2000, 136), 7.0, device="cuda")
    out = big[:, 8:128]
    got = ops.spmm_proj(csr, None, x, W, bias=b, act=ops.ACT_RELU, out=out)
    assert got.data_ptr() == out.data_ptr()
    _within_bound(out, csr, None, x, W, b, act_relu=True)
    assert torch.equal(big[:, :8], torch.full_like(big[:, :8], 7.0)) and torch.equal(big[:, 128:], torch.full_like(big[:, 128:], 7.0))
    empty = (csr.rowptr[1:] == csr.rowptr[:-1]).nonzero().flatten()
    assert empty.numel() >= 7
    assert torch.equal(out[empty], torch.relu(b).expand(empty.numel(), -1))
    same = ops.spmm_proj(csr, None, x.contiguous(), W, bias=b, act=ops.ACT_RELU)
    assert torch.equal(_bits(same), _bits(out))


def test_hub_row_through_the_plan():
    csr, w, x, W, b = _case(n=5000, e=40000, hub=(42, 60000), F=100, U=128)
    assert csr.plan is not None and csr.plan.n_hubs > 0
    got = ops.spmm_proj(csr, w, x, W, bias=b)
    rs = np.random.RandomState(0)
    rows = np.concatenate([[42], rs.randint(0, 5000, 200)])
    _within_bound(got, csr, w, x, W, b, rows=rows)


def test_deterministic_and_plan_free_rows_unchanged():
    csr, w, x, W, b = _case(n=5000, e=40000, hub=(42, 60000), F=100, U=128)
    a = ops.spmm_proj(csr, w, x, W, bias=b, act=ops.ACT_RELU)
    again = ops.spmm_proj(csr, w, x, W, bias=b, act=ops.ACT_RELU)
    assert torch.equal(_bits(a), _bits(again))
    plan, csr.plan = csr.plan, None
    try:
        c = ops.spmm_proj(csr, w, x, W, bias=b, act=ops.ACT_RELU)
    finally:
        csr.plan = plan
    deg = csr.rowptr[1:] - csr.rowptr[:-1]
    plain = deg <= ops.HUB_THRESHOLD
    assert torch.equal(_bits(a[plain]), _bits(c[plain]))


def _gcn_want(x, ei, n, W, b, relu=True):
    import scipy.sparse as sp
    row, col = ei[0].astype(np.int64), ei[1].astype(np.int64)
    loops = np.arange(n)
    row, col = np.concatenate([row, loops]), np.concatenate([col, loops])
    A = sp.csr_matrix((np.ones(len(row)), (row, col)), shape=(n, n))
    d = np.asarray(A.sum(1)).ravel()
    dis = np.where(d > 0, d ** -0.5, 0.0)
    An = sp.diags(dis) @ A @ sp.diags(dis)
    h = An @ (x.astype(np.float64) @ W.astype(np.float64)) + b
    S = abs(An) @ (np.abs(x.astype(np.float64)) @ np.abs(W.astype(np.float64))) + np.abs(b)
    return (np.maximum(h, 0) if relu else h), S, np.asarray(A.getnnz(1)).ravel()


def test_gcn_layer_and_functional_on_the_route():
    n, f, units = 3000, 100, 128
    ei = random_graph(n, 40000, seed=21)
    rs = np.random.RandomState(2)
    x = rs.randn(n, f).astype(np.float32)
    graph = tfg.Graph(x, ei).to_device()
    layer = tfg.layers.GCN(units, activation=tfg.nn.relu, seed=4)
    layer.build_cache_for_graph(graph)
    h, trace = _traced(lambda: layer([graph.x, graph.edge_index], cache=graph.cache))
    assert trace.counts.get("tfgk_spmm_proj_f32", 0) == 1 and "tfgk_gemm_f32" not in trace.counts
    W, b = layer.kernel.data.cpu().numpy(), rs.randn(units).astype(np.float32)
    want, S, deg = _gcn_want(x, ei, n, W, np.zeros(units))
    assert np.all(np.abs(h.cpu().numpy() - want) <= (deg[:, None] + f + 1) * U24 * S + 1e-30)
    dev_b = torch.tensor(b, device="cuda")
    hf = tfg.nn.gcn(graph.x, tfg.SparseMatrix(graph.edge_index, None, [n, n]), layer.kernel.data, dev_b, activation=None,
                    cache=graph.cache)
    want, S, deg = _gcn_want(x, ei, n, W, b, relu=False)
    assert np.all(np.abs(hf.cpu().numpy() - want) <= (deg[:, None] + f + 1) * U24 * S + 1e-30)
    # the projection-first composition, within the suite's fp32 tolerance
    normed = tfg.nn.conv.gcn.gcn_norm_adj(tfg.SparseMatrix(graph.edge_index, None, [n, n]), cache=graph.cache)
    old = normed.matmul(ops.gemm(graph.x, layer.kernel.data), bias=dev_b)
    assert_close(hf.cpu().numpy(), old.cpu().numpy(), what="aggregate-first vs project-first")


def test_products_shape_sampled_rows():
    """The bench's headline GCN layer (products-shaped graph, F = 100, U = 128), 300 sampled rows against float64."""
    import bench
    torch.manual_seed(0)
    n, pairs = bench.PRODUCTS_NODES, bench.PRODUCTS_UNDIRECTED
    ei = bench.make_graph_device(n, pairs, 0, torch.device("cuda"))
    graph = tfg.Graph(torch.randn(n, 100, device="cuda"), ei)
    layer = tfg.layers.GCN(128, activation=tfg.nn.relu, seed=2)
    layer.build_cache_for_graph(graph)
    h = layer([graph.x, graph.edge_index, graph.edge_weight], cache=graph.cache)
    normed = tfg.nn.conv.gcn.gcn_norm_adj(tfg.SparseMatrix(graph.edge_index, None, [n, n]), cache=graph.cache)
    rows = np.random.RandomState(1).randint(0, n, 300)
    _within_bound(h, normed.csr, normed.value_csr, graph.x, layer.kernel.data, layer.bias.data, rows=rows, act_relu=True)


@pytest.mark.parametrize("F,U,routed", [(100, 128, True), (4, 8, True), (124, 128, True), (128, 128, False),
                                        (100, 100, False), (130, 256, False), (102, 128, False), (2, 8, False),
                                        (64, 200, False)])
def test_route_predicate(F, U, routed):
    x = torch.zeros((16, F), device="cuda")
    W = torch.zeros((F, U), device="cuda")
    assert ops.spmm_proj_supported(x, W) == routed
    csr = _csr(np.array([[0, 1], [1, 0]], np.int32), 16)
    if not routed:
        with pytest.raises(ValueError):
            ops.spmm_proj(csr, None, x, W)
        rc = _ffi.lib().tfgk_spmm_proj_f32(ops._p(csr.rowptr), ops._p(csr.col), None, ops._p(x), F, 16, F, ops._p(W), U,
                                           None, 0, ops._p(torch.empty((16, U), device="cuda")), U, None, None)
        assert rc == _ffi.ERR_UNSUPPORTED


def test_unsupported_shapes_keep_the_projection_first_route():
    n = 500
    ei = random_graph(n, 5000, seed=3)
    rs = np.random.RandomState(4)
    graph = tfg.Graph(rs.randn(n, 130).astype(np.float32), ei).to_device()
    layer = tfg.layers.GCN(128, activation=tfg.nn.relu, seed=1)        # F = 130 > U
    layer.build_cache_for_graph(graph)
    _, trace = _traced(lambda: layer([graph.x, graph.edge_index], cache=graph.cache))
    assert "tfgk_spmm_proj_f32" not in trace.counts and trace.counts.get("tfgk_spmm_f32", 0) == 1


def test_cuda_graph_capture_of_a_routed_layer():
    n, f, units = 5000, 100, 128
    ei = random_graph(n, 40000, seed=8, hub=(42, 60000))
    rs = np.random.RandomState(5)
    graph = tfg.Graph(rs.randn(n, f).astype(np.float32), ei).to_device()
    layer = tfg.layers.GCN(units, activation=tfg.nn.relu, seed=3)
    layer.build_cache_for_graph(graph)
    static_x = graph.x.clone()
    fn = lambda: layer([static_x, graph.edge_index], cache=graph.cache)   # noqa: E731
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    new_x = torch.tensor(rs.randn(n, f).astype(np.float32), device="cuda")
    static_x.copy_(new_x)
    g.replay()
    torch.cuda.synchronize()
    eager = layer([new_x, graph.edge_index], cache=graph.cache)
    assert torch.equal(_bits(out), _bits(eager))
