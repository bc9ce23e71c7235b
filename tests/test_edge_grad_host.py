# coding=utf-8
"""Edge-weight gradients without a GPU: the host logic (edge-order perm, mean scale, the normalisation backward, route
selection, caching) over the CPU fake of the kernel layer with a numpy K7, against float64 torch autograd."""
import os

import numpy as np
import pytest
import torch

import edge_grad_fake_backend
import edge_grad_ref as ref
from conftest import assert_close, random_graph, glorot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def fake(monkeypatch):
    edge_grad_fake_backend.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg


def _graph(n=60, e=400, seed=0):
    rs = np.random.RandomState(seed)
    ei = random_graph(n, e, seed=seed, symmetric=True, isolated=2)
    ei = np.concatenate([ei, [[5, 5, 7], [5, 5, 7]], ei[:, :3]], axis=1).astype(np.int32)   # self loops, duplicates
    w = (rs.rand(ei.shape[1]) + 0.2).astype(np.float32)
    return rs, ei, w


def test_ffi_declares_k7():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    assert "tfgk_sddmm_csr_f32" in _ffi.SIGNATURES and len(_ffi.SIGNATURES["tfgk_sddmm_csr_f32"]) == 13
    header = open(os.path.join(ROOT, "include", "tfgk.h")).read()
    assert "#define TFGK_ABI_VERSION 7" in header and "int tfgk_sddmm_csr_f32(" in header


def test_fake_k7_is_the_definition():
    rs = np.random.RandomState(1)
    rowptr = np.array([0, 2, 2, 5], np.int64)
    col = np.array([1, 0, 2, 2, 1], np.int32)
    perm = np.array([4, 0, 3, 1, 2], np.int32)
    G, X = rs.randn(3, 5).astype(np.float32), rs.randn(3, 5).astype(np.float32)
    scale = np.array([0.5, 1.0, 0.25], np.float32)
    csr_order = edge_grad_fake_backend.sddmm_reference(rowptr, col, perm, G, X, scale, 2.0, edge_order=False)
    want = np.array([(G[r] @ X[c]) * 2.0 * scale[r] for r, c in zip([0, 0, 2, 2, 2], col)])
    assert_close(csr_order, want)
    edge = edge_grad_fake_backend.sddmm_reference(rowptr, col, perm, G, X, scale, 2.0)
    np.testing.assert_array_equal(edge[perm], csr_order)


@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_neighbor_aggregate_edge_gradient(fake, reduce):
    from tf_geometric_b200 import autograd
    rs, ei, w = _graph()
    n = 60
    x = rs.randn(n, 7).astype(np.float32)
    gout = rs.randn(n, 7)
    wt = torch.tensor(w, requires_grad=True)
    xt = torch.tensor(x, requires_grad=True)
    y = autograd.NeighborAggregate.apply(xt, torch.tensor(ei), wt, reduce, n)
    (y * torch.tensor(gout, dtype=torch.float32)).sum().backward()
    w64, x64 = ref.t64(w, True), ref.t64(x, True)
    r, c = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    (ref.aggregate(r, c, w64, x64, n, reduce) * torch.tensor(gout)).sum().backward()
    assert_close(wt.grad.numpy(), w64.grad.numpy(), rtol=1e-4, atol_scale=1e-4, what="d w")
    assert_close(xt.grad.numpy(), x64.grad.numpy(), rtol=1e-4, atol_scale=1e-4, what="d x")


@pytest.mark.parametrize("combo", ref.NORM_COMBOS, ids=lambda c: "-".join(map(str, c)))
def test_gcn_norm_adj_backward(fake, combo):
    from tf_geometric_b200.sparse import SparseMatrix
    norm, loop, sym, renorm, improved = combo
    rs, ei, w = _graph(seed=3)
    n = 60
    wt = torch.tensor(w, requires_grad=True)
    normed = fake.nn.gcn_norm_adj(SparseMatrix(torch.tensor(ei), wt, [n, n]), norm, loop, sym, renorm, improved)
    assert normed.value.grad_fn is not None
    plain = fake.nn.gcn_norm_adj(SparseMatrix(torch.tensor(ei), torch.tensor(w), [n, n]), norm, loop, sym, renorm, improved)
    np.testing.assert_array_equal(normed.value.detach().numpy(), plain.value.numpy())      # requires_grad changes no bit
    g = rs.randn(normed.nnz)
    (normed.value * torch.tensor(g, dtype=torch.float32)).sum().backward()
    w64 = ref.t64(w, True)
    _, _, v64 = ref.gcn_norm(torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64), w64, [n, n],
                             norm, loop, sym, renorm, improved)
    assert_close(normed.value.detach().numpy(), v64.detach().numpy(), what="normed values")
    (v64 * torch.tensor(g)).sum().backward()
    assert_close(wt.grad.numpy(), w64.grad.numpy(), rtol=1e-4, atol_scale=1e-4, what="d w {}".format(combo))


def test_zero_degree_gets_zero_gradient(fake):
    from tf_geometric_b200.sparse import SparseMatrix
    ei = np.array([[0, 1, 2, 2], [1, 0, 3, 0]], np.int32)
    w = np.array([1.0, 2.0, 0.5, -0.5], np.float32)           # row 2 sums to 0, row 3 has no entry
    wt = torch.tensor(w, requires_grad=True)
    normed = fake.nn.gcn_norm_adj(SparseMatrix(torch.tensor(ei), wt, [4, 4]), add_self_loop=False)
    normed.value.sum().backward()
    assert np.all(np.isfinite(wt.grad.numpy()))
    assert wt.grad[2].item() == 0.0 and wt.grad[3].item() == 0.0


def test_sparse_matmul_value_gradient(fake):
    from tf_geometric_b200.sparse import SparseMatrix
    rs, ei, w = _graph(seed=4)
    n = 60
    h = rs.randn(n, 5).astype(np.float32)
    b = rs.randn(5).astype(np.float32)
    wt, ht, bt = (torch.tensor(a, requires_grad=True) for a in (w, h, b))
    A = SparseMatrix(torch.tensor(ei), wt, [n, n])
    from tf_geometric_b200 import ops
    y = A.matmul(ht, bias=bt, act=ops.ACT_RELU)
    g = rs.randn(n, 5)
    (y * torch.tensor(g, dtype=torch.float32)).sum().backward()
    w64, h64, b64 = ref.t64(w, True), ref.t64(h, True), ref.t64(b, True)
    r, c = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    (torch.relu(ref.spmm(r, c, w64, h64, n) + b64) * torch.tensor(g)).sum().backward()
    for name, mine, want in (("w", wt, w64), ("h", ht, h64), ("b", bt, b64)):
        assert_close(mine.grad.numpy(), want.grad.numpy(), rtol=1e-4, atol_scale=1e-4, what="d " + name)
    # only the values need grad: the product still takes the differentiable route, and h gets nothing
    h2 = torch.tensor(h)
    y2 = SparseMatrix(torch.tensor(ei), torch.tensor(w, requires_grad=True), [n, n]) @ h2
    assert y2.grad_fn is not None and h2.grad is None


def _conv_case(tfg, name, rs, ei, n, f, u):
    """(fn(x, edge_index, w, params) -> output, float64 reference, params) for one convolution."""
    r, c = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    relu = tfg.nn.relu
    if name == "gcn":
        P = dict(k=glorot(rs, f, u), b=rs.randn(u).astype(np.float32))

        def mine(x, e, w, p):
            from tf_geometric_b200.sparse import SparseMatrix
            return tfg.nn.gcn(x, SparseMatrix(e, w, [n, n]), p["k"], p["b"], relu)

        def want(x, w, p):
            nr, nc, nv = ref.gcn_norm(r, c, w, [n, n])
            return torch.relu(ref.spmm(nr, nc, nv, x @ p["k"], n) + p["b"])
    elif name == "sgc":
        P = dict(k=glorot(rs, f, u), b=rs.randn(u).astype(np.float32))

        def mine(x, e, w, p):
            return tfg.nn.sgc(x, e, w, 2, p["k"], p["b"], relu)

        def want(x, w, p):
            nr, nc, nv = ref.gcn_norm(r, c, w, [n, n])
            return torch.relu(ref.spmm(nr, nc, nv, ref.spmm(nr, nc, nv, x @ p["k"], n), n) + p["b"])
    elif name == "le_conv":
        P = {k: glorot(rs, f, u) for k in ("ws", "wa", "wn")}
        P.update({k: rs.randn(u).astype(np.float32) for k in ("bs", "ba", "bn")})

        def mine(x, e, w, p):
            return tfg.nn.le_conv(x, e, w, p["ws"], p["bs"], p["wa"], p["ba"], p["wn"], p["bn"], relu)

        def want(x, w, p):
            return torch.relu(ref.spmm(r, c, w, (x @ p["wa"] + p["ba"]) - (x @ p["wn"] + p["bn"]), n) + x @ p["ws"] + p["bs"])
    else:
        reduce = "mean" if name == "mean_graph_sage" else "sum"
        P = dict(ws=glorot(rs, f, u), wn=glorot(rs, f, u), b=rs.randn(2 * u).astype(np.float32))
        fn = getattr(tfg.nn, name)

        def mine(x, e, w, p):
            return fn(x, e, w, p["ws"], p["wn"], p["b"], relu)

        def want(x, w, p):
            return torch.relu(torch.cat([x @ p["ws"], ref.aggregate(r, c, w, x, n, reduce) @ p["wn"]], 1) + p["b"])
    return mine, want, P


@pytest.mark.parametrize("name", ["gcn", "sgc", "le_conv", "mean_graph_sage", "sum_graph_sage"])
def test_convolution_edge_gradients(fake, name):
    rs, ei, w = _graph(seed=len(name))
    n, f, u = 60, 6, 4
    x = rs.randn(n, f).astype(np.float32)
    mine, want, P = _conv_case(fake, name, rs, ei, n, f, u)
    # only the edge weights require grad: the training route is taken all the same
    wt = torch.tensor(w, requires_grad=True)
    y = mine(torch.tensor(x), torch.tensor(ei), wt, {k: torch.tensor(v) for k, v in P.items()})
    assert y.grad_fn is not None
    g = rs.randn(*y.shape)
    (y * torch.tensor(g, dtype=torch.float32)).sum().backward()
    w64 = ref.t64(w, True)
    y64 = want(ref.t64(x), w64, {k: ref.t64(v) for k, v in P.items()})
    assert_close(y.detach().numpy(), y64.detach().numpy(), what=name + " forward")
    (y64 * torch.tensor(g)).sum().backward()
    assert_close(wt.grad.numpy(), w64.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what=name + " d w")


def test_cache_hit_carries_no_gradient(fake):
    from tf_geometric_b200.sparse import SparseMatrix
    rs, ei, w = _graph(seed=9)
    n = 60
    cache = {}
    wt = torch.tensor(w, requires_grad=True)
    cold = fake.nn.gcn_norm_adj(SparseMatrix(torch.tensor(ei), wt, [n, n]), cache=cache)
    assert cold.value.grad_fn is not None                           # a cold build is differentiable ...
    assert all(not m.value.requires_grad for m in cache.values())   # ... but what it caches is not
    warm = fake.nn.gcn_norm_adj(SparseMatrix(torch.tensor(ei), wt, [n, n]), cache=cache)
    assert not warm.value.requires_grad
    np.testing.assert_array_equal(warm.value.numpy(), cold.value.detach().numpy())


def test_in_place_update_invalidates_the_csr_ordered_weights(fake):
    from tf_geometric_b200 import _structure
    rs, ei, w = _graph(seed=11)
    n = 60
    x = torch.tensor(rs.randn(n, 3).astype(np.float32))
    eit = torch.tensor(ei)
    wt = torch.tensor(w, requires_grad=True)
    csr, _ = _structure.csr_for_edge_index(eit, n)
    first = _structure.weights_in_csr_order(wt, csr).clone()
    y = fake.nn.sum_graph_sage(x, eit, wt, torch.eye(3), torch.eye(3), None, None)
    y.sum().backward()
    with torch.no_grad():
        wt -= 0.5 * wt.grad
    second = _structure.weights_in_csr_order(wt, csr)
    np.testing.assert_array_equal(second.numpy(), wt.detach().numpy()[csr.perm.numpy()])
    assert not np.array_equal(first.numpy(), second.numpy())
    y2 = fake.nn.sum_graph_sage(x, eit, wt, torch.eye(3), torch.eye(3), None, None)
    r, c = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    want = torch.cat([x.double(), ref.aggregate(r, c, wt.detach().double(), x.double(), n, "sum")], 1)
    assert_close(y2.detach().numpy(), want.numpy(), what="second forward uses the updated weights")
