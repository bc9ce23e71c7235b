# coding=utf-8
"""DiffPool / MinCutPool without a GPU: the host logic (graph layout, pooled-edge extraction, self-loop removal, the
differentiable normalisation, the losses, the layers) over the CPU fake of the kernel layer with numpy K8a / K8b, against
a float64 dense per-graph restatement."""
import numpy as np
import pytest
import torch

import cluster_pool_fake_backend as fake_k8
import cluster_pool_ref as ref
from conftest import assert_close


@pytest.fixture
def fake(monkeypatch):
    fake_k8.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg


def _case(sizes=(5, 0, 7, 1, 9), seed=0, C=3, D=4, shuffle=True):
    ei, ngi, w = ref.batch(list(sizes), seed)
    rs = np.random.RandomState(seed + 100)
    N = len(ngi)
    if shuffle:                                          # unsorted node_graph_index: relabel the nodes
        p = rs.permutation(N)
        inv = np.empty_like(p)
        inv[p] = np.arange(N)
        ngi = ngi[p]
        ei = inv[ei].astype(np.int32)
    x = rs.randn(N, D).astype(np.float32)
    logits = rs.randn(N, C).astype(np.float32)
    return ei, ngi, w, x, logits


def test_ffi_declares_k8():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    assert len(_ffi.SIGNATURES["tfgk_graph_tmm_f32"]) == 15 and len(_ffi.SIGNATURES["tfgk_graph_rmm_f32"]) == 14


def test_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    import ctypes
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_graph_tmm_f32", None, 0, None, 0, 10, 0, 4, None, None, 2, None, 4, None, 0, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "C 0" in str(err.value)
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_graph_tmm_f32", None, 3, None, 4, 10, 3, 4, None, None, 2, None, 4, None, 0, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "null gptr" in str(err.value)
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_graph_rmm_f32", None, 4, None, 10, None, 4, 2, 3, 4, 2, 0.0, None, 4, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "trans" in str(err.value)
    need = ctypes.c_size_t()
    _ffi.call("tfgk_graph_tmm_workspace_bytes", 3, 100000, 16, 128, ctypes.byref(need))
    assert need.value >= 2 * 100000 // 1024 * 16 * 128 * 4
    from tf_geometric_b200 import ops
    with pytest.raises(TypeError):
        ops.graph_tmm(torch.zeros(3, 2), torch.zeros(3, 4), torch.zeros(2, dtype=torch.int64), 1)


def test_fake_kernels_are_the_definition():
    rs = np.random.RandomState(0)
    S, Y = rs.randn(6, 2).astype(np.float32), rs.randn(6, 3).astype(np.float32)
    gptr, gnodes = np.array([0, 2, 2, 6]), np.array([5, 0, 1, 2, 3, 4])
    out = fake_k8.tmm_reference(S, Y, gptr, gnodes)
    assert_close(out[0:2], S[[5, 0]].T @ Y[[5, 0]])
    assert np.all(out[2:4] == 0)
    ng = np.array([0, 0, 2, 2, 2, 0])
    B = rs.randn(6, 3).astype(np.float32)
    r = fake_k8.rmm_reference(S, B, ng, 2)
    assert_close(r[2], S[2] @ B[4:6])
    r = fake_k8.rmm_reference(Y, B, ng, 2, trans=True)
    assert_close(r[1], Y[1] @ B[0:2].T)


@pytest.mark.parametrize("shuffle", [False, True])
def test_diff_pool_coarsen_forward_and_gradients(fake, shuffle):
    ei, ngi, w, x, logits = _case(shuffle=shuffle)
    G, C = int(ngi.max()) + 1, logits.shape[1]
    xt, lt, wt = (torch.tensor(a, requires_grad=True) for a in (x, logits, w))
    S = torch.softmax(lt, -1)
    px, pei, pw, pngi = fake.nn.diff_pool_coarsen(xt, torch.tensor(ei), wt, torch.tensor(ngi), S)
    x64, l64, w64 = ref.t64(x, True), ref.t64(logits, True), ref.t64(w, True)
    row, col = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    P, Q = ref.blocks(x64, torch.softmax(l64, -1), w64, row, col, ngi, G)
    want_ei, want_w = ref.pooled_edges(Q, C)
    np.testing.assert_array_equal(pei.numpy(), want_ei)
    np.testing.assert_array_equal(pngi.numpy(), np.repeat(np.arange(G), C).astype(np.int32))
    assert_close(px.detach().numpy(), P.detach().numpy(), what="pooled x")
    assert_close(pw.detach().numpy(), want_w.detach().numpy(), what="pooled w")
    rs = np.random.RandomState(5)
    gx, gw = rs.randn(*px.shape), rs.randn(*pw.shape)
    ((px * torch.tensor(gx, dtype=torch.float32)).sum() + (pw * torch.tensor(gw, dtype=torch.float32)).sum()).backward()
    ((P * torch.tensor(gx)).sum() + (want_w * torch.tensor(gw)).sum()).backward()
    for name, mine, want in (("x", xt, x64), ("logits", lt, l64), ("w", wt, w64)):
        assert_close(mine.grad.numpy(), want.grad.numpy(), rtol=1e-3, atol_scale=1e-4, what="d " + name)


def test_min_cut_coarsen_and_losses_gradients(fake):
    ei, ngi, w, x, logits = _case(seed=3, C=4)
    G, C = int(ngi.max()) + 1, logits.shape[1]
    N = len(ngi)
    xt, lt, wt = (torch.tensor(a, requires_grad=True) for a in (x, logits, w))
    S = torch.softmax(lt, -1)
    eit, ngt = torch.tensor(ei), torch.tensor(ngi)
    px, pei, pw, _ = fake.nn.min_cut_pool_coarsen(xt, eit, wt, ngt, S)
    cut, orth = fake.nn.min_cut_pool_compute_losses(eit, wt, ngt, S)
    x64, l64, w64 = ref.t64(x, True), ref.t64(logits, True), ref.t64(w, True)
    row, col = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    S64 = torch.softmax(l64, -1)
    normed = ref.adj_norm(row, col, w64, N)
    P, Q = ref.blocks(x64, S64, normed, row, col, ngi, G)
    want_ei, want_w = ref.pooled_edges(Q, C, drop_self_loops=True)
    want_cut, want_orth = ref.min_cut_losses(S64, normed, row, col, ngi, G)
    np.testing.assert_array_equal(pei.numpy(), want_ei)
    assert_close(pw.detach().numpy(), want_w.detach().numpy(), what="pooled w")
    assert_close(cut.item(), want_cut.item(), what="cut loss")
    assert_close(orth.item(), want_orth.item(), what="orth loss")
    rs = np.random.RandomState(7)
    gx, gw = rs.randn(*px.shape), rs.randn(*pw.shape)
    ((px * torch.tensor(gx, dtype=torch.float32)).sum() + (pw * torch.tensor(gw, dtype=torch.float32)).sum()
     + 0.7 * cut + 1.3 * orth).backward()
    ((P * torch.tensor(gx)).sum() + (want_w * torch.tensor(gw)).sum() + 0.7 * want_cut + 1.3 * want_orth).backward()
    for name, mine, want in (("x", xt, x64), ("logits", lt, l64), ("w", wt, w64)):
        assert_close(mine.grad.numpy(), want.grad.numpy(), rtol=1e-3, atol_scale=1e-4, what="d " + name)


def test_adj_norm_edge_is_differentiable_and_unchanged(fake):
    ei, ngi, w, _, _ = _case(seed=4)
    N = len(ngi)
    plain = fake.utils.adj_norm_edge(torch.tensor(ei), N, torch.tensor(w))[1]
    wt = torch.tensor(w, requires_grad=True)
    normed = fake.utils.adj_norm_edge(torch.tensor(ei), N, wt)[1]
    np.testing.assert_array_equal(normed.detach().numpy(), plain.numpy())
    g = np.random.RandomState(1).randn(len(w))
    (normed * torch.tensor(g, dtype=torch.float32)).sum().backward()
    w64 = ref.t64(w, True)
    row, col = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    (ref.adj_norm(row, col, w64, N) * torch.tensor(g)).sum().backward()
    assert_close(wt.grad.numpy(), w64.grad.numpy(), rtol=1e-4, atol_scale=1e-4, what="d w")


def test_remove_self_loop_edge_device_path_keeps_bits_and_gradient(fake):
    ei = np.array([[0, 1, 2, 2, 3], [1, 1, 0, 2, 0]], np.int32)
    w = np.array([0.5, 1.5, -2.0, 3.0, 0.25], np.float32)
    want_ei, want_w = fake.utils.remove_self_loop_edge(ei, w)              # numpy in -> the host path
    wt = torch.tensor(w, requires_grad=True)
    got_ei, got_w = fake.utils.remove_self_loop_edge(torch.tensor(ei), wt)
    np.testing.assert_array_equal(got_ei.numpy(), want_ei)
    np.testing.assert_array_equal(got_w.detach().numpy(), want_w)
    got_w.sum().backward()
    np.testing.assert_array_equal(wt.grad.numpy(), [1, 0, 1, 0, 1])


def test_dense_converters(fake):
    a = np.array([[0.0, 2.0, 0.0], [np.nan, 0.0, 1.0], [0.0, 0.0, -3.0]], np.float32)
    ei, w = fake.utils.convert_dense_adj_to_edge(a)
    np.testing.assert_array_equal(ei, [[0, 1, 1, 2], [1, 0, 2, 2]])
    at = torch.tensor(a, requires_grad=True)
    ei_t, w_t = fake.utils.convert_dense_adj_to_edge(at)
    np.testing.assert_array_equal(ei_t.numpy(), ei)
    np.testing.assert_array_equal(w_t.detach().numpy(), w)
    w_t[~torch.isnan(w_t)].sum().backward()
    assert at.grad[0, 1].item() == 1.0 and at.grad[0, 0].item() == 0.0
    s = np.arange(6, dtype=np.float32).reshape(3, 2)
    ngi = np.array([1, 0, 1], np.int32)
    ei, w = fake.utils.convert_dense_assign_to_edge(s, ngi)
    np.testing.assert_array_equal(ei, [[0, 0, 1, 1, 2, 2], [2, 3, 0, 1, 2, 3]])
    ei_t, w_t = fake.utils.convert_dense_assign_to_edge(torch.tensor(s), torch.tensor(ngi))
    np.testing.assert_array_equal(ei_t.numpy(), ei)
    np.testing.assert_array_equal(w_t.numpy(), s.reshape(-1))


def test_errors(fake):
    ei, ngi, w, x, logits = _case(shuffle=False)
    bad = np.concatenate([ei, [[0], [len(ngi) - 1]]], axis=1).astype(np.int32)     # joins the first and last graph
    S = torch.softmax(torch.tensor(logits), -1)
    with pytest.raises(ValueError):
        fake.nn.diff_pool_coarsen(torch.tensor(x), torch.tensor(bad), None, torch.tensor(ngi), S)
    with pytest.raises(Exception, match="cannot be set to True at the same time"):
        fake.nn.min_cut_pool(torch.tensor(x), torch.tensor(ei), None, torch.tensor(ngi), None, None, 3,
                             return_loss_func=True, return_losses=True)


def test_layers_train_on_the_host(fake):
    ei, ngi, w, x, logits = _case(seed=8, C=3, D=6)
    eit, ngt, xt = torch.tensor(ei), torch.tensor(ngi), torch.tensor(x)
    for cls in (fake.layers.DiffPool, fake.layers.MinCutPool):
        feat = fake.layers.GCN(5, activation=fake.nn.relu, trainable=True, seed=1)
        assign = fake.layers.GCN(3, trainable=True, seed=2)
        pool = cls(feat, assign, 5, 3, activation=fake.nn.relu, trainable=True)
        wt = torch.tensor(w, requires_grad=True)
        if cls is fake.layers.MinCutPool:
            (h, _, pw, _), (cut, orth) = pool([xt, eit, wt, ngt], return_losses=True)
            loss = h.sum() + pw.sum() + cut + orth
        else:
            h, _, pw, _ = pool([xt, eit, wt, ngt])
            loss = h.sum() + pw.sum()
        loss.backward()
        assert pool.bias is not None and pool.bias.grad is not None
        assert feat.kernel.grad is not None and assign.kernel.grad is not None and wt.grad is not None
        assert np.all(np.isfinite(wt.grad.numpy()))


def test_golden_fixture_from_the_reference(fake):
    """cluster_pool_exec.npz: the reference's own diff_pool / min_cut_pool (edgeless graph, duplicate edges and self loops,
    unsorted node_graph_index, C = 3 and C = 1, edge_weight None, both gnn_use_normed_edge values) and convert_dense_*."""
    assert ref.check_golden(fake, "cpu") == 44
