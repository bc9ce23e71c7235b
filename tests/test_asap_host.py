# coding=utf-8
"""cluster_pool, ASAP and the differentiable segment_softmax without a GPU: the host logic over the CPU fake of the kernel
layer with a numpy Gustavson-order K10, against the float64 restatement of the reference (tests/asap_ref.py)."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import asap_fake_backend as fake_k10
import asap_ref as ref
from conftest import assert_close


@pytest.fixture
def fake(monkeypatch):
    fake_k10.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg


def _params(F, seed, grad=False):
    return {k: torch.tensor(v, requires_grad=grad) for k, v in ref.random_params(F, seed).items()}


def _grads_close(pairs, rtol=1e-3, atol_scale=1e-4):
    """(name, got, want) gradients: |got - want| <= rtol |want| + atol_scale * max |want| over ALL of them (a gradient that
    is zero in exact arithmetic, such as the attention GCN bias, is then held to the scale of the others)."""
    scale = max(float(np.max(np.abs(w))) for _, _, w in pairs if np.size(w))
    for name, got, want in pairs:
        err = np.abs(np.asarray(got, np.float64) - want)
        assert np.all(err <= rtol * np.abs(want) + atol_scale * scale), "d {}: max err {:.3e} (scale {:.3e})".format(
            name, err.max(), scale)


def _call_asap(tfg, x, ei, w, ngi, p, **kw):
    return tfg.nn.asap(x, ei, w, ngi, *[p[k] for k in ref.ORDER], None, **kw)


def test_ffi_declares_k10_and_validates_without_gpu():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    need = ctypes.c_size_t()
    _ffi.call("tfgk_spgemm_rows_workspace_bytes", 1000, ctypes.byref(need))
    assert need.value >= 1000 * 24
    _ffi.call("tfgk_spgemm_rows_workspace_bytes", 0, ctypes.byref(need))
    assert need.value == 0
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_spgemm_plan_workspace_bytes", -1, ctypes.byref(need))
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_spgemm_count", None, None, None, None, 3, 1, None, None, 0, None, None, 0, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "row range" in str(err.value)


def test_chunks_cover_the_rows():
    from tf_geometric_b200 import ops
    ptr = np.array([0, 5, 5, 9, 30, 31, 31])
    assert ops._spgemm_chunks(ptr, 10) == [(0, 3), (3, 4), (4, 6)]
    assert ops._spgemm_chunks(ptr, 0) == [(r, r + 1) for r in range(6)]
    assert ops._spgemm_chunks(ptr, 1 << 40) == [(0, 6)]


def test_gustavson_restatement():
    """Columns ascending, duplicates merged in production order, exact zeros kept; against scipy in float64."""
    a = sp.random(40, 30, density=0.2, random_state=1, format="csr", dtype=np.float32)
    b = sp.random(30, 50, density=0.2, random_state=2, format="csr", dtype=np.float32)
    rp, col, val = fake_k10.spgemm_reference(a.indptr, a.indices, a.data, b.indptr, b.indices, b.data, 50)
    want = (a.astype(np.float64) @ b.astype(np.float64)).tocsr()
    got = sp.csr_matrix((val.astype(np.float64), col, rp), shape=(40, 50))
    assert_close(got.toarray(), want.toarray(), rtol=1e-5, what="A B")
    for i in range(40):
        assert np.all(np.diff(col[rp[i]:rp[i + 1]]) > 0)
    # one row: products (col 1: 0.1*3, then 0.2*5), (col 0: 0.1*2), (col 1: 0.3*-7) in production order
    rp, col, val = fake_k10.spgemm_reference([0, 3], [0, 1, 0], np.float32([0.1, 0.2, 0.3]), [0, 2, 3], [1, 0, 1],
                                             np.float32([3, 2, 5]), 2)
    f = np.float32
    assert list(col) == [0, 1]
    assert val[0] == f(0.1) * f(2) + f(0.3) * f(2)
    assert val[1] == (f(0.1) * f(3) + f(0.2) * f(5)) + f(0.3) * f(3)


def test_cluster_pool_against_the_dense_restatement(fake):
    x, ei, w, aei, aw, K, N = ref.cluster_case()
    for weight in (w, None):
        xt, awt = torch.tensor(x, requires_grad=True), torch.tensor(aw, requires_grad=True)
        px, pei, pw = fake.nn.cluster_pool(xt, torch.tensor(ei), None if weight is None else torch.tensor(weight),
                                           torch.tensor(aei), awt, K)
        x64, aw64 = ref.t64(x, True), ref.t64(aw, True)
        want_x, want_ei, want_w = ref.cluster_pool(x64, ei, ref.t64(np.ones(ei.shape[1]) if weight is None else weight),
                                                   aei, aw64, K, N)
        np.testing.assert_array_equal(pei.numpy(), want_ei)
        assert_close(pw.detach().numpy(), want_w.detach().numpy(), what="pooled w")
        assert_close(px.detach().numpy(), want_x.detach().numpy(), what="pooled x")
        g = np.random.RandomState(2).randn(*px.shape)
        (px * torch.tensor(g, dtype=torch.float32)).sum().backward()
        (want_x * torch.tensor(g)).sum().backward()
        assert_close(xt.grad.numpy(), x64.grad.numpy(), what="d x")
        assert_close(awt.grad.numpy(), aw64.grad.numpy(), what="d assign w")
        # the zero-weight edge (3, 5) makes P[1, 2] exactly 0: not an edge
        assert np.any((pei[0].numpy() == 1) & (pei[1].numpy() == 2)) == (weight is None)
    px, _, _ = fake.nn.cluster_pool(None, ei, w, aei, None, K, num_nodes=N)
    assert px is None
    with pytest.raises(Exception, match="num_nodes"):
        fake.nn.cluster_pool(None, ei, w, aei, aw, K)


def test_pooled_weight_gradient_is_refused(fake):
    x, ei, w, aei, aw, K, N = ref.cluster_case()
    wt = torch.tensor(w, requires_grad=True)
    xt = torch.tensor(x, requires_grad=True)
    px, _, pw = fake.nn.cluster_pool(xt, torch.tensor(ei), wt, torch.tensor(aei), torch.tensor(aw), K)
    px.sum().backward()                                        # the pooled weights are not in this loss: fine
    with pytest.raises(RuntimeError, match="pooled edge weights"):
        pw.sum().backward()


@pytest.mark.parametrize("two_d", [False, True])
def test_segment_softmax_carries_gradients(fake, two_d):
    rs = np.random.RandomState(4)
    seg = np.array([2, 0, 2, 1, 0, 2, 2, 4])
    data = rs.randn(8, 3).astype(np.float32) if two_d else rs.randn(8).astype(np.float32)
    plain = fake.nn.segment_softmax(torch.tensor(data), torch.tensor(seg), 5)
    dt = torch.tensor(data, requires_grad=True)
    out = fake.nn.segment_softmax(dt, torch.tensor(seg), 5)
    assert out.requires_grad
    np.testing.assert_array_equal(out.detach().numpy(), plain.numpy())
    g = rs.randn(*data.shape)
    (out * torch.tensor(g, dtype=torch.float32)).sum().backward()
    d64 = ref.t64(data, True)
    segt = torch.tensor(seg)
    want = torch.stack([ref.segment_softmax(d64[:, c], segt, 5) for c in range(3)], 1) if two_d \
        else ref.segment_softmax(d64, segt, 5)
    (want * torch.tensor(g)).sum().backward()
    assert_close(dt.grad.numpy(), d64.grad.numpy(), rtol=1e-4, atol_scale=1e-5, what="d scores")


@pytest.mark.parametrize("with_weight", [False, True])
def test_asap_forward_and_gradients(fake, with_weight):
    x, ei, w, ngi = ref.batch([5, 1, 7, 4], seed=11, F=5)
    p = _params(5, 3, grad=True)
    xt = torch.tensor(x, requires_grad=True)
    wt = torch.tensor(w, requires_grad=True) if with_weight else None
    px, pei, pw, pngi = _call_asap(fake, xt, torch.tensor(ei), wt, torch.tensor(ngi), p, ratio=0.5)
    x64 = ref.t64(x, True)
    p64 = {k: ref.t64(v.detach().numpy(), True) for k, v in p.items()}
    w64 = ref.t64(w, True) if with_weight else None
    want_x, want_ei, want_w, want_ngi, _ = ref.asap(x64, ei, w64, ngi, p64, ratio=0.5)
    np.testing.assert_array_equal(pei.numpy(), want_ei)
    np.testing.assert_array_equal(pngi.numpy(), want_ngi)
    assert_close(px.detach().numpy(), want_x.detach().numpy(), what="pooled x")
    assert_close(pw.detach().numpy(), want_w.detach().numpy(), what="pooled w")
    g = np.random.RandomState(6).randn(*px.shape)
    (px * torch.tensor(g, dtype=torch.float32)).sum().backward()
    (want_x * torch.tensor(g)).sum().backward()
    pairs = [("x", xt.grad.numpy(), x64.grad.numpy())] + [(k, p[k].grad.numpy(), p64[k].grad.numpy()) for k in ref.ORDER]
    if with_weight:
        pairs.append(("edge_weight", wt.grad.numpy(), w64.grad.numpy()))
    _grads_close(pairs)
    if with_weight:
        with pytest.raises(RuntimeError, match="pooled edge weights"):
            pw.sum().backward()


def test_asap_errors_and_layer(fake):
    x, ei, w, ngi = ref.batch([5, 6], seed=2, F=4)
    p = _params(4, 1)
    p["attention_gcn_kernel"] = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="attention_units"):
        _call_asap(fake, torch.tensor(x), torch.tensor(ei), None, torch.tensor(ngi), p, ratio=0.5)
    with pytest.raises(ValueError, match="attention_units"):
        fake.layers.ASAP(ratio=0.5, attention_units=3)([torch.tensor(x), torch.tensor(ei), None, torch.tensor(ngi)])
    layer = fake.layers.ASAP(k=2, trainable=True, seed=3)
    h, pei, pw, pngi = layer([torch.tensor(x), torch.tensor(ei), None, torch.tensor(ngi)])
    assert sorted(n for n, _ in layer.named_parameters()) == sorted(ref.ORDER)
    assert tuple(layer.attention_score_kernel.shape) == (8, 1) and h.shape == (4, 4)
    np.testing.assert_array_equal(pngi.numpy(), [0, 0, 1, 1])
    h.sum().backward()
    assert all(prm.grad is not None for prm in layer.parameters())
    assert fake.layers.ASAP(ratio=0.5, le_conv_use_bias=False).le_conv_self_bias is None


def test_golden_fixture_from_the_reference(fake):
    """asap_exec.npz: the reference's own cluster_pool.py (sparse [node, cluster] assignment with duplicates, a node in no
    cluster, an empty cluster, a self loop, a zero-weight edge, weights None) and asap.py with the two adapters (ratio and
    k, edge_weight None and given, unsorted node_graph_index, an edgeless graph, training=False)."""
    assert ref.check_golden(fake, "cpu") == 22
