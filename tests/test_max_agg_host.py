# coding=utf-8
"""K11 (max aggregation with tie counts and its transposed-CSR backward) without a GPU: the ABI entries and their
argument errors, the numpy restatement on hand-made cases, which public calls take NeighborMax and which keep the
composition, and gradients against float64 autograd through the fake kernel layer."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import max_agg_ref as ref
from conftest import random_graph

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOWEST = np.finfo(np.float32).min


@pytest.fixture
def fake(monkeypatch):
    calls = ref.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg, calls


def test_k11_is_exported_and_declared_with_its_arity():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    handle = ctypes.CDLL(_ffi.library_path())
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "tfgk.h")).read(), flags=re.S)
    for name, arity in (("tfgk_spmm_max_f32", 13), ("tfgk_spmm_max_bwd_f32", 19)):
        assert hasattr(handle, name)
        args = re.search(r"\bint\s+" + name + r"\s*\(([^;]*?)\)\s*;", text, flags=re.S).group(1)
        assert len([a for a in args.split(",") if a.strip()]) == arity == len(_ffi.SIGNATURES[name])


def test_argument_errors_without_gpu():
    from tf_geometric_b200 import _ffi

    def code(name, *args):
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(name, *args)
        return err.value.code, str(err.value)

    fwd = "tfgk_spmm_max_f32"
    assert code(fwd, None, None, None, None, 4, -1, 4, None, 4, None, 4, None, None)[0] == _ffi.ERR_INVALID_ARGUMENT
    c, msg = code(fwd, None, None, None, None, 4, 3, 4, None, 4, None, 4, None, None)
    assert c == _ffi.ERR_INVALID_ARGUMENT and "null" in msg
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    c, msg = code(fwd, p, p, None, p, 3, 3, 4, p, 4, p, 4, None, None)
    assert c == _ffi.ERR_INVALID_ARGUMENT and "leading dimension" in msg
    assert _ffi.call(fwd, None, None, None, None, 0, 0, 4, None, 0, None, 0, None, None) == 0      # nothing to do
    bwd = "tfgk_spmm_max_bwd_f32"
    c, _ = code(bwd, None, None, None, None, 4, 3, -2, 4, None, 4, None, 4, None, 4, None, None, 4, None, None)
    assert c == _ffi.ERR_INVALID_ARGUMENT
    c, msg = code(bwd, p, p, None, p, 4, 3, 3, 4, None, 4, None, 4, None, 4, None, p, 4, None, None)
    assert c == _ffi.ERR_INVALID_ARGUMENT and "null" in msg
    c, msg = code(bwd, p, p, None, p, 4, 3, 3, 4, p, 4, p, 2, p, 4, p, p, 4, None, None)
    assert c == _ffi.ERR_INVALID_ARGUMENT and "leading dimension" in msg


def test_restatement_on_hand_made_rows():
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    # rows: 0 ties and +-0, 1 NaN and a tie, 2 empty, 3 only -inf, 4 only -FLT_MAX, 5 weighted
    h = np.array([[0.0], [-0.0], [2.0], [nan], [-inf], [LOWEST], [1.5]], np.float32)
    rowptr = np.array([0, 3, 6, 6, 7, 9, 11])
    col = np.array([0, 1, 0, 3, 2, 2, 4, 5, 5, 6, 2], np.int32)
    w = np.array([1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 1.5], np.float32)
    out, cnt = ref.k11a(rowptr, col, None, h)
    assert out[:, 0].tolist()[:2] == [0.0, 2.0] and cnt[:, 0].tolist() == [3, 2, 0, 0, 2, 1]
    assert out[2, 0] == LOWEST and out[3, 0] == LOWEST and out[4, 0] == LOWEST
    out_w, cnt_w = ref.k11a(rowptr, col, w, h)
    assert out_w[5, 0] == 3.0 and cnt_w[5, 0] == 2                    # 1.5 * 2 and 2 * 1.5 tie
    # backward: ties share, NaN upstream reaches every neighbour of its row (0 * NaN), an empty row sends nothing
    rowptr_t = np.array([0, 2, 3, 6, 7, 8, 10, 11])
    dst_t = np.array([0, 0, 0, 1, 1, 5, 1, 3, 4, 4, 5], np.int32)                   # source c -> destination rows
    g = np.array([[3.0], [nan], [1.0], [1.0], [5.0], [7.0]], np.float32)
    dh = ref.k11b(rowptr_t, dst_t, None, h, out, cnt, g)
    assert dh[0, 0] == 2.0 and dh[1, 0] == 1.0                        # 3 / 3 twice for node 0, once for node 1 (-0)
    assert np.isnan(dh[2, 0]) and np.isnan(dh[3, 0])                  # row 1's g is NaN: selected or not
    assert dh[5, 0] == 5.0 and dh[4, 0] == 0.0 and dh[6, 0] == 0.0    # 5 / 2 twice; -inf is never selected


def _max_sage_args(rs, n, f, units):
    k = units // 2
    return [torch.tensor(rs.randn(*s).astype(np.float32) * 0.3, requires_grad=True)
            for s in ((f, k), (f, 4 * k), (4 * k, k), (4 * k,), (units,))]


def test_max_pool_graph_sage_takes_k11_only_when_training(fake):
    tfg, calls = fake
    rs = np.random.RandomState(0)
    ei = torch.tensor(random_graph(40, 200, seed=1))
    x = torch.tensor(rs.randn(40, 6).astype(np.float32))
    ws, wm, wn, bm, b = _max_sage_args(rs, 40, 6, 8)
    w1 = torch.ones(ei.shape[1])
    with torch.no_grad():
        tfg.nn.max_pool_graph_sage(x, ei, w1, ws, wm, wn, bm, b, activation=tfg.nn.relu)
    assert calls == {"spmm_max": 0, "spmm_max_bwd": 0}
    out = tfg.nn.max_pool_graph_sage(x, ei, w1, ws, wm, wn, bm, b, activation=tfg.nn.relu)
    out.square().sum().backward()
    assert calls == {"spmm_max": 1, "spmm_max_bwd": 1}


def test_aggregate_neighbors_routes(fake):
    tfg, calls = fake
    from tf_geometric_b200.nn.kernel import map_reduce as mr
    rs = np.random.RandomState(2)
    ei = torch.tensor(random_graph(30, 150, seed=3))
    w = torch.tensor(rs.rand(150).astype(np.float32) + 0.5)
    x = torch.tensor(rs.randn(30, 5).astype(np.float32), requires_grad=True)
    for mapper, weight, updater in ((mr.identity_mapper, None, mr.sum_updater), (mr.gcn_mapper, w, mr.identity_updater)):
        before = calls["spmm_max"]
        tfg.nn.aggregate_neighbors(x, ei, weight, mapper, mr.max_reducer, updater).sum().backward()
        assert calls["spmm_max"] == before + 1
    before = dict(calls)
    wg = w.clone().requires_grad_()
    tfg.nn.aggregate_neighbors(x, ei, wg, mr.gcn_mapper, mr.max_reducer, mr.identity_updater).sum().backward()
    assert wg.grad is not None and calls == before                   # a weight that needs its gradient: generic route
    custom = lambda rx, nx, edge_weight=None: nx * 2.0                # noqa: E731
    tfg.nn.aggregate_neighbors(x, ei, None, custom, mr.max_reducer, mr.sum_updater).sum().backward()
    assert calls == before


def test_host_tensors_keep_the_composition(monkeypatch):
    import fake_backend
    fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops
    import tf_geometric_b200 as tfg
    monkeypatch.setattr(ops, "spmm_max", lambda *a: pytest.fail("NeighborMax took host tensors"))
    rs = np.random.RandomState(0)
    ei = torch.tensor(random_graph(20, 80, seed=4))
    x = torch.tensor(rs.randn(20, 6).astype(np.float32))
    ws, wm, wn, bm, b = _max_sage_args(rs, 20, 6, 4)
    tfg.nn.max_pool_graph_sage(x, ei, torch.ones(80), ws, wm, wn, bm, b).sum().backward()
    assert ws.grad is not None


def test_k11_route_is_bit_identical_to_the_composition_on_the_fake(monkeypatch):
    """Both routes through the numpy kernels: the forward and every gradient of max_pool_graph_sage agree bit for bit."""
    rs = np.random.RandomState(5)
    ei_np = random_graph(50, 300, seed=6)
    x_np = rs.randn(50, 7).astype(np.float32)
    g_np = rs.randn(50, 8).astype(np.float32)
    runs = []
    for use_k11 in (False, True):
        import fake_backend
        if use_k11:
            ref.install(monkeypatch)
        else:
            fake_backend.install(monkeypatch)
        import tf_geometric_b200 as tfg
        prs = np.random.RandomState(1)
        params = _max_sage_args(prs, 50, 7, 8)
        x = torch.tensor(x_np, requires_grad=True)
        out = tfg.nn.max_pool_graph_sage(x, torch.tensor(ei_np), torch.ones(ei_np.shape[1]), *params,
                                         activation=tfg.nn.relu)
        (out * torch.tensor(g_np)).sum().backward()
        runs.append([out.detach()] + [t.grad for t in [x] + params])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("weighted", [False, True])
def test_gradients_against_float64_autograd(fake, weighted):
    """aggregate_neighbors(max_reducer) through NeighborMax and the numpy K11 vs torch float64 autograd (scatter_reduce
    amax, which also shares the gradient equally among ties).  ReLU'd inputs make many ties at 0."""
    tfg, calls = fake
    from tf_geometric_b200.nn.kernel import map_reduce as mr
    rs = np.random.RandomState(7)
    n, d = 60, 9
    ei = random_graph(n, 400, seed=8, isolated=2)
    x_np = np.maximum(rs.randn(n, d), 0).astype(np.float32)
    w_np = (rs.rand(ei.shape[1]) + 0.5).astype(np.float32) if weighted else None
    g_np = rs.randn(n, d).astype(np.float32)
    x = torch.tensor(x_np, requires_grad=True)
    agg = tfg.nn.aggregate_neighbors(x, torch.tensor(ei), None if w_np is None else torch.tensor(w_np),
                                     mr.gcn_mapper if weighted else mr.identity_mapper, mr.max_reducer,
                                     mr.identity_updater)
    (agg * torch.tensor(g_np)).sum().backward()
    assert calls["spmm_max_bwd"] == 1
    x64 = torch.tensor(x_np, dtype=torch.float64, requires_grad=True)
    msg = x64[torch.tensor(ei[1]).long()]
    if weighted:
        msg = msg * torch.tensor(w_np, dtype=torch.float64).unsqueeze(1)
    idx = torch.tensor(ei[0]).long().unsqueeze(1).expand(-1, d)
    want = torch.full((n, d), float(LOWEST), dtype=torch.float64).scatter_reduce(0, idx, msg, "amax", include_self=False)
    (want * torch.tensor(g_np, dtype=torch.float64)).sum().backward()
    np.testing.assert_allclose(agg.detach().numpy(), want.detach().numpy(), rtol=1e-6, atol=0)
    np.testing.assert_allclose(x.grad.numpy(), x64.grad.numpy(), rtol=1e-5, atol=1e-6)
