# coding=utf-8
"""convert_x_to_3d and LSTM GraphSAGE without a GPU: the host logic (grouping, k rules, the raises, the layer's weight
loading and sequence-major feed, the gradient routes) over the CPU fake of the kernel layer with a numpy K9, and the
golden fixture made by executing the reference's own functions replayed through the public API."""
import os

import numpy as np
import pytest
import torch

import padded_fake_backend as fake_k9
import padded_ref as ref
from conftest import assert_close, random_graph

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "padded_exec.npz"))


@pytest.fixture
def fake(monkeypatch):
    fake_k9.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg


def test_ffi_declares_k9():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    assert len(_ffi.SIGNATURES["tfgk_pad_rows_f32"]) == 12 and len(_ffi.SIGNATURES["tfgk_unpad_rows_f32"]) == 9


def test_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_pad_rows_f32", None, None, 4, 3, 2, None, 4, 4, 4, None, None, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "layout" in str(err.value)
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_pad_rows_f32", None, None, 1 << 20, 1 << 11, 1, None, 4, 4, 4, None, 8, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "int32 slot index" in str(err.value)
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_unpad_rows_f32", None, None, 4, -1, None, 4, None, 4, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT


def test_fake_kernels_are_the_definition():
    rowptr = np.array([0, 2, 2, 5])
    src = np.array([4, 1, 0, 3, 2], np.int32)
    X = np.arange(10, dtype=np.float32).reshape(5, 2)
    out, slot = fake_k9.pad_reference(rowptr, src, X, 2)
    assert np.array_equal(out[0], X[[4, 1]]) and np.all(out[1] == 0) and np.array_equal(out[2], X[[0, 3]])
    assert slot.tolist() == [0, 1, 4, 5, -1]
    step, slot_s = fake_k9.pad_reference(rowptr, src, X, 2, step_major=True)
    assert np.array_equal(step, out.transpose(1, 0, 2)) and slot_s.tolist() == [0, 3, 2, 5, -1]
    G = np.arange(12, dtype=np.float32).reshape(3, 2, 2)
    back = fake_k9.unpad_reference(rowptr, src, G)
    assert np.array_equal(back[4], G[0, 0]) and np.array_equal(back[1], G[0, 1]) and np.all(back[2] == 0)


@pytest.mark.parametrize("tag,kw", [("none", {}), ("k2", {"k": 2}), ("k6_pad", {"k": 6, "pad": True}),
                                    ("k6_nopad", {"k": 6, "pad": False})])
def test_convert_x_to_3d_golden(fake, tag, kw):
    x, sid = GOLDEN["x3d_x"], GOLDEN["x3d_sid"]
    got = fake.utils.convert_x_to_3d(x, sid, **kw)
    assert torch.is_tensor(got)
    want = GOLDEN["x3d_" + tag]
    assert got.shape == want.shape and np.array_equal(got.numpy(), want)
    assert np.array_equal(want, ref.convert_x_to_3d(x, sid, **kw))
    from tf_geometric_b200.utils.graph_utils import convert_x_to_3d
    assert np.array_equal(convert_x_to_3d(torch.tensor(x), torch.tensor(sid), **kw).numpy(), want)


def _golden_case(tag):
    g = GOLDEN
    return (g["lstm_x"], g["lstm_ei"], g["lstm_%s_ws" % tag], g["lstm_%s_wn" % tag], g["lstm_%s_bias" % tag])


@pytest.mark.parametrize("tag", ["concat", "sum"])
def test_lstm_graph_sage_golden(fake, tag):
    x, ei, ws, wn, bias = _golden_case(tag)
    lstm = ref.torch_lstm(*(torch.tensor(GOLDEN[k]) for k in ("lstm_k", "lstm_r", "lstm_b")))
    concat = tag == "concat"
    got = fake.nn.lstm_graph_sage(x, ei, lstm, ws, wn, bias=bias, activation=fake.nn.relu, concat=concat)
    assert_close(got.numpy(), GOLDEN["lstm_%s_relu" % tag], what="relu")
    got = fake.nn.lstm_graph_sage(x, ei, lstm, ws, wn, bias=bias, concat=concat, normalize=True)
    assert_close(got.numpy(), GOLDEN["lstm_%s_l2" % tag], what="l2")


@pytest.mark.parametrize("tag", ["concat", "sum"])
def test_lstm_layer_golden_with_keras_weights(fake, tag):
    x, ei, ws, wn, bias = _golden_case(tag)
    layer = fake.layers.LSTMGraphSage(8 if tag == "concat" else 4, activation=None, concat=tag == "concat",
                                      normalize=True)
    layer.load_keras_lstm_weights(GOLDEN["lstm_k"], GOLDEN["lstm_r"], GOLDEN["lstm_b"])
    with torch.no_grad():
        layer.self_kernel.copy_(torch.tensor(ws))
        layer.neighbor_kernel.copy_(torch.tensor(wn))
        layer.bias.copy_(torch.tensor(bias))
    # the edge weight is accepted and ignored, as in the reference
    got = layer([torch.tensor(x), torch.tensor(ei), torch.tensor(GOLDEN["lstm_w"])])
    assert_close(got.detach().numpy(), GOLDEN["lstm_%s_l2" % tag])


def test_layer_keras_initialisation(fake):
    layer = fake.layers.LSTMGraphSage(8, seed=3)
    x = np.random.RandomState(0).randn(6, 5).astype(np.float32)
    layer([x, np.array([[0, 1, 2], [1, 2, 0]], np.int32)])
    cell = layer.lstm
    assert tuple(cell.weight_ih_l0.shape) == (16, 5) and tuple(cell.weight_hh_l0.shape) == (16, 4)
    rec = cell.weight_hh_l0.detach().t()                                  # Keras [U, 4U], orthogonal rows
    assert_close((rec @ rec.t()).numpy(), np.eye(4), atol_scale=1e-5)
    assert cell.bias_ih_l0[4:8].eq(1).all() and cell.bias_ih_l0[:4].eq(0).all() and cell.bias_hh_l0.eq(0).all()
    limit = np.sqrt(6.0 / (5 + 16))
    assert float(cell.weight_ih_l0.abs().max()) <= limit
    assert tuple(layer.neighbor_kernel.shape) == (4, 4) and tuple(layer.self_kernel.shape) == (5, 4)
    with pytest.raises(Exception):
        fake.layers.LSTMGraphSage(7)


def test_convert_x_to_3d_gradient_is_a_gather(fake):
    rs = np.random.RandomState(1)
    sid = rs.randint(0, 5, 40).astype(np.int32)
    x = torch.tensor(rs.randn(40, 3).astype(np.float32), requires_grad=True)
    for k in (2, None, 50):
        out = fake.utils.convert_x_to_3d(x, sid, k=k)
        g = torch.tensor(rs.randn(*out.shape).astype(np.float32))
        (dx,) = torch.autograd.grad(out, x, g)
        want = torch.zeros_like(x)
        seen = np.zeros(5, np.int64)
        for i, s in enumerate(sid):
            if seen[s] < out.shape[1]:
                want[i] = g[s, seen[s]]
            seen[s] += 1
        assert torch.equal(dx, want)


@pytest.mark.parametrize("concat,normalize", [(True, False), (False, True)])
def test_lstm_graph_sage_gradients_match_float64(fake, concat, normalize):
    rs = np.random.RandomState(2)
    n, f, u = 30, 4, 3
    ei = random_graph(n, 120, 5, isolated=2, hub=(7, 25))
    params = [rs.randn(f, 4 * u) * 0.4, rs.randn(u, 4 * u) * 0.4, rs.randn(4 * u) * 0.1, rs.randn(f, u) * 0.5,
              rs.randn(u, u) * 0.5, rs.randn(2 * u if concat else u) * 0.1, rs.randn(n, f)]
    p32 = [torch.tensor(p.astype(np.float32), requires_grad=True) for p in params]
    p64 = [torch.tensor(p, requires_grad=True) for p in params]
    act = torch.tanh
    got = fake.nn.lstm_graph_sage(p32[6], ei, ref.torch_lstm(*p32[:3]), p32[3], p32[4], bias=p32[5], activation=act,
                                  concat=concat, normalize=normalize)
    want = ref.lstm_graph_sage(p64[6], ei, ref.torch_lstm(*p64[:3]), p64[3], p64[4], bias=p64[5], activation=act,
                               concat=concat, normalize=normalize)
    assert_close(got.detach().numpy(), want.detach().numpy())
    g = rs.randn(*want.shape)
    d32 = torch.autograd.grad(got, p32, torch.tensor(g.astype(np.float32)))
    d64 = torch.autograd.grad(want, p64, torch.tensor(g))
    for i, (a, b) in enumerate(zip(d32, d64)):
        assert_close(a.numpy(), b.numpy(), rtol=1e-3, atol_scale=1e-3, what="param %d" % i)


def test_raises(fake):
    lstm = ref.torch_lstm(torch.zeros(3, 8), torch.zeros(2, 8), torch.zeros(8))
    w = torch.zeros(3, 2)
    with pytest.raises(ValueError, match="at least one edge"):
        fake.nn.lstm_graph_sage(np.zeros((4, 3), np.float32), np.zeros((2, 0), np.int32), lstm, w, torch.zeros(2, 2))
    with pytest.raises(ValueError, match="rows but source_index"):
        fake.utils.convert_x_to_3d(np.zeros((4, 3), np.float32), np.array([0, 1, 1], np.int32))
    with pytest.raises(ValueError, match="negative"):
        fake.utils.convert_x_to_3d(np.zeros((3, 3), np.float32), np.array([0, -1, 1], np.int32))
    n = 1 << 21                                          # a hub of in-degree 1024: K * N = 2^31 padded slots
    ei = np.stack([np.zeros(1024, np.int32), np.arange(1024, dtype=np.int32)])
    with pytest.raises(ValueError, match="2\\^31"):
        fake.nn.lstm_graph_sage(torch.zeros((n, 1)), ei, lstm, torch.zeros(1, 2), torch.zeros(2, 2))
