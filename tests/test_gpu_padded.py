# coding=utf-8
"""K9 (padded row gather) on the H100: bit-exactness against numpy, the K1 backward of the neighbour case against
float64, determinism, the golden fixture made by executing the reference's own functions, gradients of convert_x_to_3d,
lstm_graph_sage and LSTMGraphSage against float64 autograd over the reference op sequence, the raises, and training."""
import os

import numpy as np
import pytest
import torch

import padded_fake_backend as np_k9
import padded_ref as ref
from conftest import assert_close, random_graph

pytestmark = pytest.mark.gpu

DEV = "cuda"
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "padded_exec.npz"))


def _dev(a, grad=False):
    t = torch.tensor(a, device=DEV)
    return t.requires_grad_(grad) if grad else t


def _csr(ei, n):
    from tf_geometric_b200 import ops
    e = _dev(ei)
    return ops.csr_build(e[0].contiguous(), e[1].contiguous(), n, n), e


def _np_csr(csr):
    return csr.rowptr.cpu().numpy(), csr.col.cpu().numpy(), csr.perm.cpu().numpy()


@pytest.mark.parametrize("D", [1, 3, 16, 64, 100, 128, 256, 602])
@pytest.mark.parametrize("step_major", [False, True])
@pytest.mark.parametrize("k_mode", ["below", "equal", "above"])
def test_pad_rows_bit_exact(D, step_major, k_mode):
    from tf_geometric_b200 import ops
    n = 300
    ei = random_graph(n, 1500, D, isolated=20, hub=(5, 40))            # 20 empty rows, one of in-degree >= 40
    csr, _ = _csr(ei, n)
    kmax = int(csr.degree_i64().max())
    K = {"below": kmax // 3, "equal": kmax, "above": kmax + 5}[k_mode]
    x = np.random.RandomState(D).randn(n, D).astype(np.float32)
    got, slot = ops.pad_rows(csr, _dev(x), K, step_major=step_major, slot_index=True)
    rowptr, col, _ = _np_csr(csr)
    want, want_slot = np_k9.pad_reference(rowptr, col, x, K, step_major)
    assert np.array_equal(got.cpu().numpy(), want)
    assert np.array_equal(slot.cpu().numpy(), want_slot)


@pytest.mark.parametrize("D", [3, 64, 100])
@pytest.mark.parametrize("step_major", [False, True])
def test_pad_rows_column_slice_odd_ld(D, step_major):
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(1)
    sid = rs.randint(0, 40, 500).astype(np.int32)
    sid[sid == 7] = 8                                                     # an empty group
    csr = ops.csr_build(_dev(sid), torch.zeros(500, dtype=torch.int32, device=DEV), 40, 1)
    wide = rs.randn(500, D + 7).astype(np.float32)                        # odd leading dimension D + 7
    x = _dev(wide)[:, 3:3 + D]
    rowptr, _, perm = _np_csr(csr)
    for K in (3, int(np.bincount(sid).max()) + 2):
        got = ops.pad_rows(csr, x, K, src=csr.perm, step_major=step_major)
        want, _ = np_k9.pad_reference(rowptr, perm, wide[:, 3:3 + D], K, step_major)
        assert np.array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("D", [1, 3, 64, 100, 128])
def test_unpad_rows_bit_exact_and_deterministic(D):
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(D)
    sid = rs.randint(0, 50, 3000).astype(np.int32)
    csr = ops.csr_build(_dev(sid), torch.zeros(3000, dtype=torch.int32, device=DEV), 50, 1)
    rowptr, _, perm = _np_csr(csr)
    for K in (10, int(np.bincount(sid).max())):
        G = rs.randn(50, K, D).astype(np.float32)
        got = ops.unpad_rows(csr, _dev(G))
        assert np.array_equal(got.cpu().numpy(), np_k9.unpad_reference(rowptr, perm, G))
        assert torch.equal(got, ops.unpad_rows(csr, _dev(G)))


@pytest.mark.parametrize("D", [1, 16, 100, 128])
@pytest.mark.parametrize("step_major", [False, True])
def test_neighbor_backward_matches_float64_and_is_deterministic(D, step_major):
    """dx[c] = sum over edges e with col_e = c of dPad[slot(e)]: K1 over the transposed CSR, with a source hub of
    out-degree 5000 (spread over the hub-row plan) and a destination hub of in-degree 2500."""
    from tf_geometric_b200 import autograd
    n = 3000
    rs = np.random.RandomState(D)
    ei = random_graph(n, 20000, D, hub=(11, 2500))
    ei = np.concatenate([ei, np.stack([rs.randint(0, n, 5000), np.full(5000, 17)]).astype(np.int32)], axis=1)
    csr, e = _csr(ei, n)
    K = int(csr.degree_i64().max())
    x = _dev(rs.randn(n, D).astype(np.float32), grad=True)
    out = autograd.PadRows.apply(x, csr, K, step_major, e)
    g = rs.randn(*out.shape).astype(np.float32)
    (dx,) = torch.autograd.grad(out, x, _dev(g))
    rowptr, col, _ = _np_csr(csr)
    _, slot = np_k9.pad_reference(rowptr, col, np.zeros((n, 1), np.float32), K, step_major)
    want = np.zeros((n, D))
    np.add.at(want, col, g.reshape(-1, D).astype(np.float64)[slot])
    assert_close(dx.cpu().numpy(), want)
    for _ in range(2):
        out2 = autograd.PadRows.apply(x, csr, K, step_major, e)
        assert torch.equal(out2, out)
        assert torch.equal(torch.autograd.grad(out2, x, _dev(g))[0], dx)


@pytest.mark.parametrize("tag,kw", [("none", {}), ("k2", {"k": 2}), ("k6_pad", {"k": 6, "pad": True}),
                                    ("k6_nopad", {"k": 6, "pad": False})])
def test_convert_x_to_3d_golden(tag, kw):
    import tf_geometric_b200 as tfg
    for x, sid in ((GOLDEN["x3d_x"], GOLDEN["x3d_sid"]), (_dev(GOLDEN["x3d_x"]), _dev(GOLDEN["x3d_sid"]))):
        got = tfg.utils.convert_x_to_3d(x, sid, **kw)
        assert got.is_cuda and np.array_equal(got.cpu().numpy(), GOLDEN["x3d_" + tag])


def _golden_case(tag):
    g = GOLDEN
    return (g["lstm_x"], g["lstm_ei"], g["lstm_%s_ws" % tag], g["lstm_%s_wn" % tag], g["lstm_%s_bias" % tag])


@pytest.mark.parametrize("tag", ["concat", "sum"])
def test_lstm_graph_sage_golden(tag):
    import tf_geometric_b200 as tfg
    x, ei, ws, wn, bias = _golden_case(tag)
    lstm = ref.torch_lstm(*(_dev(GOLDEN[k]) for k in ("lstm_k", "lstm_r", "lstm_b")))
    concat = tag == "concat"
    got = tfg.nn.lstm_graph_sage(_dev(x), _dev(ei), lstm, _dev(ws), _dev(wn), bias=_dev(bias), activation=tfg.nn.relu,
                                 concat=concat)
    assert_close(got.cpu().numpy(), GOLDEN["lstm_%s_relu" % tag])
    got = tfg.nn.lstm_graph_sage(x, ei, lstm, ws, wn, bias=bias, concat=concat, normalize=True)
    assert_close(got.cpu().numpy(), GOLDEN["lstm_%s_l2" % tag])


@pytest.mark.parametrize("tag", ["concat", "sum"])
def test_lstm_layer_golden_with_keras_weights(tag):
    import tf_geometric_b200 as tfg
    x, ei, ws, wn, bias = _golden_case(tag)
    layer = tfg.layers.LSTMGraphSage(8 if tag == "concat" else 4, activation=None, concat=tag == "concat", normalize=True)
    layer.load_keras_lstm_weights(GOLDEN["lstm_k"], GOLDEN["lstm_r"], GOLDEN["lstm_b"])
    with torch.no_grad():
        layer.self_kernel.copy_(_dev(ws))
        layer.neighbor_kernel.copy_(_dev(wn))
        layer.bias.copy_(_dev(bias))
    assert torch.backends.cudnn.allow_tf32                                 # torch's default is left alone
    got = layer([_dev(x), _dev(ei), _dev(GOLDEN["lstm_w"])])
    assert torch.backends.cudnn.allow_tf32
    assert_close(got.cpu().numpy(), GOLDEN["lstm_%s_l2" % tag])


def test_convert_x_to_3d_gradient_is_an_exact_gather():
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(3)
    sid = rs.randint(0, 300, 20000).astype(np.int32)
    x = _dev(rs.randn(20000, 37).astype(np.float32), grad=True)
    for k in (5, None, 200):
        out = tfg.utils.convert_x_to_3d(x, _dev(sid), k=k)
        g = _dev(rs.randn(*out.shape).astype(np.float32))
        (dx,) = torch.autograd.grad(out, x, g)
        j = np.zeros(20000, np.int64)
        seen = np.zeros(300, np.int64)
        for i, s in enumerate(sid):
            j[i] = seen[s]
            seen[s] += 1
        keep = j < out.shape[1]
        want = np.zeros((20000, 37), np.float32)
        want[keep] = g.cpu().numpy()[sid[keep], j[keep]]
        assert np.array_equal(dx.cpu().numpy(), want)
        assert torch.equal(torch.autograd.grad(tfg.utils.convert_x_to_3d(x, _dev(sid), k=k), x, g)[0], dx)


def _hub_graph(rs, n):
    ei = random_graph(n, 6 * n, 7, isolated=3, hub=(9, 2100))              # in-degree >= 2000: K > 2000 steps
    return np.concatenate([ei, ei[:, :1], np.array([[4], [4]], np.int32)], axis=1)     # a duplicate and a self loop


@pytest.mark.parametrize("concat,normalize", [(True, False), (False, True), (True, True)])
def test_lstm_graph_sage_gradients_match_float64(concat, normalize):
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(4)
    n, f, u = 2200, 6, 4
    ei = _hub_graph(rs, n)
    params = [rs.randn(f, 4 * u) * 0.3, rs.randn(u, 4 * u) * 0.3, rs.randn(4 * u) * 0.1, rs.randn(f, u) * 0.5,
              rs.randn(u, u) * 0.5, rs.randn(2 * u if concat else u) * 0.1, rs.randn(n, f)]
    p32 = [_dev(p.astype(np.float32), grad=True) for p in params]
    p64 = [_dev(p, grad=True) for p in params]
    got = tfg.nn.lstm_graph_sage(p32[6], _dev(ei), ref.torch_lstm(*p32[:3]), p32[3], p32[4], bias=p32[5],
                                 activation=torch.tanh, concat=concat, normalize=normalize)
    want = ref.lstm_graph_sage(p64[6], ei, ref.torch_lstm(*p64[:3]), p64[3], p64[4], bias=p64[5],
                               activation=torch.tanh, concat=concat, normalize=normalize)
    assert_close(got.detach().cpu().numpy(), want.detach().cpu().numpy())
    g = rs.randn(*want.shape)
    d32 = torch.autograd.grad(got, p32, _dev(g.astype(np.float32)))
    d64 = torch.autograd.grad(want, p64, _dev(g))
    for i, (a, b) in enumerate(zip(d32, d64)):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-3, atol_scale=1e-3, what="param %d" % i)


@pytest.mark.parametrize("concat,normalize", [(True, False), (False, True)])
def test_lstm_layer_gradients_match_float64_with_default_tf32(concat, normalize):
    """cuDNN's TF32 stays at torch's default (allow_tf32=True); the layer turns it off around its own forward and
    backward, so every gradient, the LSTM weights included, matches float64 autograd."""
    import tf_geometric_b200 as tfg
    assert torch.backends.cudnn.allow_tf32
    rs = np.random.RandomState(5)
    n, f = 2200, 6
    ei = _hub_graph(rs, n)
    units = 8 if concat else 4
    layer = tfg.layers.LSTMGraphSage(units, activation=torch.tanh, concat=concat, normalize=normalize, trainable=True,
                                     seed=1)
    x = _dev(rs.randn(n, f).astype(np.float32), grad=True)
    out = layer([x, _dev(ei)], training=True)
    assert torch.backends.cudnn.allow_tf32
    cell = layer.lstm
    p64 = [t.detach().double().requires_grad_(True) for t in (cell.weight_ih_l0.t(), cell.weight_hh_l0.t(),
                                                             cell.bias_ih_l0 + cell.bias_hh_l0, layer.self_kernel,
                                                             layer.neighbor_kernel, layer.bias, x)]
    want = ref.lstm_graph_sage(p64[6], ei, ref.torch_lstm(*p64[:3]), p64[3], p64[4], bias=p64[5], activation=torch.tanh,
                               concat=concat, normalize=normalize)
    assert_close(out.detach().cpu().numpy(), want.detach().cpu().numpy())
    g = rs.randn(*want.shape)
    mine = [cell.weight_ih_l0, cell.weight_hh_l0, cell.bias_ih_l0, cell.bias_hh_l0, layer.self_kernel,
            layer.neighbor_kernel, layer.bias, x]
    d32 = torch.autograd.grad(out, mine, _dev(g.astype(np.float32)))
    assert torch.backends.cudnn.allow_tf32
    d64 = torch.autograd.grad(want, p64, _dev(g))
    pairs = [(d32[0].t(), d64[0]), (d32[1].t(), d64[1]), (d32[2], d64[2]), (d32[3], d64[2]), (d32[4], d64[3]),
             (d32[5], d64[4]), (d32[6], d64[5]), (d32[7], d64[6])]
    for i, (a, b) in enumerate(pairs):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-3, atol_scale=1e-3, what="grad %d" % i)


def test_raises():
    import tf_geometric_b200 as tfg
    lstm = ref.torch_lstm(torch.zeros(3, 8, device=DEV), torch.zeros(2, 8, device=DEV), torch.zeros(8, device=DEV))
    w = _dev(np.zeros((3, 2), np.float32))
    with pytest.raises(ValueError, match="at least one edge"):
        tfg.nn.lstm_graph_sage(_dev(np.zeros((4, 3), np.float32)), _dev(np.zeros((2, 0), np.int32)), lstm, w,
                               _dev(np.zeros((2, 2), np.float32)))
    with pytest.raises(ValueError, match="rows but source_index"):
        tfg.utils.convert_x_to_3d(_dev(np.zeros((4, 3), np.float32)), _dev(np.array([0, 1, 1], np.int32)))
    with pytest.raises(ValueError, match="negative"):
        tfg.utils.convert_x_to_3d(_dev(np.zeros((3, 3), np.float32)), _dev(np.array([0, -1, 1], np.int32)))
    n = 1 << 21                                          # a hub of in-degree 1024: K * N = 2^31 padded slots
    x = torch.zeros((n, 4), device=DEV)
    ei = _dev(np.stack([np.zeros(1024, np.int32), np.arange(1024, dtype=np.int32)]))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="2\\^31"):
        tfg.nn.lstm_graph_sage(x, ei, lstm, _dev(np.zeros((4, 2), np.float32)), _dev(np.zeros((2, 2), np.float32)))
    assert torch.cuda.max_memory_allocated() - base < (256 << 20)            # nothing near K * N * F was allocated


def _planted(rs, n, k, p_in, p_out):
    labels = np.repeat(np.arange(k), n // k)
    same = labels[:, None] == labels[None, :]
    upper = np.triu(rs.rand(n, n) < np.where(same, p_in, p_out), 1)
    r, c = np.nonzero(upper)
    return np.stack([np.concatenate([r, c]), np.concatenate([c, r])]).astype(np.int32), labels


def test_two_layer_lstm_graph_sage_learns_planted_partition():
    """Node classification on a 4-community planted partition with weak, noisy features: two LSTMGraphSage layers over
    RandomNeighborSampler(k=10) neighbourhoods (the demo_graph_sage loop), trained on half the nodes, scored on the rest."""
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(0)
    n, c, f = 2000, 4, 16
    ei, labels = _planted(rs, n, c, 0.012, 0.0008)
    x = rs.randn(n, f).astype(np.float32)
    x[np.arange(n), labels] += 0.6
    x, y = _dev(x), _dev(labels.astype(np.int64))
    train = _dev(rs.permutation(n)[:n // 2].astype(np.int64))
    test = _dev(np.setdiff1d(np.arange(n), train.cpu().numpy()).astype(np.int64))
    sampler = tfg.utils.RandomNeighborSampler(_dev(ei))
    torch.manual_seed(0)
    sages = [tfg.layers.LSTMGraphSage(32, activation=tfg.nn.relu, trainable=True, seed=1),
             tfg.layers.LSTMGraphSage(32, activation=tfg.nn.relu, trainable=True, seed=2)]
    head = torch.nn.Linear(32, c, device=DEV)

    def forward(step, training):
        h = x
        for i, sage in enumerate(sages):
            sei, sw = sampler.sample(k=10, seed=1000 * step + i)
            h = sage([h, sei, sw], training=training)
        return head(h)

    forward(0, False)
    opt = torch.optim.Adam([p for s in sages for p in s.parameters()] + list(head.parameters()), lr=0.01)
    for step in range(80):
        loss = torch.nn.functional.cross_entropy(forward(step, True)[train], y[train])
        opt.zero_grad()
        loss.backward()
        opt.step()
    with torch.no_grad():
        acc = float((forward(10 ** 6, False)[test].argmax(1) == y[test]).float().mean())
    print("held-out accuracy", acc)
    assert acc >= 0.8, acc


def test_sort_pool_conv1d_classifies_community_counts():
    """The demo_sort_pool architecture: 3 x GCN -> SortPool(k) -> convert_x_to_3d with the pooled graph ids -> Conv1d ->
    MLP, separating graphs with 2 planted communities from graphs with 4 on held-out graphs."""
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(0)
    graphs = []
    for i in range(240):
        k = 2 if i % 2 == 0 else 4
        ei, _ = _planted(rs, 40, k, 0.5, 0.02)
        deg = np.minimum(np.bincount(ei[0], minlength=40), 15)
        x = np.zeros((40, 16), np.float32)
        x[np.arange(40), deg] = 1.0
        graphs.append((ei, x, k == 4))
    torch.manual_seed(0)
    kk = 10
    gcns = [tfg.layers.GCN(32, activation=tfg.nn.relu, trainable=True, seed=s) for s in (1, 2, 3)]
    pool = tfg.layers.SortPool(k=kk)
    conv = torch.nn.Conv1d(32, 32, 5, device=DEV)
    mlp = torch.nn.Sequential(torch.nn.Linear(32 * (kk - 4), 32), torch.nn.ReLU(), torch.nn.Linear(32, 2)).to(DEV)

    def forward(batch):
        eis, ngis, xs, base = [], [], [], 0
        for j, (ei, x, _) in enumerate(batch):
            eis.append(ei + base)
            ngis.append(np.full(40, j, np.int32))
            xs.append(x)
            base += 40
        ei, ngi, h = _dev(np.concatenate(eis, 1)), _dev(np.concatenate(ngis)), _dev(np.concatenate(xs))
        for gcn in gcns:
            h = gcn([h, ei])
        px, _, _, pngi = pool([h, ei, None, ngi])
        h3 = tfg.utils.convert_x_to_3d(px, pngi, k=kk)                    # [G, k, 32]
        h = torch.relu(conv(h3.transpose(1, 2)))
        return mlp(h.flatten(1))

    forward(graphs[:2])
    opt = torch.optim.Adam([p for g in gcns for p in g.parameters()] + list(conv.parameters()) + list(mlp.parameters()),
                           lr=0.01)
    train, test = graphs[:160], graphs[160:]
    for step in range(120):
        idx = np.random.RandomState(step).choice(len(train), 32, replace=False)
        batch = [train[i] for i in idx]
        y = torch.tensor([int(b[2]) for b in batch], device=DEV)
        loss = torch.nn.functional.cross_entropy(forward(batch), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
    with torch.no_grad():
        acc = float((forward(test).argmax(1).cpu().numpy() == np.array([int(b[2]) for b in test])).mean())
    print("held-out accuracy", acc)
    assert acc >= 0.8, acc
