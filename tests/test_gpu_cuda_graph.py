# coding=utf-8
"""CUDA-graph capture on the H100: captured inference forwards and whole training steps against eager runs, bit for bit.

Inference: one eager warm-up, capture, copy a new x into the static input, replay, compare with an eager forward on that x.
Training: forward, loss, backward and Adam(capturable=True).step() in one graph; replay e draws its dropout masks from the
device keys of base_e (the value of the device buffer after the replay's own advance), so an eager step run after
tfg.set_seed(base_e) must leave the same parameters."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tf_geometric_b200 as tfg
from tf_geometric_b200 import _rng, ops, autograd
from conftest import random_graph

pytestmark = pytest.mark.gpu

MASK64 = (1 << 64) - 1


def _graph(n, pairs, seed, hub=None, features=32):
    ei = random_graph(n, 2 * pairs, seed=seed, symmetric=True, hub=hub)
    rs = np.random.RandomState(seed + 1)
    x = torch.from_numpy(rs.randn(n, features).astype(np.float32)).cuda()
    return tfg.Graph(x, torch.from_numpy(ei).cuda()), x


@pytest.fixture(scope="module")
def cora():
    return _graph(2708, 5278, 3)


@pytest.fixture(scope="module")
def hub_graph():
    # a node with in-degree 60 000: the CSR gets a work plan with hub slices, and the plan path is captured
    return _graph(200000, 400000, 5, hub=(17, 60000))


def _capture(fn, x_static):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn(x_static)
    return g, out


def _assert_replay_matches_eager(fn, x):
    fn(x)                                      # eager warm-up: caches, plans, kernel attributes
    torch.cuda.synchronize()
    static_x = x.clone()
    g, out = _capture(fn, static_x)
    new_x = torch.randn_like(x)
    static_x.copy_(new_x)
    g.replay()
    torch.cuda.synchronize()
    want = fn(new_x)
    torch.cuda.synchronize()
    outs, wants = (out, want) if isinstance(out, tuple) else ((out,), (want,))
    for o_, w_ in zip(outs, wants):
        assert o_.dtype == w_.dtype and o_.shape == w_.shape
        assert torch.equal(o_, w_), "replay differs from eager: max |diff| {}".format((o_.float() - w_.float()).abs().max())


INFERENCE_LAYERS = {
    "gcn_fp32": lambda: (tfg.layers.GCN(16, activation=tfg.nn.relu, seed=1), True),
    "gcn_bf16": lambda: (tfg.layers.GCN(16, activation=tfg.nn.relu, seed=1, message_dtype=torch.bfloat16), True),
    "gcn_fp8": lambda: (tfg.layers.GCN(32, activation=tfg.nn.relu, seed=1, message_dtype=torch.float8_e4m3fn), True),
    "gat_packed": lambda: (tfg.layers.GAT(64, num_heads=8, activation=tfg.nn.relu, seed=1), False),
    "gat_dense_keys": lambda: (tfg.layers.GAT(64, num_heads=8, activation=tfg.nn.relu, seed=1), False),
    "gat_bf16": lambda: (tfg.layers.GAT(64, num_heads=8, activation=tfg.nn.relu, seed=1, message_dtype=torch.bfloat16),
                         False),
    "mean_sage": lambda: (tfg.layers.MeanGraphSage(32, seed=1), False),
    "maxpool_sage": lambda: (tfg.layers.MaxPoolGraphSage(32, seed=1), True),        # pooling variants take weights
    "appnp": lambda: (tfg.layers.APPNP([32, 7], k=10, seed=1), True),
    "sgc": lambda: (tfg.layers.SGC(7, k=2, seed=1), True),
    "gin": lambda: (tfg.layers.GIN(lambda h: h), False),
    "chebynet": lambda: (tfg.layers.ChebyNet(16, 3, seed=1), True),
}


@pytest.mark.parametrize("which", ["cora", "hub"])
@pytest.mark.parametrize("name", sorted(INFERENCE_LAYERS))
def test_captured_inference_matches_eager(name, which, cora, hub_graph, monkeypatch):
    if name == "gat_dense_keys":
        monkeypatch.setenv("TFGK_GAT_KEYS", "dense")
    graph, x = cora if which == "cora" else hub_graph
    layer, weighted = INFERENCE_LAYERS[name]()
    cache = graph.cache if weighted else None
    if isinstance(layer, tfg.layers.GIN):
        fn = lambda xd: layer([xd, graph.edge_index])                                        # noqa: E731
    elif weighted:
        fn = lambda xd: layer([xd, graph.edge_index, graph.edge_weight], cache=cache)        # noqa: E731
    else:
        fn = lambda xd: layer([xd, graph.edge_index], cache=cache)                           # noqa: E731
    _assert_replay_matches_eager(fn, x)


@pytest.mark.parametrize("which", ["cora", "hub"])
def test_captured_sparse_matmul_matches_eager(which, cora, hub_graph):
    graph, x = cora if which == "cora" else hub_graph
    n = x.shape[0]
    w = torch.rand(graph.edge_index.shape[1], device="cuda") + 0.1
    adj = tfg.SparseMatrix(graph.edge_index, w, [n, n])
    _assert_replay_matches_eager(lambda xd: adj @ xd, x)


# ---- training steps --------------------------------------------------------------------------------------------------
# Every step ends with a probe: a dropout mask drawn like the model's own masks, returned so that the test can look at a
# mask each replay really applied.

PROBE_RATE, PROBE_N = 0.3, 1 << 16


def _epoch_value(word):
    return int(word.item()) & MASK64


def _probe(ones):
    return ops.dropout(ones, PROBE_RATE, _rng.resolve(None, ones.device))


def _check_probe(got, want, prev):
    """The replay's probe mask equals the eager one, keeps a fraction within 5 binomial sigmas of 1 - rate, and differs
    from the previous replay's."""
    assert torch.equal(got, want)
    keep = got != 0
    p = 1.0 - PROBE_RATE
    frac = keep.float().mean().item()
    assert abs(frac - p) <= 5 * np.sqrt(p * (1 - p) / keep.numel()), (frac, p)
    if prev is not None:
        assert not torch.equal(keep, prev)
    return keep


def _gcn_model(graph):
    l1 = tfg.layers.GCN(16, activation=tfg.nn.relu, edge_drop_rate=0.5, seed=1, trainable=True)
    l2 = tfg.layers.GCN(7, edge_drop_rate=0.5, seed=2, trainable=True)

    def fwd(x):
        h = autograd.dropout(x, 0.5, True)
        h = l1([h, graph.edge_index, graph.edge_weight], cache=graph.cache, training=True)
        h = autograd.dropout(h, 0.5, True)
        return l2([h, graph.edge_index, graph.edge_weight], cache=graph.cache, training=True)
    return fwd, [l1, l2]


def _gat_model(graph):
    l1 = tfg.layers.GAT(64, num_heads=8, attention_units=8, activation=tfg.nn.relu, edge_drop_rate=0.3, seed=1,
                        trainable=True)
    l2 = tfg.layers.GAT(7, num_heads=1, attention_units=8, edge_drop_rate=0.3, seed=2, trainable=True)

    def fwd(x):
        h = l1([x, graph.edge_index], cache=graph.cache, training=True)
        return l2([h, graph.edge_index], cache=graph.cache, training=True)
    return fwd, [l1, l2]


def _sage_model(graph):
    l1 = tfg.layers.MeanGraphSage(16, activation=tfg.nn.relu, seed=1, trainable=True)
    l2 = tfg.layers.MeanGraphSage(7, activation=None, concat=False, seed=2, trainable=True)

    def fwd(x):
        h = autograd.dropout(x, 0.4, True)
        h = l1([h, graph.edge_index], training=True)
        h = autograd.dropout(h, 0.4, True)
        return l2([h, graph.edge_index], training=True)
    return fwd, [l1, l2]


def _params(layers):
    return [p for layer in layers for p in layer.parameters()]


@pytest.mark.parametrize("model", [_gcn_model, _gat_model, _sage_model], ids=["gcn", "gat", "mean_sage"])
def test_captured_training_step_matches_eager(model, cora):
    graph, x = cora
    labels = torch.from_numpy(np.random.RandomState(4).randint(0, 7, x.shape[0])).cuda()
    train_idx = torch.arange(0, x.shape[0], 3, device="cuda")
    ones = torch.ones(PROBE_N, device="cuda")

    def make():
        fwd, layers = model(graph)
        fwd(x)                                                             # builds the layers
        opt = torch.optim.Adam(_params(layers), lr=0.01, capturable=True)

        def step():
            loss = F.cross_entropy(fwd(x)[train_idx], labels[train_idx])
            loss.backward()
            opt.step()
            return _probe(ones)
        return step, layers, opt

    captured, cap_layers, cap_opt = make()
    eager, eager_layers, eager_opt = make()
    for step, opt in ((captured, cap_opt), (eager, eager_opt)):          # the same eager warm-up step on both
        tfg.set_seed(123)
        opt.zero_grad(set_to_none=True)
        step()
    for a, b in zip(_params(cap_layers), _params(eager_layers)):
        assert torch.equal(a, b)

    torch.cuda.synchronize()
    cap_opt.zero_grad(set_to_none=True)
    n_epochs = len(_rng.capture_epochs())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        probe = captured()
    word = _rng.capture_epochs()[n_epochs]

    prev = None
    for e in range(5):
        g.replay()
        torch.cuda.synchronize()
        base = _epoch_value(word)
        assert base == _epoch_value(_rng.key_base())                       # the only graph that draws
        tfg.set_seed(base)
        eager_opt.zero_grad(set_to_none=True)
        want = eager()
        torch.cuda.synchronize()
        for a, b in zip(_params(cap_layers), _params(eager_layers)):
            assert torch.equal(a, b), "replay {}: parameters differ from the eager step under set_seed(base_e)".format(e)
        prev = _check_probe(probe, want, prev)


class _GatStage(torch.nn.Module):
    """Dense dropout, a GAT layer with attention dropout, and a probe mask.  make_graphed_callables takes tensor arguments:
    the graph and its cache live on the module."""

    def __init__(self, graph, units, heads, seed):
        super().__init__()
        self.graph = graph
        self.layer = tfg.layers.GAT(units, num_heads=heads, attention_units=8, activation=tfg.nn.relu if heads > 1 else None,
                                    edge_drop_rate=0.3, seed=seed, trainable=True)
        self.ones = torch.ones(PROBE_N, device="cuda")

    def forward(self, x):
        h = autograd.dropout(x, 0.5, True)
        h = self.layer([h, self.graph.edge_index], cache=self.graph.cache, training=True)
        return h, _probe(self.ones)


class _GatNet(torch.nn.Module):
    def __init__(self, graph):
        super().__init__()
        self.s1, self.s2 = _GatStage(graph, 64, 8, 1), _GatStage(graph, 7, 1, 2)

    def forward(self, x):
        h, p1 = self.s1(x)
        out, p2 = self.s2(h)
        return out, p1, p2


def _two_nets(graph, x):
    nets = []
    for _ in range(2):
        net = _GatNet(graph)
        net(x)                                                             # builds the layers
        nets.append(net)
    for a, b in zip(nets[0].parameters(), nets[1].parameters()):
        assert torch.equal(a, b)
    torch.cuda.synchronize()
    return nets


def test_make_graphed_callables_gat_matches_eager(cora):
    graph, x = cora
    labels = torch.from_numpy(np.random.RandomState(4).randint(0, 7, x.shape[0])).cuda()
    graphed_net, eager_net = _two_nets(graph, x)
    n_epochs = len(_rng.capture_epochs())
    graphed = torch.cuda.make_graphed_callables(graphed_net, (x,))
    (word,) = _rng.capture_epochs()[n_epochs:]                            # the forward graph draws, the backward does not
    opts = [torch.optim.Adam(n.parameters(), lr=0.01) for n in (graphed_net, eager_net)]
    prev = None
    for e in range(5):
        opts[0].zero_grad(set_to_none=True)
        out, p1, p2 = graphed(x)
        F.cross_entropy(out, labels).backward()
        opts[0].step()
        torch.cuda.synchronize()
        tfg.set_seed(_epoch_value(word))
        opts[1].zero_grad(set_to_none=True)
        out_e, q1, q2 = eager_net(x)
        F.cross_entropy(out_e, labels).backward()
        opts[1].step()
        torch.cuda.synchronize()
        for a, b in zip(graphed_net.parameters(), eager_net.parameters()):
            assert torch.equal(a, b), "replay {}: parameters differ from the eager step under set_seed(base_e)".format(e)
        assert torch.equal(p1, q1)
        prev = _check_probe(p2, q2, prev)


def test_make_graphed_callables_over_two_modules_matches_eager(cora):
    # torch replays the forward graphs of both modules before either backward graph: module 1's backward must still
    # regenerate module 1's masks, not the ones module 2's forward drew after it
    graph, x = cora
    labels = torch.from_numpy(np.random.RandomState(4).randint(0, 7, x.shape[0])).cuda()
    graphed_net, eager_net = _two_nets(graph, x)
    h_sample = graphed_net.s1(x)[0].detach().requires_grad_(True)
    n_epochs = len(_rng.capture_epochs())
    g1, g2 = torch.cuda.make_graphed_callables((graphed_net.s1, graphed_net.s2), ((x,), (h_sample,)))
    w1, w2 = _rng.capture_epochs()[n_epochs:]                              # one word per drawing forward graph
    opts = [torch.optim.Adam(n.parameters(), lr=0.01) for n in (graphed_net, eager_net)]
    prev = None
    for e in range(5):
        opts[0].zero_grad(set_to_none=True)
        h, p1 = g1(x)
        out, p2 = g2(h)
        F.cross_entropy(out, labels).backward()
        opts[0].step()
        torch.cuda.synchronize()
        b1, b2 = _epoch_value(w1), _epoch_value(w2)
        assert b1 != b2
        opts[1].zero_grad(set_to_none=True)
        tfg.set_seed(b1)
        h_e, q1 = eager_net.s1(x)
        tfg.set_seed(b2)
        out_e, q2 = eager_net.s2(h_e)
        F.cross_entropy(out_e, labels).backward()
        opts[1].step()
        torch.cuda.synchronize()
        for a, b in zip(graphed_net.parameters(), eager_net.parameters()):
            assert torch.equal(a, b), "replay {}: parameters differ from the eager steps under set_seed(b1), set_seed(b2)" \
                .format(e)
        assert torch.equal(p2, q2)
        prev = _check_probe(p1, q1, prev)


def test_set_seed_is_refused_under_capture(cora):
    graph, x = cora
    autograd.dropout(x, 0.5, True)                                         # an eager draw creates the device-key base
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="set_seed cannot be captured"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            tfg.set_seed(7)


# ---- refusals --------------------------------------------------------------------------------------------------------

def test_capture_refuses_host_synchronising_ops(cora):
    graph, x = cora
    layer = tfg.layers.GCN(16, seed=1)
    layer([x, graph.edge_index, graph.edge_weight], cache=graph.cache)
    fresh = graph.edge_index.clone()                                       # no cached CSR for this tensor
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="cannot be captured in a CUDA graph"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            layer([x, fresh])
    score = torch.rand(x.shape[0], device="cuda")
    source = torch.from_numpy(np.repeat(np.arange(10), (x.shape[0] + 9) // 10)[:x.shape[0]].astype(np.int32)).cuda()
    with pytest.raises(RuntimeError, match="topk_pool cannot be captured in a CUDA graph"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            tfg.nn.topk_pool(source, score, ratio=0.5)
    # the process is still usable eagerly
    got = layer([x, fresh])
    want = layer([x, graph.edge_index])
    assert torch.equal(got, want)
    assert tfg.nn.topk_pool(source, score, ratio=0.5).numel() == sum((c + 1) // 2 for c in np.bincount(source.cpu().numpy()))
