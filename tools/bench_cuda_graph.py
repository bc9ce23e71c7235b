# coding=utf-8
"""Eager calls against CUDA-graph replays of the same step, on one GPU.

Workloads:
  cfg1_forward   Cora-shaped 2-layer GCN forward with sparse bag-of-words features (bench.py cfg1): launch-bound
  gcn_train      demo_gcn training step: GCN(16, relu) -> GCN(7), dropout 0.5, Adam, Cora-shaped graph, dense x
  gat_train      demo_gat training step: GAT(64, 8 heads, attention_units=8, relu, attention dropout 0.6) -> GAT(7, 1 head)
  products_fwd   GCN(128, relu) + GAT(128, 8 heads, relu) forward, ogbn-products shape (bench.py headline): kernel-bound,
                 where eager and replay should agree within noise

Each workload first checks that a replay computes the same bits as the eager call (training: the parameters after one
replay equal those of an eager step run after tfg.set_seed(base), base read from the device-key buffer), then times
eager and replay alternately with CUDA events and reports medians.  The card's name and power limit are read in the
same run.  Prints one JSON object.

    python tools/bench_cuda_graph.py [--iters 200] [--skip-products]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import tf_geometric_b200 as tfg                                   # noqa: E402
from tf_geometric_b200 import _rng, autograd                      # noqa: E402
from bench import make_graph_device, PRODUCTS_NODES, PRODUCTS_UNDIRECTED   # noqa: E402

MASK64 = (1 << 64) - 1


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = [v.strip() for v in q.stdout.strip().split(",")]
        out.update(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as err:                                       # the numbers are still reported, without the limit
        out["power_limit"] = "unavailable ({})".format(err)
    return out


def time_alternating(eager, replay, iters):
    """Median ms of eager() and replay() over `iters` alternating pairs, each bracketed by CUDA events."""
    te, tr = [], []
    for _ in range(iters):
        for fn, acc in ((eager, te), (replay, tr)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            acc.append(a.elapsed_time(b))
    return float(np.median(te)), float(np.median(tr))


def capture(fn):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def forward_case(fn, static_x, new_x, iters):
    fn()                                                           # warm-up: caches, plans, kernel attributes
    torch.cuda.synchronize()
    g, out = capture(fn)
    static_x.copy_(new_x)
    g.replay()
    want = fn()
    torch.cuda.synchronize()
    same = all(torch.equal(a, b) for a, b in zip(out, want))
    eager_ms, replay_ms = time_alternating(fn, g.replay, iters)
    return {"bit_identical": same, "eager_ms": eager_ms, "replay_ms": replay_ms, "speedup": eager_ms / replay_ms}


def training_case(make, iters):
    """make() -> (step, params, optimizer); two identical models, the same eager warm-up step, one captured.  The
    captured step allocates its gradients inside the graph, as the eager step does after zero_grad(set_to_none=True)."""
    (cap_step, cap_params, cap_opt), (eager_step, eager_params, _) = make(), make()
    for step in (cap_step, eager_step):
        tfg.set_seed(1)
        step(zero=True)
    torch.cuda.synchronize()
    cap_opt.zero_grad(set_to_none=True)
    g, _ = capture(lambda: cap_step(zero=False))
    g.replay()
    torch.cuda.synchronize()
    tfg.set_seed(int(_rng.key_base(torch.device("cuda")).item()) & MASK64)
    eager_step(zero=True)
    torch.cuda.synchronize()
    same = all(torch.equal(a, b) for a, b in zip(cap_params, eager_params))
    eager_ms, replay_ms = time_alternating(lambda: eager_step(zero=True), g.replay, iters)
    return {"bit_identical": same, "eager_ms": eager_ms, "replay_ms": replay_ms, "speedup": eager_ms / replay_ms}


def cora_graph(device):
    return tfg.Graph(torch.zeros((2708, 1), device=device), make_graph_device(2708, 5278, 0, device))


def cfg1_forward(device, iters):
    n, feats = 2708, 1433
    graph = cora_graph(device)
    gen = torch.Generator(device="cpu").manual_seed(1)
    dense = (torch.rand((n, feats), generator=gen) < 18.0 / feats).float()
    dense = dense / dense.sum(1, keepdim=True).clamp(min=1.0)
    nz = torch.nonzero(dense, as_tuple=True)
    pattern = tfg.SparseMatrix(torch.stack(nz).to(torch.int32).to(device), dense[nz].to(device), [n, feats])
    pattern.csr
    static_x = dense[nz].to(device)
    l1 = tfg.layers.GCN(16, activation=tfg.nn.relu, seed=2)
    l2 = tfg.layers.GCN(7, seed=3)
    l1.build_cache_for_graph(graph)

    def fn():
        h = l1([pattern.with_value(static_x), graph.edge_index, graph.edge_weight], cache=graph.cache)
        return (l2([h, graph.edge_index, graph.edge_weight], cache=graph.cache),)
    return forward_case(fn, static_x, torch.rand_like(static_x), iters)


def _train_step(fwd, layers, x, labels, idx):
    fwd(x)                                                         # builds the layers
    params = [p for layer in layers for p in layer.parameters()]
    opt = torch.optim.Adam(params, lr=0.01, capturable=True)

    def step(zero):
        if zero:
            opt.zero_grad(set_to_none=True)
        loss = F.cross_entropy(fwd(x)[idx], labels[idx])
        loss.backward()
        opt.step()
        return loss
    return step, params, opt


def gcn_train(device, iters):
    graph = cora_graph(device)
    gen = torch.Generator(device="cpu").manual_seed(2)
    x = (torch.rand((2708, 1433), generator=gen) < 18.0 / 1433).float().to(device)
    labels = torch.randint(0, 7, (2708,), generator=gen).to(device)
    idx = torch.arange(140, device=device)                        # Planetoid's 20 training nodes per class

    def make():
        l1 = tfg.layers.GCN(16, activation=tfg.nn.relu, seed=1, trainable=True)
        l2 = tfg.layers.GCN(7, seed=2, trainable=True)

        def fwd(xd):
            h = autograd.dropout(xd, 0.5, True)
            h = l1([h, graph.edge_index, graph.edge_weight], cache=graph.cache, training=True)
            h = autograd.dropout(h, 0.5, True)
            return l2([h, graph.edge_index, graph.edge_weight], cache=graph.cache, training=True)
        return _train_step(fwd, [l1, l2], x, labels, idx)
    return training_case(make, iters)


def gat_train(device, iters):
    graph = cora_graph(device)
    gen = torch.Generator(device="cpu").manual_seed(3)
    x = (torch.rand((2708, 1433), generator=gen) < 18.0 / 1433).float().to(device)
    labels = torch.randint(0, 7, (2708,), generator=gen).to(device)
    idx = torch.arange(140, device=device)

    def make():
        l1 = tfg.layers.GAT(64, num_heads=8, attention_units=8, activation=tfg.nn.relu, edge_drop_rate=0.6, seed=1,
                            trainable=True)
        l2 = tfg.layers.GAT(7, num_heads=1, attention_units=8, edge_drop_rate=0.6, seed=2, trainable=True)

        def fwd(xd):
            h = autograd.dropout(xd, 0.6, True)
            h = l1([h, graph.edge_index], cache=graph.cache, training=True)
            h = autograd.dropout(h, 0.6, True)
            return l2([h, graph.edge_index], cache=graph.cache, training=True)
        return _train_step(fwd, [l1, l2], x, labels, idx)
    return training_case(make, iters)


def products_fwd(device, iters):
    n = PRODUCTS_NODES
    edge_index = make_graph_device(n, PRODUCTS_UNDIRECTED, 0, device)
    gen = torch.Generator(device="cpu").manual_seed(1)
    static_x = torch.randn((n, 100), generator=gen).to(device)
    graph = tfg.Graph(static_x, edge_index)
    gcn = tfg.layers.GCN(128, activation=tfg.nn.relu, seed=2)
    gat = tfg.layers.GAT(128, num_heads=8, activation=tfg.nn.relu, seed=3)
    gcn.build_cache_for_graph(graph)

    def fn():
        return (gcn([static_x, graph.edge_index, graph.edge_weight], cache=graph.cache),
                gat([static_x, graph.edge_index], cache=graph.cache))
    return forward_case(fn, static_x, torch.randn_like(static_x), iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--products-iters", type=int, default=20)
    ap.add_argument("--skip-products", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cuda_graph.py needs a CUDA device")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    result = {"card": card(), "iters": args.iters}
    result["cfg1_forward"] = cfg1_forward(device, args.iters)
    result["gcn_train"] = gcn_train(device, args.iters)
    result["gat_train"] = gat_train(device, args.iters)
    if not args.skip_products:
        result["products_fwd"] = products_fwd(device, args.products_iters)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
