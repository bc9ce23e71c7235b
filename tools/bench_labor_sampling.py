#!/usr/bin/env python
# coding=utf-8
"""Layer-neighbour (LABOR-0) against uniform neighbour sampling: sample_blocks(labor=True), with and without
layer_dependency, against labor=False, batches of 1 024 random seeds with fan-outs [15, 10, 5], on two graphs:
- the products shape (2 449 029 nodes, 61 859 140 pairs mirrored, bench.make_graph_device);
- an RMAT(0.57, 0.19, 0.19, 0.05) graph of 2^21 nodes and the same number of pairs, mirrored
  (tools/bench_feature_cache.py's rmat_graph), whose skewed degrees let rows share neighbours.
For each graph, the three arms alternate with the same keys:
- hop sizes and sampled edges per hop (means over the batches);
- sample_blocks on RandomNeighborSampler and on HostNeighborSampler (CUDA events around each call, which ends in a
  synchronisation);
- the layer-0 source-row gather from a HostFeatureTable of 100 features, float32 and bfloat16;
- a MeanGraphSage(256) -> MeanGraphSage(256) -> MeanGraphSage(47, concat=False) Adam step, sampling (device sampler) and
  the float32 or bfloat16 host-table gather included.
Prints one JSON line with medians, min and max, and the card's name and power limit.
    python tools/bench_labor_sampling.py [--batches 10] [--steps 8]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import bench                                   # noqa: E402
import tf_geometric_b200 as tfg                # noqa: E402
from bench_host_sampler import BATCH, CLASSES, FANOUTS, card, forward, model, stats  # noqa: E402
from bench_feature_cache import rmat_graph     # noqa: E402

F = 100
ARMS = {"uniform": {}, "labor": dict(labor=True), "labor_layer_dep": dict(labor=True, layer_dependency=True)}


def timed(fn):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e), out


def run_graph(ei_dev, args, dev, gen):
    N = int(ei_dev.max().item()) + 1                 # the samplers' node count: ids past the largest are not nodes
    res = {"nodes": N, "edges": int(ei_dev.shape[1])}
    dsamp = tfg.utils.RandomNeighborSampler(ei_dev)
    hsamp = tfg.utils.HostNeighborSampler(ei_dev.cpu().numpy())
    x = torch.randn((N, F), generator=gen)
    tables = {"f32": tfg.utils.HostFeatureTable(x), "bf16": tfg.utils.HostFeatureTable(x.to(torch.bfloat16),
                                                                                         dtype=torch.bfloat16)}
    labels = torch.randint(0, CLASSES, (N,), generator=gen).to(dev)
    seeds = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(args.batches + 1)]
    for kw in ARMS.values():                         # warm-up; both samplers give the same batch for the same key
        a = dsamp.sample_blocks(seeds[0], FANOUTS, seed=0, **kw)
        b = hsamp.sample_blocks(seeds[0], FANOUTS, seed=0, **kw)
        assert torch.equal(a.node_index, b.node_index) and all(torch.equal(p.edge_index, q.edge_index)
                                                               for p, q in zip(a.blocks, b.blocks))
        for t in tables.values():
            t._gather(a.node_index)
    times = {arm: {"device_sample": [], "host_sample": [], "gather_f32": [], "gather_bf16": []} for arm in ARMS}
    hops = {arm: [] for arm in ARMS}
    edges = {arm: [] for arm in ARMS}
    for i in range(1, args.batches + 1):
        for arm, kw in ARMS.items():
            ms, b = timed(lambda: dsamp.sample_blocks(seeds[i], FANOUTS, seed=i, **kw))
            times[arm]["device_sample"].append(ms)
            hops[arm].append(list(b.hop_sizes))
            edges[arm].append([int(blk.edge_index.shape[1]) for blk in b.blocks[::-1]])    # hop order
            times[arm]["host_sample"].append(timed(lambda: hsamp.sample_blocks(seeds[i], FANOUTS, seed=i, **kw))[0])
            for t in tables:
                times[arm]["gather_" + t].append(timed(lambda: tables[t]._gather(b.node_index))[0])
    res["hop_sizes_mean"] = {arm: [round(float(v), 1) for v in np.mean(hops[arm], axis=0)] for arm in ARMS}
    res["edges_per_hop_mean"] = {arm: [round(float(v), 1) for v in np.mean(edges[arm], axis=0)] for arm in ARMS}
    res["layer0_rows_over_uniform"] = {arm: round(float(np.mean(hops[arm], axis=0)[-1] /
                                                       np.mean(hops["uniform"], axis=0)[-1]), 3) for arm in ARMS}
    res["time"] = {arm: {k: stats(v) for k, v in t.items()} for arm, t in times.items()}

    steps = {}
    for tname, table in tables.items():
        models = {arm: model() for arm in ARMS}
        opts = {}
        ts = {arm: [] for arm in ARMS}
        for i in range(args.steps + 2):
            for arm, kw in ARMS.items():
                def step():
                    b = dsamp.sample_blocks(seeds[i % len(seeds)], FANOUTS, seed=1000 + i, **kw)
                    h = forward(models[arm], b, b.source_rows(table), True)
                    loss = torch.nn.functional.cross_entropy(h, labels[b.node_index[:BATCH].long()])
                    if arm not in opts:
                        opts[arm] = torch.optim.Adam([p for layer in models[arm] for p in layer.parameters()],
                                                     lr=1e-3)
                    opts[arm].zero_grad()
                    loss.backward()
                    opts[arm].step()
                ms, _ = timed(step)
                if i >= 2:
                    ts[arm].append(ms)
        steps[tname] = {arm: stats(v) for arm, v in ts.items()}
    res["train_step"] = steps
    hsamp.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--steps", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_labor_sampling needs a GPU")
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device="cpu").manual_seed(0)
    res = {"card": card(), "batch": BATCH, "fanouts": FANOUTS, "features": F}
    res["products"] = run_graph(bench.make_graph_device(bench.PRODUCTS_NODES, bench.PRODUCTS_UNDIRECTED, 0, dev),
                                args, dev, gen)
    torch.cuda.empty_cache()
    res["rmat"] = run_graph(rmat_graph(1 << 21, bench.PRODUCTS_UNDIRECTED, 0, dev), args, dev, gen)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
