#!/usr/bin/env python
# coding=utf-8
"""Weighted against uniform neighbour sampling (sample_blocks(weighted=True) against weighted=False), batches of 1 024
random seeds with fan-outs [15, 10, 5], on RandomNeighborSampler and on HostNeighborSampler.

Products shape (2 449 029 nodes, 61 859 140 pairs mirrored to 123 718 280 edges, bench.make_graph_device) with random
positive float32 weights in (0.01, 1]:
- per-batch sample_blocks, the routes alternating with the same keys (CUDA events around each call, which ends in a
  synchronisation), after the first weighted call has made the positive degrees; sampled edges per batch.  The uniform
  routes run on the weighted graph and on the same graph built without weights (DESIGN.md §4's figure): a uniform batch
  over a weighted host CSR also reads every sampled edge's weight over the host link;
- a MeanGraphSage(256) -> MeanGraphSage(256) -> MeanGraphSage(47, concat=False) Adam step on a fresh batch per step,
  sampling included, features on the device: weighted against uniform on each sampler.
Prints one JSON line with medians, min and max, and the card's name and power limit.
    python tools/bench_weighted_sampling.py [--batches 20] [--steps 10]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import bench                                   # noqa: E402
import tf_geometric_b200 as tfg                # noqa: E402
from bench_host_sampler import BATCH, CLASSES, FANOUTS, card, forward, model, sampled_edges, stats  # noqa: E402


def time_batch(sampler, seeds, key, weighted):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    b = sampler.sample_blocks(seeds, FANOUTS, seed=key, weighted=weighted)
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e), b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_weighted_sampling needs a GPU")
    dev = torch.device("cuda", 0)
    res = {"card": card()}
    N = bench.PRODUCTS_NODES
    ei_dev = bench.make_graph_device(N, bench.PRODUCTS_UNDIRECTED, 0, dev)
    E = ei_dev.shape[1]
    gen = torch.Generator(device="cpu").manual_seed(0)
    w = (torch.rand((E,), generator=gen) * 0.99 + 0.01).to(torch.float32)
    res.update({"nodes": N, "edges": int(E), "batch": BATCH, "fanouts": FANOUTS})
    dsamp = tfg.utils.RandomNeighborSampler(ei_dev, w.to(dev))
    ei = ei_dev.cpu().numpy()
    hsamp = tfg.utils.HostNeighborSampler(ei, w.numpy())
    dsamp_u = tfg.utils.RandomNeighborSampler(ei_dev)
    hsamp_u = tfg.utils.HostNeighborSampler(ei)
    del ei_dev, ei
    seeds = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(args.batches + 2)]
    routes = [("device_uniform", dsamp, False), ("device_weighted", dsamp, True), ("host_uniform", hsamp, False),
              ("host_weighted", hsamp, True), ("device_uniform_unweighted_graph", dsamp_u, False),
              ("host_uniform_unweighted_graph", hsamp_u, False)]
    for _, s, wt in routes:                          # warm-up, and the positive degrees of the weighted routes
        s.sample_blocks(seeds[0], FANOUTS, seed=0, weighted=wt)
    a = dsamp.sample_blocks(seeds[1], FANOUTS, seed=1, weighted=True)
    b = hsamp.sample_blocks(seeds[1], FANOUTS, seed=1, weighted=True)
    assert torch.equal(a.node_index, b.node_index) and all(torch.equal(x.edge_index, y.edge_index)
                                                           for x, y in zip(a.blocks, b.blocks))
    times = {name: [] for name, _, _ in routes}
    edges = {name: [] for name, _, _ in routes}
    for i in range(2, 2 + args.batches):
        for name, s, wt in routes:
            ms, blk = time_batch(s, seeds[i], i, wt)
            times[name].append(ms)
            edges[name].append(sampled_edges(blk))
    res["sample_blocks"] = {name: dict(stats(times[name]), edges=int(np.median(edges[name]))) for name in times}
    res["weighted_over_uniform"] = {
        "device": round(float(np.median(times["device_weighted"]) / np.median(times["device_uniform"])), 3),
        "host": round(float(np.median(times["host_weighted"]) / np.median(times["host_uniform"])), 3)}

    x = torch.randn((N, 100), generator=gen).to(dev)
    labels = torch.randint(0, CLASSES, (N,), generator=gen).to(dev)
    step_times = {}
    for (name, samp), wt in [(r, wt) for r in (("device", dsamp), ("host", hsamp)) for wt in (False, True)]:
        layers = model()
        opt = None
        ts = []
        for i in range(args.steps + 2):
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            b = samp.sample_blocks(seeds[i % len(seeds)], FANOUTS, seed=1000 + i, weighted=wt)
            h = forward(layers, b, x[b.node_index.long()], True)
            loss = torch.nn.functional.cross_entropy(h, labels[b.node_index[:BATCH].long()])
            if opt is None:
                opt = torch.optim.Adam([p for layer in layers for p in layer.parameters()], lr=1e-3)
            opt.zero_grad()
            loss.backward()
            opt.step()
            e.record()
            torch.cuda.synchronize()
            if i >= 2:
                ts.append(a.elapsed_time(e))
        step_times["{}_{}".format(name, "weighted" if wt else "uniform")] = stats(ts)
    res["train_step"] = step_times
    hsamp.close()
    hsamp_u.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
