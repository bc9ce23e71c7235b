#!/usr/bin/env python
# coding=utf-8
"""Mini-batch GCN on sampled blocks against the full graph at the products shape (2 449 029 nodes, 123.7 M edges, x of
100 features), batches of 1024 random seeds with fan-outs [15, 10, 5]:
- one Adam training step of GCN(256, activation=relu) -> the same -> GCN(47), the loss over the batch's seeds:
  (a) blocks, on a FRESH batch per step, sampling included: sample_blocks, Block.with_gcn_norm, source_rows(x), the
      layers over the GcnBlocks (the full graph's degrees, neighbour sums rescaled by degree over fan-out);
  (b) the full graph: the same layers over every node with the cached normalised adjacency, the loss at the same seeds;
  before timing, a batch drawn with every neighbour is checked to give the full graph's logits at its seeds within 1e-5
  relative with the same weights;
- the peak allocated memory of each route's training step;
- the device time of tfgk_block_gcn_values_f32 per batch (its three launches, CUDA events).
Wall clock around synchronised calls.  Prints one JSON line with medians, min and max, and the card's name and power
limit.
    python tools/bench_block_gcn.py [--steps 20]"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import bench                                   # noqa: E402
import tf_geometric_b200 as tfg                # noqa: E402
from tf_geometric_b200 import _ffi             # noqa: E402

FANOUTS = [15, 10, 5]
BATCH = 1024
CLASSES = 47
VALUES = "tfgk_block_gcn_values_f32"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3)}


def model():
    return [tfg.layers.GCN(256, activation=tfg.nn.relu, seed=1, trainable=True),
            tfg.layers.GCN(256, activation=tfg.nn.relu, seed=2, trainable=True),
            tfg.layers.GCN(CLASSES, seed=3, trainable=True)]


def forward_blocks(layers, sampler, x, seeds, key, training, fanouts=FANOUTS):
    b = sampler.sample_blocks(seeds, fanouts, seed=key)
    h = b.source_rows(x)
    for layer, blk in zip(layers, b.blocks):
        h = layer([h, blk.with_gcn_norm()], training=training)
    return h


def forward_full(layers, adj, cache, x, seeds, training):
    h = x
    for layer in layers:
        h = layer([h, adj], cache=cache, training=training)
    return h[seeds.long()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    N = bench.PRODUCTS_NODES
    ei = bench.make_graph_device(N, bench.PRODUCTS_UNDIRECTED, 0, dev)
    gen = torch.Generator(device="cpu").manual_seed(0)
    x = torch.randn((N, 100), generator=gen).to(dev)
    labels = torch.randint(0, CLASSES, (N,), generator=gen).to(dev)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    sampler._gcn_degrees()
    adj = tfg.SparseMatrix(ei, None, [N, N])
    cache = tfg.nn.gcn_build_cache_by_adj(adj)               # the full graph's normalised adjacency, built once
    torch.cuda.synchronize()
    batches = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(args.steps + 6)]

    # the block values alone: three launches per batch, timed with CUDA events
    values_ms = []
    for i, seeds in enumerate(batches[:args.steps]):
        b = sampler.sample_blocks(seeds, FANOUTS, seed=i)
        for blk in b.blocks:
            blk.with_self_loops()
        trace = _ffi.CallTrace(timed=(VALUES,))
        prev = _ffi.set_trace(trace)
        try:
            for blk in b.blocks:
                blk.with_gcn_norm().normalized()
        finally:
            _ffi.set_trace(prev)
        torch.cuda.synchronize()
        if i >= 3:
            values_ms.append(sum(trace.elapsed_ms(VALUES)))

    # the same weights on both routes; with every neighbour the block logits are the full graph's
    routes = {"blocks": model(), "full_graph": model()}
    with torch.no_grad():
        small = batches[0][:4]
        got = forward_blocks(routes["blocks"], sampler, x, small, 0, False, fanouts=[None, None, None])
        forward_full(routes["full_graph"], adj, cache, x, small, False)
        for a, c in zip(routes["blocks"], routes["full_graph"]):
            c.load_state_dict(copy.deepcopy(a.state_dict()))
        want = forward_full(routes["full_graph"], adj, cache, x, small, False)
    err = float((got - want).abs().max() / want.abs().max())
    assert err <= 1e-5, "the block and full-graph logits differ: {}".format(err)
    opts = {k: torch.optim.Adam([p for layer in v for p in layer.parameters()], lr=0.01) for k, v in routes.items()}

    def step(route, i):
        seeds = batches[i]
        if route == "blocks":
            h = forward_blocks(routes[route], sampler, x, seeds, 1000 + i, True)
        else:
            h = forward_full(routes[route], adj, cache, x, seeds, True)
        loss = torch.nn.functional.cross_entropy(h, labels[seeds.long()])
        opts[route].zero_grad()
        loss.backward()
        opts[route].step()

    train = {k: [] for k in routes}
    peak = {}
    for route in routes:
        for i in range(3):
            step(route, i)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        for i in range(3, 6):
            step(route, i)
        torch.cuda.synchronize()
        peak[route] = {"peak_allocated_mb": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1),
                       "resident_before_mb": round(base / 2 ** 20, 1)}
    for i in range(6, 6 + args.steps):
        for route in routes:                       # alternating, the same seeds for both
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(route, i)
            torch.cuda.synchronize()
            train[route].append((time.perf_counter() - t0) * 1e3)

    res = {"card": card(), "nodes": N, "edges": int(ei.shape[1]), "batch": BATCH, "fanouts": FANOUTS,
           "every_neighbour_logits_max_rel_diff": err,
           "block_gcn_values_per_batch": stats(values_ms),
           "train_step_gcn_256_256_47_adam": {k: {**stats(v), **peak[k]} for k, v in train.items()},
           "train_speedup_median": round(float(np.median(train["full_graph"]) / np.median(train["blocks"])), 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
