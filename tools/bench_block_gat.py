#!/usr/bin/env python
# coding=utf-8
"""Mini-batch GAT on self-looped blocks against the single index space at the products shape (2 449 029 nodes, 123.7 M
edges, x of 100 features), batches of 1024 random seeds with fan-outs [15, 10, 5]:
- one Adam training step of GAT(128, num_heads=4, activation=relu) -> the same -> GAT(47, num_heads=1) on a FRESH batch
  per step, sampling included, the two routes alternating over the same seeds and keys:
  (a) blocks: sample_blocks, Block.with_self_loops, source_rows(x), the layers over the looped blocks;
  (b) the single index space: sample_neighborhood, x[node_index], the layers over edge_index_list[i];
  before timing, the seeds' logits of the two routes are checked to agree within 1e-5 relative with the same weights;
- the peak allocated memory of each route's training step;
- the device time of tfgk_block_self_loops_i32 per batch (its three launches, CUDA events).
Wall clock around synchronised calls.  Prints one JSON line with medians, min and max, and the card's name and power
limit.
    python tools/bench_block_gat.py [--steps 20]"""
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
LOOPS = "tfgk_block_self_loops_i32"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3)}


def model():
    return [tfg.layers.GAT(128, num_heads=4, activation=tfg.nn.relu, seed=1, trainable=True),
            tfg.layers.GAT(128, num_heads=4, activation=tfg.nn.relu, seed=2, trainable=True),
            tfg.layers.GAT(CLASSES, num_heads=1, seed=3, trainable=True)]


def forward_blocks(layers, sampler, x, seeds, key, training):
    b = sampler.sample_blocks(seeds, FANOUTS, seed=key)
    h = b.source_rows(x)
    for layer, blk in zip(layers, b.blocks):
        h = layer([h, blk.with_self_loops()], training=training)
    return h


def forward_single(layers, sampler, x, seeds, key, training):
    nb = sampler.sample_neighborhood(seeds, FANOUTS, seed=key)
    h = x[nb.node_index.long()]
    for layer, e in zip(layers, nb.edge_index_list):
        h = layer([h, e], training=training)
    return h[:seeds.numel()]


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
    sampler._neighborhood_structure()
    torch.cuda.synchronize()
    batches = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(args.steps + 6)]

    # the looped blocks alone: three launches per batch, timed with CUDA events
    loops_ms = []
    for i, seeds in enumerate(batches[:args.steps]):
        b = sampler.sample_blocks(seeds, FANOUTS, seed=i)
        trace = _ffi.CallTrace(timed=(LOOPS,))
        prev = _ffi.set_trace(trace)
        try:
            for blk in b.blocks:
                blk.with_self_loops()
        finally:
            _ffi.set_trace(prev)
        torch.cuda.synchronize()
        if i >= 3:
            loops_ms.append(sum(trace.elapsed_ms(LOOPS)))

    # the same weights on both routes; the logits agree before anything is timed
    routes = {"blocks": (model(), forward_blocks), "single_index_space": (model(), forward_single)}
    with torch.no_grad():
        got = forward_blocks(routes["blocks"][0], sampler, x, batches[0], 0, False)
        forward_single(routes["single_index_space"][0], sampler, x, batches[0], 0, False)
        for a, c in zip(routes["blocks"][0], routes["single_index_space"][0]):
            c.load_state_dict(copy.deepcopy(a.state_dict()))
        want = forward_single(routes["single_index_space"][0], sampler, x, batches[0], 0, False)
    err = float((got - want).abs().max() / want.abs().max())
    assert err <= 1e-5, "the two routes' logits differ: {}".format(err)
    opts = {k: torch.optim.Adam([p for layer in v[0] for p in layer.parameters()], lr=0.01) for k, v in routes.items()}

    def step(route, i):
        layers, fwd = routes[route]
        seeds = batches[i]
        h = fwd(layers, sampler, x, seeds, 1000 + i, True)
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
        for route in routes:                       # alternating, the same seeds and key for both
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(route, i)
            torch.cuda.synchronize()
            train[route].append((time.perf_counter() - t0) * 1e3)

    res = {"card": card(), "nodes": N, "edges": int(ei.shape[1]), "batch": BATCH, "fanouts": FANOUTS,
           "logits_max_rel_diff": err,
           "block_self_loops_per_batch": stats(loops_ms),
           "train_step_gat_128x4_128x4_47_adam": {k: {**stats(v), **peak[k]} for k, v in train.items()},
           "train_speedup_median": round(float(np.median(train["single_index_space"]) / np.median(train["blocks"])), 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
