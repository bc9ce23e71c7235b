#!/usr/bin/env python
# coding=utf-8
"""Bipartite blocks against the single index space at the products shape (2 449 029 nodes, 123.7 M edges, x of 100
features), batches of 1024 random seeds with fan-outs [15, 10, 5]:
- time per batch of RandomNeighborSampler.sample_blocks against sample_neighborhood (same keys, so the same sample),
  alternating, and the library calls per batch that return values to the host (_ffi.CallTrace);
- one training step of MeanGraphSage(256) -> MeanGraphSage(256) -> MeanGraphSage(47, concat=False) with Adam on a
  FRESH batch per step, sampling included: blocks (sample_blocks, source_rows(x), the layers) against today's route
  (sample_neighborhood, x[node_index], the layers, which build their CSRs); before timing, the seeds' logits of the two
  routes are checked to agree within 1e-4 relative with the same weights and key;
- the peak allocated memory of each training step.
Wall clock around synchronised calls.  Prints one JSON line with medians, min and max, and the card's name and power
limit.
    python tools/bench_blocks.py [--steps 20]"""
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
# library entries that copy a result to the host and synchronise
HOST_ENTRIES = ("tfgk_neighbor_sample_rows_count", "tfgk_reindex_i32", "tfgk_frontier_i32", "tfgk_csr_build",
                "tfgk_plan_build", "tfgk_block_sample_read_total", "tfgk_block_sample_end")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3)}


def model():
    layers = [tfg.layers.MeanGraphSage(256, seed=1, trainable=True), tfg.layers.MeanGraphSage(256, seed=2, trainable=True),
              tfg.layers.MeanGraphSage(CLASSES, seed=3, trainable=True, activation=None, concat=False)]
    return layers


def forward_blocks(layers, sampler, x, seeds, key, training):
    b = sampler.sample_blocks(seeds, FANOUTS, seed=key)
    h = b.source_rows(x)
    for layer, blk in zip(layers, b.blocks):
        h = layer([h, blk], training=training)
    return h


def forward_today(layers, sampler, x, seeds, key, training):
    nb = sampler.sample_neighborhood(seeds, FANOUTS, seed=key)
    h = x[nb.node_index.long()]
    for layer, e, w in zip(layers, nb.edge_index_list, nb.edge_weight_list):
        h = layer([h, e, w], training=training)
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
    batches = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(2 * args.steps + 6)]

    # sampling, alternating; the same key gives both routes the same sample
    times = {"sample_blocks": [], "sample_neighborhood": []}
    host_calls = {}
    for i, seeds in enumerate(batches):
        for name in ("sample_blocks", "sample_neighborhood"):
            trace = _ffi.CallTrace()
            prev = _ffi.set_trace(trace)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            getattr(sampler, name)(seeds, FANOUTS, seed=i)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            _ffi.set_trace(prev)
            if i >= 3:
                times[name].append(ms)
                host_calls[name] = sum(trace.counts.get(n, 0) for n in HOST_ENTRIES)

    # training: the same weights on both routes; the logits agree before anything is timed
    blocks_layers, today_layers = model(), model()
    with torch.no_grad():
        got = forward_blocks(blocks_layers, sampler, x, batches[0], 0, False)
        want = forward_today(today_layers, sampler, x, batches[0], 0, False)
    for a, c in zip(blocks_layers, today_layers):
        c.load_state_dict(copy.deepcopy(a.state_dict()))
    with torch.no_grad():
        want = forward_today(today_layers, sampler, x, batches[0], 0, False)
    err = float((got - want).abs().max() / want.abs().max())
    assert err <= 1e-4, "the two routes' logits differ: {}".format(err)
    routes = {"blocks": (blocks_layers, forward_blocks), "today": (today_layers, forward_today)}
    opts = {k: torch.optim.Adam([p for layer in v[0] for p in layer.parameters()], lr=0.01) for k, v in routes.items()}

    def step(route, i):
        layers, fwd = routes[route]
        seeds = batches[i]
        h = fwd(layers, sampler, x, seeds, 1000 + i, True)
        loss = torch.nn.functional.cross_entropy(h, labels[seeds.long()])
        opts[route].zero_grad()
        loss.backward()
        opts[route].step()

    train = {"blocks": [], "today": []}
    peak = {}
    for route in ("blocks", "today"):
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
    for i in range(6, 6 + 2 * args.steps, 2):
        for j, route in enumerate(("blocks", "today")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(route, i + j)
            torch.cuda.synchronize()
            train[route].append((time.perf_counter() - t0) * 1e3)

    res = {"card": card(), "nodes": N, "edges": int(ei.shape[1]), "batch": BATCH, "fanouts": FANOUTS,
           "sampling": {k: stats(v) for k, v in times.items()},
           "host_round_trips_per_batch": host_calls,
           "logits_max_rel_diff": err,
           "train_step_mean_sage_256_256_47_adam": {k: {**stats(v), **peak[k]} for k, v in train.items()},
           "train_speedup_median": round(float(np.median(train["today"]) / np.median(train["blocks"])), 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
