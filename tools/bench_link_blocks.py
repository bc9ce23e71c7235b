#!/usr/bin/env python
# coding=utf-8
"""Link prediction on sampled blocks against the full graph at the products shape (2 449 029 nodes, 123.7 M edges, x of
100 features): a GAE encoder GCN(256, activation=relu) -> GCN(256), batches of 1024 positive edges drawn from the graph
with one tail-corrupted negative each, fan-outs [15, 10]:
- one Adam training step, BCE over the batch's pairs:
  (a) link blocks, on a FRESH batch per step, sampling included: sample_link_blocks (exclude=None and "reverse"),
      with_gcn_norm, source_rows(x), the layers, LinkBlocks.predict_edge;
  (b) the full graph: the same layers over every node with the cached normalised adjacency, the same pairs scored;
- the peak allocated memory of each route's training step;
- the device time of the exclusion build per batch (its two sorts and the count and fill passes, CUDA events), for
  RandomNeighborSampler and for HostNeighborSampler (whose fill reads the targeted rows over the host link).
Wall clock around synchronised calls.  Prints one JSON line with medians, min and max, and the card's name and power
limit.
    python tools/bench_link_blocks.py [--steps 20]"""
import argparse
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

FANOUTS = [15, 10]
BATCH = 1024
EXCLUSION = ("tfgk_stable_argsort_u32", "tfgk_block_exclusion_count", "tfgk_block_exclusion_fill",
             "tfgk_block_exclusion_fill_mapped")


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
            tfg.layers.GCN(256, seed=2, trainable=True)]


def exclusion_ms(sampler, batches, steps):
    out = []
    for i, pos in enumerate(batches[:steps + 3]):
        trace = _ffi.CallTrace(timed=EXCLUSION)
        prev = _ffi.set_trace(trace)
        try:
            sampler.sample_link_blocks(pos, FANOUTS, exclude="reverse", seed=i)
        finally:
            _ffi.set_trace(prev)
        torch.cuda.synchronize()
        if i >= 3:
            out.append(sum(sum(trace.elapsed_ms(name)) for name in EXCLUSION))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    N = bench.PRODUCTS_NODES
    ei = bench.make_graph_device(N, bench.PRODUCTS_UNDIRECTED, 0, dev)
    gen = torch.Generator(device="cpu").manual_seed(0)
    x = torch.randn((N, 100), generator=gen).to(dev)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    sampler._gcn_degrees()
    adj = tfg.SparseMatrix(ei, None, [N, N])
    cache = tfg.nn.gcn_build_cache_by_adj(adj)
    torch.cuda.synchronize()
    E = ei.shape[1]
    batches = [ei[:, torch.randint(0, E, (BATCH,), generator=gen).to(dev)].contiguous() for _ in range(args.steps + 6)]

    excl = {"random_sampler": exclusion_ms(sampler, batches, args.steps)}
    ei_host = ei.cpu()
    with tfg.utils.HostNeighborSampler(ei_host) as hs:
        excl["host_sampler"] = exclusion_ms(hs, batches, args.steps)
    del ei_host

    routes = {"blocks": model(), "blocks_exclude_reverse": model(), "full_graph": model()}
    with torch.no_grad():
        b = sampler.sample_link_blocks(batches[0][:, :4], FANOUTS, seed=0)
        for name, layers in routes.items():
            h = b.source_rows(x) if name != "full_graph" else x
            for layer, blk in zip(layers, b.blocks):
                h = layer([h, blk.with_gcn_norm()] if name != "full_graph" else [h, adj],
                          cache=None if name != "full_graph" else cache)
    for layers in list(routes.values())[1:]:
        for a, c in zip(routes["blocks"], layers):
            c.load_state_dict(a.state_dict())
    opts = {k: torch.optim.Adam([p for layer in v for p in layer.parameters()], lr=0.01) for k, v in routes.items()}
    bce = torch.nn.functional.binary_cross_entropy_with_logits

    def step(route, i):
        layers = routes[route]
        if route == "full_graph":
            b = sampler.sample_link_blocks(batches[i], [], seed=1000 + i)       # the pairs alone: no hop
            h = x
            for layer in layers:
                h = layer([h, adj], cache=cache, training=True)
            h = h[b.node_index.long()]
        else:
            b = sampler.sample_link_blocks(batches[i], FANOUTS, exclude="reverse" if "exclude" in route else None,
                                           seed=1000 + i)
            h = b.source_rows(x)
            for layer, blk in zip(layers, b.blocks):
                h = layer([h, blk.with_gcn_norm()], training=True)
        pl, nl = b.predict_edge(h)
        loss = bce(pl, torch.ones_like(pl)) + bce(nl, torch.zeros_like(nl))
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
        for route in routes:                       # alternating, the same pairs for every route
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(route, i)
            torch.cuda.synchronize()
            train[route].append((time.perf_counter() - t0) * 1e3)

    res = {"card": card(), "nodes": N, "edges": int(E), "batch_positive_edges": BATCH, "negatives_per_edge": 1,
           "fanouts": FANOUTS,
           "exclusion_build_per_batch": {k: stats(v) for k, v in excl.items()},
           "train_step_gae_gcn_256_256_adam": {k: {**stats(v), **peak[k]} for k, v in train.items()},
           "train_speedup_median": round(float(np.median(train["full_graph"]) / np.median(train["blocks"])), 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
