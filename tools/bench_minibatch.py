#!/usr/bin/env python
# coding=utf-8
"""Seed-node mini-batches at the products shape (2 449 029 nodes, 123.7 M edges, x of 100 features): batches of 1024
seeds with fan-outs [15, 10, 5].
- time per batch of RandomNeighborSampler.sample_neighborhood (K13 + tfgk_frontier_i32), alternating with the same hops
  composed from sample(k, sampled_node_index=(list, all nodes)) plus torch unique and relabel (different draws: that
  route keys its draws by the virtual row);
- K13's fill kernel alone (CUDA events) against its byte floor (28 B per listed row: the id, two rowptr words, the
  output offset; 8 B per sampled edge: its list position and CSR position) over 3.35 TB/s;
- how many rows per layer the single index space computes beyond the ones the next layer reads;
- a MeanGraphSage(256) x 2 forward + backward on the sampled subgraph.
Wall clock around synchronised calls (the samplers synchronise for their output sizes).  Prints one JSON line with
medians, min and max, and the card's name and power limit.
    python tools/bench_minibatch.py [--batches 30]"""
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

HBM = 3.35e12
FANOUTS = [15, 10, 5]
BATCH = 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def composed_route(sampler, seeds, N, seed):
    """Today's route: per hop, sample() restricted to (current list, every node), then torch unique + relabel."""
    dev = seeds.device
    nodes = seeds
    all_nodes = torch.arange(N, dtype=torch.int32, device=dev)
    edges = []
    for h, k in enumerate(reversed(FANOUTS)):
        ei, w = sampler.sample(k=k, sampled_node_index=(nodes, all_nodes), seed=seed + h)
        cols = ei[1]
        known = torch.zeros(N, dtype=torch.bool, device=dev)
        known[nodes.long()] = True
        cand = cols[~known[cols.long()]]
        uniq, inv = torch.unique(cand, return_inverse=True)
        first = torch.full((uniq.numel(),), cand.numel(), dtype=torch.int64, device=dev)
        first.scatter_reduce_(0, inv, torch.arange(cand.numel(), device=dev), reduce="amin")
        nodes = torch.cat([nodes, uniq[torch.argsort(first)].to(torch.int32)])
        where = torch.full((N,), -1, dtype=torch.int32, device=dev)
        where[nodes.long()] = torch.arange(nodes.numel(), dtype=torch.int32, device=dev)
        edges.append((torch.stack([ei[0], where[cols.long()]]), w))
    return nodes, edges[::-1]


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=30)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    N = bench.PRODUCTS_NODES
    ei = bench.make_graph_device(N, bench.PRODUCTS_UNDIRECTED, 0, dev)
    x = torch.randn((N, 100), device=dev)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    sampler._neighborhood_structure()
    torch.cuda.synchronize()
    gen = torch.Generator(device="cpu").manual_seed(0)
    batches = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(args.batches + 3)]

    new_t, old_t, sizes = [], [], []
    for i, seeds in enumerate(batches):
        for route in ("new", "old"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if route == "new":
                b = sampler.sample_neighborhood(seeds, FANOUTS, seed=i)
            else:
                composed_route(sampler, seeds, N, seed=i)
            torch.cuda.synchronize()
            if i >= 3:
                (new_t if route == "new" else old_t).append((time.perf_counter() - t0) * 1e3)
        if i >= 3:
            sizes.append(b.hop_sizes)

    # K13's fill kernel alone, per hop, over the recorded batches
    trace = _ffi.CallTrace(timed=("tfgk_neighbor_sample_rows_fill",))
    rows_edges = []
    prev = _ffi.set_trace(trace)
    try:
        for i, seeds in enumerate(batches[3:]):
            b = sampler.sample_neighborhood(seeds, FANOUTS, seed=i)
            for h in range(len(FANOUTS)):
                rows_edges.append((b.hop_sizes[h], b.edge_index_list[-1 - h].shape[1]))
    finally:
        _ffi.set_trace(prev)
    torch.cuda.synchronize()
    fill_ms = trace.elapsed_ms("tfgk_neighbor_sample_rows_fill")
    per_hop = []
    for h in range(len(FANOUTS)):
        ms = fill_ms[h::len(FANOUTS)]
        re = rows_edges[h::len(FANOUTS)]
        floor = [(28 * r + 8 * s) / HBM * 1e3 for r, s in re]
        per_hop.append({"fanout": FANOUTS[-1 - h], "median_rows": int(np.median([r for r, _ in re])),
                        "median_edges": int(np.median([s for _, s in re])), **stats(ms),
                        "byte_floor_ms": round(float(np.median(floor)), 5),
                        "share_of_floor": round(float(np.median(floor) / np.median(ms)), 4)})

    sizes = np.asarray(sizes)
    n_total = float(np.median(sizes[:, -1]))
    waste = [{"layer": i, "rows_computed": int(n_total), "rows_read_next": int(np.median(sizes[:, -2 - i])),
              "wasted_share": round(1.0 - float(np.median(sizes[:, -2 - i])) / n_total, 4)}
             for i in range(len(FANOUTS))]

    # MeanGraphSage(256) x 2 forward + backward on a sampled subgraph
    l1 = tfg.layers.MeanGraphSage(256, seed=1, trainable=True)
    l2 = tfg.layers.MeanGraphSage(256, seed=2, trainable=True, activation=None)
    b = sampler.sample_neighborhood(batches[0], FANOUTS[1:], seed=0)
    h0 = x[b.node_index.long()]

    def step():
        h = l2([l1([h0, b.edge_index_list[0], b.edge_weight_list[0]], training=True), b.edge_index_list[1],
                b.edge_weight_list[1]], training=True)
        h[:BATCH].sum().backward()

    for _ in range(3):
        step()
    train_t = []
    for _ in range(args.batches):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        train_t.append((time.perf_counter() - t0) * 1e3)

    res = {"card": card(), "nodes": N, "edges": int(ei.shape[1]), "batch": BATCH, "fanouts": FANOUTS,
           "hop_sizes_median": [int(v) for v in np.median(sizes, axis=0)],
           "sample_neighborhood": stats(new_t), "composed_sample_unique_relabel": stats(old_t),
           "speedup_median": round(float(np.median(old_t) / np.median(new_t)), 2),
           "k13_fill_per_hop": per_hop, "single_index_space_rows": waste,
           "train_step_2x_mean_sage256_fanouts_10_5": {"nodes": int(b.node_index.numel()), **stats(train_t)}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
