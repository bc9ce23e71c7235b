#!/usr/bin/env python
# coding=utf-8
"""Mini-batch sampling from a graph in host memory (utils.HostNeighborSampler) against the device sampler
(RandomNeighborSampler), batches of 1 024 random seeds with fan-outs [15, 10, 5].

Products shape (2 449 029 nodes, 61 859 140 pairs mirrored to 123 718 280 edges, bench.make_graph_device):
- build: HostNeighborSampler's constructor against RandomNeighborSampler._structure() (wall clock around synchronised
  calls), with the bytes the build reads over the host link (computed from E, the ranges and the weights) and the rate;
- per-batch sample_blocks, host and device alternating with the same keys, after checking that the batches are the same
  bit for bit (CUDA events around each call, which ends in a synchronisation); sampled edges per second;
- a MeanGraphSage(256) -> MeanGraphSage(256) -> MeanGraphSage(47, concat=False) Adam step on a fresh batch per step,
  sampling included, with the features in a HostFeatureTable: host sampler against device sampler, alternating in
  rounds, after checking the seeds' logits of the two agree bit for bit;
- the peak allocated device memory of each route's step, and the memory each sampler keeps.

--papers (111 059 956 nodes, 1 615 685 872 pairs mirrored to 3 231 371 744 edges, 128 features in a HostFeatureTable):
the edges are generated in device chunks into a host array, then the build (time, device memory kept), per-batch
sampling and one training step (sample + source_rows(table) + three MeanGraphSage layers + Adam).  It needs about 26 GB
of host memory for the edges, 13 GB for the CSR and 57 GB for the features, and exits with a message when the machine
has less.
Prints one JSON line with medians, min and max, and the card's name and power limit.
    python tools/bench_host_sampler.py [--batches 20] [--rounds 6] [--steps-per-round 5] [--papers]"""
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

FANOUTS = [15, 10, 5]
BATCH = 1024
CLASSES = 47
PAPERS_NODES, PAPERS_PAIRS, PAPERS_F = 111059956, 1615685872, 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3)}


def model(F_out=CLASSES):
    return [tfg.layers.MeanGraphSage(256, seed=1, trainable=True), tfg.layers.MeanGraphSage(256, seed=2, trainable=True),
            tfg.layers.MeanGraphSage(F_out, seed=3, trainable=True, activation=None, concat=False)]


def forward(layers, b, h, training):
    for layer, blk in zip(layers, b.blocks):
        h = layer([h, blk], training=training)
    return h


def build_link_bytes(s, weighted):
    """bytes the build reads over the host link: the id range (rows and columns), the row counts, and per range the rows
    twice (count and emit) and the selected columns (and weights) once"""
    E = s.num_edges
    return 8 * E + 4 * E + len(s._ranges) * 8 * E + 4 * E + (4 * E if weighted else 0)


def sampled_edges(b):
    return sum(int(blk.edge_index.shape[1]) for blk in b.blocks)


def time_batch(sampler, seeds, key):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    b = sampler.sample_blocks(seeds, FANOUTS, seed=key)
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e), b


def same_batch(a, b):
    return torch.equal(a.node_index, b.node_index) and a.hop_sizes == b.hop_sizes and all(
        torch.equal(x.edge_index, y.edge_index) and torch.equal(x.edge_weight, y.edge_weight) and
        torch.equal(x.global_col, y.global_col) for x, y in zip(a.blocks, b.blocks))


def available_host_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def products(args, res):
    dev = torch.device("cuda", 0)
    N = bench.PRODUCTS_NODES
    ei_dev = bench.make_graph_device(N, bench.PRODUCTS_UNDIRECTED, 0, dev)
    ei = ei_dev.cpu().numpy()
    gen = torch.Generator(device="cpu").manual_seed(0)
    x = torch.randn((N, 100), generator=gen)
    labels = torch.randint(0, CLASSES, (N,), generator=gen).to(dev)
    res.update({"nodes": N, "edges": int(ei.shape[1]), "batch": BATCH, "fanouts": FANOUTS})

    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    dsamp = tfg.utils.RandomNeighborSampler(ei_dev)
    dsamp._neighborhood_structure()
    torch.cuda.synchronize()
    t_dev = time.perf_counter() - t0
    dev_kept = torch.cuda.memory_allocated() - base
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    hsamp = tfg.utils.HostNeighborSampler(ei)
    torch.cuda.synchronize()
    t_host = time.perf_counter() - t0
    host_kept = torch.cuda.memory_allocated() - base
    link = build_link_bytes(hsamp, False)
    res["build"] = {"host_s": round(t_host, 3), "device_structure_s": round(t_dev, 3), "ranges": len(hsamp._ranges),
                    "host_link_gb": round(link / 1e9, 2), "host_link_gb_per_s": round(link / t_host / 1e9, 2),
                    "device_mb_kept_host_sampler": round(host_kept / 2 ** 20, 1),
                    "device_mb_kept_device_sampler": round(dev_kept / 2 ** 20, 1)}

    n_keys = args.batches + 3 + 2 * args.rounds * args.steps_per_round + 8
    seeds = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(n_keys)]
    for i in range(3):
        assert same_batch(hsamp.sample_blocks(seeds[i], FANOUTS, seed=i), dsamp.sample_blocks(seeds[i], FANOUTS, seed=i))
    times = {"host": [], "device": []}
    edges = []
    for i in range(3, 3 + args.batches):
        for name, s in (("host", hsamp), ("device", dsamp)):
            ms, b = time_batch(s, seeds[i], i)
            times[name].append(ms)
        edges.append(sampled_edges(b))
    e_mean = float(np.mean(edges))
    res["sample_blocks"] = {k: {**stats(v), "sampled_edges_per_s": round(e_mean / (float(np.median(v)) * 1e-3))}
                            for k, v in times.items()}
    res["sample_blocks"]["sampled_edges_per_batch"] = int(np.median(edges))
    res["sample_blocks"]["host_link_mb_per_batch"] = round(e_mean * 4 / 1e6, 2)

    table = tfg.utils.HostFeatureTable(x)
    variants = {"host": (hsamp, model()), "device": (dsamp, model())}
    with torch.no_grad():
        b = dsamp.sample_blocks(seeds[0], FANOUTS, seed=0)
        outs = [forward(ls, b, b.source_rows(table), False) for _, ls in variants.values()]
        hb = hsamp.sample_blocks(seeds[0], FANOUTS, seed=0)
        got = forward(variants["device"][1], hb, hb.source_rows(table), False)
        assert torch.equal(got, outs[1]), "host and device samplers give different logits"
    opts = {v: torch.optim.Adam([p for layer in ls for p in layer.parameters()], lr=0.01) for v, (_, ls) in variants.items()}

    def run(v, keys):
        s, layers = variants[v]
        for k in keys:
            b = s.sample_blocks(seeds[k], FANOUTS, seed=k)
            out = forward(layers, b, b.source_rows(table), True)
            loss = torch.nn.functional.cross_entropy(out, labels[b.node_index[:BATCH].long()])
            opts[v].zero_grad()
            loss.backward()
            opts[v].step()

    first = 3 + args.batches
    peak = {}
    for v in variants:
        run(v, [first, first + 1])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        run(v, [first + 2, first + 3])
        torch.cuda.synchronize()
        peak[v] = round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)
    first += 4
    train = {v: [] for v in variants}
    for r in range(args.rounds):
        for v in variants:
            keys = list(range(first, first + args.steps_per_round))
            first += args.steps_per_round
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(v, keys)
            torch.cuda.synchronize()
            train[v].append((time.perf_counter() - t0) * 1e3 / len(keys))
    res["train_step_mean_sage_256_256_47_adam_host_features"] = {
        v: {**stats(t), "peak_allocated_mb": peak[v]} for v, t in train.items()}
    table.close()
    hsamp.close()


def papers(args, res):
    E = 2 * PAPERS_PAIRS
    need = 4 * 2 * E + 4 * E + 4 * PAPERS_NODES * PAPERS_F
    res.update({"nodes": PAPERS_NODES, "edges": E, "features": PAPERS_F, "host_bytes_needed_gb": round(need / 1e9, 1)})
    avail = available_host_bytes()
    if avail < need + (16 << 30):               # the process, its page tables and the rest of the host need room too
        res["skipped"] = "needs about {:.0f} GB of host memory (26 GB of edges, 13 GB of CSR, 57 GB of features) plus " \
                         "16 GiB of headroom; {:.0f} GB available".format(need / 1e9, avail / 1e9)
        return
    dev = torch.device("cuda", 0)
    ei = np.empty((2, E), np.int32)
    chunk = 1 << 27
    t0 = time.perf_counter()
    for c0 in range(0, PAPERS_PAIRS, chunk):
        n = min(chunk, PAPERS_PAIRS - c0)
        part = bench.make_graph_device(PAPERS_NODES, n, c0 // chunk, dev).cpu().numpy()
        ei[:, c0:c0 + n] = part[:, :n]
        ei[:, PAPERS_PAIRS + c0:PAPERS_PAIRS + c0 + n] = part[:, n:]
        del part
    res["generate_s"] = round(time.perf_counter() - t0, 1)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    s = tfg.utils.HostNeighborSampler(ei)
    torch.cuda.synchronize()
    t_build = time.perf_counter() - t0
    del ei
    link = build_link_bytes(s, False)
    res["build"] = {"s": round(t_build, 1), "ranges": len(s._ranges), "host_link_gb": round(link / 1e9, 1),
                    "host_link_gb_per_s": round(link / t_build / 1e9, 2),
                    "device_gb_kept": round((torch.cuda.memory_allocated() - base) / 1e9, 3)}
    gen = torch.Generator(device="cpu").manual_seed(0)
    x = torch.empty((PAPERS_NODES, PAPERS_F))
    for r0 in range(0, PAPERS_NODES, 1 << 24):
        x[r0:r0 + (1 << 24)] = torch.randn((min(1 << 24, PAPERS_NODES - r0), PAPERS_F), generator=gen)
    labels = torch.randint(0, CLASSES, (PAPERS_NODES,), generator=gen).to(dev)
    table = tfg.utils.HostFeatureTable(x)
    seeds = [torch.randperm(PAPERS_NODES, generator=gen)[:BATCH].to(torch.int32).to(dev)
             for _ in range(args.batches + 3 + args.steps_per_round + 2)]
    times, edges = [], []
    for i in range(args.batches + 3):
        ms, b = time_batch(s, seeds[i], i)
        if i >= 3:
            times.append(ms)
            edges.append(sampled_edges(b))
    res["sample_blocks"] = {**stats(times), "sampled_edges_per_batch": int(np.median(edges)),
                            "sampled_edges_per_s": round(float(np.mean(edges)) / (float(np.median(times)) * 1e-3))}
    layers = model()
    with torch.no_grad():                       # the seeds' logits against the same layers over rows gathered by torch
        b = s.sample_blocks(seeds[0], FANOUTS, seed=0)
        got = forward(layers, b, b.source_rows(table), False)
        want = forward(layers, b, x[b.node_index.long().cpu()].to(dev), False)
        assert torch.equal(got, want), "host-table logits differ"
    opt = torch.optim.Adam([p for layer in layers for p in layer.parameters()], lr=0.01)
    steps = []
    for i in range(args.batches + 3, len(seeds)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b = s.sample_blocks(seeds[i], FANOUTS, seed=i)
        out = forward(layers, b, b.source_rows(table), True)
        loss = torch.nn.functional.cross_entropy(out, labels[b.node_index[:BATCH].long()])
        opt.zero_grad()
        loss.backward()
        opt.step()
        torch.cuda.synchronize()
        steps.append((time.perf_counter() - t0) * 1e3)
    res["train_step_mean_sage_256_256_47_adam"] = stats(steps[2:])
    table.close()
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps-per-round", type=int, default=5)
    ap.add_argument("--papers", action="store_true")
    args = ap.parse_args()
    res = {"card": card(), "shape": "papers100M" if args.papers else "products"}
    (papers if args.papers else products)(args, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
