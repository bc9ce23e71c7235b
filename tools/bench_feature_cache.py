#!/usr/bin/env python
# coding=utf-8
"""Device rows of a host feature table (HostFeatureTable(x, device_rows=...)) at the products shape: x [2 449 029, 100]
float32 in host memory, batches of 1 024 seeds with fan-outs [15, 10, 5], seeds drawn from a fixed random 10 %
"training" subset of the nodes.  Two graphs: the bench's uniform random pairs (near-Poisson degrees) and an
RMAT(0.57, 0.19, 0.19, 0.05) graph with as many pairs, generated as tools/bench_rmat.py does (scale 22, pairs with an
end at or past N dropped).  For each graph the rows are ranked by rank_source_rows over 20 batches whose keys are
disjoint from the timed ones; rows never read follow in id order.
- For cached fractions 0 (no cache), 1, 5, 10, 25, 50 and 100 % of the rows (the top of the ranking): layer 0's source
  rows of a batch gathered by the table (tfgk_gather_rows_mapped_f32 without a cache, tfgk_gather_rows_cached_f32
  with one), with the hit rate counted from the slot map, the bytes over the link (misses * F * 4), the gather's
  median, min and max over the timed batches (CUDA events), and the time the miss fraction predicts from the uncached
  median.  Also ops.permute over a device copy of x on the same ids: at 100 % both read only HBM.
- Uniform graph only: a MeanGraphSage(256) -> MeanGraphSage(256) -> MeanGraphSage(47, concat=False) Adam step on a
  fresh batch per step, sampling included (arm (e) of tools/bench_host_features.py, gathered on the main stream): x on
  the device, and the host table with no cache, 10 % and 100 % cached; variants alternate in rounds with the same keys.
Arms alternate per batch, and every table's rows are checked bit for bit against x_dev[node_index] first.  Prints one
JSON line with the card's name and power limit.
    python tools/bench_feature_cache.py [--batches 20] [--rank-batches 20] [--rounds 8] [--steps-per-round 5]"""
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
from tf_geometric_b200 import ops              # noqa: E402

FANOUTS = [15, 10, 5]
BATCH = 1024
CLASSES = 47
F = 100
FRACTIONS = [0.0, 0.01, 0.05, 0.10, 0.25, 0.50, 1.0]
RANK_KEY0 = 100000                             # ranking keys: disjoint from the timed and training keys


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3)}


def rmat_graph(num_nodes, pairs, seed, dev):
    """RMAT(0.57, 0.19, 0.19, 0.05) pairs over 2^22 ids, kept below num_nodes and off the diagonal, mirrored."""
    scale_bits = 22
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    u = torch.zeros((pairs,), dtype=torch.int32, device=dev)
    v = torch.zeros((pairs,), dtype=torch.int32, device=dev)
    a, b, c = 0.57, 0.19, 0.19
    for bit in range(scale_bits):
        r = torch.rand((pairs,), generator=gen, device=dev)
        u |= (r >= a + b).to(torch.int32) << bit                                   # quadrants c, d -> row bit 1
        v |= (((r >= a) & (r < a + b)) | (r >= a + b + c)).to(torch.int32) << bit  # quadrants b, d -> col bit 1
    keep = (u != v) & (u < num_nodes) & (v < num_nodes)
    u, v = u[keep], v[keep]
    return torch.stack([torch.cat([u, v]), torch.cat([v, u])]).contiguous()


def model():
    return [tfg.layers.MeanGraphSage(256, seed=1, trainable=True), tfg.layers.MeanGraphSage(256, seed=2, trainable=True),
            tfg.layers.MeanGraphSage(CLASSES, seed=3, trainable=True, activation=None, concat=False)]


def forward(layers, b, h, training):
    for layer, blk in zip(layers, b.blocks):
        h = layer([h, blk], training=training)
    return h


def gather_sweep(sampler, x, x_dev, train_nodes, gen, args, dev):
    """Rank, build one table per cached fraction, check, and time the gathers; returns (result, tables by fraction)."""
    N = x.shape[0]

    def seeds():
        return train_nodes[torch.randperm(train_nodes.numel(), generator=gen)[:BATCH]].to(dev)

    t0 = time.perf_counter()
    ids, counts = tfg.utils.rank_source_rows(
        sampler.sample_blocks(seeds(), FANOUTS, seed=RANK_KEY0 + k) for k in range(args.rank_batches))
    torch.cuda.synchronize()
    rank_s = time.perf_counter() - t0
    never = torch.nonzero(counts == 0).reshape(-1).to(torch.int32)
    order = torch.cat([ids, never])                              # every row, most-read first
    tables = {f: tfg.utils.HostFeatureTable(x, device_rows=order[:int(round(f * N))]) for f in FRACTIONS}
    batches = [sampler.sample_blocks(seeds(), FANOUTS, seed=k).node_index for k in range(args.batches + 3)]
    for f, t in tables.items():                                 # every table gives x[node_index] first
        assert torch.equal(t._gather(batches[0]), x_dev[batches[0].long()]), f
    assert torch.equal(ops.permute(x_dev, batches[0]), x_dev[batches[0].long()])

    arms = {f: (lambda idx, out, t=t: t._gather(idx, out=out)) for f, t in tables.items()}
    arms["permute_device_x"] = lambda idx, out: ops.permute(x_dev, idx)
    times = {k: [] for k in arms}
    hits = {f: 0 for f in FRACTIONS}
    rows = []
    for i, idx in enumerate(batches):
        out = torch.empty((idx.numel(), F), device=dev)
        for name, fn in arms.items():
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn(idx, out)
            b.record()
            torch.cuda.synchronize()
            if i >= 3:
                times[name].append(a.elapsed_time(b))
        if i >= 3:
            rows.append(int(idx.numel()))
            for f, t in tables.items():
                if t._slot is not None:
                    hits[f] += int((t._slot[idx.long()] >= 0).sum())
    total = sum(rows)
    base = float(np.median(times[0.0]))
    sweep = []
    for f in FRACTIONS:
        t = tables[f]
        hit = hits[f] / total
        sweep.append({"fraction": f, "cached_rows": 0 if t.device_rows is None else int(t.device_rows.numel()),
                      "device_mb": round(t.device_bytes / 1e6, 1), "hit_rate": round(hit, 4),
                      "link_mb_per_batch": round((1 - hit) * total / len(rows) * F * 4 / 1e6, 1),
                      "predicted_ms": round((1 - hit) * base, 3), **stats(times[f])})
    res = {"edges": None, "rank_batches": args.rank_batches, "rank_s": round(rank_s, 3),
           "rows_read_by_ranking_batches": int(ids.numel()),
           "source_rows_per_batch": {"median": int(np.median(rows)), "min": min(rows), "max": max(rows)},
           "gather": sweep, "permute_device_x": stats(times["permute_device_x"])}
    res["full_cache_over_permute"] = round(float(np.median(times[1.0])) / float(np.median(times["permute_device_x"])), 3)
    return res, tables


def training(sampler, x, x_dev, tables, train_nodes, gen, labels, args, dev):
    variants = {"device": x_dev, "host_no_cache": tables[0.0], "host_cache_10pct": tables[0.10],
                "host_cache_100pct": tables[1.0]}
    models = {v: model() for v in variants}
    n_keys = 3 + args.rounds * args.steps_per_round
    seeds = [train_nodes[torch.randperm(train_nodes.numel(), generator=gen)[:BATCH]].to(dev) for _ in range(n_keys)]
    key0 = 50000
    with torch.no_grad():                                        # the layers create their weights on first call
        b = sampler.sample_blocks(seeds[0], FANOUTS, seed=key0)
        want = forward(models["device"], b, b.source_rows(x_dev), False)
        exact = {}
        for v, src in variants.items():                          # same seeds in every model: the same logits
            got = forward(models[v], b, b.source_rows(src), False)
            err = float((got - want).abs().max() / want.abs().max())
            assert err <= 1e-4, "{} logits differ from the device's: {}".format(v, err)
            exact[v] = bool(torch.equal(got, want))
    opts = {v: torch.optim.Adam([p for layer in ls for p in layer.parameters()], lr=0.01) for v, ls in models.items()}

    def run(v, keys):
        for k in keys:
            b = sampler.sample_blocks(seeds[k], FANOUTS, seed=key0 + k)
            out = forward(models[v], b, b.source_rows(variants[v]), True)
            loss = torch.nn.functional.cross_entropy(out, labels[b.node_index[:BATCH].long()])
            opts[v].zero_grad()
            loss.backward()
            opts[v].step()

    for v in variants:
        run(v, [0, 1, 2])
    train = {v: [] for v in variants}
    for r in range(args.rounds):
        keys = list(range(3 + r * args.steps_per_round, 3 + (r + 1) * args.steps_per_round))
        for v in variants:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(v, keys)
            torch.cuda.synchronize()
            train[v].append((time.perf_counter() - t0) * 1e3 / len(keys))
    return {"logits_equal_to_device": exact, **{v: stats(t) for v, t in train.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--rank-batches", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--steps-per-round", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    N = bench.PRODUCTS_NODES
    gen = torch.Generator(device="cpu").manual_seed(0)
    x = torch.randn((N, F), generator=gen)                       # host memory
    x_dev = x.to(dev)
    labels = torch.randint(0, CLASSES, (N,), generator=gen).to(dev)
    train_nodes = torch.randperm(N, generator=gen)[:N // 10].to(torch.int32)
    res = {"card": card(), "nodes": N, "features": F, "batch": BATCH, "fanouts": FANOUTS,
           "seeds_from": "a fixed random 10% of the nodes", "table_gb": round(x.numel() * 4 / 1e9, 3), "graphs": {}}
    for name in ("uniform", "rmat"):
        if name == "uniform":
            ei = bench.make_graph_device(N, bench.PRODUCTS_UNDIRECTED, 0, dev)
        else:
            ei = rmat_graph(N, bench.PRODUCTS_UNDIRECTED, 7, dev)
        sampler = tfg.utils.RandomNeighborSampler(ei)
        sampler._neighborhood_structure()
        g, tables = gather_sweep(sampler, x, x_dev, train_nodes, gen, args, dev)
        g["edges"] = int(ei.shape[1])
        if name == "uniform":
            g["train_step_mean_sage_256_256_47_adam"] = training(sampler, x, x_dev, tables, train_nodes, gen, labels,
                                                                 args, dev)
        for t in tables.values():
            t.close()
        res["graphs"][name] = g
        del sampler, ei, tables
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
