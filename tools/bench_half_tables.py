#!/usr/bin/env python
# coding=utf-8
"""16-bit host feature tables (HostFeatureTable(x, dtype=torch.bfloat16 / torch.float16)) at the products shape: x
[2 449 029, 100] in host memory, batches of 1 024 random seeds with fan-outs [15, 10, 5], the same graph, keys and batches
as tools/bench_host_features.py.  Layer 0's source rows of a batch gathered by the table (CUDA events), arms alternating
per batch:
- (a) float32 table (tfgk_gather_rows_mapped_f32, 400-byte rows, 16-byte loads);
- (b) bfloat16 table, ld = 100 (tfgk_gather_rows_mapped_16, 200-byte rows: 8-byte loads);
- (c) bfloat16 table with F = 104, rows padded to 208 bytes (16-byte loads; gather only);
- (d) float16 table, ld = 100;
each with the bytes over the link (n * F * itemsize) and the rate, every arm checked bit for bit against
x.float()[node_index] first.
- (e) On the RMAT graph of tools/bench_feature_cache.py, seeds from a fixed random 10 % of the nodes, the top 10 % of
  rank_source_rows over 20 batches with their own keys cached: the bfloat16 table against the float32 table with the
  same rows cached (tfgk_gather_rows_cached_16 / _f32), with hit rate and link bytes.
- A MeanGraphSage(256) -> MeanGraphSage(256) -> MeanGraphSage(47, concat=False) Adam step on a fresh batch per step,
  sampling included, from the float32 host table and from the bfloat16 host table (uniform graph, no cache); variants
  alternate in rounds with the same keys; the bfloat16 table's logits are checked bit for bit against the same layers on
  x.to(bfloat16).float() on the device first.
Prints one JSON line with medians, min and max, and the card's name and power limit.
    python tools/bench_half_tables.py [--batches 20] [--rank-batches 20] [--rounds 8] [--steps-per-round 5]"""
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
from bench_feature_cache import rmat_graph     # noqa: E402

FANOUTS = [15, 10, 5]
BATCH = 1024
CLASSES = 47
F = 100
RANK_KEY0 = 100000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3)}


def model():
    return [tfg.layers.MeanGraphSage(256, seed=1, trainable=True), tfg.layers.MeanGraphSage(256, seed=2, trainable=True),
            tfg.layers.MeanGraphSage(CLASSES, seed=3, trainable=True, activation=None, concat=False)]


def forward(layers, b, h, training):
    for layer, blk in zip(layers, b.blocks):
        h = layer([h, blk], training=training)
    return h


def time_arms(arms, batches, widths, dev, hit_of=None):
    """Per batch, each arm in turn, timed by CUDA events; the first 3 batches warm up.  Returns (times, rows, hits)."""
    times = {k: [] for k in arms}
    hits = {k: 0 for k in arms}
    rows = []
    for i, idx in enumerate(batches):
        for name, fn in arms.items():
            out = torch.empty((idx.numel(), widths[name]), device=dev)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn(idx, out)
            b.record()
            torch.cuda.synchronize()
            if i >= 3:
                times[name].append(a.elapsed_time(b))
                if hit_of is not None:
                    hits[name] += hit_of[name](idx)
        if i >= 3:
            rows.append(int(idx.numel()))
    return times, rows, hits


def summarise(times, rows, bytes_per_row, hits=None):
    total = sum(rows)
    out = {}
    for k, t in times.items():
        miss = 1.0 - (hits[k] / total if hits else 0.0)
        link = miss * total / len(rows) * bytes_per_row[k]
        med = float(np.median(t))
        out[k] = {**stats(t), "link_mb_per_batch": round(link / 1e6, 1), "gb_per_s": round(link / (med * 1e-3) / 1e9, 2)}
        if hits:
            out[k]["hit_rate"] = round(hits[k] / total, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--rank-batches", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--steps-per-round", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    N = bench.PRODUCTS_NODES
    HFT = tfg.utils.HostFeatureTable
    ei = bench.make_graph_device(N, bench.PRODUCTS_UNDIRECTED, 0, dev)
    gen = torch.Generator(device="cpu").manual_seed(0)
    x = torch.randn((N, F), generator=gen)                       # host memory only
    labels = torch.randint(0, CLASSES, (N,), generator=gen).to(dev)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    sampler._neighborhood_structure()
    n_keys = args.batches + 6 + args.rounds * args.steps_per_round + 2
    seeds = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(n_keys)]
    x_bf16, x_f16 = x.to(torch.bfloat16), x.to(torch.float16)
    x_pad = torch.zeros((N, 104), dtype=torch.bfloat16)
    x_pad[:, :F] = x_bf16
    tables = {"a_f32": HFT(x), "b_bf16": HFT(x_bf16, dtype=torch.bfloat16),
              "c_bf16_f104": HFT(x_pad, dtype=torch.bfloat16), "d_f16": HFT(x_f16, dtype=torch.float16)}
    sources = {"a_f32": x, "b_bf16": x_bf16, "c_bf16_f104": x_pad, "d_f16": x_f16}
    widths = {k: t.num_features for k, t in tables.items()}
    res = {"card": card(), "nodes": N, "features": F, "edges": int(ei.shape[1]), "batch": BATCH, "fanouts": FANOUTS,
           "table_gb": {k: round(t.x.numel() * t.x.element_size() / 1e9, 3) for k, t in tables.items()}}

    # ---- (a)-(d): layer 0's source rows of one batch -------------------------------------------------------------
    batches = [sampler.sample_blocks(seeds[i], FANOUTS, seed=i).node_index for i in range(args.batches + 3)]
    for k, t in tables.items():                                  # every table gives x.float()[node_index] first
        got = t._gather(batches[0])
        assert torch.equal(got.cpu(), sources[k][batches[0].long().cpu()].float()), k
    arms = {k: (lambda idx, out, t=t: t._gather(idx, out=out)) for k, t in tables.items()}
    times, rows, _ = time_arms(arms, batches, widths, dev)
    res["source_rows_per_batch"] = {"median": int(np.median(rows)), "min": min(rows), "max": max(rows)}
    res["gather"] = summarise(times, rows, {k: widths[k] * t.x.element_size() for k, t in tables.items()})
    med = {k: float(np.median(v)) for k, v in times.items()}
    res["gather_time_over_f32"] = {k: round(med[k] / med["a_f32"], 3) for k in med}
    del batches

    # ---- training steps: float32 against bfloat16 host table ------------------------------------------------------
    variants = {"host_f32": tables["a_f32"], "host_bf16": tables["b_bf16"]}
    models = {v: model() for v in variants}
    key0 = args.batches + 3
    with torch.no_grad():                                        # the layers create their weights on first call
        b = sampler.sample_blocks(seeds[key0], FANOUTS, seed=key0)
        for v, src in variants.items():
            forward(models[v], b, b.source_rows(src), False)
        x_wide = x_bf16.to(dev).float()
        want = forward(models["host_bf16"], b, b.source_rows(x_wide), False)
        got = forward(models["host_bf16"], b, b.source_rows(tables["b_bf16"]), False)
        assert torch.equal(got, want), "bf16 table logits differ from the widened device x's"
        del x_wide, want, got, b
    opts = {v: torch.optim.Adam([p for layer in ls for p in layer.parameters()], lr=0.01) for v, ls in models.items()}

    def run(v, keys):
        for k in keys:
            b = sampler.sample_blocks(seeds[k], FANOUTS, seed=k)
            out = forward(models[v], b, b.source_rows(variants[v]), True)
            loss = torch.nn.functional.cross_entropy(out, labels[b.node_index[:BATCH].long()])
            opts[v].zero_grad()
            loss.backward()
            opts[v].step()

    for v in variants:
        run(v, list(range(key0, key0 + 3)))
    train = {v: [] for v in variants}
    first = key0 + 3
    for r in range(args.rounds):
        keys = list(range(first + r * args.steps_per_round, first + (r + 1) * args.steps_per_round))
        for v in variants:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(v, keys)
            torch.cuda.synchronize()
            train[v].append((time.perf_counter() - t0) * 1e3 / len(keys))
    res["train_step_mean_sage_256_256_47_adam"] = {v: stats(t) for v, t in train.items()}
    for t in tables.values():
        t.close()
    del sampler, ei, tables, models, opts
    torch.cuda.empty_cache()

    # ---- (e): 10 % of the rows cached, RMAT graph -------------------------------------------------------------------
    ei = rmat_graph(N, bench.PRODUCTS_UNDIRECTED, 7, dev)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    sampler._neighborhood_structure()
    train_nodes = torch.randperm(N, generator=gen)[:N // 10].to(torch.int32)

    def pick():
        return train_nodes[torch.randperm(train_nodes.numel(), generator=gen)[:BATCH]].to(dev)

    ids, counts = tfg.utils.rank_source_rows(
        sampler.sample_blocks(pick(), FANOUTS, seed=RANK_KEY0 + k) for k in range(args.rank_batches))
    order = torch.cat([ids, torch.nonzero(counts == 0).reshape(-1).to(torch.int32)])
    keep = order[:N // 10]
    cached = {"f32_cache_10pct": HFT(x, device_rows=keep), "bf16_cache_10pct": HFT(x_bf16, device_rows=keep,
                                                                                    dtype=torch.bfloat16)}
    src = {"f32_cache_10pct": x, "bf16_cache_10pct": x_bf16}
    batches = [sampler.sample_blocks(pick(), FANOUTS, seed=k).node_index for k in range(args.batches + 3)]
    for k, t in cached.items():
        assert torch.equal(t._gather(batches[0]).cpu(), src[k][batches[0].long().cpu()].float()), k
    arms = {k: (lambda idx, out, t=t: t._gather(idx, out=out)) for k, t in cached.items()}
    hit_of = {k: (lambda idx, t=t: int((t._slot[idx.long()] >= 0).sum())) for k, t in cached.items()}
    times, rows, hits = time_arms(arms, batches, {k: F for k in cached}, dev, hit_of)
    res["rmat_cached"] = {"edges": int(ei.shape[1]), "cached_rows": int(keep.numel()),
                          "device_mb": {k: round(t.device_bytes / 1e6, 1) for k, t in cached.items()},
                          "source_rows_per_batch": {"median": int(np.median(rows)), "min": min(rows), "max": max(rows)},
                          **summarise(times, rows, {"f32_cache_10pct": F * 4, "bf16_cache_10pct": F * 2}, hits)}
    for t in cached.values():
        t.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
