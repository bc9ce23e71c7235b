#!/usr/bin/env python
# coding=utf-8
"""Mini-batch features from a table in host memory at the products shape (x [2 449 029, 100] float32 kept in host
memory, page-locked in place by utils.HostFeatureTable), batches of 1 024 random seeds with fan-outs [15, 10, 5]:
- (a) tfgk_gather_rows_mapped_f32: layer 0's source rows of a batch gathered over the host link (CUDA events), with the
  bytes (n * F * 4) and the rate;
- (b) a bulk copy_ of the same byte count from the page-locked table to the device (CUDA events): the link's bulk rate,
  the floor (a) is judged against;
- (c) tfgk_permute_f32 over the same mapped pointer (no bounds check, no stride; CUDA events);
- (d) the torch route: node_index to the host, torch.index_select into a page-locked staging buffer, a non_blocking
  copy to the device (wall clock around synchronised calls);
- (e) a MeanGraphSage(256) -> MeanGraphSage(256) -> MeanGraphSage(47, concat=False) Adam step on a fresh batch per
  step, sampling included, in three variants: x resident on the device, the host table gathered on the main stream,
  and the host table gathered one batch ahead on a side stream; variants alternate in rounds with the same keys, the
  seeds' logits of the device and host variants are checked to agree first, and the peak allocated device memory of
  each is reported (the host variants' before x is ever copied to the device).
Arms (a)-(d) alternate per batch and are checked bit for bit against x[node_index] first.  Page-locks the table and
one staging buffer only, and releases both before exit.  Prints one JSON line with medians, min and max, and the
card's name and power limit.
    python tools/bench_host_features.py [--batches 20] [--rounds 8] [--steps-per-round 5]"""
import argparse
import ctypes
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
from tf_geometric_b200 import ops, _ffi        # noqa: E402

FANOUTS = [15, 10, 5]
BATCH = 1024
CLASSES = 47
F = 100


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3)}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    return a, b


def model():
    return [tfg.layers.MeanGraphSage(256, seed=1, trainable=True), tfg.layers.MeanGraphSage(256, seed=2, trainable=True),
            tfg.layers.MeanGraphSage(CLASSES, seed=3, trainable=True, activation=None, concat=False)]


def forward(layers, b, h, training):
    for layer, blk in zip(layers, b.blocks):
        h = layer([h, blk], training=training)
    return h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--steps-per-round", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    N = bench.PRODUCTS_NODES
    ei = bench.make_graph_device(N, bench.PRODUCTS_UNDIRECTED, 0, dev)
    gen = torch.Generator(device="cpu").manual_seed(0)
    x = torch.randn((N, F), generator=gen)                       # host memory only
    labels = torch.randint(0, CLASSES, (N,), generator=gen).to(dev)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    sampler._neighborhood_structure()
    n_keys = args.batches + 6 + args.rounds * args.steps_per_round + 2
    seeds = [torch.randperm(N, generator=gen)[:BATCH].to(torch.int32).to(dev) for _ in range(n_keys)]
    table = tfg.utils.HostFeatureTable(x)
    res = {"card": card(), "nodes": N, "features": F, "edges": int(ei.shape[1]), "batch": BATCH, "fanouts": FANOUTS,
           "table_gb": round(x.numel() * 4 / 1e9, 3)}

    # ---- (a)-(d): layer 0's source rows of one batch -------------------------------------------------------------
    batches = [sampler.sample_blocks(seeds[i], FANOUTS, seed=i).node_index for i in range(args.batches + 3)]
    cap = max(int(b.numel()) for b in batches)
    staging = torch.empty((cap, F))                              # page-locked in place: exactly cap rows
    staging_dev = ops.host_register(staging.data_ptr(), staging.numel() * 4)
    assert staging_dev and staging.is_pinned()
    flat = x.view(-1)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def arm_a(idx, out):
        table._gather(idx, out=out)

    def arm_b(idx, out):
        out.view(-1)[:idx.numel() * F].copy_(flat[:idx.numel() * F], non_blocking=True)

    def arm_c(idx, out):
        _ffi.call("tfgk_permute_f32", ctypes.c_void_p(table._ptr), ctypes.c_void_p(idx.data_ptr()), idx.numel(), F,
                  ctypes.c_void_p(out.data_ptr()), stream)

    def arm_d(idx, out):
        idx_host = idx.cpu().long()
        n = idx_host.numel()
        torch.index_select(x, 0, idx_host, out=staging[:n])
        out.copy_(staging[:n], non_blocking=True)

    for name, fn in (("a", arm_a), ("c", arm_c), ("d", arm_d)):   # every route gives x[node_index] first
        idx = batches[0]
        out = torch.full((idx.numel(), F), float("nan"), device=dev)
        fn(idx, out)
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), x[idx.long().cpu()]), name
    arms = {"a_gather_rows_mapped": arm_a, "b_bulk_copy": arm_b, "c_permute_f32": arm_c, "d_torch_index_select_copy": arm_d}
    times = {k: [] for k in arms}
    rows = []
    for i, idx in enumerate(batches):
        out = torch.empty((idx.numel(), F), device=dev)
        for name, fn in arms.items():
            torch.cuda.synchronize()
            if name.startswith("d"):
                t0 = time.perf_counter()
                fn(idx, out)
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3
            else:
                ev = timed(lambda: fn(idx, out))
                torch.cuda.synchronize()
                ms = ev[0].elapsed_time(ev[1])
            if i >= 3:
                times[name].append(ms)
        if i >= 3:
            rows.append(int(idx.numel()))
    mean_bytes = float(np.mean(rows)) * F * 4
    res["source_rows_per_batch"] = {"median": int(np.median(rows)), "min": min(rows), "max": max(rows)}
    res["bytes_per_batch_mb"] = round(mean_bytes / 1e6, 1)
    res["arms"] = {k: {**stats(v), "gb_per_s": round(mean_bytes / (float(np.median(v)) * 1e-3) / 1e9, 2)}
                   for k, v in times.items()}
    med = {k: float(np.median(v)) for k, v in times.items()}
    res["a_share_of_bulk_rate"] = round(med["b_bulk_copy"] / med["a_gather_rows_mapped"], 3)
    res["c_share_of_bulk_rate"] = round(med["b_bulk_copy"] / med["c_permute_f32"], 3)
    del batches

    # ---- (e): training steps --------------------------------------------------------------------------------------
    x_dev = None
    side = torch.cuda.Stream()
    main_stream = torch.cuda.current_stream()
    variants = {v: model() for v in ("device", "host", "host_prefetch")}
    with torch.no_grad():                                        # the layers create their weights on first call
        b = sampler.sample_blocks(seeds[0], FANOUTS, seed=0)
        h = b.source_rows(table)
        for layers in variants.values():
            forward(layers, b, h, False)
        del b, h
    opts = {v: torch.optim.Adam([p for layer in ls for p in layer.parameters()], lr=0.01) for v, ls in variants.items()}

    def step(v, b, h):
        out = forward(variants[v], b, h, True)
        loss = torch.nn.functional.cross_entropy(out, labels[b.node_index[:BATCH].long()])
        opts[v].zero_grad()
        loss.backward()
        opts[v].step()

    def run(v, keys):
        """len(keys) steps of variant v, a fresh batch each; the prefetch variant gathers batch j + 1 on the side stream
        while batch j computes"""
        if v != "host_prefetch":
            for k in keys:
                b = sampler.sample_blocks(seeds[k], FANOUTS, seed=k)
                step(v, b, b.source_rows(x_dev if v == "device" else table))
            return
        b = sampler.sample_blocks(seeds[keys[0]], FANOUTS, seed=keys[0])
        with torch.cuda.stream(side):
            h = b.source_rows(table)
        for j, k in enumerate(keys):
            main_stream.wait_stream(side)
            h.record_stream(main_stream)
            nxt = None
            if j + 1 < len(keys):
                nxt = sampler.sample_blocks(seeds[keys[j + 1]], FANOUTS, seed=keys[j + 1])
                with torch.cuda.stream(side):
                    h_next = nxt.source_rows(table)
            step(v, b, h)
            if nxt is not None:
                b, h = nxt, h_next

    peak = {}
    base_key = args.batches + 3
    for v in ("host", "host_prefetch", "device"):
        if v == "device":
            x_dev = x.to(dev)
        run(v, list(range(base_key, base_key + 3)))
        torch.cuda.synchronize()
        resident = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        run(v, list(range(base_key, base_key + 3)))
        torch.cuda.synchronize()
        peak[v] = {"peak_allocated_mb": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1),
                   "resident_before_mb": round(resident / 2 ** 20, 1)}

    with torch.no_grad():                                        # same layers, same batch: device vs host rows
        b = sampler.sample_blocks(seeds[0], FANOUTS, seed=0)
        want = forward(variants["device"], b, b.source_rows(x_dev), False)
        got = forward(variants["device"], b, b.source_rows(table), False)
    err = float((got - want).abs().max() / want.abs().max())
    assert err <= 1e-4, "device and host logits differ: {}".format(err)
    res["logits_max_rel_diff"] = err

    train = {v: [] for v in variants}
    first = base_key + 3
    for r in range(args.rounds):
        keys = list(range(first + r * args.steps_per_round, first + (r + 1) * args.steps_per_round))
        for v in variants:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(v, keys)
            torch.cuda.synchronize()
            train[v].append((time.perf_counter() - t0) * 1e3 / len(keys))
    res["train_step_mean_sage_256_256_47_adam"] = {v: {**stats(t), **peak[v]} for v, t in train.items()}

    table.close()
    ops.host_unregister(staging.data_ptr())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
