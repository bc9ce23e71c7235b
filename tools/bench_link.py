#!/usr/bin/env python
# coding=utf-8
"""Graph-autoencoder training step (demo/demo_gae.py) on the synthetic ogbn-products graph of bench.py:
encoder GCN 100 -> 128 (relu) -> 64, positives = the graph's edges, as many negatives from
negative_sampling(edge_index=None), loss = mean sigmoid-BCE, step = forward + backward.
Reports per-call CUDA-event times of the link-prediction entry points, K6's algorithmic bytes E * (8 D + 12) over its
time as a share of 3.35 TB/s (H100 SXM HBM3 data sheet), and the step time next to the same step with predict_edge
written as torch indexing (gather, multiply, sum; index_add_ backward), alternating, in the same run.
    python tools/bench_link.py [--scale 1.0] [--steps 10]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import tf_geometric_b200 as tfg  # noqa: E402
from tf_geometric_b200 import _ffi  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12
TIMED = ("tfgk_edge_dot_f32", "tfgk_csr_build", "tfgk_spmm_f32", "tfgk_random_pairs_i32", "tfgk_permute_f32")


def torch_predict_edge(h, edge_index):
    row, col = edge_index[0].long(), edge_index[1].long()
    return (h.index_select(0, row) * h.index_select(0, col)).sum(-1)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    n, pairs = int(bench.PRODUCTS_NODES * args.scale), int(bench.PRODUCTS_UNDIRECTED * args.scale)
    edge_index = bench.make_graph_device(n, pairs, 0, device)
    x = torch.randn((n, bench.FEATURES), generator=torch.Generator().manual_seed(1), dtype=torch.float32).to(device)
    graph = tfg.Graph(x, edge_index)
    gcn0 = tfg.layers.GCN(128, activation=tfg.nn.relu, seed=2, trainable=True)
    gcn1 = tfg.layers.GCN(64, seed=3, trainable=True)
    gcn0.build_cache_for_graph(graph)
    E = edge_index.shape[1]
    bce = torch.nn.functional.binary_cross_entropy_with_logits

    def step(score, seed):
        for layer in (gcn0, gcn1):
            for p in layer.parameters():
                p.grad = None
        h = gcn0([graph.x, graph.edge_index, graph.edge_weight], cache=graph.cache, training=True)
        h = gcn1([h, graph.edge_index, graph.edge_weight], cache=graph.cache, training=True)
        neg = tfg.utils.negative_sampling(E, n, None, seed=seed)
        pos_logits, neg_logits = score(h, graph.edge_index), score(h, neg)
        loss = bce(pos_logits, torch.ones_like(pos_logits)) + bce(neg_logits, torch.zeros_like(neg_logits))
        loss.backward()

    # K6 against the torch path on the same seeded inputs before anything is timed
    with torch.no_grad():
        h = torch.randn((n, 64), generator=torch.Generator().manual_seed(4), dtype=torch.float32).to(device)
        sub = edge_index[:, :1 << 22].contiguous()
        got, want = tfg.nn.predict_edge(h, sub), torch_predict_edge(h, sub)
        scale = float(want.abs().max())
        err = float((got - want).abs().max()) / scale
        assert bool(((got - want).abs() <= 1e-4 * want.abs() + 1e-4 * scale).all()), \
            "K6 disagrees with the torch path: max error {} of max|logit|".format(err)

    result = {"card": card(), "nodes": n, "edges": int(E), "steps": args.steps, "k6_check_max_err_over_max_logit": err}
    arms = {"k6": tfg.nn.predict_edge, "torch": torch_predict_edge}
    times = {"k6": [], "torch": []}
    for i in range(args.steps + 1):                               # round 0 warms both arms up
        for arm in list(arms):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            try:
                ev[0].record()
                step(arms[arm], 100 + i)
                ev[1].record()
                torch.cuda.synchronize()
            except torch.cuda.OutOfMemoryError:                   # the [E, D] temporaries of the torch arm
                del arms[arm]
                result["step_ms_torch_indexing"] = "out of memory"
                torch.cuda.empty_cache()
                continue
            if i:
                times[arm].append(ev[0].elapsed_time(ev[1]))
    for arm, key in (("k6", "step_ms_k6"), ("torch", "step_ms_torch_indexing")):
        if times[arm] and arm in arms:
            result[key] = sorted(times[arm])[len(times[arm]) // 2]
    result["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30

    # per-call times in a separate pass (the events add host work); the half-edge CSR is memoised per edge tensor, so
    # the positives' CSR is built once and the fresh negatives' CSR every step
    trace = _ffi.CallTrace(timed=TIMED)
    _ffi.set_trace(trace)
    for i in range(args.steps):
        step(tfg.nn.predict_edge, 1000 + i)
    torch.cuda.synchronize()
    _ffi.set_trace(None)
    calls = {}
    for name in TIMED:
        ms = trace.elapsed_ms(name)
        if ms:
            calls[name] = {"calls_per_step": len(ms) / args.steps, "ms_per_step": sum(ms) / args.steps}
    result["calls"] = calls
    dot_ms = trace.elapsed_ms("tfgk_edge_dot_f32")               # two launches per step: positives, negatives (D = 64)
    k6_bytes = 2 * E * (8 * 64 + 12)
    k6_s = sum(dot_ms) / args.steps / 1e3
    result["k6_bytes_per_step"] = k6_bytes
    result["k6_share_of_3.35TBps"] = k6_bytes / k6_s / PEAK_BYTES_PER_S
    print(json.dumps(result))


if __name__ == "__main__":
    main()
