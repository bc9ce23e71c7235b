#!/usr/bin/env python
# coding=utf-8
"""Edge-weight gradients on the synthetic ogbn-products graph of bench.py (BASELINE cfg4 shape: 2 449 029 nodes,
123 718 280 directed edges).
  1. K7 (tfgk_sddmm_csr_f32) alone, D = 100 and 128, with perm and the mean scale: CUDA-event time per launch and its
     algorithmic bytes  E * (4 D + 12) + N * (4 D + 8)  over that time as a share of 3.35 TB/s (H100 SXM HBM3 data sheet).
     The result is checked against a float64 restatement on a sample of edges first.
  2. MeanGraphSage(256) forward + backward (x: 100 features, trainable weights and x), with edge_weight.requires_grad
     False and True, alternating in the same run: the difference is what the edge gradient costs.
    python tools/bench_edge_grad.py [--scale 1.0] [--steps 10]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import tf_geometric_b200 as tfg  # noqa: E402
from tf_geometric_b200 import ops, _structure  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def timed(fn, steps):
    """Median CUDA-event time (ms) of fn() over `steps` calls after one warm-up call."""
    fn()
    out = []
    for _ in range(steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        out.append(ev[0].elapsed_time(ev[1]))
    return sorted(out)[len(out) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    n, pairs = int(bench.PRODUCTS_NODES * args.scale), int(bench.PRODUCTS_UNDIRECTED * args.scale)
    edge_index = bench.make_graph_device(n, pairs, 0, device)
    E = int(edge_index.shape[1])
    csr, _ = _structure.csr_for_edge_index(edge_index, n)
    gen = torch.Generator().manual_seed(1)
    cnt = (csr.rowptr[1:] - csr.rowptr[:-1]).clamp(min=1).to(torch.float32)
    scale = torch.reciprocal(cnt)
    result = {"card": card(), "nodes": n, "edges": E, "steps": args.steps, "k7": {}}

    for D in (100, 128):
        G = torch.randn((n, D), generator=gen, dtype=torch.float32).to(device)
        X = torch.randn((n, D), generator=gen, dtype=torch.float32).to(device)
        out = ops.sddmm_csr(csr, G, X, row_scale=scale)
        idx = torch.randint(0, E, (1 << 16,), generator=gen).to(device)
        r, c = edge_index[0].long()[idx], edge_index[1].long()[idx]
        want = (G[r].double() * X[c].double()).sum(-1) * scale[r].double()
        err = float(((out[idx].double() - want).abs() / (want.abs() + 1e-4 * want.abs().max())).max())
        assert err < 1e-3, "K7 disagrees with float64 (relative error {})".format(err)
        ms = timed(lambda: ops.sddmm_csr(csr, G, X, row_scale=scale, out=out), args.steps)
        nbytes = E * (4 * D + 12) + n * (4 * D + 8)
        result["k7"]["D{}".format(D)] = {"ms": ms, "bytes": nbytes, "share_of_3.35TBps": nbytes / (ms / 1e3) / PEAK_BYTES_PER_S,
                                         "check_max_rel_err": err}
        del G, X, out

    x = torch.randn((n, bench.FEATURES), generator=gen, dtype=torch.float32).to(device).requires_grad_(True)
    w_plain = torch.rand((E,), generator=gen, dtype=torch.float32).to(device)
    w_train = w_plain.clone().requires_grad_(True)
    layer = tfg.layers.MeanGraphSage(256, seed=2, trainable=True)
    layer([x, edge_index, w_plain])
    g = torch.randn((n, 256), generator=gen, dtype=torch.float32).to(device)

    def step(w):
        x.grad = None
        w.grad = None
        for p in layer.parameters():
            p.grad = None
        layer([x, edge_index, w], training=True).backward(g)

    arms = {"edge_weight_fixed": lambda: step(w_plain), "edge_weight_trainable": lambda: step(w_train)}
    times = {k: [] for k in arms}
    for i in range(args.steps + 1):                              # round 0 warms both arms up
        for name, fn in arms.items():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            fn()
            ev[1].record()
            torch.cuda.synchronize()
            if i:
                times[name].append(ev[0].elapsed_time(ev[1]))
    sage = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
    sage["edge_gradient_cost_ms"] = sage["edge_weight_trainable"] - sage["edge_weight_fixed"]
    result["mean_graph_sage_256_fwd_bwd_ms"] = sage
    result["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    print(json.dumps(result))


if __name__ == "__main__":
    main()
