# coding=utf-8
"""GCN inference at the products shape (N = 2,449,029, F = 100, U = 128), three routes timed alternately with CUDA events:

  project_first  K4 (x -> x W, [N, 128]) then K1 at D = 128 with bias + relu     (the route before aggregate-first)
  unfused        K1 at D = 100 ([N, 100] aggregate stored) then K4 with bias + relu (a reference point only)
  fused          tfgk_spmm_proj_f32: K1's ring at F = 100, projection in its epilogue

Every route's output is checked against float64 on sampled rows before timing.  Prints one JSON line with the medians,
the spread, each route's byte floor over 3.35 TB/s (H100 SXM data sheet) and the card's name and power limit.
Usage: python tools/bench_gcn_agg_first.py [--reps 15]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import bench                                   # noqa: E402
import tf_geometric_b200 as tfg                # noqa: E402
from tf_geometric_b200 import ops              # noqa: E402

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def check(name, got, rowptr, col, w, x, W, b, rows):
    xh, Wh, bh = x.double(), W.double().cpu().numpy(), b.double().cpu().numpy()
    got = got[torch.as_tensor(rows, device=got.device)].double().cpu().numpy()
    worst = 0.0
    for i, r in enumerate(rows):
        e0, e1 = int(rowptr[r]), int(rowptr[r + 1])
        c = torch.as_tensor(col[e0:e1], device=x.device).long()
        ww = torch.as_tensor(w[e0:e1], device=x.device).double()[:, None]
        agg = (ww * xh[c]).sum(0).cpu().numpy()
        agg_abs = (ww.abs() * xh[c].abs()).sum(0).cpu().numpy()
        want = np.maximum(agg @ Wh + bh, 0.0)
        S = agg_abs @ np.abs(Wh) + np.abs(bh)
        ratio = np.abs(got[i] - want) / (((e1 - e0) + W.shape[0] + 1) * 2.0 ** -24 * S + 1e-30)
        worst = max(worst, float(ratio.max()))
    assert worst <= 1.0, "{}: error {} x the float64 bound".format(name, worst)
    return worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    dev = torch.device("cuda")
    n, pairs, F, U = bench.PRODUCTS_NODES, bench.PRODUCTS_UNDIRECTED, 100, 128
    ei = bench.make_graph_device(n, pairs, 0, dev)
    gen = torch.Generator(device="cpu")
    gen.manual_seed(1)
    x = torch.randn((n, F), generator=gen).to(dev)
    graph = tfg.Graph(x, ei)
    layer = tfg.layers.GCN(U, activation=tfg.nn.relu, seed=2)
    layer.build_cache_for_graph(graph)
    layer([graph.x, graph.edge_index], cache=graph.cache)
    W = layer.kernel.data
    b = torch.randn(U, generator=gen).to(dev)
    normed = tfg.nn.conv.gcn.gcn_norm_adj(tfg.SparseMatrix(graph.edge_index, None, [n, n]), cache=graph.cache)
    csr, w = normed.csr, normed.value_csr
    E = csr.nnz
    routes = {
        "project_first": lambda: ops.spmm(csr, w, ops.gemm(x, W), bias=b, act=ops.ACT_RELU),
        "unfused": lambda: ops.gemm(ops.spmm(csr, w, x), W, bias=b, act=ops.ACT_RELU),
        "fused": lambda: ops.spmm_proj(csr, w, x, W, bias=b, act=ops.ACT_RELU),
    }
    floors = {                                                     # DESIGN.md K1 / K4 byte counts, weighted CSR
        "project_first": (n * F * 4 + n * U * 4) + E * (4 * U + 8) + n * (4 * U + 8),
        "unfused": E * (4 * F + 8) + n * (4 * F + 8) + (n * F * 4 + n * U * 4),
        "fused": E * (4 * F + 8) + n * (4 * U + 8),
    }
    rowptr, col, wh = csr.rowptr.cpu().numpy(), csr.col.cpu().numpy(), w.cpu().numpy()
    rows = np.random.RandomState(0).randint(0, n, 200)
    err = {k: check(k, f(), rowptr, col, wh, x, W, b, rows) for k, f in routes.items()}
    for f in routes.values():
        f()
    times = {k: [] for k in routes}
    for _ in range(args.reps):
        for k, f in routes.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            torch.cuda.synchronize()
            times[k].append(s.elapsed_time(e))
    res = {"card": card(), "n": n, "edges_with_loops": E, "F": F, "U": U, "reps": args.reps, "routes": {}}
    for k, t in times.items():
        t = np.array(t)
        med = float(np.median(t))
        res["routes"][k] = {"median_ms": round(med, 3), "min_ms": round(float(t.min()), 3), "max_ms": round(float(t.max()), 3),
                            "floor_gb": round(floors[k] / 1e9, 2), "floor_share_of_3.35TBps": round(floors[k] / HBM * 1e3 / med, 3),
                            "max_err_over_bound": round(err[k], 4)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
