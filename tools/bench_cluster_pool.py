# coding=utf-8
"""K8 (DiffPool / MinCutPool coarsening) on the device: per-call CUDA-event times of K8a, K8b, K1 and K7 for one
ClusterPool forward + backward, K8a's and K8b's byte floors as a share of 3.35 TB/s, and an alternating comparison with a
torch-ops composition of the same math (checked equal first).

Workloads:
  tu       4096 graphs of 10-50 nodes, about 2.2 N_g symmetric edges each, C = 20, D = 128 (a TU-dataset batch)
  products one graph of 2 449 029 nodes, bench.py's generator (123.7 M edges), C = 16, D = 128 (a one-graph MinCut)

    python tools/bench_cluster_pool.py [--steps 10] [--workloads tu,products]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tf_geometric_b200 import _ffi, autograd          # noqa: E402
from tf_geometric_b200.nn.pool import cluster_pool    # noqa: E402

HBM = 3.35e12
TIMED = ("tfgk_graph_tmm_f32", "tfgk_graph_rmm_f32", "tfgk_spmm_f32", "tfgk_sddmm_csr_f32")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as err:                            # the number is reported as unknown, never guessed
        return "unknown ({})".format(err)


def tu_batch(dev, seed=0):
    rs = np.random.RandomState(seed)
    sizes = rs.randint(10, 51, 4096)
    rows, cols, base = [], [], 0
    for n in sizes:
        half = int(1.1 * n)
        u, v = rs.randint(0, n, half), rs.randint(0, n, half)
        keep = u != v
        rows.append(base + np.concatenate([u[keep], v[keep]]))
        cols.append(base + np.concatenate([v[keep], u[keep]]))
        base += n
    ei = torch.tensor(np.stack([np.concatenate(rows), np.concatenate(cols)]).astype(np.int32), device=dev)
    ngi = torch.tensor(np.repeat(np.arange(len(sizes)), sizes).astype(np.int32), device=dev)
    return ei, ngi, 20


def products(dev):
    import bench
    ei = bench.make_graph_device(bench.PRODUCTS_NODES, bench.PRODUCTS_UNDIRECTED, 0, dev)
    return ei, torch.zeros(bench.PRODUCTS_NODES, dtype=torch.int32, device=dev), 16


def torch_composition(x, S, w, ei, ngi, G, C):
    """The same P, Q with torch ops: T = A S as an index_add_ of w_e S[col_e] (torch.sparse.mm would backpropagate a dense
    N x N gradient to the values); per-graph S^T Y as padded bmm (or one mm for G = 1)."""
    N = S.shape[0]
    row, col = ei[0].long(), ei[1].long()
    T = torch.zeros((N, C), device=S.device).index_add_(0, row, w.unsqueeze(1) * S[col])
    if G == 1:
        return S.t() @ x, S.t() @ T
    counts = torch.bincount(ngi.long(), minlength=G)
    m = int(counts.max())
    start = torch.cumsum(counts, 0) - counts
    rank = torch.arange(N, device=S.device) - start[ngi.long()]
    idx = (ngi.long(), rank)
    Sp = torch.zeros((G, m, C), device=S.device).index_put(idx, S)
    Xp = torch.zeros((G, m, x.shape[1]), device=S.device).index_put(idx, x)
    Tp = torch.zeros((G, m, C), device=S.device).index_put(idx, T)
    return torch.bmm(Sp.transpose(1, 2), Xp).reshape(G * C, -1), torch.bmm(Sp.transpose(1, 2), Tp).reshape(G * C, C)


def run(name, ei, ngi, C, D, steps, dev):
    N, E = ngi.numel(), ei.shape[1]
    G = int(ngi.max()) + 1
    gen = torch.Generator(device=dev)
    gen.manual_seed(1)
    x = torch.randn((N, D), generator=gen, device=dev).requires_grad_(True)
    logits = torch.randn((N, C), generator=gen, device=dev).requires_grad_(True)
    w = (torch.rand((E,), generator=gen, device=dev) + 0.5).requires_grad_(True)
    _, layout = cluster_pool.cluster_layout(ei, ngi, N, C, G)

    def ours():
        S = torch.softmax(logits, -1)
        P, Q = autograd.ClusterPool.apply(x, S, w, layout)
        (P.sum() + Q.sum()).backward()
        return P, Q

    def theirs():
        S = torch.softmax(logits, -1)
        P, Q = torch_composition(x, S, w, ei, ngi, G, C)
        (P.sum() + Q.sum()).backward()
        return P, Q

    with torch.no_grad():
        S = torch.softmax(logits, -1)
        P, Q = autograd.ClusterPool.apply(x, S, w, layout)
        P2, Q2 = torch_composition(x, S, w, ei, ngi, G, C)
    err = max(float((P - P2).abs().max() / P2.abs().max()), float((Q - Q2).abs().max() / Q2.abs().max()))
    assert err < 1e-4, "torch composition differs: {}".format(err)

    for _ in range(2):
        ours()
        theirs()
    torch.cuda.synchronize()
    trace = _ffi.CallTrace(timed=TIMED)
    prev = _ffi.set_trace(trace)
    ours()
    torch.cuda.synchronize()
    _ffi.set_trace(prev)
    calls = {k: [round(t, 4) for t in trace.elapsed_ms(k)] for k in TIMED}
    # byte floors of the K8 calls of one forward + backward, in launch order
    f = 4
    tmm = [N * f * (C + C) + G * C * C * f + G * 8, N * f * (C + D) + G * C * D * f + G * 8]
    rmm = [N * f * (C + D + 1) + G * C * D * f,       # dX = S dP
           N * f * (C + C + 1) + G * C * C * f,       # T dQ^T
           N * f * (D + C + 1) + G * C * D * f,       # X dP^T (beta = 1 reads out too)
           N * f * (C + C + 1) + G * C * C * f,       # U dQ
           N * f * (C + C + 1) + G * C * C * f]       # S dQ
    rmm[2:4] = [b + N * C * f for b in rmm[2:4]]
    share = {}
    for key, floors in (("tfgk_graph_tmm_f32", tmm), ("tfgk_graph_rmm_f32", rmm)):
        ts = calls[key]
        share[key] = [round(b / HBM / (t * 1e-3), 3) for b, t in zip(floors, ts)]

    times = {"ours": [], "torch": []}
    for _ in range(steps):
        for label, fn in (("ours", ours), ("torch", theirs)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[label].append((time.perf_counter() - t0) * 1e3)
    return {"workload": name, "N": N, "E": E, "G": G, "C": C, "D": D, "call_ms": calls, "hbm_share": share,
            "fwd_bwd_ms_median": {k: round(float(np.median(v)), 3) for k, v in times.items()},
            "fwd_bwd_ms_all": {k: [round(t, 3) for t in v] for k, v in times.items()}, "torch_rel_err": err}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--workloads", default="tu,products")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cluster_pool needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {"card": card()}
    for name in args.workloads.split(","):
        ei, ngi, C = tu_batch(dev) if name == "tu" else products(dev)
        out[name] = run(name, ei, ngi, C, 128, args.steps, dev)
        print(json.dumps(out[name]), flush=True)
    print(json.dumps({"card": out["card"]}))


if __name__ == "__main__":
    main()
