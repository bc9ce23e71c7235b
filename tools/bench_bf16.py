# coding=utf-8
"""bf16 message rows against fp32 at the ogbn-products shape (2 449 029 nodes, 123.7M directed edges + self loops, 100
features): CUDA-event times of K4 (the GAT projection, Q fp32 next to K | V fp32 or bf16), K1 (weighted, D = 128), K3 (8
heads, A = 128 on the TMA ring, and A = 256 on the single-pass kernel) and the whole GCN(128, relu) + GAT(128, 8 heads, relu) forward, fp32 and bf16 alternating in one run.
Every output is checked against its contract first (K1, K4 bit for bit; K3 against float64 on sampled rows).  Bytes over
each kernel's byte floor are reported as a share of the 3.35 TB/s data-sheet bandwidth, with the card's name and power limit.

    python tools/bench_bf16.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench                                          # noqa: E402
import tf_geometric_b200 as tfg                       # noqa: E402
from tf_geometric_b200 import ops, _structure        # noqa: E402
from tf_geometric_b200.nn.conv.gat import project    # noqa: E402

HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as err:                            # reported as unknown, never guessed
        return "unknown ({})".format(err)


def same_bits(a, b, what):
    ia = a.contiguous().view(torch.int16 if a.dtype == torch.bfloat16 else torch.int32)
    ib = b.contiguous().view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32)
    if not torch.equal(ia, ib):
        raise SystemExit("{}: bf16 result breaks its contract".format(what))


def timed(fn, steps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bf16 needs a GPU")
    dev = torch.device("cuda")
    n, f, a, heads = bench.PRODUCTS_NODES, bench.FEATURES, bench.UNITS, bench.HEADS
    ei = bench.make_graph_device(n, bench.PRODUCTS_UNDIRECTED, 0, dev)
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    x = torch.randn((n, f), generator=g, device=dev)
    graph = tfg.Graph(x, ei)
    gcn = tfg.layers.GCN(a, activation=tfg.nn.relu, seed=1)
    gat = tfg.layers.GAT(a, num_heads=heads, activation=tfg.nn.relu, seed=2)
    gcn16 = tfg.layers.GCN(a, activation=tfg.nn.relu, seed=1, message_dtype=torch.bfloat16)
    gat16 = tfg.layers.GAT(a, num_heads=heads, activation=tfg.nn.relu, seed=2, message_dtype=torch.bfloat16)
    gcn.build_cache_for_graph(graph)

    def forward(l1, l2):
        return l1([graph.x, graph.edge_index], cache=graph.cache), l2([graph.x, graph.edge_index], cache=graph.cache)
    forward(gcn, gat)
    forward(gcn16, gat16)
    for a32, a16 in ((gcn, gcn16), (gat, gat16)):
        for (_, p32), (_, p16) in zip(a32.named_parameters(), a16.named_parameters()):
            p16.data.copy_(p32.data)

    normed = tfg.nn.conv.gcn.gcn_norm_adj(tfg.SparseMatrix(graph.edge_index, None, [n, n]), cache=graph.cache)
    csr, w = normed.csr, normed.value_csr
    E = csr.nnz
    gat_csr, _ = _structure.csr_for_edge_index(graph.edge_index, n, add_self_loop=True, cache=graph.cache)
    E3 = gat_csr.nnz

    # ---- inputs of the kernels, and the contract checks -----------------------------------------------------------------
    wq, wk, wv = (p.data for p in (gat.query_kernel, gat.key_kernel, gat.kernel))
    bq, bk = gat.query_bias.data, gat.key_bias.data
    Q = torch.empty((n, a), device=dev)
    kv32 = torch.empty((n, 2 * a), device=dev)
    kv16 = torch.empty((n, 2 * a), dtype=torch.bfloat16, device=dev)

    def k4(kv):
        return lambda: project(x, [(wq, bq, ops.ACT_RELU, Q), (wk, bk, ops.ACT_RELU, kv[:, :a]), (wv, None, ops.ACT_NONE,
                                                                                                  kv[:, a:])])
    k4(kv32)()
    k4(kv16)()
    same_bits(kv16, kv32.to(torch.bfloat16), "K4")
    h32 = kv32[:, a:].contiguous()
    h16 = kv16[:, a:].contiguous()
    out1 = torch.empty((n, a), device=dev)

    def k1(h):
        return lambda: ops.spmm(csr, w, h, reduce="sum", act=ops.ACT_RELU, out=out1)
    k1(h16)()
    ref1 = out1.clone()
    ops.spmm(csr, w, h16.float(), reduce="sum", act=ops.ACT_RELU, out=out1)
    same_bits(ref1, out1, "K1")
    del ref1
    out3 = torch.empty((n, a), device=dev)

    def k3(kv):
        return lambda: ops.gat_fused(gat_csr, Q, kv[:, :a], kv[:, a:], heads, act=ops.ACT_RELU, out=out3)
    k3(kv16)()
    rows = torch.randint(0, n, (64,), generator=g, device=dev)
    rp, col = gat_csr.rowptr.cpu().numpy(), gat_csr.col.cpu().numpy()
    qd, kd, vd = Q.double().cpu().numpy(), kv16[:, :a].double().cpu().numpy(), kv16[:, a:].double().cpu().numpy()
    got = out3.double().cpu().numpy()
    dh = a // heads
    worst = 0.0
    for r in rows.cpu().numpy():
        c = col[rp[r]:rp[r + 1]]
        want = []
        for h in range(heads):
            s = kd[c, h * dh:(h + 1) * dh] @ qd[r, h * dh:(h + 1) * dh] / np.sqrt(np.float32(dh))
            p = np.exp(s - s.max())
            want.append((p / (p.sum() + 1e-8)) @ vd[c, h * dh:(h + 1) * dh])
        want = np.maximum(np.concatenate(want), 0)
        worst = max(worst, float(np.max(np.abs(got[r] - want) / (2e-5 * np.abs(want) + 2e-6 * np.abs(want).max() + 1e-30))))
    if worst > 1.0:
        raise SystemExit("K3: bf16 result breaks its contract (worst error / bound {:.3g})".format(worst))

    # K3 with 8 heads over A = 256 (the register-staged single-pass kernel in both modes), random Q, K, V
    aw = 2 * a
    Qw = torch.randn((n, aw), generator=g, device=dev)
    kvw32 = torch.randn((n, 2 * aw), generator=g, device=dev)
    kvw16 = kvw32.to(torch.bfloat16)
    outw = torch.empty((n, aw), device=dev)

    def k3w(kv):
        return lambda: ops.gat_fused(gat_csr, Qw, kv[:, :aw], kv[:, aw:], heads, act=ops.ACT_RELU, out=outw)
    k3w(kvw16)()
    ref3w = outw.clone()
    wf = kvw16.float()
    ops.gat_fused(gat_csr, Qw, wf[:, :aw], wf[:, aw:], heads, act=ops.ACT_RELU, out=outw)
    same_bits(ref3w, outw, "K3 (A = 256)")
    del ref3w, wf

    # ---- byte floors -------------------------------------------------------------------------------------------------
    floors = {
        "K4": {"fp32": n * (4 * f + 4 * 3 * a), "bf16": n * (4 * f + 4 * a + 2 * 2 * a)},
        "K1": {"fp32": E * (4 * a + 8) + n * (4 * a + 8), "bf16": E * (2 * a + 8) + n * (4 * a + 8)},
        "K3": {"fp32": E3 * (8 * a + 4) + n * (8 * a + 8), "bf16": E3 * (4 * a + 4) + n * (8 * a + 8)},
        "K3_A256": {"fp32": E3 * (8 * aw + 4) + n * (8 * aw + 8), "bf16": E3 * (4 * aw + 4) + n * (8 * aw + 8)},
    }
    work = {"K4": (k4(kv32), k4(kv16)), "K1": (k1(h32), k1(h16)), "K3": (k3(kv32), k3(kv16)),
            "K3_A256": (k3w(kvw32), k3w(kvw16)),
            "forward": (lambda: forward(gcn, gat), lambda: forward(gcn16, gat16))}
    for fns in work.values():
        for fn in fns:
            for _ in range(args.warmup):
                fn()
    torch.cuda.synchronize()
    times = {k: {"fp32": [], "bf16": []} for k in work}
    for _ in range(args.steps):                          # fp32 and bf16 alternate, one call each per round
        for k, (f32, f16) in work.items():
            times[k]["fp32"] += timed(f32, 1)
            times[k]["bf16"] += timed(f16, 1)
    res = {"card": card(), "nodes": n, "edges_k1": E, "edges_k3": E3, "steps": args.steps, "k3_worst_over_bound": worst}
    for k, t in times.items():
        row = {}
        for mode in ("fp32", "bf16"):
            ms = float(np.median(t[mode]))
            row[mode + "_ms"] = round(ms, 4)
            row[mode + "_spread_ms"] = [round(float(np.min(t[mode])), 4), round(float(np.max(t[mode])), 4)]
            if k in floors:
                row[mode + "_floor_bytes"] = floors[k][mode]
                row[mode + "_share_of_hbm"] = round(floors[k][mode] / (ms * 1e-3) / HBM, 4)
        row["speedup"] = round(row["fp32_ms"] / row["bf16_ms"], 4)
        res[k] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()
