# coding=utf-8
"""fp8 message rows against bf16 and fp32 at the ogbn-products shape (2 449 029 nodes, 123.7M directed edges + self loops,
100 features): CUDA-event times of K4 (the GCN projection, and the GAT projection Q | K | V with K | V in each mode), K1
(weighted, D = 128), K3 (8 heads, A = 128) and the whole GCN(128, relu) + GAT(128, 8 heads, relu) forward, the three
modes alternating in one run.  Every fp8 output is checked against its contract
first (K4 against the quantised fp32 projection, K1 and K3 bit for bit against the fp32 kernels over the dequantised
rows).  Bytes over each kernel's byte floor are reported as a share of the 3.35 TB/s data-sheet bandwidth, with the card's
name and power limit.

    python tools/bench_fp8.py [--steps 20] [--warmup 3]
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

HBM = 3.35e12
FP8 = torch.float8_e4m3fn


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as err:                            # reported as unknown, never guessed
        return "unknown ({})".format(err)


def same_bits(a, b, what):
    if not torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)):
        raise SystemExit("{}: fp8 result breaks its contract".format(what))


def deq(t, groups):
    return t.data.contiguous().view(FP8).float() * torch.exp2(t.exps.float()[:, groups])


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
        raise SystemExit("bench_fp8 needs a GPU")
    dev = torch.device("cuda")
    n, f, a, heads = bench.PRODUCTS_NODES, bench.FEATURES, bench.UNITS, bench.HEADS
    ei = bench.make_graph_device(n, bench.PRODUCTS_UNDIRECTED, 0, dev)
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    x = torch.randn((n, f), generator=g, device=dev)
    graph = tfg.Graph(x, ei)
    modes = {"fp32": None, "bf16": torch.bfloat16, "fp8": FP8}
    layers = {m: (tfg.layers.GCN(a, activation=tfg.nn.relu, seed=1, message_dtype=md),
                  tfg.layers.GAT(a, num_heads=heads, activation=tfg.nn.relu, seed=2, message_dtype=md))
              for m, md in modes.items()}
    layers["fp32"][0].build_cache_for_graph(graph)

    def forward(l1, l2):
        return l1([graph.x, graph.edge_index], cache=graph.cache), l2([graph.x, graph.edge_index], cache=graph.cache)
    for m in modes:
        forward(*layers[m])
    for m in ("bf16", "fp8"):
        for ref, other in zip(layers["fp32"], layers[m]):
            for (_, p32), (_, pm) in zip(ref.named_parameters(), other.named_parameters()):
                pm.data.copy_(p32.data)
    gcn, gat = layers["fp32"]

    normed = tfg.nn.conv.gcn.gcn_norm_adj(tfg.SparseMatrix(graph.edge_index, None, [n, n]), cache=graph.cache)
    csr, w = normed.csr, normed.value_csr
    E = csr.nnz
    gat_csr, _ = _structure.csr_for_edge_index(graph.edge_index, n, add_self_loop=True, cache=graph.cache)
    E3 = gat_csr.nnz

    # ---- inputs of the kernels, and the contract checks -----------------------------------------------------------------
    wg = gcn.kernel.data
    wq, wk, wv = (p.data for p in (gat.query_kernel, gat.key_kernel, gat.kernel))
    bq, bk = gat.query_bias.data, gat.key_bias.data
    Q = torch.empty((n, a), device=dev)
    kv = {"fp32": torch.empty((n, 2 * a), device=dev), "bf16": torch.empty((n, 2 * a), dtype=torch.bfloat16, device=dev),
          "fp8": ops.fp8_table(n, 2 * a, dev, groups=2)}
    gh = {"fp32": torch.empty((n, a), device=dev), "bf16": ops.bf16_table(n, a, dev), "fp8": ops.fp8_table(n, a, dev)}

    def kv_blocks(m):
        t = kv[m]
        return (t.block(0, a, group=0), t.block(a, 2 * a, group=1)) if m == "fp8" else (t[:, :a], t[:, a:])

    def k4(m):
        kb, vb = kv_blocks(m)
        return lambda: ops.gemm_proj(x, [(wq, bq, ops.ACT_RELU, Q), (wk, bk, ops.ACT_RELU, kb), (wv, None, ops.ACT_NONE, vb)])

    def k4g(m):
        return lambda: ops.gemm_proj(x, [(wg, None, ops.ACT_NONE, gh[m])])
    for m in modes:
        k4(m)()
        k4g(m)()
    grp2 = torch.cat([torch.zeros(a, dtype=torch.long), torch.ones(a, dtype=torch.long)]).to(dev)
    grp1 = torch.zeros(a, dtype=torch.long, device=dev)
    ref8 = ops.quantize_fp8(kv["fp32"][:, a:].contiguous())
    if not (torch.equal(ref8.data, kv["fp8"].data[:, a:]) and torch.equal(ref8.exps[:, 0], kv["fp8"].exps[:, 1])):
        raise SystemExit("K4: fp8 V block breaks its contract")
    ref8 = ops.quantize_fp8(gh["fp32"])
    if not (torch.equal(ref8.data, gh["fp8"].data) and torch.equal(ref8.exps, gh["fp8"].exps)):
        raise SystemExit("K4: fp8 GCN block breaks its contract")
    del ref8
    out1 = torch.empty((n, a), device=dev)

    def k1(m):
        return lambda: ops.spmm(csr, w, gh[m], reduce="sum", act=ops.ACT_RELU, out=out1)
    k1("fp8")()
    got1 = out1.clone()
    ops.spmm(csr, w, deq(gh["fp8"], grp1), reduce="sum", act=ops.ACT_RELU, out=out1)
    same_bits(got1, out1, "K1")
    del got1
    out3 = torch.empty((n, a), device=dev)

    def k3(m):
        if m == "fp8":
            return lambda: ops.gat_fused(gat_csr, Q, kv[m], None, heads, act=ops.ACT_RELU, out=out3)
        kb, vb = kv_blocks(m)
        return lambda: ops.gat_fused(gat_csr, Q, kb, vb, heads, act=ops.ACT_RELU, out=out3)
    k3("fp8")()
    got3 = out3.clone()
    kvh = deq(kv["fp8"], grp2)
    ops.gat_fused(gat_csr, Q, kvh[:, :a], kvh[:, a:], heads, act=ops.ACT_RELU, out=out3)
    same_bits(got3, out3, "K3")
    del got3, kvh

    # ---- byte floors -------------------------------------------------------------------------------------------------
    floors = {
        "K4_gat": {"fp32": n * (4 * f + 4 * 3 * a), "bf16": n * (4 * f + 4 * a + 2 * 2 * a),
                   "fp8": n * (4 * f + 4 * a + 2 * a + 2)},
        "K4_gcn": {"fp32": n * (4 * f + 4 * a), "bf16": n * (4 * f + 2 * a), "fp8": n * (4 * f + a + 1)},
        "K1": {"fp32": E * (4 * a + 8) + n * (4 * a + 8), "bf16": E * (2 * a + 8) + n * (4 * a + 8),
               "fp8": E * (a + 1 + 8) + n * (4 * a + 8)},
        "K3": {"fp32": E3 * (8 * a + 4) + n * (8 * a + 8), "bf16": E3 * (4 * a + 4) + n * (8 * a + 8),
               "fp8": E3 * (2 * a + 2 + 4) + n * (8 * a + 8)},
    }
    work = {"K4_gat": k4, "K4_gcn": k4g, "K1": k1, "K3": k3, "forward": lambda m: (lambda: forward(*layers[m]))}
    fns = {k: {m: mk(m) for m in modes} for k, mk in work.items()}
    for per in fns.values():
        for fn in per.values():
            for _ in range(args.warmup):
                fn()
    torch.cuda.synchronize()
    times = {k: {m: [] for m in modes} for k in fns}
    for _ in range(args.steps):                          # the three modes alternate, one call each per round
        for k, per in fns.items():
            for m, fn in per.items():
                times[k][m] += timed(fn, 1)
    res = {"card": card(), "nodes": n, "edges_k1": E, "edges_k3": E3, "steps": args.steps}
    for k, t in times.items():
        row = {}
        for m in modes:
            ms = float(np.median(t[m]))
            row[m + "_ms"] = round(ms, 4)
            row[m + "_spread_ms"] = [round(float(np.min(t[m])), 4), round(float(np.max(t[m])), 4)]
            if k in floors:
                row[m + "_floor_bytes"] = floors[k][m]
                row[m + "_share_of_hbm"] = round(floors[k][m] / (ms * 1e-3) / HBM, 4)
        row["fp8_over_bf16_speedup"] = round(row["bf16_ms"] / row["fp8_ms"], 4)
        res[k] = row

    print(json.dumps(res))


if __name__ == "__main__":
    main()
