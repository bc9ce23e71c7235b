# coding=utf-8
"""Packed keys against the dense K | V table for the fused GAT aggregation (K3) at the ogbn-products shape (2 449 029 nodes,
123.7M directed edges + self loops, 100 features, 8 heads, A = 128): CUDA-event times of K3 dense (gat_tma4_kernel<2>), K3
packed (gat_tma4_packed_kernel<2>) and the pack kernel, alternating in one run, first with the
layer's own keys (ReLU of x W_k, glorot W_k, zero bias) and then with a worst case without zeros (ReLU of x W_k + 10).
Every packed output is checked bit for bit against the dense one first.  Prints the zero fraction of K, each kernel's byte
floor (the packed one from the actual copy sizes) and its share of the 3.35 TB/s data-sheet bandwidth, with the card's name
and power limit.

    python tools/bench_gat_packed.py [--steps 20] [--warmup 3]
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
from tf_geometric_b200 import ops, _structure        # noqa: E402
from tf_geometric_b200.nn.conv.gat import project    # noqa: E402

HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as err:                            # reported as unknown, never guessed
        return "unknown ({})".format(err)


def timed_once(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    return a, b


def run_alternating(variants, steps, warmup):
    """variants: {name: fn}; one launch of each per round, rounds alternate the order; returns {name: [ms]}."""
    names = list(variants)
    for _ in range(warmup):
        for name in names:
            variants[name]()
    torch.cuda.synchronize()
    events = {name: [] for name in names}
    for i in range(steps):
        for name in (names if i % 2 == 0 else names[::-1]):
            events[name].append(timed_once(variants[name]))
    torch.cuda.synchronize()
    return {name: [a.elapsed_time(b) for a, b in ev] for name, ev in events.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gat_packed needs a GPU")
    dev = torch.device("cuda")
    n, f, a, heads = bench.PRODUCTS_NODES, bench.FEATURES, bench.UNITS, bench.HEADS
    ei = bench.make_graph_device(n, bench.PRODUCTS_UNDIRECTED, 0, dev)
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    x = torch.randn((n, f), generator=g, device=dev)
    csr, _ = _structure.csr_for_edge_index(ei, n, add_self_loop=True)
    E = csr.nnz
    wq, wk, wv = (bench.glorot((f, a), s).to(dev) for s in (11, 12, 13))
    zero = torch.zeros((a,), device=dev)
    Q = torch.empty((n, a), device=dev)
    kv = torch.empty((n, 2 * a), device=dev)
    table, sizes = ops.packed_key_table(n, a, dev)
    out_d = torch.empty((n, a), device=dev)
    out_p = torch.empty((n, a), device=dev)
    col = csr.col.long()
    info = {"card": card(), "nodes": n, "edges_with_self_loops": E, "heads": heads, "A": a}
    print(json.dumps(info), flush=True)

    for case, key_bias in (("relu_keys", 0.0), ("no_zeros", 10.0)):
        project(x, [(wq, zero, ops.ACT_RELU, Q), (wk, zero + key_bias, ops.ACT_RELU, kv[:, :a]),
                    (wv, None, ops.ACT_NONE, table[:, :a])])
        kv[:, a:].copy_(table[:, :a])
        K = kv[:, :a]

        def pack():
            ops.gat_pack_keys(K, table, sizes)

        def dense():
            ops.gat_fused(csr, Q, K, kv[:, a:], heads, act=ops.ACT_RELU, out=out_d)

        def packed():
            ops.gat_fused_packed(csr, Q, table, sizes, heads, act=ops.ACT_RELU, out=out_p)

        pack()
        dense()
        out_p.zero_()
        packed()
        if not torch.equal(out_p.view(torch.int32), out_d.view(torch.int32)):
            raise SystemExit("{}: packed K3 is not bit-identical to dense K3".format(case))
        zero_frac = float((K.contiguous().view(torch.int32) == 0).double().mean())
        copy_bytes = float((sizes.long()[col] * 16).sum())
        node_bytes = n * (4 * a + 4 * a + 8)                       # Q and the output once per node, rowptr
        floor_dense = E * (8 * a + 4) + node_bytes                 # DESIGN.md K3
        floor_packed = copy_bytes + E * (4 + 1) + node_bytes       # the slot bytes copied, col and ksize per edge
        floor_pack = n * 4 * a + float((sizes.long() * 16 - 4 * a).sum()) + n   # read K, write mask + keys, ksize

        ms = run_alternating({"k3_dense": dense, "pack": pack, "k3_packed": packed}, args.steps, args.warmup)
        res = {"case": case, "key_zero_fraction": zero_frac, "avg_packed_copy_bytes_per_edge": copy_bytes / E,
               "floor_bytes": {"k3_dense": floor_dense, "k3_packed": floor_packed, "pack": floor_pack}, "ms": {}}
        for name, v in ms.items():
            med = float(np.median(v))
            floor = floor_dense if name == "k3_dense" else floor_pack if name == "pack" else floor_packed
            res["ms"][name] = {"median": med, "min": float(np.min(v)), "max": float(np.max(v)),
                               "share_of_3.35TBps": floor / (med * 1e-3) / HBM}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
