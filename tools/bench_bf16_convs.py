# coding=utf-8
"""bf16 message rows against fp32 for the GraphSAGE, GIN, LEConv, APPNP, SGC, SSGC, TAGCN and ChebyNet forwards at the
ogbn-products shape (2 449 029 nodes, 123.7M directed edges, 100 features; hidden width 128, APPNP and SGC also with 47
outputs, APPNP and SSGC with k = 10), fp32 and bf16 alternating in one run, CUDA-event times.  Before anything is timed,
every bf16 output is checked bit for bit against the fp32 kernels applied with each gathered table replaced by its
widened bf16 rounding (DESIGN.md section 5), and each K1 variant against its contract.  K1 launches (D = 100, 128, 47)
are also reported as a share of the 3.35 TB/s data-sheet bandwidth by their byte floors:
fp32 E(4D + 8) + N(4D + 8), bf16 gather with an fp32 store E(2D + 8) + N(4D + 8), bf16-only store E(2D + 8) + N(2D + 8).

    python tools/bench_bf16_convs.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench                                                   # noqa: E402
import tf_geometric_b200 as tfg                                # noqa: E402
from tf_geometric_b200 import ops, _structure                 # noqa: E402
from tf_geometric_b200.nn.conv import graph_sage as gs        # noqa: E402
from tf_geometric_b200.nn.conv.gcn import gcn_norm_adj        # noqa: E402
from tf_geometric_b200.nn.conv.propagation import chebynet_norm_edge   # noqa: E402
from bench_bf16 import HBM, card, same_bits, timed           # noqa: E402

B16 = torch.bfloat16


def bf(t):
    return t.to(B16).float()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bf16_convs needs a GPU")
    dev = torch.device("cuda")
    n, f, hid = bench.PRODUCTS_NODES, bench.FEATURES, bench.UNITS
    ei = bench.make_graph_device(n, bench.PRODUCTS_UNDIRECTED, 0, dev)
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    x = torch.randn((n, f), generator=g, device=dev)
    ew = torch.rand((ei.shape[1],), generator=g, device=dev)

    def w(*shape):
        return torch.randn(shape, generator=g, device=dev) * (1.0 / np.sqrt(shape[0]))

    half = hid // 2
    ws, wn, b = w(f, half), w(f, half), w(hid)
    wm, bm, wpn = w(f, hid), w(hid), w(hid, half)
    wk, bk = w(f, hid), w(hid)
    wl = [w(f, hid) for _ in range(3)]
    bl = [w(hid) for _ in range(3)]
    wt, wc = w(4 * f, hid), [w(f, hid) for _ in range(3)]
    apw = {u: ([w(f, hid), w(hid, u)], [w(hid), w(u)]) for u in (47, 128)}
    sgw = {u: (w(f, u), w(u)) for u in (47, 128)}
    cache = {}
    relu = tfg.nn.relu
    csr, _ = _structure.csr_for_edge_index(ei, n)
    w_csr = _structure.weights_in_csr_order(ew, csr)
    normed = gcn_norm_adj(tfg.SparseMatrix(ei, None, [n, n]), cache=cache)
    normed_t = gcn_norm_adj(tfg.SparseMatrix(ei, None, [n, n]), renorm=False)
    E = csr.nnz

    # ---- the forwards, fp32 (md=None) and bf16 (md=B16) ----------------------------------------------------------------
    fns = {
        "mean_graph_sage": lambda md: tfg.nn.mean_graph_sage(x, ei, ew, ws, wn, b, relu, message_dtype=md),
        "sum_graph_sage": lambda md: tfg.nn.sum_graph_sage(x, ei, ew, ws, wn, b, relu, message_dtype=md),
        "gcn_graph_sage": lambda md: tfg.nn.gcn_graph_sage(x, ei, None, wk, bk, relu, message_dtype=md),
        "mean_pool_graph_sage": lambda md: tfg.nn.mean_pool_graph_sage(x, ei, ew, ws, wm, wpn, bm, b, relu,
                                                                       message_dtype=md),
        "max_pool_graph_sage": lambda md: tfg.nn.max_pool_graph_sage(x, ei, ew, ws, wm, wpn, bm, b, relu,
                                                                     message_dtype=md),
        "gin": lambda md: tfg.nn.gin(x, ei, lambda h: h, eps=0.1, message_dtype=md),
        "le_conv": lambda md: tfg.nn.le_conv(x, ei, ew, wl[0], bl[0], wl[1], bl[1], wl[2], bl[2], relu, message_dtype=md),
        "appnp_47": lambda md: tfg.nn.appnp(x, ei, None, *apw[47], k=10, alpha=0.1, cache=cache, message_dtype=md),
        "appnp_128": lambda md: tfg.nn.appnp(x, ei, None, *apw[128], k=10, alpha=0.1, cache=cache, message_dtype=md),
        "sgc_47": lambda md: tfg.nn.sgc(x, ei, None, 2, *sgw[47], cache=cache, message_dtype=md),
        "sgc_128": lambda md: tfg.nn.sgc(x, ei, None, 2, *sgw[128], cache=cache, message_dtype=md),
        "ssgc": lambda md: tfg.nn.ssgc(x, ei, None, [apw[128][0][0]], [apw[128][1][0]], k=10, alpha=0.1, cache=cache,
                                       message_dtype=md),
        "tagcn": lambda md: tfg.nn.tagcn(x, ei, None, 3, wt, b, relu, message_dtype=md),
        "chebynet": lambda md: tfg.nn.chebynet(x, ei, None, 3, wc, b, message_dtype=md),
    }

    # ---- the compositions the bf16 forwards must equal bit for bit ------------------------------------------------------
    def appnp_ref(kernels, biases):
        h = ops.gemm(ops.gemm(x, kernels[0], bias=biases[0], act=ops.ACT_RELU), kernels[1], bias=biases[1])
        cur = bf(h)
        for _ in range(10):
            out = normed.matmul(cur, alpha=0.9, addend=h, beta=0.1)
            cur = bf(out)
        return out

    def sgc_ref(kern, bias):
        h = bf(ops.gemm_proj(x, [(kern, None, ops.ACT_NONE, None)])[0])
        return normed.matmul(bf(normed.matmul(h)), bias=bias)

    def ssgc_ref():
        h = ops.gemm(x, apw[128][0][0], bias=apw[128][1][0])
        output, cur = h * 0.1, h
        for _ in range(10):
            cur = normed.matmul(bf(cur))
            output = output + 0.9 * cur / 10
        return output

    def tagcn_ref():
        hops = torch.empty((n, 4 * f), device=dev)
        hops[:, :f].copy_(x)
        for i in range(3):
            normed_t.matmul(bf(hops[:, i * f:(i + 1) * f]), out=hops[:, (i + 1) * f:(i + 2) * f])
        return ops.gemm(hops, wt, bias=b, act=ops.ACT_RELU)

    def cheb_ref():
        idx, val = chebynet_norm_edge(ei, n, torch.ones((ei.shape[1],), device=dev))
        adj = tfg.SparseMatrix(idx, val, [n, n])
        t1 = adj.matmul(bf(x))
        out = ops.gemm(x, wc[0])
        ops.gemm(t1, wc[1], beta=1.0, out=out)
        ops.gemm(adj.matmul(bf(t1), alpha=2.0, addend=x, beta=-1.0), wc[2], beta=1.0, out=out)
        return out + b

    def pool_ref(reduce):
        h_node = ops.gemm_proj(x, [(wm, bm, ops.ACT_RELU, None)])[0]
        return gs._project_pair(x, ops.spmm(csr, None, bf(h_node), reduce=reduce), ws, wpn, b, relu, True,
                                False)

    refs = {
        "mean_graph_sage": lambda: gs._project_pair(x, ops.spmm(csr, w_csr, bf(x), reduce="mean"), ws, wn, b, relu, True,
                                                    False),
        "sum_graph_sage": lambda: gs._project_pair(x, ops.spmm(csr, w_csr, bf(x), reduce="sum"), ws, wn, b, relu, True,
                                                   False),
        "gcn_graph_sage": lambda: ops.gemm(tfg.SparseMatrix(*gs._norm_edge_as_matrix(ei, n, None, renorm=False)).matmul(
            bf(x)), wk, bias=bk, act=ops.ACT_RELU),
        "mean_pool_graph_sage": lambda: pool_ref("mean"),
        "max_pool_graph_sage": lambda: pool_ref("max"),
        "gin": lambda: ops.spmm(csr, None, bf(x), reduce="sum", alpha=1.0, addend=x, beta=1.1),
        "le_conv": lambda: ops.spmm(csr, w_csr, bf(ops.gemm(x, wl[1], bias=bl[1]) - ops.gemm(x, wl[2], bias=bl[2])),
                                    reduce="sum", alpha=1.0, addend=ops.gemm(x, wl[0], bias=bl[0]), beta=1.0,
                                    act=ops.ACT_RELU),
        "appnp_47": lambda: appnp_ref(*apw[47]),
        "appnp_128": lambda: appnp_ref(*apw[128]),
        "sgc_47": lambda: sgc_ref(*sgw[47]),
        "sgc_128": lambda: sgc_ref(*sgw[128]),
        "ssgc": ssgc_ref,
        "tagcn": tagcn_ref,
        "chebynet": cheb_ref,
    }
    for name, fn in fns.items():
        same_bits(fn(B16), refs[name](), name)
    del refs

    # ---- K1 launches: fp32, bf16 gather with fp32 store, bf16-only store; each checked first --------------------------
    k1 = {}
    floors = {}
    for d in (100, 128, 47):
        t32 = torch.randn((n, d), generator=g, device=dev)
        t16 = ops.round_bf16_table(t32)
        o32 = torch.empty((n, d), device=dev)
        ob = ops.bf16_table(n, d, dev)
        ops.spmm(csr, w_csr, t16.float(), out=o32)
        want = o32.clone()
        ops.spmm(csr, w_csr, t16, out=o32)
        same_bits(o32, want, "K1 D={} (fp32 store)".format(d))
        ops.spmm(csr, w_csr, t16, out_bf16=ob)
        same_bits(ob, want.to(B16), "K1 D={} (bf16 store)".format(d))
        del want
        k1["K1_D{}".format(d)] = (lambda t=t32, o=o32: ops.spmm(csr, w_csr, t, out=o),
                                  lambda t=t16, o=o32: ops.spmm(csr, w_csr, t, out=o),
                                  lambda t=t16, o=ob: ops.spmm(csr, w_csr, t, out_bf16=o))
        floors["K1_D{}".format(d)] = (E * (4 * d + 8) + n * (4 * d + 8), E * (2 * d + 8) + n * (4 * d + 8),
                                      E * (2 * d + 8) + n * (2 * d + 8))

    work = {k: (lambda fn=fn: fn(None), lambda fn=fn: fn(B16)) for k, fn in fns.items()}
    for k, (f32, f16, f16only) in k1.items():
        work[k] = (f32, f16, f16only)
    for fns_ in work.values():
        for fn in fns_:
            for _ in range(args.warmup):
                fn()
    torch.cuda.synchronize()
    modes = ("fp32", "bf16", "bf16_only")
    times = {k: {m: [] for m in modes[:len(v)]} for k, v in work.items()}
    for _ in range(args.steps):                                # the modes alternate, one call each per round
        for k, fns_ in work.items():
            for m, fn in zip(modes, fns_):
                times[k][m] += timed(fn, 1)
    res = {"card": card(), "nodes": n, "edges": E, "features": f, "steps": args.steps,
           "command": "python tools/bench_bf16_convs.py --steps {} --warmup {}".format(args.steps, args.warmup)}
    for k, t in times.items():
        row = {}
        for i, (m, v) in enumerate(t.items()):
            ms = float(np.median(v))
            row[m + "_ms"] = round(ms, 3)
            row[m + "_spread_ms"] = [round(float(np.min(v)), 3), round(float(np.max(v)), 3)]
            if k in floors:
                row[m + "_share_of_hbm"] = round(floors[k][i] / (ms * 1e-3) / HBM, 3)
        row["speedup"] = round(row["fp32_ms"] / row["bf16_ms"], 3)
        res[k] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()
