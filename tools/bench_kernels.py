#!/usr/bin/env python
# coding=utf-8
"""Kernel micro-benchmark at the bench workload's shape (ogbn-products size): times each hot kernel alone with CUDA events
(inputs >> L2): K1 (weighted sum at D = 128, mean at D = 100), K3 with K | V in one buffer (TMA ring) and in two (cp.async
ring), and the projection GEMM with and without tensor cores (TFGK_GEMM_TC=0).  Development tool: the numbers that count
are bench.py's."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as B  # noqa: E402
from tf_geometric_b200 import ops, _structure  # noqa: E402
import tf_geometric_b200 as tfg  # noqa: E402

scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
iters = 5
dev = torch.device("cuda")
n = int(B.PRODUCTS_NODES * scale)
pairs = int(B.PRODUCTS_UNDIRECTED * scale)
ei = B.make_graph_device(n, pairs, 0, dev)
E = ei.shape[1]
gen = torch.Generator(device=dev); gen.manual_seed(1)
x = torch.randn((n, B.FEATURES), generator=gen, device=dev)
h = torch.randn((n, B.UNITS), generator=gen, device=dev)
csr, _ = _structure.csr_for_edge_index(ei, n, add_self_loop=True)
w = torch.rand((csr.nnz,), generator=gen, device=dev)
peak, _ = B.measured_peak_gbs()
results = {}


def timed(fn, label, nbytes=None):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    rec = {"ms": ms}
    if nbytes:
        rec["GBps"] = nbytes / ms / 1e6
        rec["frac_of_measured_peak"] = rec["GBps"] / peak
    results[label] = rec
    print(label, json.dumps(rec), flush=True)


D = B.UNITS
out = torch.empty((n, D), device=dev)
timed(lambda: ops.spmm(csr, w, h, out=out), "spmm_D128", csr.nnz * (4 * D + 8) + n * (4 * D + 8))
timed(lambda: ops.spmm(csr, None, x, reduce="mean"), "spmm_mean_D100", csr.nnz * (4 * 100 + 4) + n * (4 * 100 + 8))

q = torch.randn((n, D), generator=gen, device=dev)
kv = torch.randn((n, 2 * D), generator=gen, device=dev)
k_sep, v_sep = kv[:, :D].contiguous(), kv[:, D:].contiguous()
gat_bytes = csr.nnz * (8 * D + 4) + n * (8 * D + 8)
timed(lambda: ops.gat_fused(csr, q, kv[:, :D], kv[:, D:], B.HEADS), "gat_tma_interleaved", gat_bytes)
timed(lambda: ops.gat_fused(csr, q, k_sep, v_sep, B.HEADS), "gat_async_separate", gat_bytes)
assert torch.equal(ops.gat_fused(csr, q, kv[:, :D], kv[:, D:], B.HEADS), ops.gat_fused(csr, q, k_sep, v_sep, B.HEADS)), \
    "the TMA and cp.async rings gave different bits"

wmat = B.glorot((B.FEATURES, B.UNITS), 2).to(dev)
gemm_bytes = 4 * (n * B.FEATURES + B.FEATURES * B.UNITS + n * B.UNITS)
for tc in ("1", "0"):
    os.environ["TFGK_GEMM_TC"] = tc
    timed(lambda: ops.gemm(x, wmat, out=out), "gemm_100x128_" + ("tc" if tc == "1" else "simt"), gemm_bytes)
    if tc == "1":
        tc_out = out.clone()
    else:
        print("   tc vs simt max rel diff:", float((tc_out - out).abs().max() / out.abs().max()), flush=True)
os.environ.pop("TFGK_GEMM_TC")
print(json.dumps(results, indent=1))
