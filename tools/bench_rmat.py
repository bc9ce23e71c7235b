#!/usr/bin/env python
# coding=utf-8
"""Secondary workload of SURVEY.md 8d: an RMAT(0.57, 0.19, 0.19, 0.05) graph of ogbn-products size (skewed degrees).
Times K1 and K3 alone and reports the degree skew; development tool (hub rows run through the work plan of DESIGN.md section 4)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as B  # noqa: E402
from tf_geometric_b200 import ops, _structure  # noqa: E402

dev = torch.device("cuda")
scale_bits = 21
n = 1 << scale_bits
pairs = B.PRODUCTS_UNDIRECTED
gen = torch.Generator(device=dev); gen.manual_seed(7)
u = torch.zeros((pairs,), dtype=torch.int32, device=dev)
v = torch.zeros((pairs,), dtype=torch.int32, device=dev)
a, b, c = 0.57, 0.19, 0.19
for bit in range(scale_bits):
    r = torch.rand((pairs,), generator=gen, device=dev)
    ubit = (r >= a + b).to(torch.int32)                         # quadrants c, d -> row bit 1
    vbit = (((r >= a) & (r < a + b)) | (r >= a + b + c)).to(torch.int32)   # quadrants b, d -> col bit 1
    u |= ubit << bit
    v |= vbit << bit
keep = u != v
u, v = u[keep], v[keep]
ei = torch.stack([torch.cat([u, v]), torch.cat([v, u])]).contiguous()
E = ei.shape[1]
csr, _ = _structure.csr_for_edge_index(ei, n, add_self_loop=True)
deg = csr.rowptr[1:] - csr.rowptr[:-1]
print("RMAT: n=%d E=%d max degree=%d mean=%.1f  rows>4096: %d" % (n, E, int(deg.max()), float(deg.float().mean()),
                                                                 int((deg > 4096).sum())), flush=True)
D = 128
h = torch.randn((n, D), generator=gen, device=dev)
q = torch.randn((n, D), generator=gen, device=dev)
kv = torch.randn((n, 2 * D), generator=gen, device=dev)
w = torch.rand((csr.nnz,), generator=gen, device=dev)
peak, _ = B.measured_peak_gbs()
res = {"n": n, "edges": E, "max_degree": int(deg.max())}


def timed(fn, label, nbytes):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(5):
        fn()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / 5
    res[label] = {"ms": ms, "GBps": nbytes / ms / 1e6, "frac_of_measured_peak": nbytes / ms / 1e6 / peak}
    print(label, json.dumps(res[label]), flush=True)


print("plan:", None if csr.plan is None else (csr.plan.n_tasks, csr.plan.n_hubs, csr.plan.n_slots), flush=True)
timed(lambda: ops.spmm(csr, w, h), "rmat_spmm_D128", csr.nnz * (4 * D + 8) + n * (4 * D + 8))
timed(lambda: ops.gat_fused(csr, q, kv[:, :D], kv[:, D:], 8), "rmat_gat", csr.nnz * (8 * D + 4) + n * (8 * D + 8))
print(json.dumps(res, indent=1))
