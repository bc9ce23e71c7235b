#!/usr/bin/env python
# coding=utf-8
"""BASELINE config 5 (GCN fwd, ogbn-papers100M shape: 111,059,956 nodes / 1,615,685,872 edges / 128 features, destination-
partitioned over 8 GPUs) at an arbitrary rank count with the SAME per-GPU load: every rank owns 13.9 M destination rows and
generates its own ~202 M in-edges on the device (seed 1000 + rank; the global graph is never materialised), x is generated
per owner rank.  sym=False is not needed here: the GCN normalisation uses row degrees locally and the all-gathered deg^-1/2.
Run:  torchrun --nproc-per-node R tools/dist_cfg5.py        (R = 8 is the real config; R = 2 keeps the per-GPU sizes)
Checks sampled destination rows bit-exactly against the oracle arithmetic and prints the timing of one GCN forward."""
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tf_geometric_b200 import dist as tdist, ops  # noqa: E402
from oracle import c_oracle  # noqa: E402

ROWS_PER_RANK = 111059956 // 8 + 1          # 13,882,495
EDGES_PER_RANK = 1615685872 // 8            # 201,960,734
F = U = 128

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
os.environ.setdefault("NCCL_DEBUG", "WARN")
dist.init_process_group("nccl", device_id=dev)

rows = int(ROWS_PER_RANK * scale)
edges = int(EDGES_PER_RANK * scale)
n_global = rows * world
part = tdist.RowPartition(n_global, world, rank)
assert part.n_local == rows
gen = torch.Generator(device=dev)
gen.manual_seed(1000 + rank)
row_local = torch.randint(0, rows, (edges,), generator=gen, device=dev, dtype=torch.int32)
col_global = torch.randint(0, n_global, (edges,), generator=gen, device=dev, dtype=torch.int32)
pg = tdist.PartitionedGraph(part, torch.stack([row_local, col_global]).contiguous(), None)
del row_local, col_global
x_local = torch.randn((rows, F), generator=gen, device=dev, dtype=torch.float32)
wgen = torch.Generator(device="cpu"); wgen.manual_seed(2)
limit = (6.0 / (F + U)) ** 0.5
W = ((torch.rand((F, U), generator=wgen) * 2 - 1) * limit).to(dev)
bias = torch.zeros((U,), device=dev)

torch.cuda.synchronize(); dist.barrier()
t0 = time.perf_counter()
csr, value_csr = pg.gcn_normed()                      # self loops + CSR + degrees + all-gather of deg^-1/2 (one-off)
torch.cuda.synchronize()
t_cache = time.perf_counter() - t0

def step():
    return tdist.gcn_partitioned(pg, x_local, W, bias, ops.relu)

for _ in range(2):
    out = step()
torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
ev[0].record()
steps = 3
for _ in range(steps):
    out = step()
ev[1].record()
torch.cuda.synchronize(); dist.barrier()
t = torch.tensor([ev[0].elapsed_time(ev[1]) / steps], dtype=torch.float64, device=dev)
dist.all_reduce(t, op=dist.ReduceOp.MAX)
ms = float(t.item())

# parity: sampled destination rows, explicit oracle arithmetic on the gathered table (bit-exact aggregation + bias + relu)
h_local = ops.gemm(x_local, W)
h_full = pg.all_gather_rows(h_local)
sample = np.random.RandomState(rank).randint(0, rows, 64)
rp = csr.rowptr[torch.as_tensor(np.stack([sample, sample + 1]), device=dev)].cpu().numpy()
ok = True
for r, s, e in zip(sample, rp[0], rp[1]):
    cols = csr.col[s:e].long()
    hw = h_full[cols].cpu().numpy()
    ww = value_csr[s:e].cpu().numpy()
    want = c_oracle.aggregate(np.zeros(e - s, np.int32), np.arange(e - s, dtype=np.int32), ww, hw, 1, "sum")[0]
    want = np.maximum(want + 0.0, 0.0)
    ok &= bool(np.array_equal(out[r].cpu().numpy(), want))
flag = torch.tensor([int(ok)], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
mem = torch.cuda.max_memory_allocated(dev) / 2**30
if rank == 0:
    total_edges = edges * world
    print(json.dumps({"config": "GCN fwd, papers100M-shaped partition per rank", "world": world, "rows_per_rank": rows,
                      "edges_per_rank": edges, "nodes_total": n_global, "edges_total": total_edges, "ms_per_forward": ms,
                      "edges_per_s": total_edges / (ms * 1e-3), "cache_build_s": t_cache, "sampled_rows_bit_exact": bool(flag.item()),
                      "max_memory_GiB_rank0": mem,
                      "halo_bytes_in_per_rank": (world - 1) * part.block * U * 4}), flush=True)
dist.destroy_process_group()
sys.exit(0 if int(flag.item()) == 1 else 1)
