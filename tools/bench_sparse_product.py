# coding=utf-8
"""SparseMatrix @ SparseMatrix and its gradient on the device: CUDA-event times of K10 (the product) and of both K12
modes (the gradients with respect to the left and the right operand's values), after a check of K12 against float64 on
sampled entries; K12's algorithmic bytes (include/tfgk.h) over its time as a share of 3.35 TB/s; the peak allocated
memory of one forward + backward through the public product; the card's name and power limit.

Workloads (the left and right operands of each product):
  nci1      cluster_pool's two products S^T A and (S^T A) S of tools/bench_asap.py's NCI1-shaped batch
  large     the same two products on bench_asap.py's 200 000-node graph
  products  A S on bench.py's ogbn-products-shaped graph (2 449 029 nodes, 123.7 M edges), S a random sparse
            [node, cluster] assignment with 1-3 clusters per node and N / 10 clusters

    python tools/bench_sparse_product.py [--steps 10] [--workloads nci1,large,products]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import tf_geometric_b200 as tfg                       # noqa: E402
from tf_geometric_b200 import _ffi, ops               # noqa: E402
import bench_asap                                     # noqa: E402

HBM = 3.35e12
SLICE = 64                                            # TFGK_SPGEMM_GRAD_SLICE
K10 = ("tfgk_spgemm_plan", "tfgk_spgemm_count", "tfgk_spgemm_rowptr", "tfgk_spgemm_fill_f32")
K12 = ("tfgk_spgemm_grad_plan", "tfgk_spgemm_grad_f32")


def timed_calls(fn, names, steps):
    """Median CUDA-event time (ms) per ABI name, summed over the calls of one fn() (K10 runs one count and one fill per
    row chunk)."""
    per = {k: [] for k in names}
    for _ in range(steps):
        trace = _ffi.CallTrace(timed=names)
        prev = _ffi.set_trace(trace)
        fn()
        torch.cuda.synchronize()
        _ffi.set_trace(prev)
        for k in names:
            per[k].append(sum(trace.elapsed_ms(k)))
    return {k: round(float(np.median(v)), 4) for k, v in per.items()}


def walk(x_rowptr, x_col, y_rowptr, left):
    """Per X entry: the length of the Y row it walks (left: row x_col; right: X's own row)."""
    ylen = y_rowptr[1:] - y_rowptr[:-1]
    if left:
        return ylen[x_col.long()]
    rows = torch.repeat_interleave(torch.arange(x_rowptr.numel() - 1, device=x_rowptr.device), x_rowptr[1:] - x_rowptr[:-1])
    return ylen[rows]


def k12_bytes(n_x_rows, lens, left):
    """Algorithmic bytes of tfgk_spgemm_grad_f32 with perm (include/tfgk.h)."""
    nnz, products = lens.numel(), int(lens.sum())
    slices = int(torch.where(lens > SLICE, (lens + SLICE - 1) // SLICE, torch.zeros_like(lens)).sum())
    per_entry = 20 + 16 + (16 if left else 0)
    per_product = 16 + (0 if left else 16)
    return n_x_rows * 8 + nnz * per_entry + products * per_product + slices * 8, products, slices


def check_float64(x, y, c_rowptr, c_col, g, left, samples, rs):
    """max |K12 - float64| / sum |terms| over sampled X entries (CSR slots), the float64 sums taken on the device."""
    x_rowptr, x_col, got = x
    y_rowptr, y_col, y_val = y
    dev = x_rowptr.device
    p = torch.tensor(rs.choice(x_col.numel(), min(samples, x_col.numel()), replace=False), device=dev)
    x_rows = torch.searchsorted(x_rowptr, p, right=True) - 1
    yr = x_col[p].long() if left else x_rows
    lens = y_rowptr[yr + 1] - y_rowptr[yr]
    ent = torch.repeat_interleave(torch.arange(p.numel(), device=dev), lens)
    q = torch.repeat_interleave(y_rowptr[yr], lens) + torch.arange(int(lens.sum()), device=dev) - \
        torch.repeat_interleave(torch.cumsum(lens, 0) - lens, lens)
    c_row = x_rows[ent] if left else y_col[q].long()
    c_c = y_col[q].long() if left else x_col[p][ent].long()
    lo, hi = c_rowptr[c_row], c_rowptr[c_row + 1]
    # binary search of every term's column in its C row, vectorised
    while True:
        active = lo < hi
        if not bool(active.any()):
            break
        mid = (lo + hi) // 2
        less = c_col[torch.where(active, mid, torch.zeros_like(mid))].long() < c_c
        lo = torch.where(active & less, mid + 1, lo)
        hi = torch.where(active & ~less, mid, hi)
    hit = (lo < c_rowptr[c_row + 1]) & (c_col[torch.clamp(lo, max=c_col.numel() - 1)].long() == c_c)
    term = torch.where(hit, y_val[q].double() * g[torch.clamp(lo, max=g.numel() - 1)].double(),
                       torch.zeros((), dtype=torch.float64, device=dev))
    want = torch.zeros(p.numel(), dtype=torch.float64, device=dev).index_add_(0, ent, term)
    mag = torch.zeros(p.numel(), dtype=torch.float64, device=dev).index_add_(0, ent, term.abs())
    err = (got[p].double() - want).abs() / torch.clamp(mag, min=1e-30)
    return float(err.max()) if err.numel() else 0.0


def measure(name, A, B, steps, rs):
    m, k, n = A.shape[0], A.shape[1], B.shape[1]
    a_val = ops.permute(A.value.detach(), A.csr.perm)
    b_val = ops.permute(B.value.detach(), B.csr.perm)
    at = A._transposed_csr()
    at_val = ops.permute(A.value.detach(), at.perm)

    def k10():
        return ops.spgemm(A.csr.rowptr, A.csr.col, a_val, B.csr.rowptr, B.csr.col, b_val, n)

    c_rowptr, c_col, c_val = k10()
    g = torch.randn(c_col.numel(), device=c_col.device)

    def left():
        return ops.spgemm_grad("left", A.csr.rowptr, A.csr.col, B.csr.rowptr, B.csr.col, b_val, c_rowptr, c_col, g, m, k,
                               n)

    def right():
        return ops.spgemm_grad("right", B.csr.rowptr, B.csr.col, at.rowptr, at.col, at_val, c_rowptr, c_col, g, m, k, n)

    d_left, d_right = left(), right()
    err_left = check_float64((A.csr.rowptr, A.csr.col, d_left), (B.csr.rowptr, B.csr.col, b_val), c_rowptr, c_col, g, True,
                             4000, rs)
    err_right = check_float64((B.csr.rowptr, B.csr.col, d_right), (at.rowptr, at.col, at_val), c_rowptr, c_col, g, False,
                              4000, rs)
    assert err_left <= 1e-4 and err_right <= 1e-4, (err_left, err_right)
    for _ in range(2):
        k10(), left(), right()
    t10 = timed_calls(k10, K10, steps)
    tl, tr = timed_calls(left, K12, steps), timed_calls(right, K12, steps)
    bl, pl, sl = k12_bytes(m, walk(A.csr.rowptr, A.csr.col, B.csr.rowptr, True), True)
    br, pr, sr = k12_bytes(k, walk(B.csr.rowptr, B.csr.col, at.rowptr, False), False)
    del d_left, d_right, c_rowptr, c_col, c_val, g

    # one forward + backward through the public product, from a state holding only the operands and their CSRs
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    av, bv = A.value.detach().clone().requires_grad_(), B.value.detach().clone().requires_grad_()
    C = A.with_value(av) @ tfg.SparseMatrix(B.index, bv, B.shape, _csr=B.csr)
    (C.value * C.value).sum().backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    nnz_c = C.nnz
    del C, av, bv

    def share(b, ms):
        return round(b / HBM / (ms * 1e-3), 3) if ms > 0 else None

    return {"workload": name, "shape": [m, k, n], "nnz_A": A.nnz, "nnz_B": B.nnz, "nnz_C": nnz_c,
            "k10_ms": t10, "k10_total_ms": round(sum(t10.values()), 4),
            "k12_left_ms": tl, "k12_right_ms": tr,
            "k12_left": {"products": pl, "hub_slices": sl, "bytes": bl, "hbm_share": share(bl, tl["tfgk_spgemm_grad_f32"])},
            "k12_right": {"products": pr, "hub_slices": sr, "bytes": br,
                          "hbm_share": share(br, tr["tfgk_spgemm_grad_f32"])},
            "float64_max_rel_err": {"left": err_left, "right": err_right},
            "fwd_bwd_peak_allocated_bytes": int(peak), "operands_allocated_bytes": int(base)}


def cluster_products(name, rs, dev):
    ei, ngi, _ = bench_asap.nci1(rs) if name == "nci1" else bench_asap.large(rs)
    ei_sl, aei, aw, K = bench_asap.assignment(rs, ei, ngi)
    n = len(ngi)
    A = tfg.SparseMatrix(torch.tensor(ei_sl, device=dev), None, [n, n])
    St = tfg.SparseMatrix(torch.tensor(aei[::-1].copy(), device=dev), torch.tensor(aw, device=dev), [K, n])
    S = St.transpose()
    T = St @ A
    return [("S^T A", St, A), ("(S^T A) S", tfg.SparseMatrix(T.index, T.value, T.shape, _csr=T.csr), S)]


def products_graph(rs, dev):
    import bench
    n = bench.PRODUCTS_NODES
    ei = bench.make_graph_device(n, bench.PRODUCTS_UNDIRECTED, 0, dev)
    A = tfg.SparseMatrix(ei, torch.ones(ei.shape[1], device=dev), [n, n])
    per = torch.tensor(rs.randint(1, 4, n), device=dev)
    rows = torch.repeat_interleave(torch.arange(n, device=dev, dtype=torch.int32), per)
    cols = torch.tensor(rs.randint(0, n // 10, rows.numel()).astype(np.int32), device=dev)
    S = tfg.SparseMatrix(torch.stack([rows, cols]), torch.tensor(rs.uniform(0.1, 1, rows.numel()).astype(np.float32),
                                                                 device=dev), [n, n // 10])
    return [("A S", A, S)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--workloads", default="nci1,large,products")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sparse_product needs a CUDA device")
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": bench_asap.card()}), flush=True)
    for name in args.workloads.split(","):
        rs = np.random.RandomState(0)
        pairs = products_graph(rs, dev) if name == "products" else cluster_products(name, rs, dev)
        for label, A, B in pairs:
            print(json.dumps(dict(measure(name, A, B, args.steps, rs), product=label)), flush=True)
        del pairs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
