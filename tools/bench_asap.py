# coding=utf-8
"""K10 (the CSR x CSR product of cluster_pool) and the ASAP layer on the device: CUDA-event times of every K10 call of
cluster_pool's two products (T = S^T A, then P = T S), the algorithmic bytes of the fill pass as a share of 3.35 TB/s,
the same two products through torch.sparse CSR @ CSR (cuSPARSE SpGEMM) as a reference point, and the forward + backward
step time of tfg.layers.ASAP.

Workloads:
  nci1   128 graphs of 20-40 nodes with about 32 undirected edges each, F = 37 (a demo_asap batch of NCI1)
  large  one graph of 200 000 nodes with average in-degree 10 (uniform), F = 16
The assignment has ASAP's structure: half of every graph's nodes are clusters, and every self-looped edge whose target is a
cluster assigns its source to that cluster with a positive weight.

    python tools/bench_asap.py [--steps 20] [--workloads nci1,large]
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

import tf_geometric_b200 as tfg                       # noqa: E402
from tf_geometric_b200 import _ffi, ops               # noqa: E402

HBM = 3.35e12
TIMED = ("tfgk_spgemm_plan", "tfgk_spgemm_count", "tfgk_spgemm_rowptr", "tfgk_spgemm_fill_f32")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as err:                            # the number is reported as unknown, never guessed
        return "unknown ({})".format(err)


def nci1(rs):
    sizes = rs.randint(20, 41, 128)
    rows, cols, base = [], [], 0
    for n in sizes:
        u, v = rs.randint(0, n, 32), rs.randint(0, n, 32)
        keep = u != v
        rows.append(base + np.concatenate([u[keep], v[keep]]))
        cols.append(base + np.concatenate([v[keep], u[keep]]))
        base += n
    return np.stack([np.concatenate(rows), np.concatenate(cols)]).astype(np.int32), np.repeat(np.arange(128), sizes), 37


def large(rs):
    n = 200000
    return rs.randint(0, n, (2, 10 * n)).astype(np.int32), np.repeat(np.arange(200), n // 200), 16


def assignment(rs, ei, ngi):
    n = len(ngi)
    keep = ei[0] != ei[1]
    ei_sl = np.concatenate([ei[:, keep], np.stack([np.arange(n), np.arange(n)])], axis=1).astype(np.int32)
    sel = np.sort(np.concatenate([rs.permutation(np.nonzero(ngi == g)[0])[:(np.sum(ngi == g) + 1) // 2]
                                  for g in range(int(ngi.max()) + 1)]))
    cl = -np.ones(n, np.int64)
    cl[sel] = np.arange(len(sel))
    m = cl[ei_sl[0]] >= 0
    aei = np.stack([ei_sl[1][m], cl[ei_sl[0][m]]]).astype(np.int32)
    return ei_sl, aei, rs.uniform(0.05, 1.0, aei.shape[1]).astype(np.float32), len(sel)


def fill_bytes(a_rowptr, a_nnz, products, c_rows, c_nnz):
    """The fill pass reads A (rowptr, col, val), B's two row offsets per A entry and column + value per product, and writes
    C (col, val) and reads its rowptr."""
    return (a_rowptr + c_rows + 2) * 8 + a_nnz * (4 + 4 + 16) + products * 8 + c_nnz * 8


def run(name, ei, ngi, F, steps, dev, rs):
    n = len(ngi)
    ei_sl, aei, aw, K = assignment(rs, ei, ngi)
    e, a, w = (torch.tensor(v, device=dev) for v in (ei_sl, aei, aw))
    ones = torch.ones(ei_sl.shape[1], dtype=torch.float32, device=dev)
    a_csr = ops.csr_build(e[0].contiguous(), e[1].contiguous(), n, n)
    s_csr = ops.csr_build(a[0].contiguous(), a[1].contiguous(), n, K)
    st_csr = ops.csr_build(a[1].contiguous(), a[0].contiguous(), K, n)
    A = (a_csr.rowptr, a_csr.col, ones)
    S = (s_csr.rowptr, s_csr.col, ops.permute(w, s_csr.perm))
    St = (st_csr.rowptr, st_csr.col, ops.permute(w, st_csr.perm))

    def ours():
        t = ops.spgemm(*St, *A, n)
        return t, ops.spgemm(*t, *S, K)

    def cusparse():
        def m(p, r, c):                                 # torch.sparse CSR @ CSR is cuSPARSE's SpGEMM
            return torch.sparse_csr_tensor(p[0], p[1], p[2], size=(r, c))
        return m(St, K, n) @ m(A, n, n) @ m(S, n, K)

    t, p = ours()
    ref = cusparse().to_sparse_coo().coalesce()
    mine = torch.sparse_csr_tensor(*p, size=(K, K)).to_sparse_coo().coalesce()
    assert torch.equal(mine.indices(), ref.indices()), "cuSPARSE has another pattern"
    ref_err = float((mine.values() - ref.values()).abs().max() / ref.values().abs().max())
    for _ in range(2):
        ours()
        cusparse()
    torch.cuda.synchronize()
    calls = []                                          # per product: the CUDA-event times of its K10 calls (chunks)
    for left, right, n_cols in ((St, A, n), (t, S, K)):
        trace = _ffi.CallTrace(timed=TIMED)
        prev = _ffi.set_trace(trace)
        ops.spgemm(*left, *right, n_cols)
        torch.cuda.synchronize()
        _ffi.set_trace(prev)
        calls.append({k: [round(v, 4) for v in trace.elapsed_ms(k)] for k in TIMED})
    prods = []
    for (a_rp, a_c, _), (b_rp, _, _) in ((St, A), (t, S)):
        prods.append(int((b_rp[1:] - b_rp[:-1])[a_c.long()].sum()))
    floors = [fill_bytes(St[0].numel(), St[1].numel(), prods[0], K, t[1].numel()),
              fill_bytes(t[0].numel(), t[1].numel(), prods[1], K, p[1].numel())]
    share = [round(b / HBM / (sum(c["tfgk_spgemm_fill_f32"]) * 1e-3), 3) for b, c in zip(floors, calls)]

    times = {"k10": [], "cusparse": []}
    for _ in range(steps):
        for label, fn in (("k10", ours), ("cusparse", cusparse)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[label].append((time.perf_counter() - t0) * 1e3)

    out = {"workload": name, "N": n, "E_self_looped": int(ei_sl.shape[1]), "clusters": K, "assignments": int(aei.shape[1]),
           "products": prods, "nnz_T": int(t[1].numel()), "nnz_P": int(p[1].numel()), "call_ms": calls,
           "fill_bytes": floors, "fill_hbm_share": share, "cusparse_rel_err": ref_err,
           "two_products_ms_median": {k: round(float(np.median(v)), 3) for k, v in times.items()},
           "two_products_ms_all": {k: [round(v, 3) for v in vs] for k, vs in times.items()}}

    if name == "nci1":
        x = torch.tensor(rs.randn(n, F).astype(np.float32), device=dev, requires_grad=True)
        eit, ngit = torch.tensor(ei, device=dev), torch.tensor(ngi.astype(np.int32), device=dev)
        layer = tfg.layers.ASAP(ratio=0.5, trainable=True, seed=0)

        def step():
            h, _, _, _ = layer([x, eit, None, ngit], training=True)
            h.sum().backward()

        for _ in range(3):
            step()
        st = []
        for _ in range(steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step()
            torch.cuda.synchronize()
            st.append((time.perf_counter() - t0) * 1e3)
        out["asap_fwd_bwd_ms_median"] = round(float(np.median(st)), 3)
        out["asap_fwd_bwd_ms_all"] = [round(v, 3) for v in st]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--workloads", default="nci1,large")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_asap needs a CUDA device")
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    for name in args.workloads.split(","):
        rs = np.random.RandomState(0)
        ei, ngi, F = nci1(rs) if name == "nci1" else large(rs)
        print(json.dumps(run(name, ei, ngi, F, args.steps, dev, rs)), flush=True)


if __name__ == "__main__":
    main()
