# coding=utf-8
"""TEST DOUBLE for K10 (ops.spgemm, the CSR x CSR product of cluster_pool and ASAP): the CPU fake kernel layer of
tests/cluster_pool_fake_backend.py plus a numpy restatement of tfgk_spgemm_* in Gustavson order, so that the host logic of
cluster_pool and ASAP runs without a GPU.  Injected with monkeypatch; the product has no such path."""
import numpy as np

import cluster_pool_fake_backend
from fake_backend import _np, _t


def spgemm_reference(a_rowptr, a_col, a_val, b_rowptr, b_col, b_val, n_cols):
    """C = A B as (rowptr int64, col int32, val float32): ascending columns per row, every entry the float32 sum of its
    products a_ik * b_kj in production order (A's row left to right, then B's row left to right)."""
    a_rowptr, b_rowptr = np.asarray(a_rowptr, np.int64), np.asarray(b_rowptr, np.int64)
    a_col, b_col = np.asarray(a_col, np.int64), np.asarray(b_col, np.int64)
    a_val, b_val = np.asarray(a_val, np.float32), np.asarray(b_val, np.float32)
    M = len(a_rowptr) - 1
    lens = np.diff(b_rowptr)[a_col]
    total = int(lens.sum())
    ent = np.repeat(np.arange(len(a_col)), lens)                          # A entry of every product, production order
    kb = np.repeat(b_rowptr[a_col], lens) + (np.arange(total) - np.repeat(np.cumsum(lens) - lens, lens))
    row = np.repeat(np.arange(M), np.diff(a_rowptr))[ent]
    col = b_col[kb]
    p = (a_val[ent] * b_val[kb]).astype(np.float32)
    order = np.lexsort((col, row))                                        # stable: equal (row, col) keep production order
    row, col, p = row[order], col[order], p[order]
    head = np.ones(total, bool)
    head[1:] = (row[1:] != row[:-1]) | (col[1:] != col[:-1])
    start = np.nonzero(head)[0]
    run = np.diff(np.append(start, total))
    acc = p[start].copy()
    for d in range(1, int(run.max()) if total else 0):
        m = run > d
        acc[m] = (acc[m] + p[start[m] + d]).astype(np.float32)
    rowptr = np.zeros(M + 1, np.int64)
    rowptr[1:] = np.cumsum(np.bincount(row[start], minlength=M))
    return rowptr, col[start].astype(np.int32), acc.astype(np.float32)


def install(monkeypatch):
    cluster_pool_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def spgemm(a_rowptr, a_col, a_val, b_rowptr, b_col, b_val, n_cols, budget=None):
        return tuple(_t(a) for a in spgemm_reference(_np(a_rowptr), _np(a_col), _np(a_val), _np(b_rowptr), _np(b_col),
                                                     _np(b_val), n_cols))

    monkeypatch.setattr(ops, "spgemm", spgemm)
