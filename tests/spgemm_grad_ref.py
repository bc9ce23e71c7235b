# coding=utf-8
"""Numpy restatement of K12 (tfgk_spgemm_grad_*, ops.spgemm_grad), the gradient of K10's C = A B with respect to one
operand's values, in the summation order include/tfgk.h fixes: for every CSR entry p of X, the products Y.val[q] * dC
(each rounded once to float32) of the Y row it walks, summed from +0 in Y's order within slices of SLICE entries, and
the slice sums added from +0 in slice order.  A (row, column) that C does not hold contributes 0.  Also the TEST DOUBLE
that puts it behind ops.spgemm_grad for the host tests (injected with monkeypatch; the product has no such path)."""
import numpy as np

SLICE = 64          # TFGK_SPGEMM_GRAD_SLICE


def _lookup(c_rowptr, c_col, rows, cols):
    """Position of (rows[t], cols[t]) in C, or -1 when C's row does not hold the column."""
    c_rowptr, c_col = np.asarray(c_rowptr, np.int64), np.asarray(c_col, np.int64)
    n_cols = int(c_col.max()) + 1 if len(c_col) else 1
    n_cols = max(n_cols, int(cols.max()) + 1 if len(cols) else 1)
    c_rows = np.repeat(np.arange(len(c_rowptr) - 1), np.diff(c_rowptr))
    keys = c_rows * n_cols + c_col                                  # ascending: rows ascending, columns ascending per row
    want = rows.astype(np.int64) * n_cols + cols
    pos = np.searchsorted(keys, want)
    hit = pos < len(keys)
    hit[hit] = keys[pos[hit]] == want[hit]
    return np.where(hit, pos, -1)


def spgemm_grad_reference(mode, x_rowptr, x_col, y_rowptr, y_col, y_val, c_rowptr, c_col, grad_c, perm=None,
                          slice_size=SLICE):
    """One float32 per entry of X: X's CSR order, or out[perm[p]] with perm."""
    x_rowptr, y_rowptr = np.asarray(x_rowptr, np.int64), np.asarray(y_rowptr, np.int64)
    x_col, y_col = np.asarray(x_col, np.int64), np.asarray(y_col, np.int64)
    y_val, grad_c = np.asarray(y_val, np.float32), np.asarray(grad_c, np.float32)
    nnz = len(x_col)
    x_row = np.repeat(np.arange(len(x_rowptr) - 1), np.diff(x_rowptr))
    yr = x_col if mode == "left" else x_row                        # the Y row every X entry walks
    lens = np.diff(y_rowptr)[yr]
    total = int(lens.sum())
    ent = np.repeat(np.arange(nnz), lens)                          # X entry of every product, in Y order
    within = np.arange(total) - np.repeat(np.cumsum(lens) - lens, lens)
    q = np.repeat(y_rowptr[yr], lens) + within
    if mode == "left":
        pos = _lookup(c_rowptr, c_col, x_row[ent], y_col[q])
    else:
        pos = _lookup(c_rowptr, c_col, y_col[q], x_col[ent])
    term = np.where(pos >= 0, y_val[q] * grad_c[np.maximum(pos, 0)], np.float32(0)).astype(np.float32)
    # slice sums: products grouped by (entry, slice), each group summed from +0 in Y order
    n_sl = np.maximum((lens + slice_size - 1) // slice_size, 1)
    sl_base = np.cumsum(n_sl) - n_sl
    group = sl_base[ent] + within // slice_size
    part = np.zeros(int(n_sl.sum()), np.float32)
    for d in range(slice_size):
        m = (within % slice_size) == d
        part[group[m]] = (part[group[m]] + term[m]).astype(np.float32)
    acc = np.zeros(nnz, np.float32)
    for s in range(int(n_sl.max()) if nnz else 0):
        m = n_sl > s
        acc[m] = (acc[m] + part[sl_base[m] + s]).astype(np.float32)
    if perm is None:
        return acc
    out = np.empty_like(acc)
    out[np.asarray(perm, np.int64)] = acc
    return out


def install(monkeypatch):
    """ops.spgemm_grad on the CPU, on top of the numpy K10 of tests/asap_fake_backend.py."""
    import asap_fake_backend
    from fake_backend import _np, _t
    asap_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def spgemm_grad(mode, x_rowptr, x_col, y_rowptr, y_col, y_val, c_rowptr, c_col, grad_c, m, k, n, perm=None):
        return _t(spgemm_grad_reference(mode, _np(x_rowptr), _np(x_col), _np(y_rowptr), _np(y_col), _np(y_val),
                                        _np(c_rowptr), _np(c_col), _np(grad_c), _np(perm)))

    monkeypatch.setattr(ops, "spgemm_grad", spgemm_grad)
    monkeypatch.setattr(ops, "build_plan", lambda csr: None)
