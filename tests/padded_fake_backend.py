# coding=utf-8
"""TEST DOUBLE for K9 (ops.pad_rows / ops.unpad_rows, the padded row gather of lstm_graph_sage and convert_x_to_3d): the
CPU fake kernel layer of tests/cluster_pool_fake_backend.py plus numpy restatements of tfgk_pad_rows_f32 and
tfgk_unpad_rows_f32, so that the host logic of the padded API runs without a GPU.  Injected with monkeypatch; the
product has no such path."""
import numpy as np

import cluster_pool_fake_backend
from fake_backend import _np, _t


def pad_reference(rowptr, src, X, K, step_major=False):
    """(out, slot): out[r, j] = X[src[rowptr[r] + j]] for j < min(deg, K), zeros up to K ([R, K, D], or [K, R, D]);
    slot[p] = the flat output row of CSR slot p (-1 past K)."""
    X = np.asarray(X, np.float32)
    R, D = len(rowptr) - 1, X.shape[1]
    out = np.zeros((R, K, D), np.float32)
    slot = np.full(int(rowptr[-1]), -1, np.int32)
    for r in range(R):
        for j in range(int(rowptr[r + 1] - rowptr[r])):
            p = rowptr[r] + j
            if j < K:
                out[r, j] = X[src[p]]
                slot[p] = j * R + r if step_major else r * K + j
    return (np.ascontiguousarray(out.transpose(1, 0, 2)) if step_major else out), slot


def unpad_reference(rowptr, perm, G):
    """out[perm[p]] = G[r, j] for j = p - rowptr[r] < K, else 0."""
    G = np.asarray(G, np.float32)
    R, K, D = G.shape
    out = np.zeros((int(rowptr[-1]), D), np.float32)
    for r in range(R):
        for j in range(int(rowptr[r + 1] - rowptr[r])):
            out[perm[rowptr[r] + j]] = G[r, j] if j < K else 0.0
    return out


def install(monkeypatch):
    cluster_pool_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def pad_rows(csr, X, K, src=None, step_major=False, slot_index=False, out=None):
        res, slot = pad_reference(_np(csr.rowptr), _np(csr.col if src is None else src), _np(X), int(K), step_major)
        res = _t(res)
        if out is not None:
            out.copy_(res)
            res = out
        return (res, _t(slot)) if slot_index else res

    def unpad_rows(csr, G, out=None):
        res = _t(unpad_reference(_np(csr.rowptr), _np(csr.perm), _np(G)))
        if out is not None:
            out.copy_(res)
            return out
        return res

    monkeypatch.setattr(ops, "pad_rows", pad_rows)
    monkeypatch.setattr(ops, "unpad_rows", unpad_rows)
