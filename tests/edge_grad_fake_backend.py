# coding=utf-8
"""TEST DOUBLE for K7 (ops.sddmm_csr, the edge-weight gradient kernel): the CPU fake kernel layer of
tests/fake_backend.py plus a numpy restatement of tfgk_sddmm_csr_f32, so that the host logic of the edge-weight
gradients (edge-order perm, mean scale, the normalisation backward, route selection) runs without a GPU.
It lives under tests/ and is injected with monkeypatch; the product has no such path."""
import numpy as np

import fake_backend
from fake_backend import _np, _t


def sddmm_reference(rowptr, col, perm, G, X, row_scale=None, alpha=1.0, edge_order=True):
    """out[perm[p] or p] = alpha * row_scale[r] * <G[r], X[col[p]]> in float32 (numpy)."""
    rows = np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))
    f = np.float32(alpha) * (np.ones(len(rowptr) - 1, np.float32) if row_scale is None else row_scale.astype(np.float32))
    s = (G[rows].astype(np.float32) * X[col].astype(np.float32)).sum(-1, dtype=np.float32) * f[rows]
    if not edge_order:
        return s.astype(np.float32)
    out = np.empty_like(s)
    out[perm] = s
    return out.astype(np.float32)


def install(monkeypatch):
    fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def sddmm_csr(csr, G, X, row_scale=None, alpha=1.0, edge_order=True, out=None):
        res = _t(sddmm_reference(_np(csr.rowptr), _np(csr.col), _np(csr.perm), _np(G), _np(X), _np(row_scale), alpha,
                                 edge_order))
        if out is not None:
            out.copy_(res)
            return out
        return res

    monkeypatch.setattr(ops, "sddmm_csr", sddmm_csr)
