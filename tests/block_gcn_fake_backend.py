# coding=utf-8
"""TEST DOUBLE for tfgk_block_gcn_values_f32 (ops.block_gcn_values): the fakes of tests/block_gat_fake_backend.py plus a
numpy statement of the kernel (the full graph's degree factors as the fake deg_inv computes them, products in
scale_edges' order, then s_r = n_g / k_r), so that the host logic of Block.with_gcn_norm and of GCN over a GcnBlock runs
without a GPU.  Injected with monkeypatch; the product has no such path.  `calls` counts the fake kernel entries."""
import numpy as np

import block_gat_fake_backend
from fake_backend import _np, _t
from oracle import tfg_oracle as o

NORM_BOTH, NORM_LEFT, NORM_RIGHT = 0, 1, 2
LOOP_NONE, LOOP_NORMED, LOOP_FILL = 0, 1, 2


def degree_factor(rowsum, deg_fill, norm):
    """f(v) for every node: the fake deg_inv over rowsum + deg_fill."""
    d = (np.asarray(rowsum, np.float32) + np.float32(deg_fill)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return o._remove_inf_and_nan(np.power(d, np.float32(-0.5 if norm == NORM_BOTH else -1))).astype(np.float32)


def block_gcn_values_np(rowptr, gcol, w, dst, g_rowptr, g_rowsum, norm, loop, deg_fill, fill, factor=degree_factor):
    """The kernel's values in numpy: float32 [S + n_dst] in the looped layout with a loop mode, else [S]."""
    n_dst, S = dst.size, gcol.size
    rowptr = np.asarray(rowptr, np.int64)[:n_dst + 1]
    k = np.diff(rowptr)
    row = np.repeat(np.arange(n_dst), k)
    f = factor(g_rowsum, deg_fill, norm)
    g = dst[row].astype(np.int64)
    v = np.ones(S, np.float32) if w is None else np.asarray(w, np.float32).copy()
    if norm != NORM_RIGHT:
        v = (f[g] * v).astype(np.float32)
    if norm != NORM_LEFT:
        v = (v * f[gcol]).astype(np.float32)
    n = np.diff(np.asarray(g_rowptr, np.int64))[g]
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (n.astype(np.float32) / k[row].astype(np.float32)).astype(np.float32)
    v = (s * v).astype(np.float32)
    if loop == LOOP_NONE:
        return v
    out = np.empty(S + n_dst, np.float32)
    out[np.arange(S) + row] = v
    fl = np.full(n_dst, fill, np.float32)
    if loop == LOOP_NORMED:
        fd = f[dst.astype(np.int64)]
        if norm != NORM_RIGHT:
            fl = (fd * fl).astype(np.float32)
        if norm != NORM_LEFT:
            fl = (fl * fd).astype(np.float32)
    out[rowptr[1:] + np.arange(n_dst)] = fl
    return out


def install(monkeypatch):
    calls = block_gat_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops
    calls.update({"block_gcn_values": 0, "gemm": 0})

    def block_gcn_values(rowptr, gcol, w, dst, g_rowptr, g_rowsum, norm, loop, deg_fill, fill):
        calls["block_gcn_values"] += 1
        return _t(block_gcn_values_np(_np(rowptr), _np(gcol), _np(w), _np(dst), _np(g_rowptr), _np(g_rowsum), norm,
                                      loop, deg_fill, fill))

    plain_gemm = ops.gemm

    def gemm(*args, **kwargs):
        calls["gemm"] += 1
        return plain_gemm(*args, **kwargs)

    monkeypatch.setattr(ops, "block_gcn_values", block_gcn_values)
    monkeypatch.setattr(ops, "gemm", gemm)
    return calls
