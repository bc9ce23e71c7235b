# coding=utf-8
"""TEST DOUBLE for tfgk_block_self_loops_i32 (ops.block_self_loops): the fakes of tests/block_fake_backend.py plus a numpy
statement of the kernel's index arithmetic (edge p of row r to p + r, row r's self edge to rowptr[r + 1] + r), so that
the host logic of Block.with_self_loops and of GAT over a SelfLoopBlock runs without a GPU.  Injected with monkeypatch;
the product has no such path.  `calls` counts the fake kernel entries GAT on a block reaches."""
import numpy as np

import block_fake_backend
from fake_backend import _np, _t


def block_self_loops_np(rowptr, row, col, n_dst):
    """The kernel's scatter, in numpy: (out_rowptr int64 [n_dst + 1], out_row, out_col int32 [S + n_dst])."""
    rowptr = np.asarray(rowptr, np.int64)[:n_dst + 1]
    S = row.size
    out_row = np.full(S + n_dst, -1, np.int32)
    out_col = np.full(S + n_dst, -1, np.int32)
    p = np.arange(S)
    out_row[p + row], out_col[p + row] = row, col
    r = np.arange(n_dst)
    out_row[rowptr[1:] + r], out_col[rowptr[1:] + r] = r, r
    return rowptr + np.arange(n_dst + 1), out_row, out_col


def install(monkeypatch):
    calls = block_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops
    calls.update({"block_self_loops": 0, "gemm_proj": 0, "gat_fused": 0})

    def block_self_loops(rowptr, edge_index, n_dst):
        calls["block_self_loops"] += 1
        e = _np(edge_index)
        rp, r, c = block_self_loops_np(_np(rowptr), e[0], e[1], int(n_dst))
        return _t(rp), _t(np.stack([r, c]))

    def counted(name, fn):
        def wrapped(*args, **kwargs):
            calls[name] += 1
            return fn(*args, **kwargs)
        return wrapped

    monkeypatch.setattr(ops, "block_self_loops", block_self_loops)
    monkeypatch.setattr(ops, "gemm_proj", counted("gemm_proj", ops.gemm_proj))
    monkeypatch.setattr(ops, "gat_fused", counted("gat_fused", ops.gat_fused))
    return calls
