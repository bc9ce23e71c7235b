# coding=utf-8
"""TEST DOUBLE for the row-block entry (ops.row_block) and the bulk copy (ops.copy_async) on top of
tests/host_sampler_fake_backend.py, so that row_block of both samplers runs without a GPU.  The row block is restated row
by row in numpy; the copy reads through the address it is given and refuses a read outside every registered range, as
the device would fault on it.  `calls` records the fake entries in order.  Injected with monkeypatch; the product has no
such path."""
import ctypes

import numpy as np

import host_sampler_fake_backend
from fake_backend import _np, _t


def restate_row_block(rowptr, cols, r0, r1):
    """(nodes, out_rowptr, out_row, local) of rows [r0, r1) of a CSR with row pointer rowptr, whose columns in that range
    are `cols`, row by row: the rows first, then every column outside them in the order the edges first reach it."""
    n = r1 - r0
    nodes = list(range(r0, r1))
    where = {v: i for i, v in enumerate(nodes)}
    local = []
    for v in cols.tolist():
        if v not in where:
            where[v] = len(nodes)
            nodes.append(v)
        local.append(where[v])
    out_rowptr = (rowptr[r0:r1 + 1] - rowptr[r0]).astype(np.int64)
    out_row = np.repeat(np.arange(n, dtype=np.int32), np.diff(out_rowptr))
    return np.array(nodes, np.int32), out_rowptr, out_row, np.array(local, np.int32)


def install(monkeypatch):
    calls, registered = host_sampler_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def row_block(rowptr, r0, r1, cols, node_map):
        assert np.all(_np(node_map) == -1), "the map must be clean between calls"
        rp, c = _np(rowptr), _np(cols)
        calls.append(("row_block", r0, r1, c.size))
        assert rp.size == node_map.numel() + 1 and c.size == rp[r1] - rp[r0]
        return tuple(_t(a) for a in restate_row_block(rp, c, r0, r1))

    def copy_async(dst, src_address, nbytes):
        calls.append(("copy_async", nbytes))
        if nbytes:
            assert any(base <= src_address and src_address + nbytes <= base + size for base, size in registered.items()), \
                "copy from outside every registered range"
            ctypes.memmove(dst.data_ptr(), src_address, nbytes)

    def build_plan(csr):                     # a full-neighbour block's plan: hub rows here are short of HUB_THRESHOLD
        calls.append(("build_plan", csr.n_rows))
        assert int(_np(csr.rowptr)[-1] - _np(csr.rowptr)[0]) == 0 or np.diff(_np(csr.rowptr)).max() <= ops.HUB_THRESHOLD
        return None

    monkeypatch.setattr(ops, "build_plan", build_plan)
    monkeypatch.setattr(ops, "row_block", row_block)
    monkeypatch.setattr(ops, "copy_async", copy_async)
    return calls, registered
