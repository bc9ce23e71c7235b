# coding=utf-8
"""TEST DOUBLE for the host-CSR entries (ops.mapped_id_range, ops.mapped_rowptr, ops.mapped_csr_range) and the mapped
block sampler (ops.block_sample_mapped) on top of tests/host_table_fake_backend.py, so that the host logic of
utils.HostNeighborSampler runs without a GPU.  As there, a registered range's "device address" is its host address: the
fakes read the edge list and the CSR through the addresses they are given, refusing any read outside a registered range
as the device would fault on it.  `calls` records every fake entry in order.  Injected with monkeypatch; the product has
no such path."""
import ctypes

import numpy as np

import host_table_fake_backend
from fake_backend import _np, _t


def install(monkeypatch):
    calls, registered, _ = host_table_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops
    block_sample = ops.block_sample                     # block_fake_backend's restatement

    def read(ptr, n, ctype):
        assert any(base <= ptr and ptr + 4 * n <= base + size for base, size in registered.items()), \
            "read outside every registered range"
        return np.ctypeslib.as_array((ctype * n).from_address(ptr)).copy()

    def mapped_id_range(row_ptr, col_ptr, num_edges, device):
        calls.append(("id_range", num_edges))
        row, col = read(row_ptr, num_edges, ctypes.c_int32), read(col_ptr, num_edges, ctypes.c_int32)
        return int(row.min()), int(row.max()), int(col.min()), int(col.max())

    def mapped_rowptr(row_ptr, num_edges, n_rows, device):
        calls.append(("rowptr", num_edges, n_rows))
        row = read(row_ptr, num_edges, ctypes.c_int32)
        return _t(np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n_rows))]).astype(np.int64))

    def mapped_csr_range(row_ptr, col_ptr, w_ptr, num_edges, r0, r1, n_range, n_cols, device):
        calls.append(("range", r0, r1, n_range))
        row, col = read(row_ptr, num_edges, ctypes.c_int32), read(col_ptr, num_edges, ctypes.c_int32)
        sel = np.flatnonzero((row >= r0) & (row < r1))
        assert sel.size == n_range
        perm = sel[np.argsort(row[sel], kind="stable")]
        w = None if w_ptr is None else _t(read(w_ptr, num_edges, ctypes.c_float)[perm])
        return _t(col[perm]), w

    def block_sample_mapped(rowptr, col_ptr, w_ptr, seeds, fanouts, keys, node_map, padding=False, rng_stream=1):
        E = int(_np(rowptr)[-1])
        calls.append(("block_sample_mapped", E))
        col = _t(read(col_ptr, E, ctypes.c_int32))
        w = _t(np.ones(E, np.float32) if w_ptr is None else read(w_ptr, E, ctypes.c_float))
        return block_sample(rowptr, col, w, seeds, fanouts, keys, node_map, padding, rng_stream)

    monkeypatch.setattr(ops, "mapped_id_range", mapped_id_range)
    monkeypatch.setattr(ops, "mapped_rowptr", mapped_rowptr)
    monkeypatch.setattr(ops, "mapped_csr_range", mapped_csr_range)
    monkeypatch.setattr(ops, "block_sample_mapped", block_sample_mapped)
    return calls, registered
