# coding=utf-8
"""TEST DOUBLE for the host feature-table entries (ops.host_register, ops.host_unregister, ops.gather_rows_mapped) on top
of tests/block_fake_backend.py, so that the host logic of utils.HostFeatureTable and of SampledBlocks.source_rows runs
without a GPU.  The "device address" of a registered range is its host address, and the fake gather reads the table
through that address, refusing any read outside a registered range as the device would fault on it.  `calls` records
every fake entry in order.  Injected with monkeypatch; the product has no such path."""
import ctypes

import numpy as np

import block_fake_backend
from fake_backend import _np, _t


def install(monkeypatch):
    block_calls = block_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops, _ffi
    from tf_geometric_b200.utils import sampling
    monkeypatch.setattr(sampling, "_host_registered", {})
    calls = []
    registered = {}                                     # base address -> bytes

    def host_register(ptr, nbytes):
        calls.append(("register", ptr, nbytes))
        for base, size in registered.items():
            if ptr < base + size and base < ptr + nbytes:
                raise _ffi.TfgkError("tfgk_host_register", _ffi.ERR_CUDA, "part of the range is already registered")
        registered[ptr] = nbytes
        return ptr

    def host_unregister(ptr):
        calls.append(("unregister", ptr))
        if ptr not in registered:
            raise _ffi.TfgkError("tfgk_host_unregister", _ffi.ERR_CUDA, "not registered")
        del registered[ptr]

    def gather_rows_mapped(table_ptr, ld, n_rows, num_features, index, out=None):
        idx = _np(index)
        assert idx.dtype == np.int32
        calls.append(("gather", table_ptr, ld, n_rows, num_features, idx.size))
        res = np.full((idx.size, num_features), np.nan, np.float32)
        ok = (idx >= 0) & (idx < n_rows)
        if ok.any():
            last = int(idx[ok].max())                  # the furthest byte the device would read
            end = table_ptr + (last * ld + num_features) * 4
            assert any(base <= table_ptr and end <= base + size for base, size in registered.items()), \
                "read outside every registered range"
            flat = np.ctypeslib.as_array((ctypes.c_float * (last * ld + num_features)).from_address(table_ptr))
            rows = np.lib.stride_tricks.as_strided(flat, shape=(last + 1, num_features), strides=(ld * 4, 4))
            res[ok] = rows[idx[ok]]
        if out is not None:
            out.copy_(_t(res))
            return out
        return _t(res)

    monkeypatch.setattr(ops, "host_register", host_register)
    monkeypatch.setattr(ops, "host_unregister", host_unregister)
    monkeypatch.setattr(ops, "gather_rows_mapped", gather_rows_mapped)
    return calls, registered, block_calls
