# coding=utf-8
"""TEST DOUBLE for the cached host-table gather (ops.gather_rows_cached) on top of tests/host_table_fake_backend.py, so
that the host logic of HostFeatureTable(x, device_rows=...) and of rank_source_rows runs without a GPU.  The fake is a
numpy restatement of tfgk_gather_rows_cached_f32: an id outside [0, n_rows) gives a NaN row, a row whose slot is >= 0
is read from the cache, and every other row is read from the registered host table through its address, as the
uncached fake does.  `calls` (shared with the host-table fake) records ("gather_cached", table_ptr, ld, n_rows, F,
cache rows, n) for every cached gather.  Injected with monkeypatch; the product has no such path."""
import ctypes

import numpy as np

import host_table_fake_backend
from fake_backend import _np, _t


def gather_cached_ref(table, cache, slot, index):
    """out[i] = table[index[i]] with cached rows taken from cache[slot[index[i]]] and NaN rows for ids outside the
    table: the kernel's result, in numpy."""
    n_rows, F = table.shape
    out = np.full((index.size, F), np.nan, np.float32)
    for i, r in enumerate(index.tolist()):
        if 0 <= r < n_rows:
            out[i] = cache[slot[r]] if slot[r] >= 0 else table[r]
    return out


def install(monkeypatch):
    calls, registered, block_calls = host_table_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def host_rows(table_ptr, ld, n_rows, num_features):
        """The registered host table at table_ptr as an [n_rows, F] numpy view (checked against the registrations)."""
        if n_rows == 0:
            return np.zeros((0, num_features), np.float32)
        end = table_ptr + ((n_rows - 1) * ld + num_features) * 4
        assert any(base <= table_ptr and end <= base + size for base, size in registered.items()), \
            "read outside every registered range"
        flat = np.ctypeslib.as_array((ctypes.c_float * ((n_rows - 1) * ld + num_features)).from_address(table_ptr))
        return np.lib.stride_tricks.as_strided(flat, shape=(n_rows, num_features), strides=(ld * 4, 4))

    def gather_rows_cached(table_ptr, ld, n_rows, num_features, cache, slot, index, out=None):
        idx, c, s = _np(index), _np(cache), _np(slot)
        assert idx.dtype == np.int32 and s.dtype == np.int32 and s.shape == (n_rows,)
        assert c.dtype == np.float32 and c.shape[1] == num_features
        calls.append(("gather_cached", table_ptr, ld, n_rows, num_features, c.shape[0], idx.size))
        res = gather_cached_ref(host_rows(table_ptr, ld, n_rows, num_features), c, s, idx)
        if out is not None:
            out.copy_(_t(res))
            return out
        return _t(res)

    monkeypatch.setattr(ops, "gather_rows_cached", gather_rows_cached)
    return calls, registered, block_calls
