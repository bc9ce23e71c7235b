# coding=utf-8
"""TEST DOUBLE for the 16-bit host-table gathers (ops.gather_rows_mapped_16, ops.gather_rows_cached_16) on top of
tests/feature_cache_fake_backend.py, so that the host logic of HostFeatureTable(x, dtype=torch.float16 / bfloat16) runs
without a GPU.  The fakes are numpy restatements of tfgk_gather_rows_mapped_16 / _cached_16: the registered host table
is read as 16-bit patterns through its address (a read outside every registration fails, as the device would fault),
an id outside [0, n_rows) gives a NaN row, and each element is widened exactly to float32 (or copied unchanged when
out_dtype is the table's dtype).  `calls` (shared with the other fakes) records ("gather16", table_ptr, dtype, ld,
n_rows, F, n, out_dtype) and ("gather_cached16", table_ptr, dtype, ld, n_rows, F, cache rows, n).  Injected with
monkeypatch; the product has no such path."""
import ctypes

import numpy as np
import torch

import feature_cache_fake_backend

NAN16 = {torch.bfloat16: 0x7FC0, torch.float16: 0x7E00}


def widen(bits, dtype):
    """float32 values of 16-bit patterns (uint16 numpy array) of dtype, exactly."""
    if dtype == torch.bfloat16:
        return (bits.astype(np.uint32) << 16).view(np.float32)
    return bits.view(np.float16).astype(np.float32)


def bits16(t):
    """The 16-bit patterns of a float16 / bfloat16 tensor as a uint16 numpy array."""
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def from_bits16(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).view(dtype)


def install(monkeypatch):
    calls, registered, block_calls = feature_cache_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def host_bits(table_ptr, ld, n_rows, num_features):
        """The registered host table at table_ptr as an [n_rows, F] uint16 view (checked against the registrations)."""
        if n_rows == 0:
            return np.zeros((0, num_features), np.uint16)
        count = (n_rows - 1) * ld + num_features
        end = table_ptr + count * 2
        assert any(base <= table_ptr and end <= base + size for base, size in registered.items()), \
            "read outside every registered range"
        flat = np.ctypeslib.as_array((ctypes.c_uint16 * count).from_address(table_ptr))
        return np.lib.stride_tricks.as_strided(flat, shape=(n_rows, num_features), strides=(ld * 2, 2))

    def finish(res, out):
        if out is not None:
            out.copy_(res)
            return out
        return res

    def gather_rows_mapped_16(table_ptr, dtype, ld, n_rows, num_features, index, out=None, out_dtype=torch.float32):
        assert dtype in NAN16 and out_dtype in (torch.float32, dtype)
        idx = index.numpy()
        assert idx.dtype == np.int32
        calls.append(("gather16", table_ptr, dtype, ld, n_rows, num_features, idx.size, out_dtype))
        ok = (idx >= 0) & (idx < n_rows)
        res = np.full((idx.size, num_features), NAN16[dtype], np.uint16)
        if ok.any():
            last = int(idx[ok].max())                  # the furthest row the device would read
            res[ok] = host_bits(table_ptr, ld, last + 1, num_features)[idx[ok]]
        if out_dtype == dtype:
            return finish(from_bits16(res, dtype), out)
        f = widen(res, dtype)
        f[~ok] = np.nan
        return finish(torch.from_numpy(np.ascontiguousarray(f)), out)

    def gather_rows_cached_16(table_ptr, ld, n_rows, num_features, cache, slot, index, out=None):
        dtype = cache.dtype
        assert dtype in NAN16 and cache.shape[1] == num_features
        idx, s, c = index.numpy(), slot.numpy(), bits16(cache)
        assert idx.dtype == np.int32 and s.dtype == np.int32 and s.shape == (n_rows,)
        calls.append(("gather_cached16", table_ptr, dtype, ld, n_rows, num_features, c.shape[0], idx.size))
        table = host_bits(table_ptr, ld, n_rows, num_features)
        res = np.full((idx.size, num_features), np.nan, np.float32)
        for i, r in enumerate(idx.tolist()):
            if 0 <= r < n_rows:
                res[i] = widen(c[s[r]] if s[r] >= 0 else table[r], dtype)
        return finish(torch.from_numpy(res), out)

    monkeypatch.setattr(ops, "gather_rows_mapped_16", gather_rows_mapped_16)
    monkeypatch.setattr(ops, "gather_rows_cached_16", gather_rows_cached_16)
    return calls, registered, block_calls
