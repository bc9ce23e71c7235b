# coding=utf-8
"""16-bit host feature tables without a GPU: the ABI declarations and argument checks of tfgk_gather_rows_mapped_16 and
tfgk_gather_rows_cached_16, the ops wrappers' own refusals, and HostFeatureTable(x, dtype=...) over the numpy fake of
tests/half_table_fake_backend.py: the dtype keyword and its refusals, a float32 table's unchanged call log, the routing
of 16-bit tables (cache fill included), device_bytes and the dtype property, numpy float16 wrapped without a copy, and
source_rows of SampledBlocks and LinkBlocks."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import half_table_fake_backend as fake_half
from conftest import random_graph

MAPPED16, CACHED16 = "tfgk_gather_rows_mapped_16", "tfgk_gather_rows_cached_16"
DTYPES = [torch.float16, torch.bfloat16]


def _header_arity(name):
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "tfgk.h")).read()
    m = re.search(r"int {}\(([^;]*)\);".format(name), header)
    assert m, name
    return len(m.group(1).split(","))


@pytest.fixture
def fake(monkeypatch):
    calls, registered, _ = fake_half.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg, calls, registered


def _x(n=40, F=6, seed=0, dtype=torch.float32):
    x = torch.from_numpy(np.random.RandomState(seed).randn(n, F).astype(np.float32))
    return x.to(dtype)


def _widened(x, index):
    return x.float().numpy()[np.asarray(index)]


def test_entries_are_declared_and_exported():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    assert (_ffi.DTYPE_F32, _ffi.DTYPE_BF16, _ffi.DTYPE_FP8_E4M3, _ffi.DTYPE_F16) == (0, 1, 2, 3)
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "tfgk.h")).read()
    assert "TFGK_DTYPE_F16 = 3" in header
    assert len(_ffi.SIGNATURES[MAPPED16]) == _header_arity(MAPPED16) == 11
    assert len(_ffi.SIGNATURES[CACHED16]) == _header_arity(CACHED16) == 13
    for name in (MAPPED16, CACHED16):
        assert hasattr(_ffi.lib(), name)
        assert name not in _ffi.NOT_CAPTURABLE                              # no host value, no host key


def test_mapped_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    buf = (ctypes.c_uint16 * 16)()
    p = ctypes.addressof(buf)
    names = ["table", "dtype", "ld", "n_rows", "F", "index", "n", "out", "out_dtype", "ldo"]
    ok = [p, _ffi.DTYPE_BF16, 4, 10, 4, p, 1, p, _ffi.DTYPE_F32, 4, None]

    def args(**kw):
        a = list(ok)
        for k, v in kw.items():
            a[names.index(k)] = v
        return a
    cases = [(args(dtype=_ffi.DTYPE_F32), "dtype"), (args(dtype=_ffi.DTYPE_FP8_E4M3), "dtype"), (args(dtype=7), "dtype"),
             (args(out_dtype=_ffi.DTYPE_FP8_E4M3), "out_dtype"), (args(out_dtype=_ffi.DTYPE_F16), "out_dtype"),
             (args(dtype=_ffi.DTYPE_F16, out_dtype=_ffi.DTYPE_BF16), "out_dtype"),
             (args(F=0), "size"), (args(n_rows=-1), "size"), (args(n=-1), "size"), (args(ld=3), "ld"),
             (args(ldo=3), "ldo"), (args(index=None), "null"), (args(out=None), "null"), (args(table=None), "null"),
             (args(dtype=_ffi.DTYPE_F32, n=0), "dtype")]                      # the dtype is checked even with nothing to do
    for a, words in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(MAPPED16, *a)
        assert err.value.code == _ffi.ERR_INVALID_ARGUMENT, a
        assert words in str(err.value), (a, str(err.value))
    for dt in (_ffi.DTYPE_BF16, _ffi.DTYPE_F16):                              # nothing to gather: no launch
        _ffi.call(MAPPED16, None, dt, 4, 10, 4, None, 0, None, _ffi.DTYPE_F32, 4, None)
        _ffi.call(MAPPED16, None, dt, 4, 10, 4, None, 0, None, dt, 4, None)


def test_cached_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    buf = (ctypes.c_uint16 * 16)()
    p = ctypes.addressof(buf)
    names = ["table", "dtype", "ld", "n_rows", "F", "cache", "ldc", "slot", "index", "n", "out", "ldo"]
    ok = [p, _ffi.DTYPE_F16, 4, 10, 4, p, 4, p, p, 1, p, 4, None]

    def args(**kw):
        a = list(ok)
        for k, v in kw.items():
            a[names.index(k)] = v
        return a
    cases = [(args(dtype=_ffi.DTYPE_F32), "dtype"), (args(dtype=_ffi.DTYPE_FP8_E4M3), "dtype"), (args(dtype=-1), "dtype"),
             (args(F=0), "size"), (args(n_rows=-1), "size"), (args(n=-1), "size"), (args(ld=3), "ld"),
             (args(ldc=3), "ldc"), (args(ldo=3), "ldo"), (args(cache=None), "null"), (args(slot=None), "null"),
             (args(index=None), "null"), (args(out=None), "null"), (args(table=None), "null")]
    for a, words in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(CACHED16, *a)
        assert err.value.code == _ffi.ERR_INVALID_ARGUMENT, a
        assert words in str(err.value), (a, str(err.value))
    _ffi.call(CACHED16, None, _ffi.DTYPE_BF16, 4, 10, 4, None, 4, None, None, 0, None, 4, None)


class _OnDevice(torch.Tensor):                          # a CPU stand-in for a CUDA tensor
    @property
    def is_cuda(self):
        return True


def _dev(t):
    return t.as_subclass(_OnDevice)


def test_wrapper_refusals():
    """ops.gather_rows_mapped_16's and ops.gather_rows_cached_16's own checks, before any launch."""
    from tf_geometric_b200 import ops
    n_rows, F = 10, 4
    index = _dev(torch.zeros(5, dtype=torch.int32))
    for kw, err, words in [(dict(dtype=torch.float32), ValueError, "bfloat16"),
                           (dict(dtype=torch.int16), ValueError, "float16"),
                           (dict(out_dtype=torch.float64), ValueError, "out_dtype"),
                           (dict(dtype=torch.float16, out_dtype=torch.bfloat16), ValueError, "out_dtype"),
                           (dict(index=_dev(torch.zeros(5, dtype=torch.int64))), TypeError, "index"),
                           (dict(out=_dev(torch.zeros(5, F + 1))), TypeError, "out"),
                           (dict(out=_dev(torch.zeros(5, F, dtype=torch.bfloat16))), TypeError, "out"),
                           (dict(out=torch.zeros(5, F)), TypeError, "out"),                       # a host tensor
                           (dict(out=_dev(torch.zeros(5, F)), out_dtype=torch.bfloat16), TypeError, "out")]:
        a = dict(dtype=torch.bfloat16, index=index, out=None, out_dtype=torch.float32)
        a.update(kw)
        with pytest.raises(err, match=words):
            ops.gather_rows_mapped_16(0, a["dtype"], F, n_rows, F, a["index"], out=a["out"], out_dtype=a["out_dtype"])

    cache, slot = _dev(torch.zeros(3, F, dtype=torch.float16)), _dev(torch.full((n_rows,), -1, dtype=torch.int32))
    elsewhere = torch.zeros(3, F, dtype=torch.float16, device="meta").as_subclass(_OnDevice)
    for kw, err, words in [(dict(cache=_dev(torch.zeros(3, F))), TypeError, "cache"),                 # float32 cache
                           (dict(cache=torch.zeros(3, F, dtype=torch.float16)), TypeError, "cache"),  # a host tensor
                           (dict(cache=_dev(torch.zeros(3, F + 1, dtype=torch.float16))), TypeError, "cache"),
                           (dict(cache=_dev(torch.zeros(3 * F, dtype=torch.float16))), TypeError, "cache"),
                           (dict(slot=_dev(torch.full((n_rows - 1,), -1, dtype=torch.int32))), ValueError, "slot"),
                           (dict(slot=_dev(torch.full((n_rows,), -1, dtype=torch.int64))), TypeError, "slot"),
                           (dict(index=_dev(torch.zeros(5, dtype=torch.int64))), TypeError, "index"),
                           (dict(out=_dev(torch.zeros(5, F, dtype=torch.float16))), TypeError, "out"),
                           (dict(cache=elsewhere), ValueError, "one device")]:
        a = dict(cache=cache, slot=slot, index=index, out=None)
        a.update(kw)
        with pytest.raises(err, match=words):
            ops.gather_rows_cached_16(0, F, n_rows, F, a["cache"], a["slot"], a["index"], out=a["out"])


def test_dtype_keyword_refusals(fake):
    tfg, calls, registered = fake
    HFT = tfg.utils.HostFeatureTable
    x = _x()
    for bad in (torch.float64, torch.int16, torch.float8_e4m3fn, "bfloat16", np.float16, None):
        with pytest.raises(ValueError, match="dtype"):
            HFT(x.to(torch.bfloat16), dtype=bad)
    for table, dtype in [(x, torch.bfloat16), (x, torch.float16), (x.half(), torch.bfloat16),
                         (x.to(torch.bfloat16), torch.float16), (x.numpy(), torch.float16),
                         (x.numpy().astype(np.float16), torch.bfloat16)]:
        got = table.dtype if torch.is_tensor(table) else torch.from_numpy(table).dtype
        with pytest.raises(TypeError) as err:
            HFT(table, dtype=dtype, device_rows=[1, 2])
        assert str(dtype) in str(err.value) and str(got) in str(err.value), str(err.value)
    for table in (x.half(), x.to(torch.bfloat16), x.numpy().astype(np.float16)):    # the default stays float32
        with pytest.raises(TypeError, match="float32 features"):
            HFT(table)
    assert calls == [] and registered == {}                 # refused before registering or gathering


def _session(tfg, x, dtype, rows):
    """The same sequence of table operations for any dtype: construction (with a cache when rows), three gathers."""
    HFT = tfg.utils.HostFeatureTable
    kw = {} if dtype is None else dict(dtype=dtype)
    with HFT(x, device_rows=rows, **kw) as t:
        a = t.gather([5, 1, 5, 39])
        out = torch.full((2, x.shape[1]), 7.0)
        b = t.gather([0, 17], out=out)
        assert b is out
        c = t.gather(np.zeros(0, np.int32))
    return t, a, b, c


def test_float32_call_log_is_unchanged(fake):
    tfg, calls, _ = fake
    x = _x()
    ptr, nbytes = x.untyped_storage().data_ptr(), x.untyped_storage().nbytes()
    for dtype in (None, torch.float32):
        del calls[:]
        _session(tfg, x, dtype, None)
        assert calls == [("register", ptr, nbytes), ("gather", ptr, 6, 40, 6, 4), ("gather", ptr, 6, 40, 6, 2),
                         ("unregister", ptr)]
        del calls[:]
        _session(tfg, x, dtype, [3, 9])
        assert calls == [("register", ptr, nbytes), ("gather", ptr, 6, 40, 6, 2),
                         ("gather_cached", ptr, 6, 40, 6, 2, 4), ("gather_cached", ptr, 6, 40, 6, 2, 2),
                         ("unregister", ptr)]


@pytest.mark.parametrize("dtype", DTYPES)
def test_16_bit_tables_are_routed_to_the_new_entries(fake, dtype):
    tfg, calls, _ = fake
    x = _x(dtype=dtype)
    ptr, nbytes = x.untyped_storage().data_ptr(), x.untyped_storage().nbytes()
    t, a, b, c = _session(tfg, x, dtype, None)
    assert calls == [("register", ptr, nbytes), ("gather16", ptr, dtype, 6, 40, 6, 4, torch.float32),
                     ("gather16", ptr, dtype, 6, 40, 6, 2, torch.float32), ("unregister", ptr)]
    for got, ids in ((a, [5, 1, 5, 39]), (b, [0, 17])):
        assert got.dtype == torch.float32
        np.testing.assert_array_equal(got.numpy(), _widened(x, ids))
    assert c.shape == (0, 6) and c.dtype == torch.float32
    del calls[:]
    t, a, b, c = _session(tfg, x, dtype, [3, 9, 5])
    # the cache is filled by the copy mode of the mapped entry, in the table's dtype
    assert calls == [("register", ptr, nbytes), ("gather16", ptr, dtype, 6, 40, 6, 3, dtype),
                     ("gather_cached16", ptr, dtype, 6, 40, 6, 3, 4), ("gather_cached16", ptr, dtype, 6, 40, 6, 3, 2),
                     ("unregister", ptr)]
    np.testing.assert_array_equal(a.numpy(), _widened(x, [5, 1, 5, 39]))
    np.testing.assert_array_equal(b.numpy(), _widened(x, [0, 17]))
    assert not any(k[0] in ("gather", "gather_cached") for k in calls)


@pytest.mark.parametrize("dtype", DTYPES)
def test_cache_device_bytes_and_dtype(fake, dtype):
    tfg, _, _ = fake
    x = _x(50, 7, seed=1, dtype=dtype)
    rows = np.array([31, 2, 49, 0, 17], np.int64)
    with tfg.utils.HostFeatureTable(x, device_rows=rows, dtype=dtype) as t:
        assert t.dtype == dtype
        assert t._cache.dtype == dtype and t._cache.shape == (5, 7)
        np.testing.assert_array_equal(fake_half.bits16(t._cache), fake_half.bits16(x)[rows])
        assert t.device_bytes == rows.size * 7 * 2 + 50 * 4
    with tfg.utils.HostFeatureTable(x, dtype=dtype) as t:
        assert t.dtype == dtype and t.device_bytes == 0
    x32 = _x(50, 7, seed=1)
    with tfg.utils.HostFeatureTable(x32, device_rows=rows) as t:
        assert t.dtype == torch.float32 and t.device_bytes == rows.size * 7 * 4 + 50 * 4


def test_numpy_float16_is_wrapped_without_a_copy(fake):
    tfg, _, _ = fake
    a = np.random.RandomState(2).randn(30, 5).astype(np.float16)
    t = tfg.utils.HostFeatureTable(a, dtype=torch.float16)
    assert t.x.data_ptr() == a.ctypes.data and t.x.untyped_storage().data_ptr() == a.ctypes.data
    a[4] = 7.0                                              # the table reads the array itself
    np.testing.assert_array_equal(t.gather([4]).numpy(), a[[4]].astype(np.float32))
    sliced = a[:, 1:4]                                      # a strided numpy view: row stride 5 > F = 3
    t2 = tfg.utils.HostFeatureTable(sliced, dtype=torch.float16)
    assert t2._ld == 5
    np.testing.assert_array_equal(t2.gather([0, 29, 3]).numpy(), sliced[[0, 29, 3]].astype(np.float32))
    t.close()
    t2.close()


def test_special_values_widen_exactly(fake):
    """The fake's widening is x.float(): the reference the GPU tests hold the kernels to."""
    tfg, _, _ = fake
    for dtype in DTYPES:
        info = torch.finfo(dtype)
        vals = torch.tensor([0.0, -0.0, info.tiny, info.tiny / 4, -info.tiny / 8, info.max, -info.max,
                             float("inf"), -float("inf"), 1.0], dtype=dtype).reshape(2, 5)
        with tfg.utils.HostFeatureTable(vals, dtype=dtype) as t:
            got = t.gather([1, 0])
            assert torch.equal(got.view(torch.int32), vals.float()[[1, 0]].view(torch.int32))


def _batch(tfg, n_nodes=300):
    ei = random_graph(n_nodes, 2400, seed=5, isolated=20, hub=(7, 400)).astype(np.int32)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    return sampler.sample_blocks(np.array([7, 0, 299, 3, 150, 42, 77], np.int32), [4, 3], seed=2)


@pytest.mark.parametrize("dtype", DTYPES)
def test_source_rows_routing(fake, dtype):
    tfg, calls, _ = fake
    b = _batch(tfg)
    x = _x(300, 12, seed=3, dtype=dtype)
    ni = b.node_index.numpy()
    want = _widened(x, ni)
    pairs = torch.tensor([[0, 1, 2], [3, 4, 5]], dtype=torch.int32)
    link = tfg.utils.LinkBlocks(b.node_index, b.hop_sizes, b.blocks, b.num_nodes, pairs, 2)
    by_hand = tfg.utils.SampledBlocks(b.node_index, b.hop_sizes, b.blocks)
    with tfg.utils.HostFeatureTable(x, dtype=dtype) as t:
        for batch in (b, link, by_hand):
            n = len(calls)
            rows = batch.source_rows(t)
            assert rows.dtype == torch.float32
            np.testing.assert_array_equal(rows.numpy(), want)
            assert calls[n:] == [("gather16", t._ptr, dtype, 12, 300, 12, ni.size, torch.float32)]
    cached = ni[::2].copy()
    with tfg.utils.HostFeatureTable(x, device_rows=cached, dtype=dtype) as t:
        for batch in (b, link, by_hand):
            n = len(calls)
            np.testing.assert_array_equal(batch.source_rows(t).numpy(), want)
            assert calls[n:] == [("gather_cached16", t._ptr, dtype, 12, 300, 12, cached.size, ni.size)]
    with tfg.utils.HostFeatureTable(x[:299], dtype=dtype) as short, pytest.raises(ValueError, match="rows"):
        b.source_rows(short)
