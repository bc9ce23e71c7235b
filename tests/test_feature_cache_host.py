# coding=utf-8
"""Device rows of a host feature table without a GPU: the ABI declaration and argument checks of
tfgk_gather_rows_cached_f32, and HostFeatureTable(x, device_rows=...) and rank_source_rows over the numpy fake of
tests/feature_cache_fake_backend.py: the slot map, the refusals of device_rows, the routing of gathers between the
cached and the uncached entry, device_bytes, release on close, and the ranking against a numpy restatement."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import feature_cache_fake_backend as fake_cache
from conftest import random_graph

CACHED = "tfgk_gather_rows_cached_f32"


def _header_arity(name):
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "tfgk.h")).read()
    m = re.search(r"int {}\(([^;]*)\);".format(name), header)
    assert m, name
    return len(m.group(1).split(","))


@pytest.fixture
def fake(monkeypatch):
    calls, registered, _ = fake_cache.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg, calls, registered


def _x(n=40, F=6, seed=0):
    return torch.from_numpy(np.random.RandomState(seed).randn(n, F).astype(np.float32))


def test_entry_is_declared_and_exported():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    assert len(_ffi.SIGNATURES[CACHED]) == _header_arity(CACHED) == 12
    assert hasattr(_ffi.lib(), CACHED)
    assert CACHED not in _ffi.NOT_CAPTURABLE                                 # no host value, no host key


def test_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    buf = (ctypes.c_float * 8)()
    p = ctypes.addressof(buf)
    #        table ld  n_rows F  cache ldc slot index n  out ldo stream
    ok = [p, 4, 10, 4, p, 4, p, p, 1, p, 4, None]

    def args(**kw):
        a = list(ok)
        for k, v in kw.items():
            a[["table", "ld", "n_rows", "F", "cache", "ldc", "slot", "index", "n", "out", "ldo"].index(k)] = v
        return a
    cases = [(args(F=0), "size"), (args(n_rows=-1), "size"), (args(n=-1), "size"), (args(ld=3), "ld"),
             (args(ldc=3), "ldc"), (args(ldo=3), "ldo"), (args(cache=None), "null"), (args(slot=None), "null"),
             (args(index=None), "null"), (args(out=None), "null"), (args(table=None), "null")]
    for a, words in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(CACHED, *a)
        assert err.value.code == _ffi.ERR_INVALID_ARGUMENT, a
        assert words in str(err.value), (a, str(err.value))
    _ffi.call(CACHED, None, 4, 10, 4, None, 4, None, None, 0, None, 4, None)        # nothing to gather: no launch


def test_slot_map_and_cache(fake):
    tfg, calls, _ = fake
    x = _x(50, 7, seed=1)
    rows = np.array([31, 2, 49, 0, 17], np.int64)
    with tfg.utils.HostFeatureTable(x, device_rows=rows) as t:
        want_slot = np.full(50, -1, np.int32)
        want_slot[rows] = np.arange(rows.size)
        np.testing.assert_array_equal(t._slot.numpy(), want_slot)
        np.testing.assert_array_equal(t._cache.numpy(), x.numpy()[rows])
        assert t.device_rows.dtype == torch.int32
        np.testing.assert_array_equal(t.device_rows.numpy(), rows)
        assert t.device_bytes == rows.size * 7 * 4 + 50 * 4
        # the cache was filled by the uncached host gather, with its old arguments
        assert ("gather", x.data_ptr(), 7, 50, 7, rows.size) in calls


@pytest.mark.parametrize("kind", ["list", "numpy32", "torch64", "torch32"])
def test_device_rows_kinds(fake, kind):
    tfg, _, _ = fake
    x = _x()
    ids = [3, 39, 0]
    rows = {"list": ids, "numpy32": np.array(ids, np.int32), "torch64": torch.tensor(ids),
            "torch32": torch.tensor(ids, dtype=torch.int32)}[kind]
    with tfg.utils.HostFeatureTable(x, device_rows=rows) as t:
        np.testing.assert_array_equal(t.device_rows.numpy(), ids)


def test_refusals_of_device_rows(fake):
    tfg, calls, registered = fake
    HFT = tfg.utils.HostFeatureTable
    x = _x()
    for bad, err, words in [([40], IndexError, "outside"), ([-1], IndexError, "outside"),
                            ([0, 40, 40], IndexError, "outside"),
                            (np.array([2 ** 32 + 5], np.int64), IndexError, "outside"),
                            (np.array([-(2 ** 32) + 5], np.int64), IndexError, "outside"),
                            ([3, 5, 3], ValueError, "repeated"), (np.array([[1, 2], [3, 4]]), ValueError, "vector"),
                            (torch.tensor(3), ValueError, "vector"),
                            (np.array([1.0, 2.0]), TypeError, "integer"), (torch.tensor([True]), TypeError, "integer")]:
        with pytest.raises(err, match=words):
            HFT(x, device_rows=bad)
    assert calls == [] and registered == {}                 # refused before registering or gathering
    with pytest.raises(TypeError, match="float32"):         # the table's own refusals come first
        HFT(x.double(), device_rows=[40])


def test_device_rows_are_the_tables_own(fake):
    tfg, _, _ = fake
    x = _x()
    ranked = torch.tensor([9, 4, 30, 2], dtype=torch.int32)
    with tfg.utils.HostFeatureTable(x, device_rows=ranked[:3]) as t:
        ranked.fill_(0)                                     # the caller reuses its buffer
        np.testing.assert_array_equal(t.device_rows.numpy(), [9, 4, 30])
        np.testing.assert_array_equal(t.gather([30, 1]).numpy(), x.numpy()[[30, 1]])


def test_wrapper_refusals():
    """ops.gather_rows_cached's own checks, before any launch (CPU tensors stand in for CUDA ones)."""
    from tf_geometric_b200 import ops

    class OnDevice(torch.Tensor):
        @property
        def is_cuda(self):
            return True

    def dev(t):
        return t.as_subclass(OnDevice)
    n_rows, F = 10, 4
    cache, slot, index = dev(torch.zeros(3, F)), dev(torch.full((n_rows,), -1, dtype=torch.int32)), \
        dev(torch.zeros(5, dtype=torch.int32))
    elsewhere = torch.zeros(3, F, device="meta").as_subclass(OnDevice)
    cases = [(dict(cache=dev(torch.zeros(3, F, dtype=torch.float64))), TypeError, "cache"),
             (dict(cache=torch.zeros(3, F)), TypeError, "cache"),                       # a host tensor
             (dict(cache=dev(torch.zeros(3, F + 1))), TypeError, "cache"),
             (dict(cache=dev(torch.zeros(3 * F))), TypeError, "cache"),
             (dict(slot=dev(torch.full((n_rows - 1,), -1, dtype=torch.int32))), ValueError, "slot"),
             (dict(slot=dev(torch.full((n_rows,), -1, dtype=torch.int64))), TypeError, "slot"),
             (dict(index=dev(torch.zeros(5, dtype=torch.int64))), TypeError, "index"),
             (dict(out=dev(torch.zeros(5, F + 1))), TypeError, "out"),
             (dict(cache=elsewhere), ValueError, "one device")]
    for kw, err, words in cases:
        a = dict(cache=cache, slot=slot, index=index, out=None)
        a.update(kw)
        with pytest.raises(err, match=words):
            ops.gather_rows_cached(0, F, n_rows, F, a["cache"], a["slot"], a["index"], out=a["out"])


def test_no_cache_behaves_as_before(fake):
    tfg, calls, _ = fake
    x = _x()
    for rows in (None, [], np.zeros(0, np.int64), torch.zeros(0, dtype=torch.int32)):
        with tfg.utils.HostFeatureTable(x, device_rows=rows) as t:
            assert t.device_rows is None and t.device_bytes == 0
            np.testing.assert_array_equal(t.gather([5, 1, 5]).numpy(), x.numpy()[[5, 1, 5]])
            assert calls[-1] == ("gather", x.data_ptr(), 6, 40, 6, 3)
    assert not any(c[0] == "gather_cached" for c in calls)


def _batch(tfg, n_nodes=300):
    ei = random_graph(n_nodes, 2400, seed=5, isolated=20, hub=(7, 400)).astype(np.int32)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    return sampler, sampler.sample_blocks(np.array([7, 0, 299, 3, 150, 42, 77], np.int32), [4, 3], seed=2)


def test_routing(fake, monkeypatch):
    tfg, calls, _ = fake
    _, b = _batch(tfg)
    x = _x(300, 12, seed=3)
    want = x.numpy()[b.node_index.numpy()]
    cached = b.node_index.numpy()[::2].copy()
    t = tfg.utils.HostFeatureTable(x, device_rows=cached)
    n = len(calls)
    rows = b.source_rows(t)                                 # on the cache's device: the cached entry
    np.testing.assert_array_equal(rows.numpy(), want)
    assert calls[n:] == [("gather_cached", x.data_ptr(), 12, 300, 12, cached.size, len(want))]
    ids = [299, 3, 3, 0, int(cached[0])]
    np.testing.assert_array_equal(t.gather(ids).numpy(), x.numpy()[ids])
    assert calls[-1][0] == "gather_cached"
    out = torch.full((5, 12), 7.0)
    assert t.gather(ids, out=out) is out
    np.testing.assert_array_equal(out.numpy(), x.numpy()[ids])
    by_hand = tfg.utils.SampledBlocks(b.node_index, b.hop_sizes, b.blocks)
    np.testing.assert_array_equal(by_hand.source_rows(t).numpy(), want)
    assert calls[-1][0] == "gather_cached"

    with monkeypatch.context() as m:                        # a cache on another device than the gather's
        m.setattr(t, "_cache", torch.empty((cached.size, 12), device="meta"))
        n = len(calls)
        np.testing.assert_array_equal(b.source_rows(t).numpy(), want)
        assert calls[n:] == [("gather", x.data_ptr(), 12, 300, 12, len(want))]    # every row over the link
    t.close()


def test_two_caches_share_one_registration(fake):
    tfg, calls, registered = fake
    x = _x()
    storage = x.untyped_storage()
    a = tfg.utils.HostFeatureTable(x, device_rows=[1, 2, 3])
    b = tfg.utils.HostFeatureTable(x, device_rows=[39])
    c = tfg.utils.HostFeatureTable(x)
    assert [k for k in calls if k[0] == "register"] == [("register", storage.data_ptr(), storage.nbytes())]
    for t in (a, b, c):
        np.testing.assert_array_equal(t.gather([39, 2, 0]).numpy(), x.numpy()[[39, 2, 0]])
    a.close()
    b.close()
    assert list(registered) == [storage.data_ptr()]
    c.close()
    assert registered == {}


def test_close_drops_cache_and_registration(fake):
    tfg, calls, registered = fake
    x = _x()
    with tfg.utils.HostFeatureTable(x, device_rows=[4, 8]) as t:
        assert registered and t.device_bytes > 0
    assert registered == {}
    assert t._cache is None and t._slot is None and t.device_rows is None and t.device_bytes == 0
    with pytest.raises(RuntimeError, match="closed"):
        t.gather([1])
    t2 = tfg.utils.HostFeatureTable(x, device_rows=[5])
    del t2                                                  # collected without close(): released
    assert registered == {}


def _rank_ref(node_indices, num_nodes):
    counts = np.zeros(num_nodes, np.int64)
    for ni in node_indices:
        counts[np.unique(ni)] += 1
    ids = np.array(sorted(np.flatnonzero(counts), key=lambda j: (-counts[j], j)), np.int64)
    return ids, counts


def test_rank_source_rows(fake):
    tfg, _, _ = fake
    sampler, _ = _batch(tfg)
    rs = np.random.RandomState(4)
    batches = [sampler.sample_blocks(rs.choice(300, 6, replace=False).astype(np.int32), [3, 2], seed=k)
               for k in range(12)]
    batches.append(batches[0])                              # the same batch twice counts twice
    ids, counts = tfg.utils.rank_source_rows(iter(batches))
    want_ids, want_counts = _rank_ref([b.node_index.numpy() for b in batches], 300)
    assert ids.dtype == counts.dtype == torch.int32 and counts.shape == (300,)
    np.testing.assert_array_equal(counts.numpy(), want_counts)
    np.testing.assert_array_equal(ids.numpy(), want_ids)
    assert (want_counts == 0).any()                         # ids never sampled are left out
    c = want_counts[want_ids]
    assert any(c[i] == c[i + 1] for i in range(c.size - 1))  # ties, broken by id
    ids2, counts2 = tfg.utils.rank_source_rows(batches)
    assert torch.equal(ids, ids2) and torch.equal(counts, counts2)
    # the ranked rows drive a cache whose gathers still give x[index]
    x = _x(300, 5, seed=8)
    with tfg.utils.HostFeatureTable(x, device_rows=ids[:40]) as t:
        np.testing.assert_array_equal(batches[3].source_rows(t).numpy(), x.numpy()[batches[3].node_index.numpy()])


def test_rank_source_rows_edge_cases(fake):
    tfg, _, _ = fake
    ids, counts = tfg.utils.rank_source_rows([])
    assert ids.shape == counts.shape == (0,) and ids.dtype == counts.dtype == torch.int32
    sampler, b = _batch(tfg)
    by_hand = tfg.utils.SampledBlocks(b.node_index, b.hop_sizes, b.blocks)
    with pytest.raises(ValueError, match="by hand"):
        tfg.utils.rank_source_rows([b, by_hand])
    other = tfg.utils.RandomNeighborSampler(random_graph(200, 1000, seed=6).astype(np.int32))
    with pytest.raises(ValueError, match="one graph"):
        tfg.utils.rank_source_rows([b, other.sample_blocks(np.array([1, 2], np.int32), [2], seed=1)])
