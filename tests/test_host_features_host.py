# coding=utf-8
"""Feature tables in host memory without a GPU: the ABI declarations and argument checks of the host-table entries, and
utils.HostFeatureTable over the numpy fake of tests/host_table_fake_backend.py: one registration per storage with a
count, release on close, every refusal before any (fake) device work, integer and numpy ids, and the routing of
SampledBlocks.source_rows for a host table, a device tensor and a CPU tensor."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import host_table_fake_backend as fake_host
from conftest import random_graph

ENTRIES = {"tfgk_host_register": 3, "tfgk_host_unregister": 1, "tfgk_gather_rows_mapped_f32": 9}


def _header_arity(name):
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "tfgk.h")).read()
    m = re.search(r"int {}\(([^;]*)\);".format(name), header)
    assert m, name
    return len(m.group(1).split(","))


@pytest.fixture
def fake(monkeypatch):
    calls, registered, _ = fake_host.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg, calls, registered


def _x(n=40, F=6, seed=0):
    return torch.from_numpy(np.random.RandomState(seed).randn(n, F).astype(np.float32))


def test_entries_are_declared_and_exported():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    lib = _ffi.lib()
    for name, n in ENTRIES.items():
        assert len(_ffi.SIGNATURES[name]) == _header_arity(name) == n, name
        assert hasattr(lib, name), name
    assert "tfgk_host_register" in _ffi.NOT_CAPTURABLE
    assert "tfgk_gather_rows_mapped_f32" not in _ffi.NOT_CAPTURABLE          # no host value, no host key


def test_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    dev = ctypes.c_void_p()
    buf = (ctypes.c_float * 8)()
    cases = [
        ("tfgk_host_register", (None, 64, ctypes.byref(dev)), "null"),
        ("tfgk_host_register", (ctypes.addressof(buf), 0, ctypes.byref(dev)), "empty"),
        ("tfgk_host_register", (ctypes.addressof(buf), 32, None), "null"),
        ("tfgk_host_unregister", (None,), "null"),
        ("tfgk_gather_rows_mapped_f32", (None, 4, 10, 0, None, 1, None, 4, None), "size"),
        ("tfgk_gather_rows_mapped_f32", (None, 4, -1, 4, None, 1, None, 4, None), "size"),
        ("tfgk_gather_rows_mapped_f32", (None, 4, 10, 4, None, -1, None, 4, None), "size"),
        ("tfgk_gather_rows_mapped_f32", (None, 3, 10, 4, None, 1, None, 4, None), "ld"),
        ("tfgk_gather_rows_mapped_f32", (None, 4, 10, 4, None, 1, None, 3, None), "ldo"),
        ("tfgk_gather_rows_mapped_f32", (None, 4, 10, 4, None, 1, None, 4, None), "null"),
    ]
    for name, args, words in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(name, *args)
        assert err.value.code == _ffi.ERR_INVALID_ARGUMENT, name
        assert words in str(err.value), (name, str(err.value))
    _ffi.call("tfgk_gather_rows_mapped_f32", None, 4, 10, 4, None, 0, None, 4, None)     # nothing to gather: no launch


def test_one_registration_per_storage(fake):
    tfg, calls, registered = fake
    x = _x()
    storage = x.untyped_storage()
    a = tfg.utils.HostFeatureTable(x)
    b = tfg.utils.HostFeatureTable(x[:, 2:5])            # a column slice: same storage, row stride 6 > F = 3
    c = tfg.utils.HostFeatureTable(x[10:20])
    assert calls == [("register", storage.data_ptr(), storage.nbytes())]
    assert (b.num_rows, b.num_features, c.num_rows, c.num_features) == (40, 3, 10, 6)
    a.close()
    b.close()
    assert list(registered) == [storage.data_ptr()]      # c still holds it
    np.testing.assert_array_equal(c.gather([0, 9]).numpy(), x.numpy()[[10, 19]])
    c.close()
    assert calls[-1] == ("unregister", storage.data_ptr()) and registered == {}
    d = tfg.utils.HostFeatureTable(x)                    # registering again after the last close
    assert calls[-1] == ("register", storage.data_ptr(), storage.nbytes())
    d.close()
    assert registered == {}


def test_close_and_use_after_close(fake):
    tfg, calls, registered = fake
    x = _x()
    with tfg.utils.HostFeatureTable(x) as t:
        assert registered
    assert registered == {}
    n = len(calls)
    t.close()                                           # a second close does nothing
    assert len(calls) == n
    with pytest.raises(RuntimeError, match="closed"):
        t.gather([1])
    sampler = tfg.utils.RandomNeighborSampler(random_graph(40, 200, seed=1))
    b = sampler.sample_blocks([3, 5], [2], seed=1)
    with pytest.raises(RuntimeError, match="closed"):
        b.source_rows(t)
    assert len(calls) == n
    t2 = tfg.utils.HostFeatureTable(x)
    del t2                                              # collected without close(): released
    assert registered == {}


def test_refusals_before_device_work(fake):
    tfg, calls, registered = fake
    HFT = tfg.utils.HostFeatureTable
    x = _x()

    class OnDevice(torch.Tensor):                       # a CPU stand-in for a CUDA tensor
        @property
        def is_cuda(self):
            return True
    for bad, err, words in [(x.clone().requires_grad_(), ValueError, "grad"), (x.double(), TypeError, "float32"),
                            (x.numpy().astype(np.float16), TypeError, "float32"), (x[0], TypeError, "2-D"),
                            (x[None], TypeError, "2-D"), (x.as_subclass(OnDevice), TypeError, "CUDA"),
                            (x.tolist(), TypeError, "numpy"), (x.t(), ValueError, "column stride"),
                            (x[:1].expand(5, 6), ValueError, "overlap")]:
        with pytest.raises(err, match=words):
            HFT(bad)
    assert calls == [] and registered == {}


def test_numpy_table_is_wrapped_without_a_copy(fake):
    tfg, calls, _ = fake
    a = np.random.RandomState(2).randn(30, 5).astype(np.float32)
    t = tfg.utils.HostFeatureTable(a)
    assert t.x.data_ptr() == a.ctypes.data and t.x.untyped_storage().data_ptr() == a.ctypes.data
    a[4] = 7.0                                          # the table reads the array itself
    np.testing.assert_array_equal(t.gather([4]).numpy(), a[[4]])
    sliced = a[:, 1:4]                                  # a strided numpy view: row stride 5 > F = 3
    t2 = tfg.utils.HostFeatureTable(sliced)
    np.testing.assert_array_equal(t2.gather([0, 29, 3]).numpy(), sliced[[0, 29, 3]])
    t.close()
    t2.close()


def test_ids(fake):
    tfg, calls, _ = fake
    x = _x()
    t = tfg.utils.HostFeatureTable(x)
    want = x.numpy()[[5, 5, 39, 0, 17]]
    for ids in ([5, 5, 39, 0, 17], np.array([5, 5, 39, 0, 17], np.int64), np.array([5, 5, 39, 0, 17], np.int32),
                torch.tensor([5, 5, 39, 0, 17]), torch.tensor([5, 5, 39, 0, 17], dtype=torch.int32),
                np.array([[5, 5], [39, 0]], np.int64)):
        got = t.gather(ids).numpy()
        np.testing.assert_array_equal(got, want[:got.shape[0]])
    n = len(calls)
    for bad in ([40], [-1], [3, 40], np.array([2 ** 32 + 5], np.int64), np.array([-(2 ** 32) + 5], np.int64)):
        with pytest.raises(IndexError, match="outside"):
            t.gather(bad)
    with pytest.raises(TypeError, match="integer"):
        t.gather(np.array([1.0, 2.0]))
    empty = t.gather(np.zeros(0, np.int64))
    assert tuple(empty.shape) == (0, 6) and empty.dtype == torch.float32
    assert len(calls) == n                              # refused and empty gathers launch nothing
    out = torch.empty(2, 6)
    assert t.gather([1, 2], out=out) is out
    np.testing.assert_array_equal(out.numpy(), x.numpy()[[1, 2]])
    t.close()


def _batch(tfg, n_nodes=300):
    ei = random_graph(n_nodes, 2400, seed=5, isolated=20, hub=(7, 400)).astype(np.int32)
    sampler = tfg.utils.RandomNeighborSampler(ei)
    return sampler.sample_blocks(np.array([7, 0, 299, 3, 150, 42, 77], np.int32), [4, 3], seed=2)


def test_source_rows_routing(fake, monkeypatch):
    tfg, calls, _ = fake
    b = _batch(tfg)
    assert b.num_nodes == 300
    x = _x(300, 12, seed=3)
    want = x.numpy()[b.node_index.numpy()]
    t = tfg.utils.HostFeatureTable(x)

    def no_checked_gather(self, index, out=None):
        raise AssertionError("a sampled batch's ids were checked by the sampler")
    with monkeypatch.context() as m:
        m.setattr(tfg.utils.HostFeatureTable, "gather", no_checked_gather)
        rows = b.source_rows(t)
    assert torch.is_tensor(rows) and not isinstance(rows, tfg.utils.SourceRows)
    np.testing.assert_array_equal(rows.numpy(), want)
    assert calls[-1] == ("gather", x.data_ptr(), 12, 300, 12, len(want))

    n = len(calls)
    with pytest.raises(ValueError, match="rows"):       # fewer rows than the sampler's nodes: refused from sizes
        b.source_rows(tfg.utils.HostFeatureTable(x[:299]))
    assert len(calls) == n

    by_hand = tfg.utils.SampledBlocks(b.node_index, b.hop_sizes, b.blocks)
    assert by_hand.num_nodes is None
    np.testing.assert_array_equal(by_hand.source_rows(t).numpy(), want)
    short = tfg.utils.HostFeatureTable(x[:int(b.node_index.max())])
    with pytest.raises(IndexError, match="outside"):    # a batch built by hand takes the checked gather
        by_hand.source_rows(short)

    for table in (x, x.numpy()):                        # tensors keep their route: SourceRows over the table
        src = b.source_rows(table)
        assert isinstance(src, tfg.utils.SourceRows) and src.shape == (len(want), 12)
        np.testing.assert_array_equal(src.gather().numpy(), want)
    t.close()
    short.close()


@pytest.mark.parametrize("kind", ["MeanGraphSage", "SumGraphSage", "MeanPoolGraphSage", "MaxPoolGraphSage"])
def test_layers_on_host_rows(fake, kind):
    tfg, _, _ = fake
    b = _batch(tfg)
    x = _x(300, 12, seed=3)
    layers = [getattr(tfg.layers, kind)(8, seed=1, trainable=True), getattr(tfg.layers, kind)(4, seed=2, trainable=True)]
    with tfg.utils.HostFeatureTable(x) as t:
        h = b.source_rows(t)
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, blk], training=True)
    h.sum().backward()
    grads = [p.grad.clone() for layer in layers for p in layer.parameters()]
    for layer in layers:
        layer.zero_grad()
    h2 = x[b.node_index.long()]
    for layer, blk in zip(layers, b.blocks):
        h2 = layer([h2, blk], training=True)
    h2.sum().backward()
    np.testing.assert_array_equal(h.detach().numpy(), h2.detach().numpy())
    for g, layer_p in zip(grads, [p for layer in layers for p in layer.parameters()]):
        np.testing.assert_array_equal(g.numpy(), layer_p.grad.numpy())
