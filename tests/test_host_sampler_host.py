# coding=utf-8
"""Sampling from a graph in host memory without a GPU: the ABI declarations and argument checks of the host-CSR entries
and of the mapped block fill, range cutting against the device budget, and utils.HostNeighborSampler over the numpy fake
of tests/host_sampler_fake_backend.py: argument checks and dtype conversion, the host CSR against the oracle's CSR, one
registration per buffer (with a HostFeatureTable over another buffer open at the same time), release of the edge list by
the constructor and of the CSR by close(), and blocks assembled by the helper RandomNeighborSampler.sample_blocks uses."""
import ctypes

import numpy as np
import pytest
import torch

import host_sampler_fake_backend as fake_host
from conftest import random_graph
from oracle import c_oracle

ENTRIES = {"tfgk_mapped_id_range_i32": 7, "tfgk_mapped_rowptr_workspace_bytes": 2, "tfgk_mapped_rowptr_i32": 7,
           "tfgk_mapped_select_rows_workspace_bytes": 2, "tfgk_mapped_select_rows_i32": 13,
           "tfgk_block_sample_mapped_workspace_bytes": 3, "tfgk_block_sample_fill_mapped": 24}


@pytest.fixture
def fake(monkeypatch):
    calls, registered = fake_host.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg, calls, registered


def test_entries_are_declared_and_refuse_capture():
    from tf_geometric_b200 import _ffi
    lib = _ffi.lib()
    for name, n in ENTRIES.items():
        assert len(_ffi.SIGNATURES[name]) == n and hasattr(lib, name), name
    for name in ("tfgk_mapped_id_range_i32", "tfgk_block_sample_fill_mapped"):     # a host read-back, a host key
        assert name in _ffi.NOT_CAPTURABLE, name


def test_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    need = ctypes.c_size_t()
    cases = [
        ("tfgk_mapped_id_range_i32", (None, None, 0, None, None, 0, None), "bad argument"),
        ("tfgk_mapped_id_range_i32", (None, None, 10, (ctypes.c_int32 * 4)(), None, 0, None), "null"),
        ("tfgk_mapped_rowptr_workspace_bytes", (-1, ctypes.byref(need)), "bad argument"),
        ("tfgk_mapped_rowptr_i32", (None, -1, 4, None, None, 0, None), "size"),
        ("tfgk_mapped_rowptr_i32", (None, 10, 4, None, None, 0, None), "null"),
        ("tfgk_mapped_select_rows_workspace_bytes", (-1, ctypes.byref(need)), "bad argument"),
        ("tfgk_mapped_select_rows_i32", (None, None, None, 10, 3, 2, None, None, None, 5, None, 0, None), "size"),
        ("tfgk_mapped_select_rows_i32", (None, None, None, 10, 0, 2, None, None, None, 1 << 31, None, 0, None), "size"),
        ("tfgk_mapped_select_rows_i32", (None, None, None, 10, 0, 2, None, None, None, 5, None, 0, None), "null"),
        ("tfgk_block_sample_mapped_workspace_bytes", (4, 1 << 31, ctypes.byref(need)), "bad argument"),
        ("tfgk_block_sample_fill_mapped", (None, 4, None, None, 4, None, None, None, 2, 2, 8, 16, 3, 0, 0, 1, None, None,
                                           None, None, None, None, 0, None), "size"),
    ]
    for name, args, words in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(name, *args)
        assert err.value.code == _ffi.ERR_INVALID_ARGUMENT, name
        assert words in str(err.value), (name, str(err.value))
    _ffi.call("tfgk_block_sample_workspace_bytes", 100, 1500, ctypes.byref(need))
    plain = need.value
    _ffi.call("tfgk_block_sample_mapped_workspace_bytes", 100, 1500, ctypes.byref(need))
    assert need.value > plain                            # int64 positions
    _ffi.call("tfgk_mapped_select_rows_i32", None, None, None, 10, 2, 2, None, None, None, 0, None, 0, None)  # nothing


def test_row_ranges():
    from tf_geometric_b200.utils.sampling import _row_ranges
    rp = np.array([0, 3, 3, 10, 5010, 5012, 5012], np.int64)
    assert _row_ranges(rp, 10 ** 9, 33) == [(0, 6)]
    got = _row_ranges(rp, 33 * 5000 + 24, 33, 12)
    assert got == [(0, 3), (3, 4), (4, 6)]               # the hub row alone
    for r0, r1 in got:                                   # every range fits
        assert 33 * (rp[r1] - rp[r0]) + 12 * (r1 - r0 + 1) <= 33 * 5000 + 24
    with pytest.raises(ValueError, match="row 3 has 5000 edges"):
        _row_ranges(rp, 33 * 5000 + 23, 33, 12)
    with pytest.raises(ValueError, match="row 0 has 3 edges"):
        _row_ranges(rp, 10, 33, 12)
    assert _row_ranges(np.zeros(1, np.int64), 10, 33) == []
    big = np.array([0, 5, (1 << 31) - 10, (1 << 31) + 100], np.int64)
    assert _row_ranges(big, 1 << 50, 1) == [(0, 2), (2, 3)]          # fewer than 2^31 edges per range
    with pytest.raises(ValueError, match="row 1 has 2147483647 edges"):
        _row_ranges(np.array([0, 5, (1 << 31) + 4], np.int64), 1 << 50, 1)


def _graph():
    ei = random_graph(300, 2400, seed=5, isolated=20, hub=(7, 400))
    ei = np.concatenate([ei, ei[:, :50], [[3, 8], [350, 8]]], axis=1).astype(np.int32)
    w = np.random.RandomState(6).rand(ei.shape[1]).astype(np.float32)
    return ei, w


def _check_csr(s, ei, w):
    rowptr, col, perm = c_oracle.csr_build(ei[0], ei[1], int(ei.max()) + 1)
    np.testing.assert_array_equal(s.rowptr.numpy(), rowptr)
    np.testing.assert_array_equal(s._col, col)
    if w is None:
        assert s._w is None
    else:
        np.testing.assert_array_equal(s._w, w[perm])


@pytest.mark.parametrize("range_bytes", [1 << 30, 30000])
def test_host_csr(fake, range_bytes):
    tfg, calls, registered = fake
    from tf_geometric_b200.utils import sampling
    ei, w = _graph()
    device_bytes = range_bytes + 8 * 352 + 8 * (ei.shape[1] // 1024 + 1) + sampling.HOST_CSR_FIXED_BYTES
    s = tfg.utils.HostNeighborSampler(ei, w, device_bytes=device_bytes)
    assert (s.num_nodes, s.num_row_nodes, s.num_edges) == (351, 300, ei.shape[1])
    _check_csr(s, ei, w)
    n_ranges = sum(1 for c in calls if c[0] == "range")
    assert (n_ranges == 1) == (range_bytes == 1 << 30) and n_ranges >= 1
    assert len(s._ranges) >= n_ranges                    # ranges without edges launch nothing
    s.close()


def test_conversions(fake):
    tfg, calls, registered = fake
    ei, w = _graph()
    HNS = tfg.utils.HostNeighborSampler
    for arg, warg in ((ei.astype(np.int64), w.astype(np.float64)), (torch.from_numpy(ei), torch.from_numpy(w)),
                      (np.asfortranarray(ei), w[:, None]), (ei.astype(np.uint16), torch.from_numpy(w).double()),
                      (ei, np.arange(ei.shape[1]) % 3)):
        with HNS(arg, warg, device_bytes=1 << 30) as s:
            _check_csr(s, ei, np.asarray(warg, np.float32).reshape(-1))
    with HNS(ei, device_bytes=1 << 30) as s:
        _check_csr(s, ei, None)
    assert registered == {}


def test_refusals_before_any_work(fake):
    tfg, calls, registered = fake
    HNS = tfg.utils.HostNeighborSampler
    ei, w = _graph()

    class OnDevice(torch.Tensor):                        # a CPU stand-in for a CUDA tensor
        @property
        def is_cuda(self):
            return True
    for args, err, words in [((ei.astype(np.float32),), TypeError, "integer"), ((ei.astype(bool),), TypeError, "integer"),
                             ((torch.from_numpy(ei).as_subclass(OnDevice),), TypeError, "RandomNeighborSampler"),
                             ((ei.tolist(),), TypeError, "numpy"), ((ei[0],), ValueError, "dimension"),
                             ((ei[:1],), ValueError, "2, E"), ((-ei.astype(np.int64),), ValueError, "negative"),
                             ((ei.astype(np.int64) << 31,), ValueError, "2\\^31"),
                             ((ei, w[1:]), ValueError, "entries"),
                             ((ei, torch.from_numpy(w).requires_grad_()), ValueError, "grad"),
                             ((ei, w.astype(np.complex64)), TypeError, "floating")]:
        with pytest.raises(err, match=words):
            HNS(*args, device_bytes=1 << 30)
    assert calls == [] and registered == {}
    for bad, words in ((0, 1), (1, 5)):                  # negative ids found by the device pass: released again
        b = ei.copy()
        b[bad, words] = -2
        with pytest.raises(ValueError, match="negative"):
            HNS(b, w, device_bytes=1 << 30)
    with pytest.raises(ValueError, match="row 7 has 4[0-9][0-9] edges"):
        HNS(ei, device_bytes=29 * 300 + 8 * 352 + 8 * 3 + (1 << 20))
    assert registered == {}
    assert [c[0] for c in calls].count("register") == [c[0] for c in calls].count("unregister")


def test_registrations_and_lifetimes(fake, monkeypatch):
    tfg, calls, registered = fake
    from tf_geometric_b200.utils import sampling
    ei, w = _graph()
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    table = tfg.utils.HostFeatureTable(x)
    assert list(registered) == [x.data_ptr()]
    s = tfg.utils.HostNeighborSampler(ei, w, device_bytes=1 << 30)
    # the edge list and weights were copied (small arrays), registered for the build and released; the CSR's two
    # arrays stay registered, each on pages of its own
    assert len(registered) == 3 and x.data_ptr() in registered
    assert all(base % 4096 == 0 for base in registered if base != x.data_ptr())
    assert s._col.ctypes.data in registered and s._w.ctypes.data in registered
    assert [c[0] for c in calls].count("register") == 5 and [c[0] for c in calls].count("unregister") == 2
    b = s.sample_blocks([7, 0, 299, 3], [4, 3], seed=2)
    with pytest.raises(ValueError, match="duplicate"):
        s.sample_blocks([4, 9, 4], [3])
    with pytest.raises(ValueError, match="outside"):
        s.sample_blocks([4, 351], [3])
    rows = b.source_rows(table)                          # the batch's ids were checked by the sampler
    np.testing.assert_array_equal(rows.numpy(), x.numpy()[b.node_index.numpy()])
    s.close()
    assert list(registered) == [x.data_ptr()]
    s.close()
    with pytest.raises(RuntimeError, match="closed"):
        s.sample_blocks([1], [2])
    assert b.blocks[0].edge_index.shape[1] > 0           # batches outlive the sampler
    table.close()
    # an int32 array of HOST_IN_PLACE_BYTES or more is read in place
    monkeypatch.setattr(sampling, "HOST_IN_PLACE_BYTES", ei.nbytes)
    with tfg.utils.HostNeighborSampler(ei, device_bytes=1 << 30) as s2:
        assert ("register", ei.ctypes.data, ei.nbytes) in calls and ei.ctypes.data not in registered
        _check_csr(s2, ei, None)
    s3 = tfg.utils.HostNeighborSampler(ei, device_bytes=1 << 30)
    del s3                                               # collected without close(): released
    assert registered == {}


@pytest.mark.parametrize("fanouts,padding", [([5, 3], False), ([2, 4, 3], True), ([4], "head"), ([], False)])
def test_blocks_through_the_shared_helper(fake, monkeypatch, fanouts, padding):
    tfg, calls, _ = fake
    from tf_geometric_b200.utils import sampling
    ei, w = _graph()
    used = []
    helper = sampling._sample_blocks

    def spy(*args):
        used.append(args[2])
        return helper(*args)
    monkeypatch.setattr(sampling, "_sample_blocks", spy)
    seeds = np.array([7, 0, 299, 350, 3, 150], np.int32)
    want = tfg.utils.RandomNeighborSampler(ei, w).sample_blocks(seeds, fanouts, padding=padding, seed=11)
    with tfg.utils.HostNeighborSampler(ei, w, device_bytes=1 << 30) as s:
        got = s.sample_blocks(seeds, fanouts, padding=padding, seed=11)
    assert used == [351, 351]                            # both samplers, with the node count of their graph
    assert any(c[0] == "block_sample_mapped" for c in calls)
    np.testing.assert_array_equal(got.node_index.numpy(), want.node_index.numpy())
    assert got.hop_sizes == want.hop_sizes and got.num_nodes == want.num_nodes == 351
    for x, y in zip(got.blocks, want.blocks):
        assert (x.num_src, x.num_dst) == (y.num_src, y.num_dst)
        for a, b in ((x.edge_index, y.edge_index), (x.edge_weight, y.edge_weight), (x.global_col, y.global_col),
                     (x.csr.rowptr, y.csr.rowptr), (x.csr.col, y.csr.col), (x.csr.perm, y.csr.perm)):
            np.testing.assert_array_equal(a.numpy(), b.numpy())
