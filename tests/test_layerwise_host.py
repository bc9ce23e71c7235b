# coding=utf-8
"""Layer-wise inference without a GPU: the ABI declarations and argument checks of the row-block entry and the bulk copy,
row_block of both samplers over the numpy fake of tests/layerwise_fake_backend.py against sample_blocks(arange, [None])
and a row-by-row restatement (empty ranges, isolated rows, 0 and 1 output rows, a hub row, first-occurrence order), the
chunk cutter and byte counts, the layer-to-block routing, output placement by budget, and the refusals."""
import ctypes

import numpy as np
import pytest
import torch

import layerwise_fake_backend as fake_lw
from conftest import random_graph
from fake_backend import _np

ENTRIES = {"tfgk_row_block_i32": 15, "tfgk_copy_async": 4}


def _graph():
    """A hub row of 600 edges, 20 isolated rows, duplicate edges, self loops and a column id past the last row."""
    ei = random_graph(400, 3000, seed=5, isolated=20, hub=(30, 600))
    ei = np.concatenate([ei, ei[:, :100], [[3, 40, 41], [450, 40, 41]]], axis=1).astype(np.int32)
    w = np.random.RandomState(6).rand(ei.shape[1]).astype(np.float32)
    return ei, w


@pytest.fixture
def fake(monkeypatch):
    calls, _ = fake_lw.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg, calls


def test_entries_are_declared_and_refuse_capture():
    from tf_geometric_b200 import _ffi
    lib = _ffi.lib()
    for name, n in ENTRIES.items():
        assert len(_ffi.SIGNATURES[name]) == n and hasattr(lib, name), name
    assert "tfgk_row_block_i32" in _ffi.NOT_CAPTURABLE             # it reads the source-row count back
    assert "tfgk_copy_async" not in _ffi.NOT_CAPTURABLE


def test_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    n = ctypes.c_int32()
    rb = ("tfgk_row_block_i32",)
    cases = [
        (rb + ((None, 10, 5, 4, None, 0, None, None, None, None, None, ctypes.byref(n), None, 0, None),), "bad range"),
        (rb + ((None, 10, -1, 4, None, 0, None, None, None, None, None, ctypes.byref(n), None, 0, None),), "bad range"),
        (rb + ((None, 10, 0, 11, None, 0, None, None, None, None, None, ctypes.byref(n), None, 0, None),), "bad range"),
        (rb + ((None, 10, 0, 4, None, 1 << 31, None, None, None, None, None, ctypes.byref(n), None, 0, None),), "2^31"),
        (rb + ((None, 10, 4, 4, None, 3, None, None, None, None, None, ctypes.byref(n), None, 0, None),), "no rows"),
        (rb + ((None, 10, 0, 4, None, 3, None, None, None, None, None, None, None, 0, None),), "null"),
        (rb + ((ctypes.c_void_p(8), 10, 0, 4, None, 3, None, None, ctypes.c_void_p(8), None, None, ctypes.byref(n), None,
                0, None),), "null"),
        (("tfgk_copy_async", (None, ctypes.c_void_p(8), 4, None)), "null"),
    ]
    for (name, args), words in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(name, *args)
        assert err.value.code == _ffi.ERR_INVALID_ARGUMENT, name
        assert words in str(err.value), (name, str(err.value))
    _ffi.call("tfgk_copy_async", None, None, 0, None)                  # nothing to copy


def test_restatement_orders_by_first_occurrence():
    rowptr = np.array([0, 3, 3, 6, 6], np.int64)
    col = np.array([7, 2, 7, 5, 1, 9], np.int32)
    nodes, out_rowptr, out_row, local = fake_lw.restate_row_block(rowptr, col[3:6], 2, 4)
    assert nodes.tolist() == [2, 3, 5, 1, 9]
    assert out_rowptr.tolist() == [0, 3, 3] and out_row.tolist() == [0, 0, 0] and local.tolist() == [2, 3, 4]
    nodes, _, out_row, local = fake_lw.restate_row_block(rowptr, col[0:6], 0, 4)
    assert nodes.tolist() == [0, 1, 2, 3, 7, 5, 9] and local.tolist() == [4, 2, 4, 5, 1, 6]
    assert out_row.tolist() == [0, 0, 0, 2, 2, 2]


def _device_calls(calls):
    return [c[0] for c in calls if c[0] in ("row_block", "copy_async")]


def _assert_same_batch(a, b):
    assert np.array_equal(_np(a.node_index), _np(b.node_index))
    assert a.hop_sizes == b.hop_sizes and a.num_nodes == b.num_nodes and len(a.blocks) == len(b.blocks) == 1
    x, y = a.blocks[0], b.blocks[0]
    assert (x.num_src, x.num_dst, x.fanout) == (y.num_src, y.num_dst, y.fanout)
    for name in ("edge_index", "global_col", "dst_ids"):
        assert np.array_equal(_np(getattr(x, name)), _np(getattr(y, name))), name
    assert np.array_equal(_np(x.edge_weight).view(np.int32), _np(y.edge_weight).view(np.int32))
    for name in ("rowptr", "col", "perm"):
        assert np.array_equal(_np(getattr(x.csr, name)), _np(getattr(y.csr, name))), name
    assert x.degrees() is not None and y.degrees is not None


def _ranges(deg):
    hub = int(np.argmax(deg))
    iso = np.flatnonzero(deg == 0)
    N = deg.size
    return [(0, 0), (N, N), (0, 1), (hub, hub + 1), (hub - 3, hub + 4), (int(iso[0]), int(iso[0]) + 3), (0, N),
            (N - 7, N), (5, 6), (17, 120)]


@pytest.mark.parametrize("weighted", [True, False])
def test_host_row_block_matches_sample_blocks(fake, weighted):
    tfg, calls = fake
    ei, w = _graph()
    with tfg.utils.HostNeighborSampler(ei, w if weighted else None, device_bytes=1 << 30) as s:
        rp = s._host_rowptr()
        assert rp.size == s.num_nodes + 1 == 452
        deg = np.diff(rp)
        assert deg[:3].sum() == 0 and deg[400:].sum() == 0            # isolated rows, and ids past the last row
        for r0, r1 in _ranges(deg):
            del calls[:]
            got = s.row_block(r0, r1)
            assert _device_calls(calls) == ["copy_async"] * (2 if weighted and rp[r1] > rp[r0] else
                                                             1 if rp[r1] > rp[r0] else 0) + ["row_block"]
            _assert_same_batch(got, s.sample_blocks(np.arange(r0, r1, dtype=np.int32), [None]))
            nodes, out_rowptr, out_row, local = fake_lw.restate_row_block(rp, s._col[rp[r0]:rp[r1]], r0, r1)
            blk = got.blocks[0]
            assert np.array_equal(_np(got.node_index), nodes) and got.hop_sizes == [r1 - r0, nodes.size]
            assert np.array_equal(_np(blk.csr.rowptr), out_rowptr)
            assert np.array_equal(_np(blk.edge_index), np.stack([out_row, local]))
            want_w = s._w[rp[r0]:rp[r1]] if weighted else np.ones(rp[r1] - rp[r0], np.float32)
            assert np.array_equal(_np(blk.edge_weight), want_w)


def test_device_sampler_row_block_matches_sample_blocks(fake):
    tfg, calls = fake
    ei, w = _graph()
    s = tfg.utils.RandomNeighborSampler(torch.from_numpy(ei), torch.from_numpy(w))
    rp = s._host_rowptr()
    for r0, r1 in _ranges(np.diff(rp)):
        del calls[:]
        got = s.row_block(r0, r1)
        assert _device_calls(calls) == ["row_block"]                    # columns read in place: no copy
        _assert_same_batch(got, s.sample_blocks(np.arange(r0, r1, dtype=np.int32), [None]))


def test_row_block_refusals(fake):
    tfg, calls = fake
    from tf_geometric_b200.utils import sampling
    ei, w = _graph()
    s = tfg.utils.HostNeighborSampler(ei, w, device_bytes=1 << 30)
    N = s.num_nodes
    del calls[:]
    for r0, r1 in ((-1, 3), (0, N + 1), (5, 4)):
        with pytest.raises(ValueError, match="0 <= r0 <= r1"):
            s.row_block(r0, r1)
    with pytest.raises(TypeError):
        s.row_block(0.0, 3)
    assert _device_calls(calls) == []                                                   # refused before any device work
    rp = np.array([0, 5, (1 << 31) + 5, (1 << 31) + 6], np.int64)
    with pytest.raises(ValueError, match=r"rows \[0, 2\) hold 2147483653 edges"):
        sampling._row_range(rp, 0, 2)
    s.close()
    with pytest.raises(RuntimeError, match="closed"):
        s.row_block(0, 3)
    assert _device_calls(calls) == []


def test_row_range_past_2_31_is_refused():
    from tf_geometric_b200.utils import sampling
    rp = np.array([0, 5, (1 << 31) + 3, (1 << 31) + 6], np.int64)
    assert sampling._row_range(rp, 1, 2) == (1, 2, 5, (1 << 31) + 3)   # 2^31 - 2 edges
    assert sampling._row_range(rp, 2, 3) == (2, 3, (1 << 31) + 3, (1 << 31) + 6)   # an int64 start
    with pytest.raises(ValueError, match=r"rows \[1, 3\) hold 2147483649 edges; a row block takes fewer than 2\^31 - 1"):
        sampling._row_range(rp, 1, 3)
    rp = np.array([0, 5, (1 << 31) + 4], np.int64)                    # exactly 2^31 - 1 edges: refused
    with pytest.raises(ValueError, match="2147483647 edges"):
        sampling._row_range(rp, 1, 2)


def test_chunks_cover_the_rows_once():
    from tf_geometric_b200.utils import sampling
    import tf_geometric_b200 as tfg
    ei, _ = _graph()
    rp = np.concatenate([[0], np.cumsum(np.bincount(ei[0], minlength=452))]).astype(np.int64)
    layer = tfg.layers.GAT(16, num_heads=4)
    eb, rb, D = sampling.layerwise_chunk_bytes(layer, 32)
    assert D == 16
    for budget in (eb * 700 + rb * 3, eb * 2000 + rb * 100, eb * rp[-1] + rb * 1000):
        ranges = sampling._row_ranges(rp, budget, eb, rb)
        assert ranges[0][0] == 0 and ranges[-1][1] == 452
        assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:])) and all(r0 < r1 for r0, r1 in ranges)
        assert all(eb * (rp[r1] - rp[r0]) + rb * (r1 - r0 + 1) <= budget for r0, r1 in ranges)
    with pytest.raises(ValueError, match="row 30 has 6"):
        sampling._row_ranges(rp, eb * 500, eb, rb)                       # the hub alone needs more
    big = np.array([0, 1 << 30, (1 << 31) - 2, (3 << 30)], np.int64)
    assert all(big[r1] - big[r0] < 1 << 31 for r0, r1 in sampling._row_ranges(big, 1 << 40, 1, 0))
    from tf_geometric_b200.utils import layerwise
    exact = np.array([0, 1 << 30, (1 << 31) - 1, (3 << 30)], np.int64)  # rows 0-1 hold exactly 2^31 - 1 edges
    ranges, _ = layerwise._plan_layer(exact, 1 << 45, 1, 0, 0)
    assert ranges[0] == (0, 1) and ranges[-1][1] == 3
    assert all(exact[r1] - exact[r0] < (1 << 31) - 1 for r0, r1 in ranges)


def test_byte_counts_follow_the_widths():
    import tf_geometric_b200 as tfg
    from tf_geometric_b200.utils import sampling as s
    F = 100
    sage = s.layerwise_chunk_bytes(tfg.layers.MeanGraphSage(256), F)
    assert sage == (s.ROW_BLOCK_EDGE_BYTES + 4 * F, s.ROW_BLOCK_ROW_BYTES + 4 * (3 * F + 2 * 256 + 2 * 256), 256)
    assert s.layerwise_chunk_bytes(tfg.layers.SumGraphSage(256), F) == sage
    gcn = s.layerwise_chunk_bytes(tfg.layers.GCN(256), F)
    assert gcn[0] == s.ROW_BLOCK_EDGE_BYTES + s.LOOPED_EDGE_BYTES + s.GCN_VALUE_BYTES + 4 * (F + 256)
    assert gcn[2] == 256 and s.layerwise_chunk_bytes(tfg.layers.GCN(256, use_kernel=False), F)[2] == F
    gat = s.layerwise_chunk_bytes(tfg.layers.GAT(128, num_heads=4), F)
    assert gat[0] == s.ROW_BLOCK_EDGE_BYTES + s.LOOPED_EDGE_BYTES + 4 * (F + 3 * 128) and gat[2] == 128
    assert s.layerwise_chunk_bytes(tfg.layers.GAT(64, num_heads=4, split_value_heads=False), F)[0] == \
        s.ROW_BLOCK_EDGE_BYTES + s.LOOPED_EDGE_BYTES + 4 * (F + 2 * 64 + 256)
    pool = s.layerwise_chunk_bytes(tfg.layers.MaxPoolGraphSage(64), F)
    assert pool[0] == s.ROW_BLOCK_EDGE_BYTES + 4 * (F + 4 * 32) and pool[2] == 64
    assert s.layerwise_chunk_bytes(tfg.layers.MeanPoolGraphSage(64), F) == pool
    with pytest.raises(TypeError, match="GCN, GAT, MeanGraphSage, SumGraphSage, MeanPoolGraphSage"):
        s.layerwise_chunk_bytes(tfg.layers.GCNGraphSage(64), F)


def test_routing():
    import tf_geometric_b200 as tfg
    from tf_geometric_b200.utils import layerwise

    class FakeBlock(object):
        def with_self_loops(self):
            return "looped"

        def with_gcn_norm(self):
            return "gcn"
    b = FakeBlock()
    assert layerwise._adapt(tfg.layers.GAT(8), b) == "looped"
    assert layerwise._adapt(tfg.layers.GCN(8), b) == "gcn"
    for layer in (tfg.layers.MeanGraphSage(8), tfg.layers.SumGraphSage(8), tfg.layers.MeanPoolGraphSage(8),
                  tfg.layers.MaxPoolGraphSage(8)):
        assert layerwise._adapt(layer, b) is b


def test_output_placement_by_budget():
    from tf_geometric_b200.utils import layerwise, sampling
    rp = np.arange(0, 1001 * 10, 10, dtype=np.int64)              # 1 000 rows of 10 edges
    eb, rb, out = 100, 50, 1 << 20
    fixed = sampling.LAYERWISE_FIXED_BYTES
    ranges, on_device = layerwise._plan_layer(rp, fixed + out + eb * 10_000 + rb * 1001, eb, rb, out)
    assert on_device and ranges == [(0, 1000)]
    ranges, on_device = layerwise._plan_layer(rp, fixed + out + eb * 1000 + rb * 101, eb, rb, out)
    assert on_device and len(ranges) == 10
    ranges, on_device = layerwise._plan_layer(rp, fixed + out // 2, eb, rb, out)     # the output does not fit: host
    assert not on_device and ranges[0][0] == 0 and ranges[-1][1] == 1000
    with pytest.raises(ValueError, match="row 0 has 10 edges"):
        layerwise._plan_layer(rp, fixed + eb * 5, eb, rb, out)


def test_layerwise_refusals(fake):
    tfg, calls = fake
    ei, w = _graph()
    s = tfg.utils.HostNeighborSampler(ei, w, device_bytes=1 << 30)
    x = torch.zeros((452, 8))
    del calls[:]
    with pytest.raises(TypeError, match="GCN, GAT, MeanGraphSage"):
        tfg.utils.layerwise_inference(s, x, [tfg.layers.MeanGraphSage(8), tfg.layers.GIN(8)])
    with pytest.raises(TypeError, match="RandomNeighborSampler or a HostNeighborSampler"):
        tfg.utils.layerwise_inference(object(), x, [tfg.layers.MeanGraphSage(8)])
    with pytest.raises(ValueError, match="at least one layer"):
        tfg.utils.layerwise_inference(s, x, [])
    s.close()
    with pytest.raises(RuntimeError, match="closed"):
        tfg.utils.layerwise_inference(s, x, [tfg.layers.MeanGraphSage(8)])
    assert _device_calls(calls) == []
