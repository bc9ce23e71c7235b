# coding=utf-8
"""Feature tables in host memory on the device: HostFeatureTable.gather bit for bit against x[index] across widths,
strides, pinned and numpy tables; the NaN guard of tfgk_gather_rows_mapped_f32 inside registered padding (a broken
guard would read finite padding, never memory outside the registration); registration and release;
SampledBlocks.source_rows over a host table without a host synchronisation; and GraphSAGE over blocks whose input came
from the host table, forward and weight gradients bit for bit against the same layers on x_dev[node_index], with the
gather on the current stream and on a side stream."""
import ctypes

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from tf_geometric_b200.utils import sampling
from conftest import random_graph

pytestmark = pytest.mark.gpu

HFT = tfg.utils.HostFeatureTable


@pytest.fixture(autouse=True)
def no_registration_left():
    yield
    assert sampling._host_registered == {}, "a test left host memory registered"


def _table(n, F, seed):
    return torch.from_numpy(np.random.RandomState(seed).randn(n, F).astype(np.float32))


def _ids(n, count, seed):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, n, count).astype(np.int32))   # repeats, unsorted


@pytest.mark.parametrize("F", [1, 3, 4, 47, 100, 128, 256, 600])
def test_gather_is_bit_exact(F):
    x = _table(1000, F, F)
    ids = _ids(1000, 3000, F + 1)
    with HFT(x) as t:
        got = t.gather(ids.cuda())
        assert got.is_cuda and got.is_contiguous() and got.shape == (3000, F)
        assert torch.equal(got.cpu(), x[ids.long()])
        empty = t.gather(torch.zeros(0, dtype=torch.int32, device="cuda"))
        assert empty.shape == (0, F) and empty.is_cuda
        out = torch.full((50, F + 5), 3.0, device="cuda")[:, 2:2 + F]        # an output with row stride > F
        assert t.gather(ids[:50].cuda(), out=out) is out
        assert torch.equal(out.cpu(), x[ids[:50].long()])


@pytest.mark.parametrize("first,F", [(3, 100), (4, 100), (0, 47), (8, 120)])
def test_column_slice_with_row_stride(first, F):
    big = _table(700, 128, 5)
    view = big[:, first:first + F]                       # row stride 128 > F; an odd offset or F take 4-byte accesses
    ids = _ids(700, 2000, 6)
    with HFT(view) as t:
        assert torch.equal(t.gather(ids).cpu(), view[ids.long()])


def test_pinned_and_numpy_tables():
    x = _table(500, 100, 7).pin_memory()
    ids = _ids(500, 1500, 8)
    with HFT(x) as t:
        assert sampling._host_registered == {}           # pinned memory is read as it is
        assert torch.equal(t.gather(ids).cpu(), x[ids.long()])
    a = np.random.RandomState(9).randn(400, 36).astype(np.float32)
    with HFT(a) as t, HFT(a[:, 1:30]) as t2:             # two views of one array: one registration
        assert len(sampling._host_registered) == 1
        idx = np.random.RandomState(10).randint(0, 400, 1200)
        np.testing.assert_array_equal(t.gather(idx).cpu().numpy(), a[idx])
        np.testing.assert_array_equal(t2.gather(idx).cpu().numpy(), a[idx, 1:30])


@pytest.mark.parametrize("F", [100, 3])
def test_guard_writes_nan_inside_registered_padding(F):
    """The table covers rows [8, N + 8) of a registered buffer of N + 16 finite rows, so ids N, N + 7 and -1 would land
    in registered padding if the guard were broken: finite values, not a fault."""
    N = 64
    buf = _table(N + 16, F, 11)
    with HFT(buf) as whole, HFT(buf[8:N + 8]) as t:
        assert len(sampling._host_registered) == 1
        ids = torch.tensor([N, N + 7, -1, 0, N - 1, 5], dtype=torch.int32, device="cuda")
        out = torch.zeros((6, F), device="cuda")
        _ffi.call("tfgk_gather_rows_mapped_f32", ctypes.c_void_p(t._ptr), t._ld, N, F, ctypes.c_void_p(ids.data_ptr()), 6,
                  ctypes.c_void_p(out.data_ptr()), F, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        got = out.cpu()
        assert torch.isnan(got[:3]).all()
        assert torch.equal(got[3:], buf[[8, N + 7, 13]])
        for bad in ([N], [N + 7], [-1], [0, N]):
            with pytest.raises(IndexError, match="outside"):
                t.gather(torch.tensor(bad, dtype=torch.int32, device="cuda"))
        assert torch.equal(whole.gather([N + 15]).cpu(), buf[[N + 15]])


def test_close_unregisters():
    x = _table(300, 20, 12)
    storage = x.untyped_storage()
    t = HFT(x)
    with pytest.raises(_ffi.TfgkError) as err:           # registered while the table is open
        ops.host_register(storage.data_ptr(), storage.nbytes())
    assert err.value.code == _ffi.ERR_CUDA
    assert torch.equal(t.gather([1, 2]).cpu(), x[[1, 2]])    # the failed call left no CUDA error behind
    t.close()
    t.close()
    with pytest.raises(RuntimeError, match="closed"):
        t.gather([1])
    assert ops.host_register(storage.data_ptr(), storage.nbytes())     # the range is free again
    ops.host_unregister(storage.data_ptr())
    with pytest.raises(TypeError, match="CUDA"):
        HFT(x.cuda())


def _graph():
    # every node has in-edges, so no max-pool row is empty (-FLT_MAX) and the gradients stay finite
    ei = random_graph(3000, 30000, seed=41, hub=(9, 3000)).astype(np.int32)
    return tfg.utils.RandomNeighborSampler(ops.as_device(ei, torch.int32))


@pytest.fixture(scope="module")
def sampler():
    return _graph()


def test_source_rows_without_synchronisation(sampler):
    x = _table(3000, 100, 13)
    x_dev = x.cuda()
    seeds = np.random.RandomState(14).permutation(3000)[:256].astype(np.int32)
    b = sampler.sample_blocks(seeds, [15, 10, 5], seed=3)
    assert b.num_nodes == 3000
    with HFT(x) as t:
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            rows = b.source_rows(t)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert torch.equal(rows, x_dev[b.node_index.long()])
        with HFT(x[:2999]) as short, pytest.raises(ValueError, match="rows"):
            b.source_rows(short)
        by_hand = tfg.utils.SampledBlocks(b.node_index, b.hop_sizes, b.blocks)
        assert torch.equal(by_hand.source_rows(t), rows)


KINDS = ["MeanGraphSage", "SumGraphSage", "MeanPoolGraphSage", "MaxPoolGraphSage"]


def _bits(t):
    return t.view(torch.int32)


def _same_bits(a, b):
    return all(torch.equal(_bits(u), _bits(v)) for u, v in zip(a, b))


def _run(layers, blocks, h):
    for layer, blk in zip(layers, blocks):
        h = layer([h, blk], training=True)
    h.square().sum().backward()
    grads = [p.grad.clone() for layer in layers for p in layer.parameters()]
    for layer in layers:
        layer.zero_grad()
    return h.detach(), grads


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fanouts", [[10, 5], [15, 10, 5]])
def test_layers_on_host_rows_match_device_rows(sampler, kind, fanouts):
    x = _table(3000, 100, 15)
    x_dev = x.cuda()
    units = [64] * (len(fanouts) - 1) + [16]
    layers = [getattr(tfg.layers, kind)(u, seed=i + 1, trainable=True) for i, u in enumerate(units)]
    seeds = np.random.RandomState(16).permutation(3000)[:200].astype(np.int32)
    b = sampler.sample_blocks(seeds, fanouts, seed=5)
    want_h, want_g = _run(layers, b.blocks, x_dev[b.node_index.long()])
    assert all(bool(torch.isfinite(t).all()) for t in [want_h] + want_g)
    with HFT(x) as t:
        got_h, got_g = _run(layers, b.blocks, b.source_rows(t))
        assert _same_bits([got_h] + got_g, [want_h] + want_g)
        # the prefetch recipe: gather on a side stream, then wait for it before layer 0
        side, main = torch.cuda.Stream(), torch.cuda.current_stream()
        with torch.cuda.stream(side):
            rows = b.source_rows(t)
        main.wait_stream(side)
        rows.record_stream(main)
        got_h, got_g = _run(layers, b.blocks, rows)
        assert _same_bits([got_h] + got_g, [want_h] + want_g)
