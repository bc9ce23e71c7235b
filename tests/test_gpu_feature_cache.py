# coding=utf-8
"""Device rows of a host feature table on the device: HostFeatureTable(x, device_rows=...) gathers bit for bit equal to
x[index] across widths, cached fractions, strides, pinned and numpy tables and both kernels of
tfgk_gather_rows_cached_f32; the NaN guard of the raw entry; source_rows of a cached table without a host
synchronisation; hits read from the cache (overwritten with sentinels); a gather on a fresh stream right after
construction; the gather captured in a CUDA graph; a side-stream gather with the table dropped under it; GraphSAGE
and GAT training from a partly cached table bit for bit against source_rows(x_dev), over both samplers; and
rank_source_rows against its numpy restatement over real batches."""
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


def _rows(n, fraction, seed):
    """A random choice of round(fraction * n) distinct rows, unsorted."""
    return np.random.RandomState(seed).permutation(n)[:int(round(fraction * n))]


def _kernel_calls(fn):
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    try:
        result = fn()
    finally:
        _ffi.set_trace(prev)
    return result, trace.counts


@pytest.mark.parametrize("F", [1, 3, 4, 47, 100, 128, 256, 600])
@pytest.mark.parametrize("fraction", [0.0, "one", 1 / 3, 1.0])
def test_gather_is_bit_exact(F, fraction):
    n = 1000
    x = _table(n, F, F)
    rows = np.array([417]) if fraction == "one" else _rows(n, fraction, F + 2)
    ids = _ids(n, 3000, F + 1)
    with HFT(x, device_rows=rows) as t:
        assert t.device_bytes == (rows.size * F * 4 + n * 4 if rows.size else 0)
        got, counts = _kernel_calls(lambda: t.gather(ids.cuda()))
        assert counts.get("tfgk_gather_rows_cached_f32", 0) == (1 if rows.size else 0)
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
    with HFT(view, device_rows=_rows(700, 0.5, 7)) as t:
        assert torch.equal(t.gather(ids).cpu(), view[ids.long()])


def test_pinned_and_numpy_tables():
    x = _table(500, 100, 7).pin_memory()
    ids = _ids(500, 1500, 8)
    with HFT(x, device_rows=torch.from_numpy(_rows(500, 0.2, 9)).cuda()) as t:
        assert sampling._host_registered == {}           # pinned memory is read as it is
        assert torch.equal(t.gather(ids).cpu(), x[ids.long()])
    a = np.random.RandomState(9).randn(400, 36).astype(np.float32)
    with HFT(a, device_rows=_rows(400, 0.3, 1)) as t, HFT(a[:, 1:30], device_rows=_rows(400, 0.6, 2)) as t2:
        assert len(sampling._host_registered) == 1       # two views, two caches: one registration
        idx = np.random.RandomState(10).randint(0, 400, 1200)
        np.testing.assert_array_equal(t.gather(idx).cpu().numpy(), a[idx])
        np.testing.assert_array_equal(t2.gather(idx).cpu().numpy(), a[idx, 1:30])


@pytest.mark.parametrize("F", [100, 3])
def test_guard_writes_nan(F):
    """Ids outside [0, n_rows) give NaN rows and read neither the map nor a table: the table covers rows [8, N + 8) of
    a registered buffer of N + 16 finite rows, so a broken guard would read finite padding, not fault."""
    N = 64
    buf = _table(N + 16, F, 11)
    with HFT(buf) as whole, HFT(buf[8:N + 8], device_rows=[0, 13, N - 1]) as t:
        ids = torch.tensor([N, N + 7, -1, 0, N - 1, 5], dtype=torch.int32, device="cuda")
        out = torch.zeros((6, F), device="cuda")
        _ffi.call("tfgk_gather_rows_cached_f32", ctypes.c_void_p(t._ptr), t._ld, N, F,
                  ctypes.c_void_p(t._cache.data_ptr()), F, ctypes.c_void_p(t._slot.data_ptr()),
                  ctypes.c_void_p(ids.data_ptr()), 6, ctypes.c_void_p(out.data_ptr()), F,
                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        got = out.cpu()
        assert torch.isnan(got[:3]).all()
        assert torch.equal(got[3:], buf[[8, N + 7, 13]])
        for bad in ([N], [-1]):
            with pytest.raises(IndexError, match="outside"):
                t.gather(torch.tensor(bad, dtype=torch.int32, device="cuda"))


def test_refusals():
    x = _table(100, 8, 3)
    for bad, err in (([100], IndexError), ([-1], IndexError), ([4, 4], ValueError), (np.array([1.5]), TypeError)):
        with pytest.raises(err):
            HFT(x, device_rows=bad)
    with pytest.raises(ValueError):
        HFT(x, device_rows=torch.tensor([7, 9, 7], device="cuda"))


def _graph():
    # every node has in-edges, so no max-pool row is empty (-FLT_MAX) and the gradients stay finite
    return random_graph(3000, 30000, seed=41, hub=(9, 3000)).astype(np.int32)


@pytest.fixture(scope="module")
def sampler():
    return tfg.utils.RandomNeighborSampler(ops.as_device(_graph(), torch.int32))


def test_source_rows_without_synchronisation(sampler):
    x = _table(3000, 100, 13)
    x_dev = x.cuda()
    seeds = np.random.RandomState(14).permutation(3000)[:256].astype(np.int32)
    b = sampler.sample_blocks(seeds, [15, 10, 5], seed=3)
    with HFT(x, device_rows=b.node_index[::3].clone()) as t:
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            rows, counts = _kernel_calls(lambda: b.source_rows(t))
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert counts == {"tfgk_gather_rows_cached_f32": 1}
        assert torch.equal(rows, x_dev[b.node_index.long()])


def test_gather_in_a_cuda_graph():
    n, F = 2000, 100
    x = _table(n, F, 21)
    with HFT(x, device_rows=_rows(n, 0.25, 22)) as t:
        static = _ids(n, 4000, 23).cuda()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            t._gather(static)                            # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = t._gather(static)
        for seed in (24, 25):
            fresh = _ids(n, 4000, seed)
            static.copy_(fresh.cuda())
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out.cpu(), x[fresh.long()])
        del graph


def test_gather_on_a_fresh_stream_right_after_construction():
    """The constructor returns with the cache and the map in place: a stream that never waited on the one that filled
    them reads them at once.  The fill crosses the link (about 50 MB), so it would still be pending otherwise."""
    n, F = 200000, 128
    x = _table(n, F, 35)
    idx = _ids(n, 100000, 36).cuda()
    torch.cuda.synchronize()
    with HFT(x, device_rows=_rows(n, 0.5, 37)) as t:
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            rows = t._gather(idx)
        side.synchronize()
        assert torch.equal(rows.cpu(), x[idx.long().cpu()])


def test_side_stream_gather_then_drop_the_table():
    n, F = 20000, 128
    x = _table(n, F, 31)
    ids = _ids(n, 60000, 32).cuda()
    torch.cuda.synchronize()
    keeper = HFT(x)                                      # holds the registration: dropping t unregisters nothing
    t = HFT(x, device_rows=_rows(n, 0.5, 33))
    side, main = torch.cuda.Stream(), torch.cuda.current_stream()
    with torch.cuda.stream(side):
        rows = t._gather(ids)
    del t                                                # cache and map freed while the gather may be pending
    junk = [torch.full((n // 2, F), -1.0, device="cuda") for _ in range(4)]   # would reuse the cache's memory
    main.wait_stream(side)
    rows.record_stream(main)
    assert torch.equal(rows.cpu(), x[ids.long().cpu()])
    del junk
    keeper.close()


@pytest.mark.parametrize("F", [100, 3])
def test_hits_are_read_from_the_cache(F):
    """With the cache overwritten by sentinels, hit rows return the sentinels and miss rows x: the slot map is used."""
    n = 3000
    x = _table(n, F, 41)
    ids = _ids(n, 5000, 42)
    with HFT(x, device_rows=_rows(n, 0.4, 43)) as t:
        C = t._cache.shape[0]
        t._cache.copy_(-torch.arange(1, C + 1, dtype=torch.float32, device="cuda")[:, None].expand(C, F))
        got = t.gather(ids.cuda()).cpu()
        slot = t._slot.cpu()[ids.long()]
        hit = slot >= 0
        assert 0 < int(hit.sum()) < ids.numel()
        assert torch.equal(got[hit], -(slot[hit] + 1).float()[:, None].expand(-1, F))
        assert torch.equal(got[~hit], x[ids[~hit].long()])


KINDS = ["MeanGraphSage", "MaxPoolGraphSage", "GAT"]


def _layers(kind, depth):
    if kind == "GAT":
        return [tfg.layers.GAT(64, num_heads=4, activation=tfg.nn.relu, seed=i + 1, trainable=True)
                for i in range(depth - 1)] + [tfg.layers.GAT(16, num_heads=1, seed=depth, trainable=True)]
    units = [64] * (depth - 1) + [16]
    return [getattr(tfg.layers, kind)(u, seed=i + 1, trainable=True) for i, u in enumerate(units)]


def _run(kind, layers, blocks, h):
    for layer, blk in zip(layers, blocks):
        h = layer([h, blk.with_self_loops() if kind == "GAT" else blk], training=True)
    h.square().sum().backward()
    grads = [p.grad.clone() for layer in layers for p in layer.parameters()]
    for layer in layers:
        layer.zero_grad()
    return [h.detach()] + grads


def _same_bits(a, b):
    return all(torch.equal(u.view(torch.int32), v.view(torch.int32)) for u, v in zip(a, b))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fanouts", [[10, 5], [15, 10, 5]])
def test_training_from_a_partly_cached_table(sampler, kind, fanouts):
    ei = _graph()
    x = _table(3000, 100, 15)
    x_dev = x.cuda()
    layers = _layers(kind, len(fanouts))
    seeds = np.random.RandomState(16).permutation(3000)[:200].astype(np.int32)
    b = sampler.sample_blocks(seeds, fanouts, seed=5)
    want = _run(kind, layers, b.blocks, b.source_rows(x_dev))
    assert all(bool(torch.isfinite(t).all()) for t in want)
    warm = [sampler.sample_blocks(np.random.RandomState(k).permutation(3000)[:200].astype(np.int32), fanouts,
                                  seed=100 + k) for k in range(4)]
    ids, _ = tfg.utils.rank_source_rows(warm)
    with HFT(x, device_rows=ids[:1000]) as t:
        assert torch.isin(b.node_index, t.device_rows).any() and not torch.isin(b.node_index, t.device_rows).all()
        assert _same_bits(_run(kind, layers, b.blocks, b.source_rows(t)), want)
        with tfg.utils.HostNeighborSampler(ei) as s:
            hb = s.sample_blocks(seeds, fanouts, seed=5)
            assert _same_bits(_run(kind, layers, hb.blocks, hb.source_rows(t)), want)


def _rank_ref(node_indices, num_nodes):
    counts = np.zeros(num_nodes, np.int64)
    for ni in node_indices:
        counts[np.unique(ni)] += 1
    order = np.lexsort((np.arange(num_nodes), -counts))
    return order[counts[order] > 0], counts


def test_rank_source_rows_over_real_batches(sampler):
    rs = np.random.RandomState(51)
    # 10 batches of at most 16 + 64 + 128 rows: some of the 3 000 rows are never read
    batches = [sampler.sample_blocks(rs.permutation(3000)[:16].astype(np.int32), [4, 2], seed=200 + k)
               for k in range(10)]
    ids, counts = tfg.utils.rank_source_rows(batches)
    want_ids, want_counts = _rank_ref([b.node_index.cpu().numpy() for b in batches], 3000)
    assert ids.is_cuda and counts.is_cuda and ids.dtype == counts.dtype == torch.int32
    np.testing.assert_array_equal(counts.cpu().numpy(), want_counts)
    np.testing.assert_array_equal(ids.cpu().numpy(), want_ids)
    assert 0 < ids.numel() < 3000 and (want_counts > 1).any()
    ids2, counts2 = tfg.utils.rank_source_rows(batches)
    assert torch.equal(ids, ids2) and torch.equal(counts, counts2)
    with tfg.utils.HostNeighborSampler(_graph()) as s:
        hb = [s.sample_blocks(rs.permutation(3000)[:64].astype(np.int32), [10, 5], seed=300 + k) for k in range(5)]
        ids, counts = tfg.utils.rank_source_rows(hb)
        want_ids, want_counts = _rank_ref([b.node_index.cpu().numpy() for b in hb], 3000)
        np.testing.assert_array_equal(counts.cpu().numpy(), want_counts)
        np.testing.assert_array_equal(ids.cpu().numpy(), want_ids)
