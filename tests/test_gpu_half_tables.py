# coding=utf-8
"""16-bit host feature tables on the device, for float16 and bfloat16: HostFeatureTable(x, dtype=...) gathers bit for
bit equal to x.float()[index] across widths, every load tier of tfgk_gather_rows_mapped_16 / _cached_16, repeated and
unsorted ids, empty and strided outputs; every 16-bit pattern widened exactly (NaN at the same positions) and copied
unchanged by the copy mode; the NaN guard inside registered padding; the device cache (0, 1, a third and all rows; hits
read from it; device_bytes); source_rows without a host synchronisation; the gather in a CUDA graph; a side-stream
gather with the table dropped under it; GraphSAGE, GAT and GCN training, a link batch's predict_edge and
layerwise_inference from 16-bit tables bit for bit against the same layers on the widened float32 x; and the refusals."""
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
DTYPES = [torch.float16, torch.bfloat16]
CODE = {torch.float16: _ffi.DTYPE_F16, torch.bfloat16: _ffi.DTYPE_BF16}
NAN16 = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0}
MAPPED16, CACHED16 = "tfgk_gather_rows_mapped_16", "tfgk_gather_rows_cached_16"


@pytest.fixture(autouse=True)
def no_registration_left():
    yield
    assert sampling._host_registered == {}, "a test left host memory registered"


def _table(n, F, seed, dtype):
    return torch.from_numpy(np.random.RandomState(seed).randn(n, F).astype(np.float32)).to(dtype)


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


def _same_bits(a, b):
    return torch.equal(a.cpu().view(torch.int32), b.cpu().view(torch.int32))


def _same_nan_bits(got, want):
    """bit for bit where want is a number, NaN where it is NaN (the widening of a NaN keeps only its NaN-ness)"""
    got, want = got.cpu(), want.cpu()
    nan = want.isnan()
    return torch.equal(got.isnan(), nan) and torch.equal(got[~nan].view(torch.int32), want[~nan].view(torch.int32))


def _bits16(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("F", [1, 2, 3, 4, 7, 8, 47, 100, 128, 256, 600, 768])
def test_gather_is_bit_exact(dtype, F):
    x = _table(1000, F, F, dtype)
    ids = _ids(1000, 3000, F + 1)
    want = x.float()[ids.long()]
    with HFT(x, dtype=dtype) as t:
        got, counts = _kernel_calls(lambda: t.gather(ids.cuda()))
        assert counts == {MAPPED16: 1}
        assert got.is_cuda and got.is_contiguous() and got.dtype == torch.float32 and got.shape == (3000, F)
        assert _same_bits(got, want)
        empty = t.gather(torch.zeros(0, dtype=torch.int32, device="cuda"))
        assert empty.shape == (0, F) and empty.is_cuda and empty.dtype == torch.float32
        out = torch.full((50, F + 5), 3.0, device="cuda")[:, 2:2 + F]        # an output with row stride > F
        assert t.gather(ids[:50].cuda(), out=out) is out
        assert _same_bits(out, want[:50])


# (first column, F) of a [700, 136] table (272-byte rows, 64-byte aligned base), and the load the offset and width allow
TIERS = [pytest.param(0, 104, id="16B-F104"), pytest.param(0, 120, id="16B-F120"),
         pytest.param(4, 100, id="8B-off4"), pytest.param(0, 100, id="8B-F100"),
         pytest.param(2, 98, id="4B-off2"), pytest.param(0, 6, id="4B-F6"),
         pytest.param(1, 100, id="2B-off1"), pytest.param(0, 47, id="2B-F47")]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("first,F", TIERS)
def test_column_slices_reach_every_load_tier(dtype, first, F):
    big = _table(700, 136, 5, dtype)
    assert big.data_ptr() % 64 == 0
    view = big[:, first:first + F]                       # row stride 136 > F
    ids = _ids(700, 2000, 6)
    want = view.float()[ids.long()]
    with HFT(view, dtype=dtype) as t, HFT(view, dtype=dtype, device_rows=_rows(700, 0.5, 7)) as c:
        assert t._ld == 136
        assert _same_bits(t.gather(ids), want)
        assert _same_bits(c.gather(ids), want)
        out = torch.zeros((2000, F + 3), device="cuda")[:, 1:1 + F]          # a 4-byte aligned output: narrower stores
        assert _same_bits(c.gather(ids, out=out), want)
        assert _same_bits(t.gather(ids, out=out), want)


def _every_pattern(dtype, width):
    """All 65 536 16-bit patterns (±0, subnormals, the largest finite values, ±inf, quiet and signalling NaNs with
    payloads), shuffled into rows of `width`."""
    bits = np.random.RandomState(3).permutation(np.arange(65536, dtype=np.int64)).astype(np.uint16)
    return torch.from_numpy(bits.view(np.int16).reshape(-1, width)).view(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("width,first", [(16, 0), (16, 1), (8, 4), (4, 2)])
def test_every_bit_pattern_widens_exactly_and_copies_unchanged(dtype, width, first):
    whole = _every_pattern(dtype, width)
    x = whole[:, first:]
    n, F = x.shape
    info = torch.finfo(dtype)
    specials = torch.tensor([0.0, -0.0, info.tiny / 2, -info.tiny / 1024, info.max, -info.max, float("inf"),
                             -float("inf")], dtype=dtype)
    assert torch.isin(_bits16(specials), _bits16(whole)).all()
    ids = torch.from_numpy(np.random.RandomState(4).permutation(n).astype(np.int32)).cuda()
    with HFT(x, dtype=dtype) as t:
        got = t.gather(ids)
        assert _same_nan_bits(got, x.float()[ids.long().cpu()])
        copied = ops.gather_rows_mapped_16(t._ptr, dtype, t._ld, n, F, ids, out_dtype=dtype)
        assert copied.dtype == dtype
        assert torch.equal(_bits16(copied.cpu()), _bits16(x[ids.long().cpu()]))         # NaN payloads included
    with HFT(x, dtype=dtype, device_rows=_rows(n, 0.5, 5)) as c:
        assert torch.equal(_bits16(c._cache.cpu()), _bits16(x[c.device_rows.long().cpu()]))
        assert _same_nan_bits(c.gather(ids), x.float()[ids.long().cpu()])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("F", [100, 3])
def test_guard_writes_nan_inside_registered_padding(dtype, F):
    """The table covers rows [8, N + 8) of a registered buffer of N + 16 finite rows, so ids N, N + 7 and -1 would land
    in registered padding if the guard were broken: finite values, not a fault."""
    N = 64
    buf = _table(N + 16, F, 11, dtype)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    with HFT(buf, dtype=dtype) as whole, HFT(buf[8:N + 8], dtype=dtype) as t, \
            HFT(buf[8:N + 8], dtype=dtype, device_rows=[0, 13, N - 1]) as c:
        assert len(sampling._host_registered) == 1
        ids = torch.tensor([N, N + 7, -1, 0, N - 1, 5], dtype=torch.int32, device="cuda")
        want = buf.float()[[8, N + 7, 13]]
        out = torch.zeros((6, F), device="cuda")
        _ffi.call(MAPPED16, ctypes.c_void_p(t._ptr), CODE[dtype], t._ld, N, F, ctypes.c_void_p(ids.data_ptr()), 6,
                  ctypes.c_void_p(out.data_ptr()), _ffi.DTYPE_F32, F, stream)
        got = out.cpu()
        assert torch.isnan(got[:3]).all() and torch.equal(got[3:], want)
        out16 = torch.zeros((6, F), dtype=dtype, device="cuda")
        _ffi.call(MAPPED16, ctypes.c_void_p(t._ptr), CODE[dtype], t._ld, N, F, ctypes.c_void_p(ids.data_ptr()), 6,
                  ctypes.c_void_p(out16.data_ptr()), CODE[dtype], F, stream)
        got16 = _bits16(out16.cpu())
        assert (got16[:3] == NAN16[dtype]).all()
        assert torch.equal(got16[3:], _bits16(buf[[8, N + 7, 13]]))
        out.zero_()
        _ffi.call(CACHED16, ctypes.c_void_p(c._ptr), CODE[dtype], c._ld, N, F, ctypes.c_void_p(c._cache.data_ptr()), F,
                  ctypes.c_void_p(c._slot.data_ptr()), ctypes.c_void_p(ids.data_ptr()), 6,
                  ctypes.c_void_p(out.data_ptr()), F, stream)
        got = out.cpu()
        assert torch.isnan(got[:3]).all() and torch.equal(got[3:], want)
        for bad in ([N], [N + 7], [-1], [0, N]):
            with pytest.raises(IndexError, match="outside"):
                t.gather(torch.tensor(bad, dtype=torch.int32, device="cuda"))
        assert torch.equal(whole.gather([N + 15]).cpu(), buf.float()[[N + 15]])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("F", [1, 3, 8, 100, 104, 256])
@pytest.mark.parametrize("fraction", [0.0, "one", 1 / 3, 1.0])
def test_cached_gather_is_bit_exact(dtype, F, fraction):
    n = 1000
    x = _table(n, F, F, dtype)
    rows = np.array([417]) if fraction == "one" else _rows(n, fraction, F + 2)
    ids = _ids(n, 3000, F + 1)
    want = x.float()[ids.long()]
    with HFT(x, device_rows=rows, dtype=dtype) as t:
        assert t.dtype == dtype
        assert t.device_bytes == (rows.size * F * 2 + n * 4 if rows.size else 0)
        if rows.size:
            assert t._cache.dtype == dtype and torch.equal(_bits16(t._cache.cpu()), _bits16(x[rows]))
        got, counts = _kernel_calls(lambda: t.gather(ids.cuda()))
        assert counts == ({CACHED16: 1} if rows.size else {MAPPED16: 1})
        assert _same_bits(got, want)
        out = torch.full((50, F + 5), 3.0, device="cuda")[:, 2:2 + F]
        assert t.gather(ids[:50].cuda(), out=out) is out
        assert _same_bits(out, want[:50])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("F", [100, 3])
def test_hits_are_read_from_the_cache(dtype, F):
    """With the cache overwritten by other values, hit rows return those and miss rows x: the slot map is used."""
    n = 3000
    x = _table(n, F, 41, dtype)
    ids = _ids(n, 5000, 42)
    with HFT(x, device_rows=_rows(n, 0.4, 43), dtype=dtype) as t:
        C = t._cache.shape[0]
        t._cache.copy_((torch.randn(C, F, device="cuda") + 50.0).to(dtype))     # far from x's N(0, 1) values
        sentinel = t._cache.float().cpu()
        got = t.gather(ids.cuda()).cpu()
        slot = t._slot.cpu()[ids.long()]
        hit = slot >= 0
        assert 0 < int(hit.sum()) < ids.numel()
        assert _same_bits(got[hit], sentinel[slot[hit].long()])
        assert _same_bits(got[~hit], x.float()[ids[~hit].long()])


def _graph():
    # every node has in-edges, so no max-pool row is empty (-FLT_MAX) and the gradients stay finite
    return random_graph(3000, 30000, seed=41, hub=(9, 3000)).astype(np.int32)


@pytest.fixture(scope="module")
def sampler():
    return tfg.utils.RandomNeighborSampler(ops.as_device(_graph(), torch.int32))


@pytest.mark.parametrize("dtype", DTYPES)
def test_source_rows_without_synchronisation(sampler, dtype):
    x = _table(3000, 100, 13, dtype)
    x_dev = x.float().cuda()
    seeds = np.random.RandomState(14).permutation(3000)[:256].astype(np.int32)
    b = sampler.sample_blocks(seeds, [15, 10, 5], seed=3)
    with HFT(x, dtype=dtype) as t, HFT(x, dtype=dtype, device_rows=b.node_index[::3].clone()) as c:
        for table, entry in ((t, MAPPED16), (c, CACHED16)):
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                rows, counts = _kernel_calls(lambda: b.source_rows(table))
            finally:
                torch.cuda.set_sync_debug_mode("default")
            assert counts == {entry: 1}
            assert _same_bits(rows, x_dev[b.node_index.long()])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fraction", [0.0, 0.25])
def test_gather_in_a_cuda_graph(dtype, fraction):
    n, F = 2000, 100
    x = _table(n, F, 21, dtype)
    with HFT(x, device_rows=_rows(n, fraction, 22), dtype=dtype) as t:
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
            assert _same_bits(out, x.float()[fresh.long()])
        del graph


@pytest.mark.parametrize("dtype", DTYPES)
def test_side_stream_gather_then_drop_the_table(dtype):
    n, F = 20000, 128
    x = _table(n, F, 31, dtype)
    ids = _ids(n, 60000, 32).cuda()
    torch.cuda.synchronize()
    keeper = HFT(x, dtype=dtype)                         # holds the registration: dropping t unregisters nothing
    t = HFT(x, device_rows=_rows(n, 0.5, 33), dtype=dtype)
    side, main = torch.cuda.Stream(), torch.cuda.current_stream()
    with torch.cuda.stream(side):
        rows = t._gather(ids)
    del t                                                # cache and map freed while the gather may be pending
    junk = [torch.full((n // 2, F), -1.0, device="cuda", dtype=dtype) for _ in range(4)]   # would reuse the cache
    main.wait_stream(side)
    rows.record_stream(main)
    assert _same_bits(rows, x.float()[ids.long().cpu()])
    del junk
    keeper.close()


# ---- models -----------------------------------------------------------------------------------------------------

KINDS = ["MeanGraphSage", "MaxPoolGraphSage", "GAT", "GCN"]


def _layers(kind, depth):
    L = tfg.layers
    if kind == "GAT":
        return [L.GAT(64, num_heads=4, activation=tfg.nn.relu, seed=i + 1, trainable=True)
                for i in range(depth - 1)] + [L.GAT(16, num_heads=1, seed=depth, trainable=True)]
    units = [64] * (depth - 1) + [16]
    if kind == "GCN":
        return [L.GCN(u, activation=tfg.nn.relu if i + 1 < depth else None, seed=i + 1, trainable=True)
                for i, u in enumerate(units)]
    return [getattr(L, kind)(u, seed=i + 1, trainable=True) for i, u in enumerate(units)]


def _adapt(kind, blk):
    return blk.with_self_loops() if kind == "GAT" else blk.with_gcn_norm() if kind == "GCN" else blk


def _forward(kind, layers, blocks, h):
    for layer, blk in zip(layers, blocks):
        h = layer([h, _adapt(kind, blk)], training=True)
    return h


def _run(kind, layers, blocks, h):
    h = _forward(kind, layers, blocks, h)
    h.square().sum().backward()
    grads = [p.grad.clone() for layer in layers for p in layer.parameters()]
    for layer in layers:
        layer.zero_grad()
    return [h.detach()] + grads


def _all_same_bits(a, b):
    return len(a) == len(b) and all(_same_bits(u, v) for u, v in zip(a, b))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fanouts", [[10, 5], [15, 10, 5]])
def test_training_from_16_bit_tables(sampler, dtype, kind, fanouts):
    ei = _graph()
    x = _table(3000, 100, 15, dtype)
    x_dev = x.float().cuda()                             # the caller's widened copy: the reference
    layers = _layers(kind, len(fanouts))
    seeds = np.random.RandomState(16).permutation(3000)[:200].astype(np.int32)
    b = sampler.sample_blocks(seeds, fanouts, seed=5)
    want = _run(kind, layers, b.blocks, b.source_rows(x_dev))
    assert all(bool(torch.isfinite(t).all()) for t in want)
    warm = [sampler.sample_blocks(np.random.RandomState(k).permutation(3000)[:200].astype(np.int32), fanouts,
                                  seed=100 + k) for k in range(4)]
    ids, _ = tfg.utils.rank_source_rows(warm)
    with HFT(x, dtype=dtype) as plain, HFT(x, device_rows=ids[:1000], dtype=dtype) as cached, \
            tfg.utils.HostNeighborSampler(ei) as s:
        assert torch.isin(b.node_index, cached.device_rows).any()
        assert not torch.isin(b.node_index, cached.device_rows).all()
        hb = s.sample_blocks(seeds, fanouts, seed=5)
        for t in (plain, cached):
            assert _all_same_bits(_run(kind, layers, b.blocks, b.source_rows(t)), want)
            assert _all_same_bits(_run(kind, layers, hb.blocks, hb.source_rows(t)), want)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["GCN", "MeanGraphSage"])
def test_link_batch_from_a_16_bit_table(sampler, dtype, kind):
    x = _table(3000, 100, 17, dtype)
    x_dev = x.float().cuda()
    layers = _layers(kind, 2)
    pos = np.random.RandomState(18).randint(0, 3000, (2, 128)).astype(np.int32)
    b = sampler.sample_link_blocks(pos, [10, 5], num_negatives=2, exclude="reverse", seed=6)

    def scores(h0):
        pl, nl = b.predict_edge(_forward(kind, layers, b.blocks, h0))
        (pl.sum() - nl.sum()).backward()
        grads = [p.grad.clone() for layer in layers for p in layer.parameters()]
        for layer in layers:
            layer.zero_grad()
        return [pl.detach(), nl.detach()] + grads
    want = scores(b.source_rows(x_dev))
    with HFT(x, dtype=dtype) as plain, HFT(x, device_rows=_rows(3000, 0.3, 19), dtype=dtype) as cached:
        for t in (plain, cached):
            assert _all_same_bits(scores(b.source_rows(t)), want)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["GCN", "GAT", "MeanGraphSage"])
def test_layerwise_inference_from_a_16_bit_table(sampler, dtype, kind):
    ei = _graph()
    x = _table(3000, 24, 23, dtype)
    x_dev = x.float().cuda()
    L = tfg.layers
    if kind == "GAT":
        layers = [L.GAT(32, num_heads=4, activation=tfg.nn.relu, seed=1), L.GAT(8, num_heads=4, seed=2)]
    else:
        layers = [getattr(L, kind)(32, activation=tfg.nn.relu, seed=1), getattr(L, kind)(8, seed=2)]
    with torch.no_grad():                                # build the weights
        b = sampler.sample_blocks(np.arange(64, dtype=np.int32), [None, None])
        h = b.source_rows(x_dev)
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, _adapt(kind, blk)], training=False)
    budget = sampling.LAYERWISE_FIXED_BYTES + (6 << 20)  # a few chunks per layer
    want = tfg.utils.layerwise_inference(sampler, x_dev, layers, device_bytes=budget)
    with HFT(x, dtype=dtype) as plain, HFT(x, device_rows=_rows(3000, 0.3, 24), dtype=dtype) as cached, \
            tfg.utils.HostNeighborSampler(ei) as s:
        for t in (plain, cached):
            got = tfg.utils.layerwise_inference(sampler, t, layers, device_bytes=budget)
            assert got.dtype == torch.float32 and _same_bits(got, want)
            assert _same_bits(tfg.utils.layerwise_inference(s, t, layers, device_bytes=budget), want)


@pytest.mark.parametrize("dtype", DTYPES)
def test_refusals(dtype):
    x = _table(100, 8, 3, dtype)
    with pytest.raises(TypeError, match="float32"):     # the default stays float32
        HFT(x)
    with pytest.raises(TypeError, match=str(dtype)):
        HFT(x.float(), dtype=dtype)
    with pytest.raises(ValueError, match="dtype"):
        HFT(x, dtype=torch.float64)
    for bad, err in (([100], IndexError), ([-1], IndexError), ([4, 4], ValueError), (np.array([1.5]), TypeError)):
        with pytest.raises(err):
            HFT(x, device_rows=bad, dtype=dtype)
    with pytest.raises(ValueError):
        HFT(x, device_rows=torch.tensor([7, 9, 7], device="cuda"), dtype=dtype)
    with pytest.raises(TypeError, match="CUDA"):
        HFT(x.cuda(), dtype=dtype)
    t = HFT(x, dtype=dtype, device_rows=[1, 2])
    t.close()
    with pytest.raises(RuntimeError, match="closed"):
        t.gather([1])
