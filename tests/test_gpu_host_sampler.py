# coding=utf-8
"""Mini-batch sampling from a graph in host memory on the device: HostNeighborSampler's host CSR bit for bit against
csr_build over the same edges (one range, about ten, a range holding only the hub row; weighted and unweighted; int32 and
int64, numpy and tensor, non-contiguous input), sample_blocks bit for bit against RandomNeighborSampler.sample_blocks with
the parametrisations of test_gpu_blocks.py, one host synchronisation per batch, CSR positions past 2^31 against the
oracle's restatement of the draws, GraphSAGE over HostNeighborSampler + HostFeatureTable against RandomNeighborSampler +
a device x, the refusals and the registrations' lifetimes."""
import gc

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from tf_geometric_b200.utils import sampling
from oracle import tfg_oracle as o
from conftest import random_graph

pytestmark = pytest.mark.gpu

HNS = tfg.utils.HostNeighborSampler
RNS = tfg.utils.RandomNeighborSampler


def _graph():
    """A hub row of 5 000 edges, 30 isolated rows, duplicate edges, self loops and a column id past the last row."""
    ei = random_graph(3000, 30000, seed=31, isolated=30, hub=(9, 5000))
    ei = np.concatenate([ei, ei[:, :500], [[3, 40, 41], [3100, 40, 41]]], axis=1).astype(np.int32)
    w = np.random.RandomState(32).rand(ei.shape[1]).astype(np.float32)
    return ei, w


def _device_structure(ei, w):
    csr, w_csr, rowptr, _ = RNS(ops.as_device(ei, torch.int32), None if w is None else ops.as_device(w))\
        ._neighborhood_structure()
    return rowptr, csr.col, w_csr


def _device_bytes(ei, budget):
    """device_bytes that leaves `budget` bytes for a range of rows"""
    N = int(ei.max()) + 1
    return budget + 8 * (N + 1) + 8 * (ei.shape[1] // 1024 + 1) + sampling.HOST_CSR_FIXED_BYTES


def _check_csr(s, ei, w):
    rowptr, col, w_csr = _device_structure(ei, w)
    assert torch.equal(s.rowptr, rowptr)
    assert np.array_equal(s._col, col.cpu().numpy())
    if w is None:
        assert s._w is None and s._w_ptr is None
    else:
        assert np.array_equal(s._w.view(np.int32), w_csr.cpu().numpy().view(np.int32))


@pytest.mark.parametrize("budget", ["one", "ten", "hub"])
@pytest.mark.parametrize("weighted", [True, False])
def test_host_csr_matches_csr_build(budget, weighted):
    ei, w = _graph()
    w = w if weighted else None
    eb = sampling.HOST_CSR_EDGE_BYTES if weighted else sampling.HOST_CSR_EDGE_BYTES_UNWEIGHTED
    rb = sampling.HOST_CSR_ROW_BYTES
    rp = np.concatenate([[0], np.cumsum(np.bincount(ei[0], minlength=int(ei.max()) + 1))])
    deg = np.diff(rp)
    # "ten": ranges of about 5 200 edges (the hub row alone has more than 5 000)
    B = {"one": None, "ten": eb * 5200 + rb * 400, "hub": eb * int(deg.max()) + 2 * rb}[budget]
    if B is not None:
        ranges = sampling._row_ranges(rp, B, eb)
        if budget == "ten":
            assert 7 <= len(ranges) <= 12, len(ranges)
        else:
            assert (9, 10) in ranges
    with HNS(ei, w, device_bytes=None if B is None else _device_bytes(ei, B)) as s:
        assert (s.num_nodes, s.num_row_nodes, s.num_edges) == (3101, 3000, ei.shape[1])
        _check_csr(s, ei, w)


@pytest.mark.parametrize("kind", ["int64 numpy", "int32 tensor", "int64 tensor", "non-contiguous"])
def test_input_kinds(kind):
    ei, w = _graph()
    if kind == "int64 numpy":
        arg, warg = ei.astype(np.int64), w.astype(np.float64)
    elif kind == "int32 tensor":
        arg, warg = torch.from_numpy(ei), torch.from_numpy(w)
    elif kind == "int64 tensor":
        arg, warg = torch.from_numpy(ei).long(), torch.from_numpy(w)[:, None]
    else:
        arg, warg = np.asfortranarray(ei), np.stack([w, w], 1)[:, 0]
        assert not arg.flags.c_contiguous and not warg.flags.c_contiguous
    with HNS(arg, warg) as s:
        _check_csr(s, ei, w)


@pytest.fixture(scope="module")
def samplers():
    ei, w = _graph()
    dev = RNS(ops.as_device(ei, torch.int32), ops.as_device(w))
    host = HNS(ei, w)
    yield dev, host
    host.close()


def _seeds(n, first=(9, 0, 3)):
    seeds = np.random.RandomState(33).permutation(3000)[:n].astype(np.int32)
    seeds[:min(n, len(first))] = first[:n]
    return seeds


def _assert_same_batch(a, b):
    assert torch.equal(a.node_index, b.node_index)
    assert a.hop_sizes == b.hop_sizes and a.num_nodes == b.num_nodes
    assert len(a.blocks) == len(b.blocks)
    for x, y in zip(a.blocks, b.blocks):
        assert (x.num_src, x.num_dst) == (y.num_src, y.num_dst)
        for name in ("edge_index", "global_col"):
            assert torch.equal(getattr(x, name), getattr(y, name)), name
        assert torch.equal(x.edge_weight.view(torch.int32), y.edge_weight.view(torch.int32))
        for name in ("rowptr", "col", "perm"):
            assert torch.equal(getattr(x.csr, name), getattr(y.csr, name)), name
        assert (x.csr.n_rows, x.csr.n_cols) == (y.csr.n_rows, y.csr.n_cols)
        assert (x.csr.plan is None) == (y.csr.plan is None)
        if x.csr.plan is not None:
            assert (x.csr.plan.n_tasks, x.csr.plan.n_hubs, x.csr.plan.n_slots) == \
                (y.csr.plan.n_tasks, y.csr.plan.n_hubs, y.csr.plan.n_slots)
            for name, t in x.csr.plan.arrays.items():
                assert torch.equal(t, y.csr.plan.arrays[name]), name


@pytest.mark.parametrize("fanouts,padding,n_seeds", [([15, 10, 5], False, 256), ([4, 25], True, 256), ([6], "head", 256),
                                                     ([3, None], False, 64), ([None, 2], True, 64), ([5, 4], False, 0),
                                                     ([5, 4], False, 1), ([None], False, 256)])
def test_sample_blocks_matches_device_sampler(samplers, fanouts, padding, n_seeds):
    dev, host = samplers
    seeds = _seeds(n_seeds)
    want = dev.sample_blocks(seeds, fanouts, padding=padding, seed=17)
    _assert_same_batch(host.sample_blocks(seeds, fanouts, padding=padding, seed=17), want)
    again = host.sample_blocks(ops.as_device(seeds, torch.int32), fanouts, padding=padding, seed=17)
    _assert_same_batch(again, want)


def test_unweighted_sample_blocks():
    ei, _ = _graph()
    dev = RNS(ops.as_device(ei, torch.int32))
    with HNS(ei) as host:
        for fanouts in ([15, 10, 5], [None, 3]):
            _assert_same_batch(host.sample_blocks(_seeds(256), fanouts, seed=3),
                               dev.sample_blocks(_seeds(256), fanouts, seed=3))


def test_one_synchronisation_per_batch(samplers):
    _, host = samplers
    seeds = ops.as_device(_seeds(512), torch.int32)
    host.sample_blocks(seeds, [15, 10, 5], seed=1)
    torch.cuda.synchronize()
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    torch.cuda.set_sync_debug_mode("error")
    try:
        host.sample_blocks(seeds, [15, 10, 5], seed=2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        _ffi.set_trace(prev)
    assert trace.counts.get("tfgk_block_sample_end") == 1 and "tfgk_block_sample_read_total" not in trace.counts
    assert trace.counts.get("tfgk_block_sample_fill_mapped") == 3 and "tfgk_block_sample_fill" not in trace.counts


def test_bad_seeds(samplers):
    dev, host = samplers
    for bad in (np.array([5, 6, 5], np.int32), np.array([5, 3101], np.int32), np.array([-1, 2], np.int32)):
        with pytest.raises(ValueError) as want:
            dev.sample_blocks(bad, [4, 3], seed=17)
        with pytest.raises(ValueError) as got:
            host.sample_blocks(bad, [4, 3], seed=17)
        assert str(got.value) == str(want.value)
    assert bool((host._node_map == -1).all())
    _assert_same_batch(host.sample_blocks(_seeds(128), [4, 3], seed=17), dev.sample_blocks(_seeds(128), [4, 3], seed=17))


# ---- CSR positions past 2^31 ---------------------------------------------------------------------------------------

BIG_E = (1 << 31) + (1 << 24)
BIG_DEG = 1024
BIG_ROWS = BIG_E // BIG_DEG


def _big_col(p):
    return ((np.asarray(p, np.int64) * 7 + 3) % BIG_ROWS).astype(np.int32)


def _available_host_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def test_positions_past_2_31():
    need = 3 * 4 * BIG_E + (4 << 30)          # edge list and CSR columns, plus room for the generation's temporaries
    if _available_host_bytes() < need:
        pytest.skip("needs about {:.0f} GB of available host memory for a graph of 2^31 + 2^24 edges".format(need / 1e9))
    # sorted by row (row p // 1024), so the CSR position of an edge is its position in the list
    ei = np.empty((2, BIG_E), np.int32)
    step = 1 << 26
    for p0 in range(0, BIG_E, step):
        p = np.arange(p0, min(p0 + step, BIG_E), dtype=np.int64)
        ei[0, p0:p0 + p.size] = p // BIG_DEG
        ei[1, p0:p0 + p.size] = _big_col(p)
    s = HNS(ei)
    del ei
    gc.collect()
    try:
        assert s.num_nodes == BIG_ROWS and s.num_edges == BIG_E
        rp = s.rowptr.cpu().numpy()
        assert np.array_equal(rp, np.arange(BIG_ROWS + 1, dtype=np.int64) * BIG_DEG)
        pos = np.concatenate([np.arange(0, 64), (1 << 31) + np.arange(-4096, 4096), np.arange(BIG_E - 64, BIG_E),
                              np.random.RandomState(1).randint(0, BIG_E, 4096)])
        assert np.array_equal(s._col[pos], _big_col(pos))
        first_past = (1 << 31) // BIG_DEG
        seeds = np.array([first_past, first_past + 5, BIG_ROWS - 1, 7, first_past - 1], np.int32)
        key = 123
        for k, padding in ((5, False), (200, False), (2000, True)):
            b = s.sample_blocks(seeds, [k], padding=padding, seed=key)
            blk = b.blocks[0]
            h_key = tfg.utils.graph_utils._batch_seed(key, 0)
            want = []
            for r in seeds.tolist():
                start, idx = r * BIG_DEG, np.arange(BIG_DEG, dtype=np.uint64)
                base = np.uint64(r) << np.uint64(32)
                if padding:                      # k >= degree: k draws with replacement
                    p = start + o.random_below(h_key, o.RNG_STREAM_SAMPLER, base + np.arange(k, dtype=np.uint64),
                                               BIG_DEG)
                else:                            # reservoir: slot j ends at the last draw i >= k that picked it
                    p = start + np.arange(k, dtype=np.int64)
                    j = o.random_below(h_key, o.RNG_STREAM_SAMPLER, base + idx[k:], idx[k:] + np.uint64(1))
                    for i, jj in zip(range(k, BIG_DEG), j.tolist()):
                        if jj < k:
                            p[jj] = start + i
                want.append(_big_col(p))
            assert np.array_equal(blk.global_col.cpu().numpy(), np.concatenate(want)), (k, padding)
            rows = blk.edge_index[0].cpu().numpy()
            assert np.array_equal(rows, np.repeat(np.arange(len(seeds)), k))
    finally:
        s.close()


# ---- end to end ----------------------------------------------------------------------------------------------------

def _run(layers, blocks, h):
    for layer, blk in zip(layers, blocks):
        h = layer([h, blk], training=True)
    h.square().sum().backward()
    grads = [p.grad.clone() for layer in layers for p in layer.parameters()]
    for layer in layers:
        layer.zero_grad()
    return h.detach(), grads


def _same_bits(a, b):
    return all(torch.equal(u.view(torch.int32), v.view(torch.int32)) for u, v in zip(a, b))


@pytest.mark.parametrize("kind", ["MeanGraphSage", "MaxPoolGraphSage"])
@pytest.mark.parametrize("fanouts", [[10, 5], [15, 10, 5]])
def test_training_over_host_graph_and_host_features(kind, fanouts):
    # every node has in-edges, so no max-pool row is empty and the gradients stay finite
    ei = random_graph(3000, 30000, seed=41, hub=(9, 3000)).astype(np.int32)
    x = torch.from_numpy(np.random.RandomState(15).randn(3000, 100).astype(np.float32))
    units = [64] * (len(fanouts) - 1) + [16]
    layers = [getattr(tfg.layers, kind)(u, seed=i + 1, trainable=True) for i, u in enumerate(units)]
    seeds = np.random.RandomState(16).permutation(3000)[:200].astype(np.int32)
    b = RNS(ops.as_device(ei, torch.int32)).sample_blocks(seeds, fanouts, seed=5)
    want_h, want_g = _run(layers, b.blocks, x.cuda()[b.node_index.long()])
    assert all(bool(torch.isfinite(t).all()) for t in [want_h] + want_g)
    with HNS(ei) as s, tfg.utils.HostFeatureTable(x) as t:
        hb = s.sample_blocks(seeds, fanouts, seed=5)
        got_h, got_g = _run(layers, hb.blocks, hb.source_rows(t))
    assert _same_bits([got_h] + got_g, [want_h] + want_g)


# ---- refusals and lifetimes ----------------------------------------------------------------------------------------

def test_refusals_leave_nothing_behind():
    ei, w = _graph()
    before = dict(sampling._host_registered)
    neg = ei.copy()
    neg[1, 77] = -3
    bad_rows = ei.copy()
    bad_rows[0, 5] = -1
    cases = [
        ((neg,), {}, ValueError, "negative"),
        ((bad_rows,), {}, ValueError, "negative"),
        ((ei.astype(np.int64) + (1 << 31),), {}, ValueError, "2\\^31"),
        ((-ei.astype(np.int64),), {}, ValueError, "negative"),
        ((ei.astype(np.float32),), {}, TypeError, "integer"),
        ((ei.astype(bool),), {}, TypeError, "integer"),
        ((torch.from_numpy(ei).cuda(),), {}, TypeError, "RandomNeighborSampler"),
        ((ei.tolist(),), {}, TypeError, "numpy"),
        ((ei[:1],), {}, ValueError, "2, E"),
        ((ei, w[:-1]), {}, ValueError, "entries"),
        ((ei, torch.from_numpy(w).requires_grad_()), {}, ValueError, "grad"),
        ((ei, torch.from_numpy(w).cuda()), {}, TypeError, "RandomNeighborSampler"),
        ((ei, w.astype(np.complex64)), {}, TypeError, "floating"),
        ((ei,), {"device_bytes": _device_bytes(ei, 29 * 4000)}, ValueError, "row 9 has 50[0-9][0-9] edges"),
    ]
    for args, kw, err, words in cases:
        with pytest.raises(err, match=words):
            HNS(*args, **kw)
        assert sampling._host_registered == before, words
    s = HNS(ei, w)
    s.close()
    with pytest.raises(RuntimeError, match="closed"):
        s.sample_blocks([1, 2], [3])
    assert sampling._host_registered == before


def test_lifetimes():
    """the edge list is released by the constructor (an array of 32 MiB or more is read in place), the CSR by close()"""
    ei = random_graph(100000, 4200000, seed=2)
    assert ei.flags.c_contiguous and ei.dtype == np.int32 and ei.nbytes >= sampling.HOST_IN_PLACE_BYTES
    w = np.random.RandomState(3).rand(ei.shape[1]).astype(np.float32)
    before = dict(sampling._host_registered)
    s = HNS(ei, w)
    assert len(sampling._host_registered) == len(before) + 2           # the CSR's columns and weights
    for a in (ei, w):                                                   # read in place, and released
        ops.host_register(a.ctypes.data, a.nbytes)
        ops.host_unregister(a.ctypes.data)
    b = s.sample_blocks(_seeds(64), [5, 5], seed=1)
    s.close()
    assert sampling._host_registered == before
    assert b.blocks[0].edge_weight.is_cuda and bool(torch.isfinite(b.blocks[0].edge_weight).all())
    s.close()
    s2 = HNS(ei)
    assert len(sampling._host_registered) == len(before) + 1           # no weights for an unweighted graph
    del s2
    gc.collect()
    assert sampling._host_registered == before
