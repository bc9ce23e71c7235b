# coding=utf-8
"""Layer-wise inference on the device: row_block of both samplers bit for bit against sample_blocks(arange(r0, r1),
[None]) (the graph of test_gpu_host_sampler.py, weighted and unweighted, host CSR built in one range and in about ten),
its host synchronisations, a clean map after every call, a range past CSR position 2^31; layerwise_inference for every
supported layer over both samplers and both kinds of x, bit for bit against the same layers on sample_blocks batches,
between budgets and between output placements, within 1e-5 of the full-graph layers, within its memory budget; and a
model trained on host-memory blocks evaluated by it."""
import gc

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from tf_geometric_b200.utils import sampling
from conftest import random_graph

pytestmark = pytest.mark.gpu

HNS = tfg.utils.HostNeighborSampler
RNS = tfg.utils.RandomNeighborSampler
N_NODES = 3101


def _graph():
    """A hub row of 5 000 edges, 30 isolated rows, duplicate edges, self loops and a column id past the last row."""
    ei = random_graph(3000, 30000, seed=31, isolated=30, hub=(9, 5000))
    ei = np.concatenate([ei, ei[:, :500], [[3, 40, 41], [3100, 40, 41]]], axis=1).astype(np.int32)
    w = np.random.RandomState(32).rand(ei.shape[1]).astype(np.float32)
    return ei, w


def _ten_ranges_bytes(ei):
    """device_bytes that builds the host CSR in about ten ranges (test_gpu_host_sampler.py's "ten")"""
    eb, rb = sampling.HOST_CSR_EDGE_BYTES, sampling.HOST_CSR_ROW_BYTES
    N = int(ei.max()) + 1
    return eb * 5200 + rb * 400 + 8 * (N + 1) + 8 * (ei.shape[1] // 1024 + 1) + sampling.HOST_CSR_FIXED_BYTES


@pytest.fixture(scope="module")
def samplers():
    ei, w = _graph()
    out = {"dev": RNS(ops.as_device(ei, torch.int32), ops.as_device(w)), "host": HNS(ei, w),
           "host10": HNS(ei, w, device_bytes=_ten_ranges_bytes(ei)), "dev_unw": RNS(ops.as_device(ei, torch.int32)),
           "host_unw": HNS(ei)}
    yield out
    for s in out.values():
        if isinstance(s, HNS):
            s.close()


def _assert_same_batch(a, b):
    assert torch.equal(a.node_index, b.node_index)
    assert a.hop_sizes == b.hop_sizes and a.num_nodes == b.num_nodes and len(a.blocks) == len(b.blocks) == 1
    x, y = a.blocks[0], b.blocks[0]
    assert (x.num_src, x.num_dst, x.fanout) == (y.num_src, y.num_dst, y.fanout)
    for name in ("edge_index", "global_col", "dst_ids"):
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
    for u, v in zip(x.degrees(), y.degrees()):
        assert torch.equal(u, v)


RANGES = [(0, 0), (N_NODES, N_NODES), (0, 1), (9, 10), (0, 40), (2990, N_NODES), (0, 30), (3000, N_NODES),
          (5, 700), (0, N_NODES), (1500, 1501)]


@pytest.mark.parametrize("name", ["dev", "host", "host10", "dev_unw", "host_unw"])
def test_row_block_matches_sample_blocks(samplers, name):
    s = samplers[name]
    for r0, r1 in RANGES:
        got = s.row_block(r0, r1)
        _assert_same_batch(got, s.sample_blocks(torch.arange(r0, r1, dtype=torch.int32, device="cuda"), [None]))
        assert bool((s._node_map == -1).all())
    if name != "dev":
        for r0, r1 in RANGES:
            _assert_same_batch(s.row_block(r0, r1), samplers["dev" if "unw" not in name else "dev_unw"].row_block(r0, r1))


def test_synchronisations_per_row_block(samplers):
    for s in (samplers["host"], samplers["dev"]):
        s.row_block(0, 700)
        torch.cuda.synchronize()
        rp = s._host_rowptr()
        for r0, r1 in ((0, 700), (0, 30), (20, 20), (1000, 1001)):
            trace = _ffi.CallTrace()
            prev = _ffi.set_trace(trace)
            torch.cuda.set_sync_debug_mode("error")
            try:
                s.row_block(r0, r1)
            finally:
                torch.cuda.set_sync_debug_mode(0)
                _ffi.set_trace(prev)
            host_returning = {k: v for k, v in trace.counts.items() if k in _ffi.NOT_CAPTURABLE}
            has_edges = rp[r1] > rp[r0]
            # the row block reads its source-row count back (when it has edges), the work plan its task counts
            assert host_returning == dict({"tfgk_row_block_i32": 1}, **({"tfgk_plan_build": 1} if has_edges else {})), \
                (r0, r1, trace.counts)
            assert trace.counts.get("tfgk_copy_async", 0) == (2 if s is samplers["host"] and has_edges else 0)


def test_refusals_leave_the_map_clean(samplers):
    for s in (samplers["host"], samplers["dev"]):
        for r0, r1 in ((-1, 3), (0, N_NODES + 1), (7, 6)):
            with pytest.raises(ValueError):
                s.row_block(r0, r1)
            assert bool((s._node_map == -1).all())
    ei, w = _graph()
    s = HNS(ei, w)
    s.close()
    with pytest.raises(RuntimeError, match="closed"):
        s.row_block(0, 5)


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


def test_row_block_past_2_31():
    need = 3 * 4 * BIG_E + (4 << 30)          # edge list and CSR columns, plus room for the generation's temporaries
    if _available_host_bytes() < need:
        pytest.skip("needs about {:.0f} GB of available host memory for a graph of 2^31 + 2^24 edges".format(need / 1e9))
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
        first_past = (1 << 31) // BIG_DEG
        for r0, r1 in ((first_past - 2, first_past + 3), (BIG_ROWS - 4, BIG_ROWS)):
            blk = s.row_block(r0, r1).blocks[0]
            pos = np.arange(r0 * BIG_DEG, r1 * BIG_DEG, dtype=np.int64)
            assert np.array_equal(blk.global_col.cpu().numpy(), _big_col(pos))
            assert np.array_equal(blk.global_col.cpu().numpy(), s._col[pos])
            assert np.array_equal(blk.edge_index[0].cpu().numpy(), np.repeat(np.arange(r1 - r0), BIG_DEG))
            assert bool((s._node_map == -1).all())
    finally:
        s.close()


# ---- layerwise_inference -------------------------------------------------------------------------------------------

F_IN = 24


def _model(kind, n_layers):
    L = tfg.layers
    widths = [32] * (n_layers - 1) + [8]
    acts = [tfg.nn.relu] * (n_layers - 1) + [None]
    if kind == "GCN":
        layers = [L.GCN(u, activation=a, seed=i) for i, (u, a) in enumerate(zip(widths, acts))]
    elif kind == "GAT":
        layers = [L.GAT(u, num_heads=4, activation=a, seed=i) for i, (u, a) in enumerate(zip(widths, acts))]
    else:
        layers = [getattr(L, kind)(u, activation=a, seed=i) for i, (u, a) in enumerate(zip(widths, acts))]
    return layers


def _x():
    return np.random.RandomState(7).randn(N_NODES, F_IN).astype(np.float32)


def _built(layers, samplers, x):
    """Build the layers on one batch so that their weights exist before any comparison."""
    b = samplers["dev"].sample_blocks(np.arange(64, dtype=np.int32), [None] * len(layers))
    with torch.no_grad():
        h = b.source_rows(x)
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, sampling_adapt(layer, blk)], training=False)
    return layers


def sampling_adapt(layer, blk):
    from tf_geometric_b200.utils.layerwise import _adapt
    return _adapt(layer, blk)


def _layer_ranges(sampler, layers, device_bytes):
    """The ranges layerwise_inference cuts for each layer at device_bytes (device outputs assumed)."""
    from tf_geometric_b200.utils.layerwise import _plan_layer
    rp = sampler._host_rowptr()
    N, F, plans = rp.size - 1, F_IN, []
    for i, layer in enumerate(layers):
        eb, rb, D = sampling.layerwise_chunk_bytes(layer, F)
        ranges, on_device = _plan_layer(rp, device_bytes - (4 * N * F if i else 0), eb, rb, 4 * N * D)
        assert on_device
        plans.append(ranges)
        F = D
    return plans


def _chunked_reference(sampler, x, layers, plans):
    """The same layers applied to sample_blocks(arange(r0, r1), [None]) batches over each layer's own chunks."""
    h = x
    for layer, ranges in zip(layers, plans):
        out = []
        for r0, r1 in ranges:
            b = sampler.sample_blocks(torch.arange(r0, r1, dtype=torch.int32, device="cuda"), [None])
            with torch.no_grad():
                out.append(layer([b.source_rows(h), sampling_adapt(layer, b.blocks[0])], training=False))
        h = torch.cat(out)
    return h


def _full_graph(ei, w, x, layers):
    """The full-graph layers over the sampler's edge list (N nodes; GAT adds self loops itself)."""
    g_ei, g_w = ops.as_device(ei, torch.int32), ops.as_device(w)
    adj = tfg.SparseMatrix(g_ei, g_w, [N_NODES if x.shape[0] == N_NODES else x.shape[0]] * 2)
    h = x
    with torch.no_grad():
        for layer in layers:
            if isinstance(layer, tfg.layers.GAT):
                h = layer([h, g_ei])
            elif isinstance(layer, tfg.layers.GCN):
                h = layer([h, adj], cache={})
            else:
                h = layer([h, g_ei, g_w])
    return h


def _same_bits(a, b):
    """bit for bit, except that NaN (a row whose max-pool has no neighbour) matches any NaN"""
    a, b = torch.as_tensor(a).cuda(), torch.as_tensor(b).cuda()
    if a.shape != b.shape or not torch.equal(a.isnan(), b.isnan()):
        return False
    keep = ~a.isnan()
    return torch.equal(a[keep].view(torch.int32), b[keep].view(torch.int32))


def _same(a, b, exact):
    """Between different chunkings, GraphSAGE rows change in their last bits: its projections go through ops.gemm
    (tfgk_gemm_f32), which takes the 3xTF32 tensor-core kernel when M * K >= 2^14 and the SIMT kernel (split-K chosen
    from M) otherwise, and M is the chunk's output rows (the pool layers' MLP: its source rows).  So do rows of chunks
    of a few rows around the 5 000-edge hub for every layer.  Those compare within 1e-6; the same chunks, and GCN and GAT
    at ordinary chunk sizes, bit for bit.  Max-pool rows without in-edges hold non-finite values that depend on the
    chunk: only finite rows are compared there."""
    if exact:
        return _same_bits(a, b)
    a, b = torch.as_tensor(a).cuda(), torch.as_tensor(b).cuda()
    finite = a.isfinite().all(1) & b.isfinite().all(1)
    if not bool(finite.all()):
        assert float(finite.float().mean()) > 0.25          # three max-pool layers spread them to most rows
        a, b = a[finite], b[finite]
    torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-6 * float(a.nan_to_num(0, 0, 0).abs().max()), equal_nan=True)
    return True


def _budget_for(sampler, layers, chunks):
    """device_bytes that cuts every layer's rows into about `chunks` ranges, with device outputs"""
    rp = sampler._host_rowptr()
    N, E = rp.size - 1, int(rp[-1])
    need = 0
    F = F_IN
    for layer in layers:
        eb, rb, D = sampling.layerwise_chunk_bytes(layer, F)
        need = max(need, (eb * E + rb * N) // chunks + eb * 5000 + 4 * N * D)
        F = D
    return need + sampling.LAYERWISE_FIXED_BYTES


KINDS = ["GCN", "GAT", "MeanGraphSage", "SumGraphSage", "MeanPoolGraphSage", "MaxPoolGraphSage"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n_layers", [2, 3])
def test_layerwise_matches_blocks_and_full_graph(samplers, kind, n_layers):
    ei, w = _graph()
    x_np = _x()
    x = torch.from_numpy(x_np).cuda()
    layers = _built(_model(kind, n_layers), samplers, x)
    dev, host = samplers["dev"], samplers["host"]
    one = tfg.utils.layerwise_inference(dev, x, layers)
    many_bytes = _budget_for(dev, layers, 10)
    many = tfg.utils.layerwise_inference(dev, x, layers, device_bytes=many_bytes)
    exact = kind in ("GCN", "GAT")
    assert one.is_cuda and one.shape == (N_NODES, 8)
    assert _same(one, many, exact)
    plans = _layer_ranges(dev, layers, many_bytes)
    assert len(plans[0]) > 3 and all(len(ranges) > 1 for ranges in plans)
    assert _same_bits(many, _chunked_reference(dev, x, layers, plans))        # the same chunks: bit for bit
    with tfg.utils.HostFeatureTable(x_np) as table, \
            tfg.utils.HostFeatureTable(x_np, device_rows=np.arange(0, N_NODES, 3)) as cached:
        assert _same_bits(tfg.utils.layerwise_inference(host, table, layers, device_bytes=many_bytes), many)
        assert _same_bits(tfg.utils.layerwise_inference(samplers["host10"], cached, layers), one)
    full = _full_graph(ei, w, x, layers)
    finite = one.isfinite().all(1) & full.isfinite().all(1)
    torch.testing.assert_close(one[finite], full[finite], rtol=1e-5, atol=1e-5 * float(full[finite].abs().max()))


@pytest.mark.parametrize("kind", KINDS)
def test_placement_gives_the_same_bits(samplers, kind):
    """One layer over the same chunks with its output on the device and in page-locked host memory."""
    from tf_geometric_b200.utils import layerwise
    x = torch.from_numpy(_x()).cuda()
    layer = _built(_model(kind, 2), samplers, x)[0]
    for name in ("dev", "host"):
        s = samplers[name]
        rp = s._host_rowptr()
        eb, rb, D = sampling.layerwise_chunk_bytes(layer, F_IN)
        ranges = sampling._row_ranges(rp, eb * 8000 + rb * 400, eb, rb)
        assert len(ranges) > 3
        on_dev, key = layerwise._run_layer(s, x, layer, ranges, rp, True, x.device)
        assert key is None and on_dev.is_cuda
        on_host, key = layerwise._run_layer(s, x, layer, ranges, rp, False, x.device)
        try:
            assert isinstance(on_host, np.ndarray) and _same_bits(torch.from_numpy(on_host), on_dev), (kind, name)
        finally:
            sampling._host_release(key)


def test_every_output_in_host_memory(samplers):
    """A budget that fits the hub row's chunk but not next to any layer's output: every output goes to host memory, the
    last comes back as a CPU tensor, and the bits are those of device outputs over the same chunks.  Every layer has 8
    inputs and 8 outputs, so every layer's chunk needs the same bytes."""
    from tf_geometric_b200.utils import layerwise
    x = torch.from_numpy(_x()[:, :8].copy()).cuda()
    L, relu = tfg.layers, tfg.nn.relu
    models = {"GAT": [L.GAT(8, num_heads=4, activation=relu, seed=i) for i in range(3)],
              "GCN": [L.GCN(8, activation=relu, seed=i) for i in range(3)],
              "MeanGraphSage": [L.MeanGraphSage(8, activation=relu, seed=i) for i in range(3)]}
    rp = samplers["host"]._host_rowptr()
    for kind, layers in models.items():
        layers = _built(layers, samplers, x)
        eb, rb, D = sampling.layerwise_chunk_bytes(layers[0], 8)
        assert all(sampling.layerwise_chunk_bytes(layer, 8) == (eb, rb, D) for layer in layers)
        small = sampling.LAYERWISE_FIXED_BYTES + eb * 5073 + 2 * rb + 4 * N_NODES * D - 1
        ranges, on_device = layerwise._plan_layer(rp, small, eb, rb, 4 * N_NODES * D)
        assert not on_device and len(ranges) > 3
        regs = dict(sampling._host_registered)
        got = tfg.utils.layerwise_inference(samplers["host"], x, layers, device_bytes=small)
        assert not got.is_cuda and got.shape == (N_NODES, 8)
        assert sampling._host_registered.keys() == regs.keys()          # every output's registration released
        h = x
        for layer in layers:                                            # the same chunks, outputs on the device
            h, _ = layerwise._run_layer(samplers["host"], h, layer, ranges, rp, True, x.device)
        assert _same_bits(got, h), kind


def test_gcn_block_values_are_the_full_graphs(samplers):
    """GCN's block values on row blocks are the full graph's gcn_norm_adj values, bit for bit (s_r = 1)."""
    ei, w = _graph()
    full = tfg.nn.gcn_norm_adj(tfg.SparseMatrix(ops.as_device(ei, torch.int32), ops.as_device(w), [N_NODES, N_NODES]))
    frp, fval = full.csr.rowptr.cpu().numpy(), full.value_csr.cpu().numpy()
    for r0, r1 in ((0, 40), (5, 700), (2990, N_NODES)):
        normed = samplers["host"].row_block(r0, r1).blocks[0].with_gcn_norm().normalized()
        want = fval[frp[r0]:frp[r1]]
        assert np.array_equal(normed.value.cpu().numpy().view(np.int32), want.view(np.int32))


def test_peak_memory_with_wide_hidden_layers(samplers):
    """Three layers with 256-wide hidden outputs at a budget that leaves each chunk little more than the hub row: the
    previous layer's output, held while it is the next layer's input, counts against device_bytes."""
    x = torch.from_numpy(_x()).cuda()
    for kind in ("GCN", "MeanGraphSage", "GAT"):
        L = tfg.layers
        if kind == "GAT":
            layers = [L.GAT(256, num_heads=4, activation=tfg.nn.relu, seed=i) for i in range(2)] + [L.GAT(8, seed=2)]
        else:
            layers = [getattr(L, kind)(256, activation=tfg.nn.relu, seed=i) for i in range(2)] + \
                [getattr(L, kind)(8, seed=2)]
        layers = _built(layers, samplers, x)
        tight, F = 0, F_IN
        for i, layer in enumerate(layers):
            eb, rb, D = sampling.layerwise_chunk_bytes(layer, F)
            tight = max(tight, 4 * N_NODES * (D + (F if i else 0)) + eb * 6000 + rb * 300)
            F = D
        tight += sampling.LAYERWISE_FIXED_BYTES
        want = tfg.utils.layerwise_inference(samplers["host"], x, layers)
        torch.cuda.synchronize()
        resident = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        got = tfg.utils.layerwise_inference(samplers["host"], x, layers, device_bytes=tight)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - resident
        print("{} 3 wide layers: peak {} of budget {}".format(kind, peak, tight))
        assert peak <= tight, (kind, peak, tight)
        assert _same(got, want, False)


def test_peak_memory_stays_within_the_budget(samplers):
    x = torch.from_numpy(_x()).cuda()
    for kind in ("GAT", "GCN", "MeanPoolGraphSage"):
        layers = _built(_model(kind, 2), samplers, x)
        budget = _budget_for(samplers["host"], layers, 6)
        torch.cuda.synchronize()
        resident = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        tfg.utils.layerwise_inference(samplers["host"], x, layers, device_bytes=budget)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - resident
        print("{}: peak {} of budget {}".format(kind, peak, budget))
        assert peak <= budget, (kind, peak, budget)


def test_synchronisations_per_chunk(samplers):
    x = torch.from_numpy(_x()).cuda()
    for kind, plans in (("MeanGraphSage", 1), ("GAT", 2)):
        layers = _built(_model(kind, 2), samplers, x)
        budget = _budget_for(samplers["host"], layers, 6)
        tfg.utils.layerwise_inference(samplers["host"], x, layers, device_bytes=budget)
        torch.cuda.synchronize()
        trace = _ffi.CallTrace()
        prev = _ffi.set_trace(trace)
        torch.cuda.set_sync_debug_mode("error")
        try:
            tfg.utils.layerwise_inference(samplers["host"], x, layers, device_bytes=budget)
        finally:
            torch.cuda.set_sync_debug_mode(0)
            _ffi.set_trace(prev)
        chunks = trace.counts["tfgk_row_block_i32"]
        assert chunks >= 6
        host_returning = sum(v for k, v in trace.counts.items() if k in _ffi.NOT_CAPTURABLE)
        assert host_returning <= (1 + plans) * chunks, trace.counts


def test_refusals(samplers):
    x = torch.from_numpy(_x()).cuda()
    with pytest.raises(TypeError, match="GCN, GAT, MeanGraphSage"):
        tfg.utils.layerwise_inference(samplers["dev"], x, [tfg.layers.GIN(8)])
    with pytest.raises(ValueError, match="x has 100 rows"):
        tfg.utils.layerwise_inference(samplers["dev"], x[:100], [tfg.layers.MeanGraphSage(8)])
    with pytest.raises(ValueError, match="row 9 has 5073 edges"):
        tfg.utils.layerwise_inference(samplers["dev"], x, _built(_model("MeanGraphSage", 2), samplers, x),
                                      device_bytes=sampling.LAYERWISE_FIXED_BYTES + 100_000)
    assert bool((samplers["dev"]._node_map == -1).all())


# ---- end to end ----------------------------------------------------------------------------------------------------

def test_trained_on_host_blocks_evaluated_layerwise():
    rs = np.random.RandomState(3)
    n, k, F = 6000, 4, 32
    label = rs.randint(0, k, n)
    src = rs.randint(0, n, 120_000)
    same = rs.rand(src.size) < 0.8
    dst = np.where(same, 0, rs.randint(0, n, src.size))
    by_class = [np.flatnonzero(label == c) for c in range(k)]
    dst[same] = [by_class[label[u]][rs.randint(len(by_class[label[u]]))] for u in src[same]]
    ei = np.stack([src, dst]).astype(np.int32)
    x_np = (np.eye(k)[label] @ rs.randn(k, F) * 0.5 + rs.randn(n, F)).astype(np.float32)
    train, test = np.arange(0, n // 2), np.arange(n // 2, n)
    torch.manual_seed(0)
    layers = [tfg.layers.MeanGraphSage(64, activation=tfg.nn.relu, seed=1, trainable=True),
              tfg.layers.MeanGraphSage(k, activation=None, seed=2, trainable=True)]
    y = torch.from_numpy(label).cuda()
    with HNS(ei) as s, tfg.utils.HostFeatureTable(x_np) as table:
        b = s.sample_blocks(train[:64].astype(np.int32), [10, 10], seed=0)
        h = b.source_rows(table)
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, blk], training=True)
        opt = torch.optim.Adam([p for layer in layers for p in layer.parameters()], lr=1e-2)
        for step in range(150):
            seeds = rs.choice(train, 256, replace=False).astype(np.int32)
            b = s.sample_blocks(seeds, [10, 10], seed=step)
            h = b.source_rows(table)
            for layer, blk in zip(layers, b.blocks):
                h = layer([h, blk], training=True)
            loss = torch.nn.functional.cross_entropy(h, y[torch.from_numpy(seeds).long().cuda()])
            opt.zero_grad()
            loss.backward()
            opt.step()
        logits = tfg.utils.layerwise_inference(s, table, layers)
    acc = float((logits[test].argmax(1) == y[test]).float().mean())
    print("held-out accuracy", acc)
    assert acc >= 0.8
    full = _full_graph(ei, np.ones(ei.shape[1], np.float32), torch.from_numpy(x_np).cuda(), layers)
    top2 = torch.topk(full, 2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-5
    assert torch.equal(logits.argmax(1)[clear], full.argmax(1)[clear])
