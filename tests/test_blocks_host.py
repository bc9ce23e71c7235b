# coding=utf-8
"""Bipartite blocks without a GPU: the ABI declarations and argument checks of the block sampler, the capacities it
allocates, RandomNeighborSampler.sample_blocks over the CPU fake of the sampler against the dict-based restatement of
tests/minibatch_ref.py, and GraphSAGE over blocks on the fake kernel layer: the four aggregators against the single
index space, the SourceRows rules and the refusals."""
import numpy as np
import pytest
import torch

import block_fake_backend as fake_blocks
import minibatch_ref as ref
from conftest import random_graph
from oracle import c_oracle

ENTRIES = {"tfgk_block_sample_workspace_bytes": 3, "tfgk_block_sample_begin": 8, "tfgk_block_sample_count": 13,
           "tfgk_block_sample_read_total": 7, "tfgk_block_sample_fill": 24, "tfgk_block_sample_end": 8,
           "tfgk_csr_build_in_range": 11}


@pytest.fixture
def fake(monkeypatch):
    calls = fake_blocks.install(monkeypatch)
    import tf_geometric_b200 as tfg

    def no_plan(csr):
        raise AssertionError("build_plan must not run for fan-outs below DENSE_ROW_DEGREE")
    monkeypatch.setattr(tfg.ops, "build_plan", no_plan)
    return tfg, calls


def test_ffi_declares_the_entries_and_refuses_capture():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    for name, n in ENTRIES.items():
        assert len(_ffi.SIGNATURES[name]) == n, name
    for name in ("tfgk_block_sample_read_total", "tfgk_block_sample_fill", "tfgk_block_sample_end"):
        assert name in _ffi.NOT_CAPTURABLE, name
    for name in ("tfgk_block_sample_begin", "tfgk_block_sample_count"):     # no host value, no host key
        assert name not in _ffi.NOT_CAPTURABLE, name


def test_argument_validation_without_gpu():
    import ctypes
    from tf_geometric_b200 import _ffi
    bad = _ffi.ERR_INVALID_ARGUMENT
    need = ctypes.c_size_t()
    cases = [
        ("tfgk_block_sample_workspace_bytes", (4, -1, ctypes.byref(need)), None),
        ("tfgk_block_sample_workspace_bytes", (4, 1 << 31, ctypes.byref(need)), None),
        ("tfgk_block_sample_begin", (None, -1, 10, None, None, None, 2, None), "size"),
        ("tfgk_block_sample_begin", (None, 3, 10, None, None, None, 2, None), "null"),
        ("tfgk_block_sample_count", (None, 4, None, None, 0, 2, 8, 3, 7, None, None, 0, None), "padding"),
        ("tfgk_block_sample_count", (None, 4, None, None, 0, 2, 8, -1, 2, None, None, 0, None), "head"),
        ("tfgk_block_sample_count", (None, 4, None, None, -1, 2, 8, 3, 0, None, None, 0, None), "size"),
        ("tfgk_block_sample_count", (None, 4, None, None, 2, 2, 8, 3, 0, None, None, 0, None), "size"),   # hop >= L
        ("tfgk_block_sample_fill", (None, 4, None, None, 4, None, None, None, 2, 2, 8, 16, 3, 0, 0, 1, None, None, None,
                                    None, None, None, 0, None), "size"),
        ("tfgk_block_sample_read_total", (None, 0, None, 4, None, None, None), None),
        ("tfgk_block_sample_end", (None, 4, 10, None, None, 2, None, None), "null"),
        ("tfgk_csr_build_in_range", (None, None, -1, 4, 4, None, None, None, None, 0, None), None),
    ]
    for name, args, words in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(name, *args)
        assert err.value.code == bad, name
        if words:
            assert words in str(err.value), (name, str(err.value))
    _ffi.call("tfgk_block_sample_workspace_bytes", 100, 1500, ctypes.byref(need))
    small = need.value
    _ffi.call("tfgk_block_sample_workspace_bytes", 100, 150000, ctypes.byref(need))
    assert need.value > small


def test_capacities():
    from tf_geometric_b200 import ops
    assert ops.block_capacities(1024, 5, 10 ** 6) == (5120, 6144)
    assert ops.block_capacities(6144, 10, 10 ** 6) == (61440, 67584)
    assert ops.block_capacities(67584, 15, 50000) == (1013760, 50000)     # the list never outgrows the graph
    assert ops.block_capacities(10, None, 100) == (None, None)             # every neighbour: read back
    assert ops.block_capacities(300, 2 ** 23, 100) == (None, None)         # 2^31 edges or more: read back
    assert ops.block_capacities(0, 7, 100) == (0, 0)


def test_block_sample_refuses_fanouts_before_any_device_work():
    """the rules the entries would apply mid-batch are applied first: nothing is read from the (here absent) tensors"""
    from tf_geometric_b200 import ops
    with pytest.raises(ValueError, match="head"):
        ops.block_sample(None, None, None, None, [3, None], [0, 1], None, padding="head")
    with pytest.raises(ValueError, match=">= 0"):
        ops.block_sample(None, None, None, None, [3, -2], [0, 1], None)


def test_sampled_inputs_are_refused_by_as_device():
    from tf_geometric_b200 import ops
    from tf_geometric_b200.utils import Block, SourceRows
    for obj in (Block(2, 1, None, None, None, None), SourceRows(None, None)):
        with pytest.raises(TypeError, match="mean_graph_sage"):
            ops.as_device(obj, torch.int32)


def _sampler_graph():
    ei = random_graph(300, 2400, seed=5, isolated=20, hub=(7, 400))
    ei = np.concatenate([ei, ei[:, :50]], axis=1)                       # duplicate edges
    ei = np.concatenate([ei, [[3], [350]]], axis=1).astype(np.int32)    # a column id past the last source row
    w = np.random.RandomState(6).rand(ei.shape[1]).astype(np.float32)
    return ei, w


@pytest.mark.parametrize("fanouts,padding", [([5, 3], False), ([2, 4, 3], True), ([4], "head"), ([], False)])
def test_sample_blocks_matches_restatement(fake, fanouts, padding):
    tfg, calls = fake
    ei, w = _sampler_graph()
    sampler = tfg.utils.RandomNeighborSampler(ei, w)
    seeds = np.array([7, 0, 299, 350, 3, 150], np.int32)
    b = sampler.sample_blocks(seeds, fanouts, padding=padding, seed=11)
    rowptr, col, perm = c_oracle.csr_build(ei[0], ei[1], int(ei[0].max()) + 1)
    nodes, edges, weights, sizes = ref.neighborhood(rowptr, col, w[perm], seeds, fanouts, padding, 11)
    np.testing.assert_array_equal(b.node_index.numpy(), nodes)
    assert b.hop_sizes == sizes and len(b.blocks) == len(fanouts)
    L = len(fanouts)
    for i, (blk, e, ww) in enumerate(zip(b.blocks, edges, weights)):
        assert (blk.num_src, blk.num_dst) == (sizes[L - i], sizes[L - 1 - i])
        np.testing.assert_array_equal(blk.edge_index.numpy(), e)
        np.testing.assert_array_equal(blk.edge_weight.numpy(), ww)
        np.testing.assert_array_equal(blk.global_col.numpy(), nodes[e[1]])
        csr = blk.csr
        assert (csr.n_rows, csr.n_cols, csr.nnz) == (blk.num_dst, blk.num_src, e.shape[1]) and csr.plan is None
        np.testing.assert_array_equal(csr.rowptr.numpy(), np.concatenate([[0], np.cumsum(np.bincount(
            e[0], minlength=blk.num_dst))]))
        np.testing.assert_array_equal(csr.col.numpy(), e[1])
        np.testing.assert_array_equal(csr.perm.numpy(), np.arange(e.shape[1]))
    built = len(calls["csr_build"])
    for blk in b.blocks:
        csr_t, w_t = blk.transposed("mean")
        e = blk.edge_index.numpy()
        rp, c, p = c_oracle.csr_build(e[1], e[0], blk.num_src)
        np.testing.assert_array_equal(csr_t.col.numpy(), c)
        cnt = np.maximum(np.bincount(e[0], minlength=blk.num_dst), 1).astype(np.float32)
        np.testing.assert_array_equal(w_t.numpy(), (np.float32(1) / cnt[e[0]] * blk.edge_weight.numpy())[p])
        assert blk.transposed("mean")[1] is w_t and blk.transposed()[0] is csr_t      # memoised on the block
    assert calls["csr_build"][built:] == [True] * len(b.blocks)


def test_sample_blocks_rejects_bad_seeds(fake):
    tfg, _ = fake
    ei, w = _sampler_graph()
    sampler = tfg.utils.RandomNeighborSampler(ei, w)
    with pytest.raises(ValueError, match="duplicate"):
        sampler.sample_blocks([4, 9, 4], [3])
    with pytest.raises(ValueError, match="outside"):
        sampler.sample_blocks([4, 351], [3])
    b = sampler.sample_blocks([4, 9], [3], seed=1)
    assert b.hop_sizes[0] == 2


# ---- GraphSAGE on blocks over the fake kernel layer -------------------------------------------------------------

KINDS = {"mean": "MeanGraphSage", "sum": "SumGraphSage", "mean_pool": "MeanPoolGraphSage", "max_pool": "MaxPoolGraphSage"}


def _batch(tfg):
    ei, w = _sampler_graph()
    sampler = tfg.utils.RandomNeighborSampler(ei, w)
    seeds = np.array([7, 0, 299, 3, 150, 42, 77], np.int32)
    return sampler.sample_blocks(seeds, [4, 3], seed=2), sampler.sample_neighborhood(seeds, [4, 3], seed=2)


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("concat,normalize", [(True, False), (False, True)])
def test_aggregators_on_blocks_match_the_single_space(fake, kind, concat, normalize):
    tfg, _ = fake
    b, nb = _batch(tfg)
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    xs = x[nb.node_index.long()].contiguous()
    layer = getattr(tfg.layers, KINDS[kind])(8, seed=1, concat=concat, normalize=normalize)
    blk = b.blocks[0]
    with torch.no_grad():
        single = layer([xs, nb.edge_index_list[0], nb.edge_weight_list[0]])
        out = layer([xs, blk])
        src = layer([b.source_rows(x), blk])
    assert out.shape == (blk.num_dst, 8)
    np.testing.assert_allclose(out.numpy(), single.numpy()[:blk.num_dst], rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(src.numpy(), out.numpy())


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_block_backward_routes(fake, kind):
    """x_src gets a gradient over num_src rows through the transposed block CSR; a SourceRows input gets none"""
    tfg, _ = fake
    b, _ = _batch(tfg)
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    l1 = getattr(tfg.layers, KINDS[kind])(8, seed=1, trainable=True)
    l2 = getattr(tfg.layers, KINDS[kind])(4, seed=2, trainable=True, activation=None)
    xs = x[b.node_index.long()].clone().requires_grad_()
    h = l2([l1([xs, b.blocks[0]], training=True), b.blocks[1]], training=True)
    assert h.shape == (b.hop_sizes[0], 4)
    h.sum().backward()
    assert xs.grad.shape == xs.shape and float(xs.grad.abs().sum()) > 0
    assert all(p.grad is not None for p in l1.parameters())
    for layer in (l1, l2):
        layer.zero_grad()
    h = l2([l1([b.source_rows(x), b.blocks[0]], training=True), b.blocks[1]], training=True)
    h.sum().backward()
    assert all(p.grad is not None for p in l1.parameters())


def test_source_rows_rules(fake):
    tfg, _ = fake
    b, _ = _batch(tfg)
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    src = b.source_rows(x)
    assert src.shape == (b.hop_sizes[-1], 12)
    np.testing.assert_array_equal(src.gather().numpy(), x.numpy()[b.node_index.numpy()])
    np.testing.assert_array_equal(src.gather(3).numpy(), x.numpy()[b.node_index.numpy()[:3]])
    xg = x.clone().requires_grad_()
    rows = b.source_rows(xg).gather()
    rows.sum().backward()                                   # differentiable through TakeRows when x requires grad
    np.testing.assert_array_equal(xg.grad.numpy(), np.bincount(b.node_index.numpy(), minlength=351)[:, None]
                                  * np.ones((1, 12), np.float32))


def test_refusals(fake):
    tfg, _ = fake
    b, _ = _batch(tfg)
    blk = b.blocks[0]
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    xs = x[b.node_index.long()].contiguous()
    for kind in KINDS.values():
        layer = getattr(tfg.layers, kind)(8, seed=1)
        with pytest.raises(ValueError, match="rows"):
            layer([xs[:-1], blk])
        with pytest.raises(ValueError):
            layer([b.source_rows(x), b.blocks[1]])
        with pytest.raises(NotImplementedError, match="edge-weight"):
            layer([xs, blk, torch.ones(blk.edge_index.shape[1], requires_grad=True)])
        with pytest.raises(ValueError, match="carries"):
            layer([xs, blk, torch.ones(blk.edge_index.shape[1])])
        with pytest.raises(NotImplementedError, match="fp32"):
            getattr(tfg.layers, kind)(8, seed=1, message_dtype=torch.bfloat16)([xs, blk])
    fns = (lambda: tfg.layers.GCN(4)([xs, blk]),
           lambda: tfg.layers.GAT(4)([xs, blk]),
           lambda: tfg.nn.gcn_graph_sage(xs, blk, None, torch.ones(12, 4)),
           lambda: tfg.layers.GCNGraphSage(4)([xs, blk]),
           lambda: tfg.layers.LSTMGraphSage(4)([xs, blk]),
           lambda: tfg.nn.gcn_graph_sage(b.source_rows(x), torch.zeros((2, 1), dtype=torch.int32), None,
                                         torch.ones(12, 4)))
    for fn in fns:
        with pytest.raises(TypeError, match="block"):
            fn()
