# coding=utf-8
"""GAT on sampled blocks without a GPU: the declaration of tfgk_block_self_loops_i32 and its argument checks, the looped
layout of Block.with_self_loops against a row-by-row restatement (empty rows, 0 and 1 output rows, no edges), its
memoisation and work-plan rule, the routing of tfg.nn.gat / tfg.layers.GAT over the fake kernel layer against the single
index space, and the refusals, all before any device work."""
import numpy as np
import pytest
import torch

import block_gat_fake_backend as fake_gat
from test_blocks_host import _batch


@pytest.fixture
def fake(monkeypatch):
    calls = fake_gat.install(monkeypatch)
    import tf_geometric_b200 as tfg
    plans = []

    def build_plan(csr):
        plans.append(csr)
        return None
    monkeypatch.setattr(tfg.ops, "build_plan", build_plan)
    return tfg, calls, plans


def test_entry_is_declared_and_checks_its_arguments():
    import tf_geometric_b200 as tfg
    from tf_geometric_b200 import _ffi
    assert "SelfLoopBlock" in dir(tfg.utils) and _ffi.ABI_VERSION == 7
    assert len(_ffi.SIGNATURES["tfgk_block_self_loops_i32"]) == 9
    assert "tfgk_block_self_loops_i32" not in _ffi.NOT_CAPTURABLE        # no host value, no host key
    cases = [((None, None, None, -1, 2, None, None, None, None), _ffi.ERR_INVALID_ARGUMENT),
             ((None, None, None, 3, -1, None, None, None, None), _ffi.ERR_INVALID_ARGUMENT),
             ((None, None, None, 3, 2, None, None, None, None), _ffi.ERR_INVALID_ARGUMENT),        # null pointers
             ((None, None, None, (1 << 31) - 4, 4, None, None, None, None), _ffi.ERR_UNSUPPORTED)]
    for args, code in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call("tfgk_block_self_loops_i32", *args)
        assert err.value.code == code, args


def _looped_restatement(e, n_dst):
    """Row by row: the sampled edges of row r in order, then (r, r)."""
    rows, cols, rowptr = [], [], [0]
    for r in range(n_dst):
        sel = np.nonzero(e[0] == r)[0]
        rows += [r] * (sel.size + 1)
        cols += e[1][sel].tolist() + [r]
        rowptr.append(len(rows))
    return np.array(rowptr, np.int64), np.array([rows, cols], np.int32).reshape(2, -1)


def _hand_block(tfg, e, n_dst, n_src, fanout=None):
    e = np.asarray(e, np.int32).reshape(2, -1)
    S = e.shape[1]
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(e[0], minlength=n_dst))]).astype(np.int64)
    csr = tfg.ops.CSR(torch.from_numpy(rowptr), torch.from_numpy(e[1].copy()), torch.arange(S, dtype=torch.int32),
                      n_dst, n_src)
    return tfg.utils.Block(n_src, n_dst, torch.from_numpy(e), torch.ones(S), torch.from_numpy(e[1].copy()), csr,
                           fanout=fanout)


def test_looped_layout_matches_the_restatement(fake):
    tfg, calls, _ = fake
    b, _ = _batch(tfg)
    blocks = list(b.blocks) + [
        _hand_block(tfg, [[0, 0, 2, 2, 2], [3, 1, 4, 0, 4]], 4, 6),      # rows 1 and 3 empty
        _hand_block(tfg, np.zeros((2, 0)), 0, 5),                        # no output rows
        _hand_block(tfg, [[0, 0], [2, 1]], 1, 3),                        # one output row
        _hand_block(tfg, np.zeros((2, 0)), 3, 3)]                        # no edges: self loops only
    for blk in blocks:
        lb = blk.with_self_loops()
        assert isinstance(lb, tfg.utils.SelfLoopBlock) and not isinstance(lb, tfg.utils.Block)
        rowptr, e = _looped_restatement(blk.edge_index.numpy(), blk.num_dst)
        assert (lb.num_src, lb.num_dst) == (blk.num_src, blk.num_dst)
        np.testing.assert_array_equal(lb.edge_index.numpy(), e)
        np.testing.assert_array_equal(lb.csr.rowptr.numpy(), rowptr)
        np.testing.assert_array_equal(lb.csr.col.numpy(), e[1])
        np.testing.assert_array_equal(lb.csr.perm.numpy(), np.arange(e.shape[1]))
        assert (lb.csr.n_rows, lb.csr.n_cols, lb.csr.nnz) == (blk.num_dst, blk.num_src, e.shape[1])
    assert calls["block_self_loops"] == len(blocks)


def test_memoised_and_plan_rule(fake):
    tfg, calls, plans = fake
    b, _ = _batch(tfg)                                   # fan-outs [4, 3]: short rows, no plan
    n_plans = len(plans)
    lb = b.blocks[0].with_self_loops()
    assert b.blocks[0].with_self_loops() is lb and calls["block_self_loops"] == 1
    assert len(plans) == n_plans and lb.csr.plan is None
    assert [blk.fanout for blk in b.blocks] == [4, 3]
    built = len(calls["csr_build"])
    csr_t = lb.transposed()
    assert lb.transposed() is csr_t and calls["csr_build"][built:] == [True]
    e = lb.edge_index.numpy()
    order = np.lexsort((np.arange(e.shape[1]), e[1]))
    np.testing.assert_array_equal(csr_t.perm.numpy(), order)
    e = [[0, 1], [1, 0]]
    k = tfg.ops.DENSE_ROW_DEGREE
    for fanout, planned in ((k - 2, False), (k - 1, True), (k, True), (None, True)):
        del plans[:]
        blk = _hand_block(tfg, e, 2, 2, fanout=fanout)
        lb = blk.with_self_loops()
        assert (plans == [lb.csr]) == planned, fanout


def _gat_layers(tfg, heads, split, act, trainable=False):
    return tfg.layers.GAT(8, attention_units=8, num_heads=heads, split_value_heads=split, activation=act, seed=1,
                          trainable=trainable)


@pytest.mark.parametrize("heads,split,act", [(1, True, None), (2, True, "relu"), (2, False, None)])
def test_gat_on_a_looped_block_matches_the_single_space(fake, heads, split, act):
    tfg, calls, _ = fake
    b, nb = _batch(tfg)
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    xs = x[nb.node_index.long()].contiguous()
    layer = _gat_layers(tfg, heads, split, tfg.nn.relu if act else None)
    blk = b.blocks[0]
    lb = blk.with_self_loops()
    with torch.no_grad():
        single = layer([xs, nb.edge_index_list[0]])
        n_proj = calls["gemm_proj"]
        out = layer([xs, lb, torch.ones(3)])              # a third input (edge weights) is ignored
        assert calls["gemm_proj"] - n_proj == 2           # Q over num_dst rows, K | V over num_src rows
        src = layer([b.source_rows(x), lb])
    assert out.shape == (blk.num_dst, 8)
    np.testing.assert_allclose(out.numpy(), single.numpy()[:blk.num_dst], rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(src.numpy(), out.numpy())
    p = {k: v.detach() for k, v in layer.named_parameters()}
    h, att = tfg.nn.gat(xs, lb, p["query_kernel"], p["query_bias"], tfg.nn.relu, p["key_kernel"], p["key_bias"],
                        tfg.nn.relu, p["kernel"], p["bias"], num_heads=heads, split_value_heads=split,
                        return_attention=True)
    _, att_s = tfg.nn.gat(xs, nb.edge_index_list[0], p["query_kernel"], p["query_bias"], tfg.nn.relu, p["key_kernel"],
                          p["key_bias"], tfg.nn.relu, p["kernel"], p["bias"], num_heads=heads,
                          split_value_heads=split, return_attention=True)
    assert att.shape == (lb.edge_index.shape[1], heads)
    np.testing.assert_allclose(att.numpy(), att_s.numpy()[_single_positions(blk)], rtol=1e-5, atol=1e-6)


def _single_positions(blk):
    """For every looped-block position, the position of the same edge in the single index space's edge list with self
    loops (its E sampled edges, then one self loop per node)."""
    e = blk.edge_index.numpy()
    rowptr = blk.csr.rowptr.numpy()
    E, n = e.shape[1], blk.num_dst
    pos = np.empty(E + n, np.int64)
    pos[np.arange(E) + e[0]] = np.arange(E)
    pos[rowptr[1:n + 1] + np.arange(n)] = E + np.arange(n)
    return pos


def test_training_two_layers_matches_the_single_space(fake):
    tfg, _, _ = fake
    b, nb = _batch(tfg)
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    grads = []
    for route in ("blocks", "single"):
        l1 = tfg.layers.GAT(8, num_heads=2, activation=tfg.nn.relu, seed=1, trainable=True)
        l2 = tfg.layers.GAT(4, num_heads=1, seed=2, trainable=True)
        xs = x[nb.node_index.long()].clone().requires_grad_()
        if route == "blocks":
            h = l2([l1([xs, b.blocks[0].with_self_loops()], training=True), b.blocks[1].with_self_loops()],
                   training=True)
        else:
            h = l2([l1([xs, nb.edge_index_list[0]], training=True), nb.edge_index_list[1]], training=True)[:b.hop_sizes[0]]
        assert h.shape == (b.hop_sizes[0], 4)
        (h * h).sum().backward()
        grads.append([xs.grad.numpy()] + [p.grad.numpy() for p in list(l1.parameters()) + list(l2.parameters())])
    for gb, gs in zip(*grads):
        np.testing.assert_allclose(gb, gs, rtol=1e-4, atol=1e-5)


def test_refusals_before_any_device_work(fake):
    tfg, calls, _ = fake
    b, _ = _batch(tfg)
    blk = b.blocks[0]
    lb, lb1 = blk.with_self_loops(), b.blocks[1].with_self_loops()
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    xs = x[b.node_index.long()].contiguous()
    before = dict(calls)
    for dt in (torch.bfloat16, torch.float8_e4m3fn):
        with pytest.raises(NotImplementedError, match="fp32"):
            tfg.layers.GAT(8, seed=1, message_dtype=dt)([xs, lb])
    with pytest.raises(ValueError, match="rows"):
        tfg.layers.GAT(8, seed=1)([xs[:-1], lb])
    with pytest.raises(ValueError, match="rows"):
        tfg.layers.GAT(8, seed=1)([b.source_rows(x), lb1])
    with pytest.raises(NotImplementedError, match="return_attention"):
        w = torch.ones(12, 8, requires_grad=True)
        tfg.nn.gat(xs, lb, w, None, None, w, None, None, w, return_attention=True)
    assert {k: calls[k] for k in ("gemm_proj", "gat_fused", "block_self_loops")} == \
        {k: before[k] for k in ("gemm_proj", "gat_fused", "block_self_loops")}
    fns = (lambda: tfg.layers.GAT(4)([xs, blk]),                    # a plain Block: no self loops defined
           lambda: tfg.layers.GCN(4)([xs, lb]),
           lambda: tfg.layers.MeanGraphSage(4)([xs, lb]),
           lambda: tfg.layers.MaxPoolGraphSage(4)([xs, lb]),
           lambda: tfg.layers.GCNGraphSage(4)([xs, lb]),
           lambda: tfg.layers.LSTMGraphSage(4)([xs, lb]),
           lambda: tfg.layers.SGC(4)([xs, lb]))
    for fn in fns:
        with pytest.raises(TypeError, match="block") as err:
            fn()
        assert "mean_graph_sage" in str(err.value)
