# coding=utf-8
"""GCN on sampled blocks without a GPU: the declaration of tfgk_block_gcn_values_f32 and its argument checks, the values
of Block.with_gcn_norm against a row-by-row restatement (empty rows, 0 and 1 output rows, no edges) and, with every
neighbour, against the full graph's gcn_norm_adj, the memoisation per configuration, the refusal of a block built by
hand, the routing of tfg.nn.gcn / tfg.layers.GCN over the fake kernel layer against the full graph, and the refusals,
all before any device work."""
import numpy as np
import pytest
import torch

import block_gcn_fake_backend as fake_gcn
from test_blocks_host import _sampler_graph

CONFIGS = [dict(), dict(improved=True), dict(renorm=False), dict(add_self_loop=False), dict(norm="left"),
           dict(norm="left", add_self_loop=False), dict(norm="right"), dict(norm="right", add_self_loop=False),
           dict(renorm=False, improved=True)]


@pytest.fixture
def fake(monkeypatch):
    calls = fake_gcn.install(monkeypatch)
    import tf_geometric_b200 as tfg
    monkeypatch.setattr(tfg.ops, "build_plan", lambda csr: None)
    return tfg, calls


def test_entry_is_declared_and_checks_its_arguments():
    import tf_geometric_b200 as tfg
    from tf_geometric_b200 import _ffi
    assert "GcnBlock" in dir(tfg.utils) and _ffi.ABI_VERSION == 7
    assert len(_ffi.SIGNATURES["tfgk_block_gcn_values_f32"]) == 14
    assert "tfgk_block_gcn_values_f32" not in _ffi.NOT_CAPTURABLE        # no host value, no host key
    assert (_ffi.GCN_NORM_BOTH, _ffi.GCN_NORM_LEFT, _ffi.GCN_NORM_RIGHT) == (0, 1, 2)
    assert (_ffi.GCN_LOOP_NONE, _ffi.GCN_LOOP_NORMED, _ffi.GCN_LOOP_FILL) == (0, 1, 2)

    def args(S=3, n_dst=2, norm=0, loop=1):
        return (None, None, None, S, None, n_dst, None, None, norm, loop, 1.0, 1.0, None, None)
    cases = [(args(S=-1), _ffi.ERR_INVALID_ARGUMENT),
             (args(n_dst=-1), _ffi.ERR_INVALID_ARGUMENT),
             (args(norm=3), _ffi.ERR_INVALID_ARGUMENT),
             (args(loop=3), _ffi.ERR_INVALID_ARGUMENT),
             (args(n_dst=0), _ffi.ERR_INVALID_ARGUMENT),                 # edges without output rows
             (args(), _ffi.ERR_INVALID_ARGUMENT),                        # null pointers
             (args(S=(1 << 31) - 4, n_dst=4), _ffi.ERR_UNSUPPORTED)]
    for a, code in cases:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call("tfgk_block_gcn_values_f32", *a)
        assert err.value.code == code, a
    _ffi.call("tfgk_block_gcn_values_f32", *args(S=0, n_dst=0))         # nothing to write
    _ffi.call("tfgk_block_gcn_values_f32", *args(S=0, n_dst=3, loop=0))  # no edges, no loops


def _batch(tfg, fanouts=(4, 3), padding=False, weighted=True):
    ei, w = _sampler_graph()
    sampler = tfg.utils.RandomNeighborSampler(ei, w if weighted else None)
    seeds = np.array([7, 0, 299, 3, 150, 42, 77, 310], np.int32)        # 310: an id with no row (an isolated node)
    return sampler, sampler.sample_blocks(seeds, list(fanouts), padding=padding, seed=2), ei, w if weighted else None


def _full_normed(tfg, ei, w, n, cfg):
    """The full graph's normalised values in its CSR order, with its rowptr (the fake gcn_norm_adj)."""
    adj = tfg.SparseMatrix(torch.from_numpy(ei), None if w is None else torch.from_numpy(w), [n, n])
    normed = tfg.nn.gcn_norm_adj(adj, **cfg)
    return normed.csr.rowptr.numpy(), normed.value_csr.numpy()


def _restatement(blk, rowsum, g_rowptr, cfg):
    """Row by row, in float32: the values the definition gives every slot of the block."""
    norm = cfg.get("norm", "both")
    loops, renorm = cfg.get("add_self_loop", True), cfg.get("renorm", True)
    fill = np.float32(2.0 if cfg.get("improved", False) else 1.0)
    deg_fill = fill if loops and (norm != "both" or renorm) else np.float32(0)
    code = {"both": 0, "left": 1, "right": 2}[norm]
    f = fake_gcn.degree_factor(rowsum, deg_fill, code)
    rp, gcol, w, dst = (t.numpy() for t in (blk.csr.rowptr, blk.global_col, blk.edge_weight, blk.dst_ids))
    out = []
    for r in range(blk.num_dst):
        g = int(dst[r])
        k = int(rp[r + 1] - rp[r])
        s = np.float32(int(g_rowptr[g + 1] - g_rowptr[g])) / np.float32(max(k, 1))
        for p in range(rp[r], rp[r + 1]):
            v = np.float32(w[p])
            if norm != "right":
                v = np.float32(f[g] * v)
            if norm != "left":
                v = np.float32(v * f[gcol[p]])
            out.append(np.float32(s * v))
        if loops:
            v = fill
            if norm != "both" or renorm:
                v = np.float32(f[g] * v) if norm != "right" else v
                v = np.float32(v * f[g]) if norm != "left" else v
            out.append(v)
    return np.array(out, np.float32)


def _hand_block(tfg, e, n_dst, n_src, dst, gcols, degrees):
    e = np.asarray(e, np.int32).reshape(2, -1)
    S = e.shape[1]
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(e[0], minlength=n_dst))]).astype(np.int64)
    csr = tfg.ops.CSR(torch.from_numpy(rowptr), torch.from_numpy(e[1].copy()), torch.arange(S, dtype=torch.int32),
                      n_dst, n_src)
    w = torch.from_numpy(np.random.RandomState(S).rand(S).astype(np.float32))
    return tfg.utils.Block(n_src, n_dst, torch.from_numpy(e), w, torch.tensor(gcols, dtype=torch.int32), csr,
                           dst_ids=torch.tensor(dst, dtype=torch.int32), degrees=degrees)


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: ",".join("{}={}".format(k, v) for k, v in c.items()) or "default")
def test_values_match_the_row_by_row_restatement(fake, cfg):
    tfg, calls = fake
    sampler, b, _, _ = _batch(tfg)
    g_rowptr, rowsum = sampler._gcn_degrees()
    deg = sampler._gcn_degrees
    blocks = list(b.blocks) + [
        _hand_block(tfg, [[0, 0, 2, 2, 2], [3, 1, 4, 0, 4]], 4, 6, [7, 0, 3, 9], [11, 0, 3, 7, 3], deg),   # rows 1, 3 empty
        _hand_block(tfg, np.zeros((2, 0)), 0, 5, [], [], deg),                                              # no output rows
        _hand_block(tfg, [[0, 0], [2, 1]], 1, 3, [7], [11, 40], deg),                                       # one output row
        _hand_block(tfg, np.zeros((2, 0)), 3, 3, [7, 0, 310], [], deg)]                                     # no edges
    for blk in blocks:
        normed = blk.with_gcn_norm().normalized(**cfg)
        want = _restatement(blk, rowsum.numpy(), g_rowptr.numpy(), cfg)
        np.testing.assert_array_equal(normed.value.numpy(), want)
        assert normed.shape == [blk.num_dst, blk.num_src]
        loops = cfg.get("add_self_loop", True)
        structure = blk.with_self_loops() if loops else blk
        assert normed.csr is structure.csr
        np.testing.assert_array_equal(normed.index.numpy(), structure.edge_index.numpy())
        np.testing.assert_array_equal(normed.value_csr.numpy(), want)
    assert calls["block_gcn_values"] == len(blocks)


@pytest.mark.parametrize("weighted", [True, False])
def test_every_neighbour_gives_the_full_graph_values(fake, weighted):
    tfg, _ = fake
    sampler, b, ei, w = _batch(tfg, fanouts=(None, None), weighted=weighted)
    n = 351
    for cfg in CONFIGS:
        rowptr, full = _full_normed(tfg, ei, w, n, cfg)
        for blk in b.blocks:
            dst = blk.dst_ids.numpy()
            want = np.concatenate([full[rowptr[g]:rowptr[g + 1]] for g in dst]) if dst.size else np.zeros(0, np.float32)
            np.testing.assert_array_equal(blk.with_gcn_norm().normalized(**cfg).value.numpy(), want, err_msg=str(cfg))


def test_memoised_per_configuration(fake):
    tfg, calls = fake
    _, b, _, _ = _batch(tfg)
    blk = b.blocks[0]
    sampled = len(calls["csr_build"])
    gb = blk.with_gcn_norm()
    assert blk.with_gcn_norm() is gb and isinstance(gb, tfg.utils.GcnBlock) and calls["block_gcn_values"] == 0
    assert not isinstance(gb, (tfg.utils.Block, tfg.utils.SelfLoopBlock)) and isinstance(gb, tfg.ops.SampledInput)
    a = gb.normalized()
    assert gb.normalized() is a and gb.normalized("both", True, True, True, False) is a
    assert calls["block_gcn_values"] == 1
    c = gb.normalized(improved=True)
    assert c is not a and gb.normalized(improved=True) is c and calls["block_gcn_values"] == 2
    d = gb.normalized(add_self_loop=False)
    assert d.csr is blk.csr and a.csr is blk.with_self_loops().csr and calls["block_self_loops"] == 1
    assert a._transposed_csr() is blk.with_self_loops().transposed()
    assert d._transposed_csr() is blk.transposed()[0]
    built = len(calls["csr_build"])
    dropped = a.dropout(0.5, training=True, seed=3)
    assert dropped._transposed_csr() is a._transposed_csr() and len(calls["csr_build"]) == built
    assert calls["csr_build"][sampled:] == [True, True]            # both transposed CSRs, without the id check
    layer = tfg.layers.GCN(4, seed=1)
    xs = torch.randn(blk.num_src, 6)
    with torch.no_grad():
        layer([xs, gb], cache={})
        layer([xs, gb])
    assert calls["block_gcn_values"] == 3


def test_a_block_built_by_hand_is_refused(fake):
    tfg, calls = fake
    from test_block_gat_host import _hand_block as plain_block
    blk = plain_block(tfg, [[0, 1], [1, 0]], 2, 2)
    with pytest.raises(ValueError, match="degrees"):
        blk.with_gcn_norm()
    assert calls["block_gcn_values"] == 0


def _model(tfg, units, trainable=False):
    return [tfg.layers.GCN(u, activation=tfg.nn.relu if i < len(units) - 1 else None, seed=1 + i, trainable=trainable)
            for i, u in enumerate(units)]


@pytest.mark.parametrize("cfg", [dict(), dict(norm="left"), dict(add_self_loop=False), dict(renorm=False)],
                         ids=["default", "left", "no_loops", "no_renorm"])
def test_gcn_on_blocks_matches_the_full_graph(fake, cfg):
    tfg, calls = fake
    sampler, b, ei, w = _batch(tfg, fanouts=(None, None))
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    layers = [tfg.layers.GCN(u, activation=tfg.nn.relu if i == 0 else None, seed=1 + i, **cfg)
              for i, u in enumerate((8, 5))]
    adj = tfg.SparseMatrix(torch.from_numpy(ei), torch.from_numpy(w), [351, 351])
    with torch.no_grad():
        h = x
        for layer in layers:
            h = layer([h, adj])
        full = h.numpy()[b.node_index.numpy()[:b.hop_sizes[0]]]
        h = b.source_rows(x)
        for layer, blk in zip(layers, b.blocks):
            h = layer([h, blk.with_gcn_norm()])
        dense = layers[0]([x[b.node_index.long()].contiguous(), b.blocks[0].with_gcn_norm()])
        src = layers[0]([b.source_rows(x), b.blocks[0].with_gcn_norm()])
    assert h.shape == (b.hop_sizes[0], 5)
    np.testing.assert_allclose(h.numpy(), full, rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(src.numpy(), dense.numpy())


def test_gcn_on_blocks_trains(fake):
    tfg, _ = fake
    _, b, _, _ = _batch(tfg, fanouts=(4, 3))
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32)).requires_grad_(True)
    layers = _model(tfg, (8, 5), trainable=True)
    h = b.source_rows(x)
    for layer, blk in zip(layers, b.blocks):
        h = layer([h, blk.with_gcn_norm()], training=True)
    assert h.shape == (b.hop_sizes[0], 5)
    h.square().sum().backward()
    assert x.grad is not None and x.grad.shape == x.shape
    for layer in layers:
        assert layer.kernel.grad is not None and layer.bias.grad is not None
    # through nn.gcn, with edge dropout and column splits
    blk = b.blocks[1]
    xs = torch.randn(blk.num_src, 6, requires_grad=True)
    W = torch.randn(6, 4, requires_grad=True)
    y = tfg.nn.gcn(xs, blk.with_gcn_norm(), W, edge_drop_rate=0.5, training=True)
    y.sum().backward()
    assert y.shape == (blk.num_dst, 4) and xs.grad.shape == xs.shape and W.grad.shape == W.shape
    with torch.no_grad():
        a = tfg.nn.gcn(xs, blk.with_gcn_norm(), W, num_or_size_splits=2)
        c = tfg.nn.gcn(xs, blk.with_gcn_norm(), W)
    np.testing.assert_array_equal(a.numpy(), c.numpy())


def test_refusals_before_any_device_work(fake):
    tfg, calls = fake
    _, b, _, _ = _batch(tfg)
    x = torch.from_numpy(np.random.RandomState(3).randn(351, 12).astype(np.float32))
    blk = b.blocks[0]
    gb, gb1 = blk.with_gcn_norm(), b.blocks[1].with_gcn_norm()
    xs = x[b.node_index.long()].contiguous()
    before = dict(calls)
    for dt in (torch.bfloat16, torch.float8_e4m3fn):
        with pytest.raises(NotImplementedError, match="fp32"):
            tfg.layers.GCN(8, seed=1, message_dtype=dt)([xs, gb])
    with pytest.raises(NotImplementedError):
        tfg.nn.gcn(xs.to_sparse(), gb, torch.ones(12, 4))
    with pytest.raises(NotImplementedError, match="sym"):
        tfg.layers.GCN(8, seed=1, sym=False)([xs, gb])
    with pytest.raises(ValueError, match="rows"):
        tfg.layers.GCN(8, seed=1)([xs[:-1], gb])
    with pytest.raises(ValueError, match="rows"):
        tfg.layers.GCN(8, seed=1)([b.source_rows(x), gb1])
    with pytest.raises(ValueError, match="carries"):
        tfg.layers.GCN(8, seed=1)([xs, gb, torch.ones(blk.edge_index.shape[1])])
    with pytest.raises(NotImplementedError, match="edge-weight"):
        tfg.layers.GCN(8, seed=1)([xs, gb, torch.ones(blk.edge_index.shape[1], requires_grad=True)])
    with pytest.raises(Exception, match="norm type"):
        tfg.nn.gcn(xs, gb, torch.ones(12, 4), norm="column")
    assert {k: calls[k] for k in ("block_gcn_values", "gemm", "block_self_loops")} == \
        {k: before[k] for k in ("block_gcn_values", "gemm", "block_self_loops")}
    fns = (lambda: tfg.layers.GCN(4)([xs, blk]),                    # a plain Block: the refusal names with_gcn_norm()
           lambda: tfg.layers.GCN(4)([xs, blk.with_self_loops()]),
           lambda: tfg.layers.GAT(4)([xs, gb]),
           lambda: tfg.layers.MeanGraphSage(4)([xs, gb]),
           lambda: tfg.layers.MaxPoolGraphSage(4)([xs, gb]),
           lambda: tfg.layers.GCNGraphSage(4)([xs, gb]),
           lambda: tfg.layers.SGC(4)([xs, gb]),
           lambda: tfg.layers.APPNP([4])([xs, gb]))
    for fn in fns:
        with pytest.raises(TypeError, match="block") as err:
            fn()
        assert "mean_graph_sage" in str(err.value) and "with_gcn_norm()" in str(err.value)
