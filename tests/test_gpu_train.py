# coding=utf-8
"""GPU parity for the training-mode extras and the device samplers (SURVEY.md 8(f)3-4):
dropout masks / per-head aggregation / GAT softmax backward against the numpy restatements, whole-layer gradients
against torch-CPU autograd over the op-for-op port of the reference (the stand-in for TensorFlow autodiff), and
drop_edge / neighbour samplers bit for bit against the oracle (same counter-based generator) and against the
fixtures produced by executing the reference's own sampler (tests/golden/ref_exec_sampler.npz)."""
import os

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _structure, _ffi
from oracle import tfg_oracle as o
from oracle import torch_cpu_port as port
from conftest import random_graph, assert_close, glorot

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def dev(a, dtype=None):
    return ops.as_device(a, dtype)


def host(t):
    return t.detach().cpu().numpy()


def _csr_of(ei, n):
    rowptr, col, perm = o.csr_build(ei[0], ei[1], n)
    csr = ops.CSR(dev(rowptr.astype(np.int64)), dev(col.astype(np.int32)), dev(perm.astype(np.int32)), n, n)
    return csr, rowptr, col, perm


# ---- kernels against their restatements -----------------------------------------------------------------------------

@pytest.mark.parametrize("n,rate", [(1, 0.5), (1000, 0.0), (100003, 0.3), (4099, 0.9)])
def test_dropout_mask_bit_exact(n, rate):
    x = np.random.RandomState(n).randn(n).astype(np.float32)
    seed = 0x1234567890ABCDEF + n
    got = host(ops.dropout(dev(x), rate, seed))
    np.testing.assert_array_equal(got, o.dropout(x, rate, seed))
    if n > 50000:
        assert abs((got != 0).mean() - (1 - rate)) < 0.01
        other = host(ops.dropout(dev(x), rate, seed + 1))
        assert 0.3 < ((got != 0) == (other != 0)).mean() < 0.8          # a different key gives a different mask
    np.testing.assert_array_equal(host(ops.dropout(dev(x), rate, seed)), got)


@pytest.mark.parametrize("H,dh,mode,with_map,rate", [
    (8, 16, "split", False, 0.0), (8, 16, "split", True, 0.25), (4, 32, "split", False, 0.5), (1, 128, "split", True, 0.0),
    (3, 5, "split", True, 0.0), (2, 40, "split", False, 0.4), (4, 8, "broadcast", True, 0.3), (3, 7, "broadcast", False, 0.0),
    (4, 8, "reduce", False, 0.2), (5, 3, "reduce", True, 0.0)])
def test_spmm_heads_bit_exact(H, dh, mode, with_map, rate):
    rs = np.random.RandomState(H * 100 + dh)
    n, e = 300, 2500
    ei = random_graph(n, e, seed=dh, isolated=3)
    csr, rowptr, col, _ = _csr_of(ei, n)
    E = ei.shape[1]
    w = rs.rand(E, H).astype(np.float32)
    emap = rs.permutation(E).astype(np.int32) if with_map else None
    src = rs.randn(n, dh if mode == "broadcast" else H * dh).astype(np.float32)
    bias = rs.randn(dh if mode == "reduce" else H * dh).astype(np.float32)
    code = {"split": ops.HEADS_SPLIT, "broadcast": ops.HEADS_BROADCAST, "reduce": ops.HEADS_REDUCE}[mode]
    want = o.spmm_heads(rowptr, col, w, src, H, mode, emap, rate, 77, 0.5, None, None)
    got = ops.spmm_heads(csr, dev(w), dev(src), H, mode=code, emap=None if emap is None else dev(emap), drop_rate=rate,
                         seed=77, alpha=0.5)
    np.testing.assert_array_equal(host(got), want)
    want = o.spmm_heads(rowptr, col, w, src, H, mode, emap, rate, 77, 1.0, bias, "relu")
    got = ops.spmm_heads(csr, dev(w), dev(src), H, mode=code, emap=None if emap is None else dev(emap), drop_rate=rate,
                         seed=77, bias=dev(bias), act=ops.ACT_RELU)
    assert_close(host(got), want, rtol=1e-6, atol_scale=1e-7, what="spmm_heads bias+relu")


@pytest.mark.parametrize("H,dv,split,rate", [(8, 16, True, 0.0), (8, 16, True, 0.3), (4, 32, True, 0.0), (32, 4, True, 0.0),
                                             (1, 128, True, 0.2), (3, 5, True, 0.0), (4, 12, False, 0.0),
                                             (2, 7, False, 0.5)])
def test_gat_softmax_bwd_matches_restatement(H, dv, split, rate):
    rs = np.random.RandomState(H + dv)
    n = 400
    ei = random_graph(n, 3000, seed=H, isolated=2)
    csr, rowptr, col, _ = _csr_of(ei, n)
    rows = np.repeat(np.arange(n), np.diff(rowptr)).astype(np.int32)
    att = np.stack([o.segment_softmax((rs.randn(ei.shape[1]) * 2).astype(np.float32), rows, n) for _ in range(H)], axis=1)
    G = rs.randn(n, H * dv if split else dv).astype(np.float32)
    V = rs.randn(n, H * dv).astype(np.float32)
    want = o.gat_softmax_bwd(rowptr, col, att, G, V, H, split, rate, 5)
    got = ops.gat_softmax_bwd(csr, dev(att), dev(G), dev(V), H, split_value_heads=split, drop_rate=rate, seed=5)
    assert_close(host(got), want, rtol=1e-4, atol_scale=1e-5, what="gat_softmax_bwd")


# ---- whole-layer gradients against autograd over the reference port -------------------------------------------------

def _port_gat(x, ei_loops, params, H, relu, split, att_scale=None):
    t = [torch.tensor(np.asarray(p, np.float64), requires_grad=True) for p in params]
    row, col = torch.from_numpy(ei_loops[0].astype(np.int64)), torch.from_numpy(ei_loops[1].astype(np.int64))
    x64 = torch.tensor(x.astype(np.float64), requires_grad=True)
    y = port.gat_forward(x64, row, col, t[0], t[1], t[2], t[3], t[4], t[5], H, relu=relu,
                         split_value_heads=split, att_scale=None if att_scale is None else torch.tensor(att_scale))
    return y, t, x64


# path: "recompute" = stats forward + tfgk_gat_bwd_* (heads split, V as wide as Q/K, no dropout, no hub row, H <= 8);
#       "table"     = coefficient table + tfgk_gat_softmax_bwd_f32 + spmm_heads (everything else)
# the first five rows keep the ids they had before `hub` and `path` were parameters
@pytest.mark.parametrize("f,a,u,H,split,relu,rate,hub,path", [
    pytest.param(24, 64, 128, 8, True, True, 0.0, False, "table", id="24-64-128-8-True-True-0.0"),   # V wider than Q/K
    pytest.param(24, 64, 128, 8, True, True, 0.4, False, "table", id="24-64-128-8-True-True-0.4"),   # attention dropout
    pytest.param(10, 12, 20, 4, True, False, 0.0, False, "table", id="10-12-20-4-True-False-0.0"),
    pytest.param(10, 12, 6, 3, False, True, 0.0, False, "table", id="10-12-6-3-False-True-0.0"),      # averaged heads
    pytest.param(10, 12, 6, 3, False, False, 0.3, False, "table", id="10-12-6-3-False-False-0.3"),
    (24, 64, 64, 8, True, True, 0.0, False, "recompute"),      # GAT(64, num_heads=8), attention_units = units
    (24, 128, 128, 8, True, True, 0.0, False, "recompute"),    # GAT(128, num_heads=8)
    (16, 32, 32, 4, True, False, 0.0, False, "recompute"),     # no output activation
    (16, 32, 32, 4, True, True, 0.0, True, "table"),           # a hub destination row: the forward has a hub plan
    (24, 64, 64, 16, True, True, 0.0, False, "table"),         # GAT(64, num_heads=16): more heads than the backward packs
    (24, 128, 128, 32, True, True, 0.0, False, "table")])      # GAT(128, num_heads=32)
def test_gat_gradients_match_reference_autodiff(f, a, u, H, split, relu, rate, hub, path):
    rs = np.random.RandomState(f + a + u)
    n = 350
    ei = random_graph(n, 2600, seed=a, symmetric=True, isolated=2, hub=(5, ops.HUB_THRESHOLD + 100) if hub else None)
    x = rs.randn(n, f).astype(np.float32)
    v_units = u if split else u * H
    params = [glorot(rs, f, a), rs.randn(a).astype(np.float32) * .1, glorot(rs, f, a), rs.randn(a).astype(np.float32) * .1,
              glorot(rs, f, v_units), rs.randn(u).astype(np.float32) * .1]
    gout = rs.randn(n, u).astype(np.float32)
    seed = 99

    ei_dev = dev(ei, torch.int32)
    tp = [dev(p).requires_grad_(True) for p in params]
    xd = dev(x).requires_grad_(True)
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    try:
        y = tfg.nn.gat(xd, ei_dev, tp[0], tp[1], tfg.nn.relu, tp[2], tp[3], tfg.nn.relu, tp[4], tp[5],
                       tfg.nn.relu if relu else None, num_heads=H, split_value_heads=split, edge_drop_rate=rate,
                       training=True, seed=seed)
        (y * dev(gout)).sum().backward()
    finally:
        _ffi.set_trace(prev)
    recompute, table = trace.counts.get("tfgk_gat_bwd_dst_f32", 0), trace.counts.get("tfgk_gat_softmax_bwd_f32", 0)
    if path == "recompute":
        assert recompute == 1 and table == 0, trace.counts
    elif path == "table":
        assert table == 1 and recompute == 0, trace.counts
    else:
        assert path is None and not trace.counts          # host-logic tests: fake kernels that never reach the C ABI

    ei_loops = o.add_self_loop_edge(ei, n)[0]
    att_scale = None
    if rate > 0.0:
        # the product draws the mask per (forward-CSR position, head); the port wants it per virtual edge, head-major
        csr, _ = _structure.csr_for_edge_index(ei_dev, n, add_self_loop=True)
        perm = host(csr.perm).astype(np.int64)
        mult_csr = o.dropout_scale(ei_loops.shape[1] * H, rate, seed).reshape(-1, H)
        mult = np.empty_like(mult_csr)
        mult[perm] = mult_csr
        att_scale = mult.T.reshape(-1).astype(np.float64)
    y_ref, t, x64 = _port_gat(x, ei_loops, params, H, relu, split, att_scale)
    (y_ref * torch.tensor(gout.astype(np.float64))).sum().backward()

    assert_close(host(y), y_ref.detach().numpy(), what="gat training forward")
    for name, mine, ref in zip(("query_kernel", "query_bias", "key_kernel", "key_bias", "kernel", "bias", "x"), tp + [xd],
                               t + [x64]):
        assert mine.grad is not None, name
        assert_close(host(mine.grad), ref.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what="d loss / d " + name)


def test_gat_layer_learns():
    rs = np.random.RandomState(3)
    n, f, classes = 400, 16, 4
    ei = random_graph(n, 3000, seed=4, symmetric=True)
    labels = rs.randint(0, classes, n)
    x = (rs.randn(n, f) * 0.3 + np.eye(classes)[labels].repeat(f // classes, axis=1)).astype(np.float32)
    layer = tfg.layers.GAT(classes, attention_units=16, num_heads=4, edge_drop_rate=0.2, seed=1, trainable=True)
    xd, eid, target = dev(x), dev(ei, torch.int32), dev(labels.astype(np.int64))
    layer([xd, eid])
    opt = torch.optim.Adam(layer.parameters(), lr=0.02)
    losses = []
    for _ in range(25):
        opt.zero_grad()
        loss = torch.nn.functional.cross_entropy(layer([xd, eid], training=True), target)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < 0.6 * losses[0], losses
    before = host(layer([xd, eid]))
    np.testing.assert_array_equal(host(layer([xd, eid])), before)          # inference: no dropout, deterministic


def test_gcn_edge_dropout_forward_and_gradients():
    rs = np.random.RandomState(8)
    n, f, u, rate, seed = 500, 20, 12, 0.35, 4242
    ei = random_graph(n, 4000, seed=9, symmetric=True, isolated=1)
    w = (rs.rand(ei.shape[1]) + .2).astype(np.float32)
    x, k, b = rs.randn(n, f).astype(np.float32), glorot(rs, f, u), rs.randn(u).astype(np.float32)
    normed = o.gcn_norm_adj(o.SparseMatrix(ei, w, [n, n]))
    dropped = o.dropout(normed.value, rate, seed)
    adj = tfg.SparseMatrix(ei, w, [n, n])
    mine = tfg.nn.gcn_norm_adj(adj).dropout(rate, training=True, seed=seed)
    np.testing.assert_array_equal(host(mine.index), normed.index)
    assert_close(host(mine.value), dropped, rtol=6e-7, atol_scale=0, what="dropped adjacency values")
    assert tfg.nn.gcn_norm_adj(adj).dropout(rate, training=False) is not None

    kd, bd = dev(k).requires_grad_(True), dev(b).requires_grad_(True)
    tfg.set_seed(11)
    y = tfg.nn.gcn(dev(x), adj, kd, bd, tfg.nn.relu, edge_drop_rate=rate, training=True)
    gout = rs.randn(n, u).astype(np.float32)
    (y * dev(gout)).sum().backward()
    tfg.set_seed(11)
    from tf_geometric_b200 import _rng
    used = o.dropout(normed.value, rate, _rng.next_seed())
    kt, bt = torch.tensor(k.astype(np.float64), requires_grad=True), torch.tensor(b.astype(np.float64), requires_grad=True)
    y_ref = port.gcn_forward(torch.tensor(x.astype(np.float64)), torch.from_numpy(normed.index[0].astype(np.int64)),
                             torch.from_numpy(normed.index[1].astype(np.int64)), torch.tensor(used.astype(np.float64)), kt, bt)
    (y_ref * torch.tensor(gout.astype(np.float64))).sum().backward()
    assert_close(host(y), y_ref.detach().numpy(), what="gcn with edge dropout")
    assert_close(host(kd.grad), kt.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what="d kernel")
    assert_close(host(bd.grad), bt.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what="d bias")


def test_appnp_training_gradients_and_dense_dropout():
    rs = np.random.RandomState(12)
    n, f, hdim, u, k, alpha = 300, 14, 10, 5, 4, 0.15
    ei = random_graph(n, 2400, seed=13, symmetric=True)
    w = (rs.rand(ei.shape[1]) + .2).astype(np.float32)
    x = rs.randn(n, f).astype(np.float32)
    ks, bs = [glorot(rs, f, hdim), glorot(rs, hdim, u)], [rs.randn(hdim).astype(np.float32), rs.randn(u).astype(np.float32)]
    gout = rs.randn(n, u).astype(np.float32)
    kd, bd = [dev(a).requires_grad_(True) for a in ks], [dev(a).requires_grad_(True) for a in bs]
    y = tfg.nn.appnp(dev(x), dev(ei, torch.int32), dev(w), kd, bd, k=k, alpha=alpha, training=True)
    assert_close(host(y), o.appnp(x, ei, w, ks, bs, k=k, alpha=alpha), what="appnp training forward")
    (y * dev(gout)).sum().backward()

    normed = o.gcn_norm_adj(o.SparseMatrix(ei, w, [n, n]))
    kt = [torch.tensor(a.astype(np.float64), requires_grad=True) for a in ks]
    bt = [torch.tensor(a.astype(np.float64), requires_grad=True) for a in bs]
    row, col = torch.from_numpy(normed.index[0].astype(np.int64)), torch.from_numpy(normed.index[1].astype(np.int64))
    val = torch.tensor(normed.value.astype(np.float64))
    h = torch.relu(torch.tensor(x.astype(np.float64)) @ kt[0] + bt[0]) @ kt[1] + bt[1]
    out = h
    for _ in range(k):
        out = port.spmm(row, col, val, out, n) * (1.0 - alpha) + h * alpha
    (out * torch.tensor(gout.astype(np.float64))).sum().backward()
    for name, mine, ref in (("k0", kd[0], kt[0]), ("k1", kd[1], kt[1]), ("b0", bd[0], bt[0]), ("b1", bd[1], bt[1])):
        assert_close(host(mine.grad), ref.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what="appnp d " + name)

    # dense dropout: a fraction of the hidden units is zeroed, the survivors are scaled, inference is untouched
    tfg.set_seed(5)
    y_drop = tfg.nn.appnp(dev(x), dev(ei, torch.int32), dev(w), [dev(a) for a in ks], [dev(a) for a in bs], k=0,
                          last_dense_drop_rate=0.5, training=True)
    y_plain = host(tfg.nn.appnp(dev(x), dev(ei, torch.int32), dev(w), [dev(a) for a in ks], [dev(a) for a in bs], k=0,
                                last_dense_drop_rate=0.5, training=False))
    yd = host(y_drop)
    kept = yd != 0
    assert 0.35 < kept.mean() < 0.65
    assert_close(yd[kept], (y_plain * 2)[kept], rtol=1e-6, atol_scale=0, what="kept units are scaled by 1/(1-rate)")


# ---- drop_edge and the samplers --------------------------------------------------------------------------------------

@pytest.mark.parametrize("force_undirected", [False, True])
def test_drop_edge_matches_oracle(force_undirected):
    rs = np.random.RandomState(21)
    n = 600
    ei = random_graph(n, 20000, seed=22, symmetric=True)
    w = rs.rand(ei.shape[1]).astype(np.float32)
    tag = np.arange(ei.shape[1], dtype=np.int32)
    feat = rs.randn(3, ei.shape[1]).astype(np.float32)
    want = o.drop_edge([ei, w, tag, feat], 0.3, force_undirected, True, seed=17)
    got = tfg.nn.drop_edge([dev(ei, torch.int32), dev(w), dev(tag), dev(feat)], 0.3, force_undirected, True, seed=17)
    for g, e in zip(got, want):
        np.testing.assert_array_equal(host(g), e)
    if force_undirected:
        gi = host(got[0])
        half = gi.shape[1] // 2
        np.testing.assert_array_equal(gi[:, half:], gi[::-1, :half])
        assert (gi[0, :half] < gi[1, :half]).all()
    else:
        assert abs(host(got[0]).shape[1] / ei.shape[1] - 0.7) < 0.02
    # inference and the host (numpy) container
    same = tfg.nn.drop_edge([ei, w], 0.3, force_undirected, False)
    assert same[0] is ei and same[1] is w
    got_np = tfg.nn.drop_edge([ei, w], 0.3, force_undirected, True, seed=17)
    assert isinstance(got_np[0], np.ndarray) and isinstance(got_np[1], np.ndarray)
    np.testing.assert_array_equal(got_np[0], want[0])
    np.testing.assert_array_equal(got_np[1], want[1])
    with pytest.raises(ValueError):
        tfg.nn.drop_edge([ei], 1.5, training=True)
    assert host(tfg.nn.drop_edge([dev(ei, torch.int32)], 1.0, training=True)[0]).shape == (2, 0)


def test_uniform_neighbor_sampler_matches_oracle():
    rs = np.random.RandomState(31)
    n = 500
    ei = random_graph(n, 12000, seed=32)
    w = rs.rand(ei.shape[1]).astype(np.float32)
    sampler = tfg.utils.UniformNeighborSampler(dev(ei, torch.int32), dev(w))
    gi, gw = sampler.sample(0.25, seed=3)
    wi, ww = o.uniform_neighbor_sample(ei, w, 0.25, seed=3)
    np.testing.assert_array_equal(host(gi), wi)
    np.testing.assert_array_equal(host(gw), ww)
    assert abs(wi.shape[1] / ei.shape[1] - 0.25) < 0.02
    subset = rs.permutation(n)[:200].astype(np.int32)
    gi, gw = sampler.sample(0.5, sampled_node_index=subset, seed=4)
    wi, ww = o.uniform_neighbor_sample(ei, w, 0.5, subset, seed=4)
    np.testing.assert_array_equal(host(gi), wi)
    np.testing.assert_array_equal(host(gw), ww)
    rows, cols = rs.permutation(n)[:150].astype(np.int32), rs.permutation(n)[:300].astype(np.int32)
    gi, gw = sampler.sample(1.0, sampled_node_index=(rows, cols), seed=4)
    wi, ww = o.uniform_neighbor_sample(ei, w, 1.0, (rows, cols), seed=4)
    np.testing.assert_array_equal(host(gi), wi)
    np.testing.assert_array_equal(host(gw), ww)
    assert wi[0].max() < 150 and wi[1].max() < 300


def _check_sample_semantics(ei, w, si, sw, k, ratio, padding):
    """What the reference guarantees whatever its generator draws (graph_utils.py:741-756)."""
    deg = np.bincount(ei[0], minlength=int(ei[0].max()) + 1)
    weight_of = {}
    for (r, c), ww in zip(ei.T, w):
        weight_of.setdefault((int(r), int(c)), set()).add(float(ww))
    for (r, c), ww in zip(si.T, sw):
        assert float(ww) in weight_of[(int(r), int(c))]                    # every sample is a real (edge, weight) pair
    assert (np.diff(si[0]) >= 0).all()                                     # rows come out in ascending order
    cnt = np.bincount(si[0], minlength=len(deg))
    for r in np.nonzero(deg)[0]:
        if ratio is not None:
            expect = int(np.ceil(deg[r] * ratio))
        elif k is None:
            expect = deg[r]
        else:
            expect = k if (padding or k < deg[r]) else deg[r]
        assert cnt[r] == expect, (r, cnt[r], expect)
    assert cnt[deg == 0].sum() == 0


@pytest.mark.parametrize("k,ratio,padding", [(None, None, False), (5, None, False), (5, None, True), (40, None, True),
                                             (1, None, False), (None, 0.3, False), (None, 1.0, False)])
def test_random_neighbor_sampler_matches_oracle(k, ratio, padding):
    rs = np.random.RandomState(41)
    n = 400
    ei = random_graph(n, 6000, seed=42, isolated=3, hub=(7, 300))
    ei = np.concatenate([ei[:, ei[0] != 11], ], axis=1)                     # node 11 has no neighbours
    w = rs.rand(ei.shape[1]).astype(np.float32)
    sampler = tfg.utils.RandomNeighborSampler(dev(ei, torch.int32), dev(w))
    gi, gw = sampler.sample(k=k, ratio=ratio, padding=padding, seed=123)
    wi, ww = o.random_neighbor_sample(ei, w, k=k, ratio=ratio, padding=padding, seed=123)
    np.testing.assert_array_equal(host(gi), wi)
    np.testing.assert_array_equal(host(gw), ww)
    _check_sample_semantics(ei, w, wi, ww, k, ratio, padding)
    if k == 5 and not padding:                                              # without replacement: no slot drawn twice
        rowptr, _, perm = o.csr_build(ei[0], ei[1], int(ei[0].max()) + 1)
        _, pos, _ = o.neighbor_sample_csr(rowptr, k, None, False, 123)
        assert len(np.unique(pos)) == len(pos)
        other, _ = sampler.sample(k=k, seed=124)
        assert not np.array_equal(host(other), wi)
    subset = rs.permutation(n)[:120].astype(np.int32)
    gi, gw = sampler.sample(k=k, ratio=ratio, padding=padding, sampled_node_index=subset, seed=9)
    wi, ww = o.random_neighbor_sample(ei, w, k=k, ratio=ratio, padding=padding, seed=9, sampled_node_index=subset)
    if wi is None:
        assert gi is None and gw is None
    else:
        np.testing.assert_array_equal(host(gi), wi)
        np.testing.assert_array_equal(host(gw), ww)
        assert wi.max() < 120
    with pytest.raises(Exception):
        sampler.sample(k=3, ratio=0.5)


# ---- every other convolution trains through the same autograd Functions ---------------------------------------------------

def _t64(a, grad=True):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=grad)


def _spmm64(index, value, h, n):
    return port.spmm(torch.from_numpy(index[0].astype(np.int64)), torch.from_numpy(index[1].astype(np.int64)),
                     torch.tensor(np.asarray(value, np.float64)), h, n)


@pytest.mark.parametrize("name", ["sgc", "ssgc", "tagcn", "gin", "le_conv", "chebynet", "gcn_graph_sage",
                                  "mean_pool_graph_sage", "max_pool_graph_sage"])
def test_conv_training_gradients_match_autodiff(name):
    """Loss gradients of the remaining convolutions against float64 torch autograd over the reference's op sequence."""
    rs = np.random.RandomState(sum(map(ord, name)))
    n, f, u = 320, 9, 6
    ei = random_graph(n, 2400, seed=len(name), symmetric=True, isolated=1)
    if name == "max_pool_graph_sage":
        # every node needs an in-edge here: an empty max is float32 lowest (reference semantics, asserted in
        # test_gpu_models), which overflows in the projection that follows and says nothing about gradients
        ring = np.arange(n, dtype=ei.dtype)
        ei = np.concatenate([ei[:, :ei.shape[1] // 2], np.stack([ring, np.roll(ring, 1)]),
                             ei[:, ei.shape[1] // 2:], np.stack([np.roll(ring, 1), ring])], axis=1)
    w = (rs.rand(ei.shape[1]) + 0.2).astype(np.float32)
    half = ei.shape[1] // 2
    w[half:] = w[:half]                                             # symmetric weights (chebynet's Laplacian)
    x = rs.randn(n, f).astype(np.float32)
    eid, wd = dev(ei, torch.int32), dev(w)
    relu = tfg.nn.relu
    P = {}                                                          # name -> numpy parameter

    def run(mine, ref, grad_x=False):
        gout = None
        tp = {k: dev(v).requires_grad_(True) for k, v in P.items()}
        xd = dev(x).requires_grad_(grad_x)
        y = mine(xd, tp)
        gout = rs.randn(*y.shape).astype(np.float32)
        (y * dev(gout)).sum().backward()
        t64 = {k: _t64(v) for k, v in P.items()}
        x64 = _t64(x, grad_x)
        y_ref = ref(x64, t64)
        (y_ref * torch.tensor(gout.astype(np.float64))).sum().backward()
        assert_close(host(y), y_ref.detach().numpy(), what=name + " forward (training path)")
        for k in P:
            assert tp[k].grad is not None, k
            assert_close(host(tp[k].grad), t64[k].grad.numpy(), rtol=1e-3, atol_scale=2e-4, what=name + " d " + k)
        if grad_x:
            assert_close(host(xd.grad), x64.grad.numpy(), rtol=1e-3, atol_scale=2e-4, what=name + " d x")

    def normed(renorm=True, improved=False, weights=w):
        m = o.gcn_norm_adj(o.SparseMatrix(ei, weights, [n, n]), renorm=renorm, improved=improved)
        return m.index, m.value

    if name == "sgc":
        P.update(k=glorot(rs, f, u), b=rs.randn(u).astype(np.float32))
        ai, av = normed()
        run(lambda xd, p: tfg.nn.sgc(xd, eid, wd, 2, p["k"], p["b"], relu),
            lambda x64, p: torch.relu(_spmm64(ai, av, _spmm64(ai, av, x64 @ p["k"], n), n) + p["b"]))
    elif name == "ssgc":
        P.update(k0=glorot(rs, f, 8), b0=rs.randn(8).astype(np.float32), k1=glorot(rs, 8, u), b1=rs.randn(u).astype(np.float32))
        ai, av = normed()

        def ref(x64, p):
            h = torch.relu(x64 @ p["k0"] + p["b0"]) @ p["k1"] + p["b1"]
            out = h * 0.2
            for _ in range(3):
                h = _spmm64(ai, av, h, n)
                out = out + (1 - 0.2) * h / 3
            return out
        run(lambda xd, p: tfg.nn.ssgc(xd, eid, wd, [p["k0"], p["k1"]], [p["b0"], p["b1"]], k=3, alpha=0.2), ref)
    elif name == "tagcn":
        P.update(k=glorot(rs, 3 * f, u), b=rs.randn(u).astype(np.float32))
        ai, av = normed(renorm=False)

        def ref(x64, p):
            a1 = _spmm64(ai, av, x64, n)
            return torch.relu(torch.cat([x64, a1, _spmm64(ai, av, a1, n)], dim=1) @ p["k"] + p["b"])
        run(lambda xd, p: tfg.nn.tagcn(xd, eid, wd, 2, p["k"], p["b"], relu), ref, grad_x=True)
    elif name == "gin":
        from tf_geometric_b200 import autograd
        P.update(m=glorot(rs, f, u), eps=np.array([0.3], np.float32))
        ones = np.ones(ei.shape[1], np.float32)
        run(lambda xd, p: tfg.nn.gin(xd, eid, lambda h, training=None: autograd.dense(h, p["m"], None, relu), eps=p["eps"]),
            lambda x64, p: torch.relu((x64 * (1.0 + p["eps"]) + _spmm64(ei, ones, x64, n)) @ p["m"]), grad_x=True)
    elif name == "le_conv":
        for k_ in ("ws", "wa", "wn"):
            P[k_] = glorot(rs, f, u)
        for k_ in ("bs", "ba", "bn"):
            P[k_] = rs.randn(u).astype(np.float32)
        run(lambda xd, p: tfg.nn.le_conv(xd, eid, wd, p["ws"], p["bs"], p["wa"], p["ba"], p["wn"], p["bn"], relu),
            lambda x64, p: torch.relu(_spmm64(ei, w, (x64 @ p["wa"] + p["ba"]) - (x64 @ p["wn"] + p["bn"]), n)
                                      + x64 @ p["ws"] + p["bs"]), grad_x=True)
    elif name == "chebynet":
        P.update(k0=glorot(rs, f, u), k1=glorot(rs, f, u), k2=glorot(rs, f, u), b=rs.randn(u).astype(np.float32))
        li, lv = o.chebynet_norm_edge(ei, n, w, "sym")

        def ref(x64, p):
            t0 = x64
            out = t0 @ p["k0"]
            t1 = _spmm64(li, lv, t0, n)
            out = out + t1 @ p["k1"]
            t2 = _spmm64(li, lv, t1, n) * 2.0 - t0
            return torch.relu(out + t2 @ p["k2"] + p["b"])
        run(lambda xd, p: tfg.nn.chebynet(xd, eid, wd, 3, [p["k0"], p["k1"], p["k2"]], p["b"], relu), ref)
    elif name == "gcn_graph_sage":
        P.update(k=glorot(rs, f, u), b=rs.randn(u).astype(np.float32))
        ai, av = normed(renorm=False, weights=np.ones_like(w))     # quirks: weights -> ones, cache=None -> renorm=False
        run(lambda xd, p: tfg.nn.gcn_graph_sage(xd, eid, wd, p["k"], p["b"], relu),
            lambda x64, p: torch.relu(_spmm64(ai, av, x64, n) @ p["k"] + p["b"]), grad_x=True)
    elif name == "max_pool_graph_sage":
        P.update(ws=glorot(rs, f, u), wm=glorot(rs, f, 8), wn=glorot(rs, 8, u), bm=rs.randn(8).astype(np.float32),
                 b=rs.randn(2 * u).astype(np.float32))
        row64 = torch.from_numpy(ei[0].astype(np.int64)).unsqueeze(1).expand(-1, 8)
        col64 = torch.from_numpy(ei[1].astype(np.int64))

        def ref(x64, p):
            h_node = torch.relu(x64 @ p["wm"] + p["bm"])
            red = torch.zeros((n, 8), dtype=torch.float64).scatter_reduce(0, row64, h_node[col64], "amax", include_self=False)
            return torch.relu(torch.cat([x64 @ p["ws"], red @ p["wn"]], dim=1) + p["b"])
        run(lambda xd, p: tfg.nn.max_pool_graph_sage(xd, eid, wd, p["ws"], p["wm"], p["wn"], p["bm"], p["b"], relu), ref,
            grad_x=True)
    else:
        P.update(ws=glorot(rs, f, u), wm=glorot(rs, f, 8), wn=glorot(rs, 8, u), bm=rs.randn(8).astype(np.float32),
                 b=rs.randn(2 * u).astype(np.float32))
        cnt = np.maximum(np.bincount(ei[0], minlength=n), 1).astype(np.float64)

        def ref(x64, p):
            h_node = torch.relu(x64 @ p["wm"] + p["bm"])
            red = _spmm64(ei, np.ones(ei.shape[1]), h_node, n) / torch.tensor(cnt).unsqueeze(1)
            return torch.relu(torch.cat([x64 @ p["ws"], red @ p["wn"]], dim=1) + p["b"])
        run(lambda xd, p: tfg.nn.mean_pool_graph_sage(xd, eid, wd, p["ws"], p["wm"], p["wn"], p["bm"], p["b"], relu), ref)


def test_every_trainable_layer_gets_gradients():
    """trainable=True layers: one forward+backward each, every registered weight receives a finite, non-zero gradient."""
    rs = np.random.RandomState(2)
    n, f = 200, 10
    ei = random_graph(n, 1500, seed=3, symmetric=True)
    xd, eid, wd = dev(rs.randn(n, f).astype(np.float32)), dev(ei, torch.int32), dev((rs.rand(ei.shape[1]) + .2).astype(np.float32))
    L = tfg.layers
    cases = [
        (L.GCN(8, activation=tfg.nn.relu, seed=1, trainable=True), [xd, eid, wd]),
        (L.GAT(8, num_heads=2, activation=tfg.nn.relu, seed=1, trainable=True), [xd, eid]),
        (L.MeanGraphSage(8, seed=1, trainable=True), [xd, eid, wd]),
        (L.SumGraphSage(8, concat=False, seed=1, trainable=True), [xd, eid, wd]),
        (L.GCNGraphSage(8, seed=1, trainable=True), [xd, eid, wd]),
        (L.MeanPoolGraphSage(8, seed=1, trainable=True), [xd, eid, wd]),
        (L.MaxPoolGraphSage(8, seed=1, trainable=True), [xd, eid, wd]),
        (L.APPNP([12, 5], k=3, seed=1, trainable=True), [xd, eid, wd]),
        (L.SGC(6, k=2, seed=1, trainable=True), [xd, eid, wd]),
        (L.SSGC([12, 5], k=3, seed=1, trainable=True), [xd, eid, wd]),
        (L.TAGCN(6, k=2, seed=1, trainable=True), [xd, eid, wd]),
        (L.LEConv(6, activation=tfg.nn.relu, seed=1, trainable=True), [xd, eid, wd]),
        (L.ChebyNet(6, k=3, seed=1, trainable=True), [xd, eid, wd]),
    ]
    for layer, inputs in cases:
        out = layer(inputs, training=True)
        assert out.requires_grad, type(layer).__name__
        (out * out).sum().backward()
        params = dict(layer.named_parameters())
        assert params, type(layer).__name__
        for pname, p in params.items():
            assert p.grad is not None and torch.isfinite(p.grad).all(), "{}.{}".format(type(layer).__name__, pname)
            if "bias" not in pname:
                assert float(p.grad.abs().sum()) > 0, "{}.{}".format(type(layer).__name__, pname)


def test_every_pool_layer_passes_gradients():
    """Round-1 advisory: pooling / reducers cut the autograd graph silently.  Gradients of the four graph poolings, the stock
    reducers, the fused aggregate_neighbors routes and of a GCN -> SAGPool -> MeanPool model against float64 autograd over
    plain torch ops."""
    rs = np.random.RandomState(3)
    n, graphs, d = 400, 9, 6
    gi = np.sort(rs.randint(0, graphs - 1, n)).astype(np.int32)          # the last graph stays empty
    x = rs.randn(n, d).astype(np.float32)
    x[5] = x[6]                                                          # a tie inside one graph for max / min
    gi[5] = gi[6]
    g = rs.randn(graphs, d).astype(np.float32)
    gid = dev(gi, torch.int32)
    seg = torch.from_numpy(gi.astype(np.int64))
    for name in ("sum", "mean", "max", "min"):
        xd = dev(x).requires_grad_(True)
        out = getattr(tfg.nn, name + "_pool")(xd, gid, graphs)
        (out * dev(g)).sum().backward()
        x64 = torch.from_numpy(x).double().requires_grad_(True)
        if name in ("sum", "mean"):
            ref = torch.zeros((graphs, d), dtype=torch.float64).index_add_(0, seg, x64)
            if name == "mean":
                ref = ref / torch.bincount(seg, minlength=graphs).clamp(min=1).double().unsqueeze(1)
        else:
            ref = torch.zeros((graphs, d), dtype=torch.float64).scatter_reduce(
                0, seg.unsqueeze(1).expand(-1, d), x64, reduce="amax" if name == "max" else "amin", include_self=False)
        (ref * torch.from_numpy(g).double()).sum().backward()
        assert xd.grad is not None, name + "_pool returned no gradient"
        assert_close(host(xd.grad), x64.grad.numpy(), rtol=1e-5, atol_scale=1e-6, what=name + "_pool gradient")
    # fused aggregate_neighbors routes with a differentiable input
    ei = random_graph(n, 3000, seed=4)
    w = (rs.rand(ei.shape[1]) + 0.1).astype(np.float32)
    gg = rs.randn(n, d).astype(np.float32)
    row, col = torch.from_numpy(ei[0].astype(np.int64)), torch.from_numpy(ei[1].astype(np.int64))
    for reducer, red in ((tfg.nn.sum_reducer, "sum"), (tfg.nn.mean_reducer, "mean"), (tfg.nn.max_reducer, "max")):
        xd = dev(x).requires_grad_(True)
        out = tfg.nn.aggregate_neighbors(xd, dev(ei, torch.int32), dev(w), tfg.nn.gcn_mapper, reducer, tfg.nn.sum_updater)
        (out * dev(gg)).sum().backward()
        x64 = torch.from_numpy(x).double().requires_grad_(True)
        msg = x64[col] * torch.from_numpy(w).double().unsqueeze(1)
        if red == "max":
            agg = torch.full((n, d), float(np.finfo(np.float32).min), dtype=torch.float64).scatter_reduce(
                0, row.unsqueeze(1).expand(-1, d), msg, reduce="amax", include_self=True)
        else:
            agg = torch.zeros((n, d), dtype=torch.float64).index_add_(0, row, msg)
            if red == "mean":
                agg = agg / torch.bincount(row, minlength=n).clamp(min=1).double().unsqueeze(1)
        ((x64 + agg) * torch.from_numpy(gg).double()).sum().backward()
        assert_close(host(xd.grad), x64.grad.numpy(), rtol=1e-5, atol_scale=1e-5, what="aggregate_neighbors({}) gradient".format(red))
    # a small trainable model: conv -> SAGPool -> MeanPool -> loss; every weight must receive a gradient
    conv = tfg.layers.GCN(d, activation=tfg.nn.relu, seed=1, trainable=True)
    score = tfg.layers.GCN(1, seed=2, trainable=True)
    xd, eid, wd = dev(x), dev(ei, torch.int32), dev(w)
    gi2 = np.sort(rs.randint(0, graphs, n)).astype(np.int32)
    gi2[-1] = graphs - 1
    h = conv([xd, eid, wd])
    px, pei, pw, pgi = tfg.layers.SAGPool(score, ratio=0.5, score_activation=torch.tanh)([h, eid, wd, dev(gi2, torch.int32)])
    pooled = tfg.layers.MeanPool()([px, pgi, graphs])
    pooled.pow(2).sum().backward()
    for layer in (conv, score):
        for name, p in layer.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), name
    assert float(conv.kernel.grad.abs().max()) > 0 and float(score.kernel.grad.abs().max()) > 0
