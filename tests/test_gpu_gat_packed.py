# coding=utf-8
"""Packed keys for the fused GAT aggregation: tfgk_gat_pack_keys_f32 round-trips K bit for bit, and
tfgk_gat_fused_packed_f32 gives the output bits of tfgk_gat_fused_f32 (TMA ring over one [N, 2A] K | V buffer) for every
shape the ring takes, for keys with no, some or only zeros, for -0.0 / NaN / inf / denormal entries, empty rows, a hub row cut
into slices by the plan and every ring depth; the GAT layer's packed route matches TFGK_GAT_KEYS=dense."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from conftest import random_graph

pytestmark = pytest.mark.gpu

SHAPES = [(h, d) for h in (1, 2, 4, 8) for d in (4, 8, 16, 32) if h * d <= 128]
KINDS = ("zero", "nonzero", "relu", "special")


def bits(t):
    """int32 view: compares NaN payloads and signed zeros exactly."""
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def make_keys(kind, n, a, seed):
    rs = np.random.RandomState(seed)
    if kind == "zero":
        k = np.zeros((n, a), np.float32)
    elif kind == "nonzero":
        k = (rs.rand(n, a) + 0.5).astype(np.float32)
    elif kind == "relu":
        k = np.maximum(rs.randn(n, a), 0.0).astype(np.float32)
    else:
        k = np.maximum(rs.randn(n, a), 0.0).astype(np.float32)
        special = np.array([-0.0, np.nan, np.inf, -np.inf, 1e-40, -1e-42, 0.0], np.float32)
        pick = rs.rand(n, a) < 0.02
        k[pick] = special[rs.randint(0, len(special), int(pick.sum()))]
    return torch.from_numpy(k).cuda()


def csr_of(n, e, seed, isolated=0, hub=None):
    ei = torch.from_numpy(random_graph(n, e, seed=seed, isolated=isolated, hub=hub)).cuda()
    return ops.csr_build(ei[0].contiguous(), ei[1].contiguous(), n)


def dense_and_packed(K, V):
    n, a = K.shape
    kv = torch.empty((n, 2 * a), dtype=torch.float32, device="cuda")
    kv[:, :a] = K
    kv[:, a:] = V
    table, sizes = ops.packed_key_table(n, a, K.device)
    table[:, :a] = V
    ops.gat_pack_keys(K, table, sizes)
    return kv, table, sizes


def both(csr, Q, K, V, heads, bias=None, act=ops.ACT_NONE):
    kv, table, sizes = dense_and_packed(K, V)
    a = K.shape[1]
    want = ops.gat_fused(csr, Q, kv[:, :a], kv[:, a:], heads, bias=bias, act=act)
    got = ops.gat_fused_packed(csr, Q, table, sizes, heads, bias=bias, act=act)
    return want, got


@pytest.mark.parametrize("a", [4, 12, 64, 128])
@pytest.mark.parametrize("kind", KINDS)
def test_pack_keys_round_trip(a, kind):
    n = 777
    K = make_keys(kind, n, a, seed=a)
    V = torch.randn((n, a), device="cuda")
    _, table, sizes = dense_and_packed(K, V)
    assert table.shape[1] % 16 == 0 and table.shape[1] >= 2 * a + 4
    t = table.cpu().numpy()
    kb = K.cpu().numpy().view(np.uint32)
    sz = sizes.cpu().numpy().astype(np.int64)
    assert same_bits(table[:, :a], V)                                    # V untouched
    mask = t[:, a:a + 4].copy().view(np.uint32)
    for r in range(n):
        nz = kb[r] != 0
        want_mask = np.zeros(4, np.uint32)
        for c in np.nonzero(nz)[0]:
            want_mask[c // 32] |= np.uint32(1) << np.uint32(c % 32)
        assert np.array_equal(mask[r], want_mask), r
        cnt = int(nz.sum())
        padded = (cnt + 3) // 4 * 4
        assert sz[r] == (a + 4 + padded) // 4, r
        packed = t[r, a + 4:a + 4 + padded].copy().view(np.uint32)
        assert np.array_equal(packed[:cnt], kb[r][nz]), r                  # same bits, column order
        assert not packed[cnt:].any(), r                                   # zero padding
        rebuilt = np.zeros(a, np.uint32)
        rebuilt[nz] = packed[:cnt]
        assert np.array_equal(rebuilt, kb[r]), r


@pytest.mark.parametrize("heads,dqk", SHAPES)
def test_packed_k3_bit_identical_to_dense(heads, dqk):
    """Every (H, dqk) of the TMA ring, every kind of key, rows with no edges, bias and ReLU epilogue."""
    n, a = 1500, heads * dqk
    csr = csr_of(n, 30000, seed=heads * 100 + dqk, isolated=7)
    Q = torch.randn((n, a), device="cuda")
    V = torch.randn((n, a), device="cuda")
    bias = torch.randn((a,), device="cuda")
    for kind in KINDS:
        K = make_keys(kind, n, a, seed=dqk)
        for b, act in ((None, ops.ACT_NONE), (bias, ops.ACT_RELU)):
            want, got = both(csr, Q, K, V, heads, bias=b, act=act)
            assert same_bits(got, want), (kind, act)
            if kind == "special" and act == ops.ACT_NONE:
                assert torch.isnan(want).any()                             # the NaN keys reached the output


@pytest.mark.parametrize("kind", KINDS)
def test_packed_ring_hub_plan(kind):
    """A hub row of in-degree 60,000 is cut into slices by the plan; empty rows."""
    n, heads, a = 4000, 8, 128
    csr = csr_of(n, 50000, seed=11, isolated=5, hub=(17, 60000))
    assert csr.plan is not None and csr.plan.n_hubs >= 1
    Q = torch.randn((n, a), device="cuda")
    V = torch.randn((n, a), device="cuda")
    bias = torch.randn((a,), device="cuda")
    K = make_keys(kind, n, a, seed=3)
    want, got = both(csr, Q, K, V, heads, bias=bias, act=ops.ACT_RELU)
    assert same_bits(got, want), kind
    assert same_bits(ops.gat_fused_packed(csr, Q, *dense_and_packed(K, V)[1:], heads, bias=bias, act=ops.ACT_RELU), got)


def test_packed_refuses_other_shapes():
    n = 64
    csr = csr_of(n, 500, seed=1)
    Q = torch.randn((n, 256), device="cuda")
    table, sizes = ops.packed_key_table(n, 128, Q.device)
    with pytest.raises(_ffi.TfgkError):
        ops.gat_fused_packed(csr, Q, table, sizes, 8)                      # A = 256
    with pytest.raises(_ffi.TfgkError):
        ops.gat_fused_packed(csr, Q[:, :96], table, sizes, 8)              # dqk = 12: dqk / 4 is not a power of two
    with pytest.raises(_ffi.TfgkError):
        ops.gat_pack_keys(torch.zeros((n, 256), device="cuda"), table, sizes)


def _layer_run(layer, x, ei, graph_cache):
    trace = _ffi.CallTrace()
    _ffi.set_trace(trace)
    try:
        out = layer([x, ei], cache=graph_cache)
    finally:
        _ffi.set_trace(None)
    return out, trace.counts


@pytest.mark.parametrize("units,heads", [(128, 8), (64, 8), (32, 2)])
def test_gat_layer_packed_route_matches_dense(units, heads, monkeypatch):
    rs = np.random.RandomState(units)
    n = 6000
    ei = torch.from_numpy(random_graph(n, 80000, seed=units, symmetric=True, hub=(3, 5000))).cuda()
    x = torch.from_numpy(rs.randn(n, 100).astype(np.float32)).cuda()
    layer = tfg.layers.GAT(units, num_heads=heads, activation=tfg.nn.relu, seed=4)
    cache = {}
    monkeypatch.delenv("TFGK_GAT_KEYS", raising=False)
    got, counts = _layer_run(layer, x, ei, cache)
    assert counts.get("tfgk_gat_fused_packed_f32") == 1 and counts.get("tfgk_gat_pack_keys_f32") == 1
    assert counts.get("tfgk_gat_fused_f32", 0) == 0 and counts.get("tfgk_gemm_proj_f32") == 1
    again, _ = _layer_run(layer, x, ei, cache)
    assert same_bits(again, got)
    monkeypatch.setenv("TFGK_GAT_KEYS", "dense")
    want, counts = _layer_run(layer, x, ei, cache)
    assert counts.get("tfgk_gat_fused_f32") == 1 and counts.get("tfgk_gat_fused_packed_f32", 0) == 0
    assert same_bits(got, want)


def test_gat_layer_without_relu_keys_stays_dense():
    rs = np.random.RandomState(0)
    n = 500
    ei = torch.from_numpy(random_graph(n, 4000, seed=2)).cuda()
    x = torch.from_numpy(rs.randn(n, 16).astype(np.float32)).cuda()
    layer = tfg.layers.GAT(32, num_heads=4, key_activation=None, seed=1)
    _, counts = _layer_run(layer, x, ei, {})
    assert counts.get("tfgk_gat_fused_f32") == 1 and counts.get("tfgk_gat_fused_packed_f32", 0) == 0
