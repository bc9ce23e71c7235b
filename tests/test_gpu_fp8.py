# coding=utf-8
"""fp8 message rows for GCN and GAT inference on the H100: K4's fp8 blocks and tfgk_quantize_fp8 write the bytes and
exponents of the numpy restatement (tests/fp8_ref.py) bit for bit; K1 and K3 over fp8 rows equal the fp32 kernels over the
dequantised rows bit for bit; the layers hold their bounds and trained models keep their accuracy."""
import os
import sys

import numpy as np
import pytest
import torch

import fp8_ref
import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from conftest import random_graph, assert_close
from test_gpu_bf16 import same_bits, hub_csr, gat_f64, _gat_graph, _planted

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn


def dev(a, dtype=None):
    return ops.as_device(a, dtype)


def host(t):
    return t.detach().cpu().numpy()


def deq(t, groups=None):
    """x^ of an Fp8Table on the device (float32, exact): float(q) * 2^k, exponent column per 128 columns or `groups`."""
    v = t.data.contiguous().view(FP8).float()
    k = t.exps.float()
    cols = (torch.arange(t.cols, device=v.device) // 128) if groups is None else groups
    return v * torch.exp2(k[:, cols])


def padded_f32(x):
    """A float32 copy of x [n, d] inside a buffer of leading dimension d rounded up to 16 (the fp8 table's, in elements)."""
    ld = max(-(-x.shape[1] // 16) * 16, 16)
    buf = torch.zeros((x.shape[0], ld), dtype=torch.float32, device=x.device)
    buf[:, :x.shape[1]] = x
    return buf[:, :x.shape[1]]


def check_table(table, src):
    """bytes and exponents of `table` equal the restatement applied to the float32 values src."""
    q, k = fp8_ref.quantize(host(src))
    assert np.array_equal(host(table.data), q), "fp8 bytes differ"
    assert np.array_equal(host(table.exps)[:, :k.shape[1]], k), "exponents differ"


# ---- K4 and the standalone quantiser ---------------------------------------------------------------------------------

def _special_rows(x):
    """Rows of x whose projections are zero, tiny (clamped exponent), huge (inf after the sum) and NaN."""
    x[0] = 0.0
    x[1] *= 1e-38
    x[2] *= 3e37
    x[3, 0] = np.nan
    x[4] = 0.0
    x[4, 0] = 3e38
    return x


@pytest.mark.parametrize("k", [1, 4, 8, 100, 128, 184])
def test_gemm_proj_fp8_blocks_are_the_restatement_of_fp32(k):
    """K = 1 (lda not a multiple of 4) is refused by the tensor-core kernel and takes ops.gemm_proj's fallback, the fp32
    GEMM followed by tfgk_quantize_fp8; every other K here runs K4's fp8 epilogue."""
    m, n = 1000, 128
    rs = np.random.RandomState(k)
    x = dev(_special_rows(rs.randn(m, k).astype(np.float32)))
    w1, w2 = dev(rs.randn(k, n).astype(np.float32)), dev(rs.randn(k, 72).astype(np.float32))
    b1 = dev(rs.randn(n).astype(np.float32))
    q32 = torch.empty((m, n), device="cuda")
    ref1, ref2 = ops.gemm_proj(x, [(w1, b1, ops.ACT_RELU, None), (w2, None, ops.ACT_NONE, None)])
    t = ops.fp8_table(m, n + 72, "cuda", groups=2)
    ops.gemm_proj(x, [(w1, b1, ops.ACT_RELU, q32), (w1, b1, ops.ACT_RELU, t.block(0, n, group=0)),
                      (w2, None, ops.ACT_NONE, t.block(n, n + 72, group=1))])
    same_bits(q32, ref1)                                 # the fp32 block of a mixed launch is unchanged
    check_table(t.block(0, n, group=0), ref1)
    check_table(t.block(n, n + 72, group=1), ref2)


def test_quantize_fp8_special_values_and_wide_gemm():
    rs = np.random.RandomState(5)
    x = rs.randn(16, 300).astype(np.float32)
    x[0] = 0.0
    x[1] = -0.0
    x[2, :5] = [np.inf, -np.inf, np.nan, -0.0, 1.0]
    x[3] *= 1e-39                                         # amax below 448 * 2^-126: the exponent clamps at -126
    x[4] *= 1e38
    x[4, 7] = 3.4e38                                      # near FLT_MAX
    x[5, 128:256] = 0.0                                   # an all-zero group
    t = ops.quantize_fp8(dev(x))
    check_table(t, dev(x))
    assert t.exps.shape[1] == 3 and int(t.exps[3, 0]) == -126
    a = dev(rs.randn(700, 600).astype(np.float32))        # K = 600: past the tensor-core kernel
    w = dev(rs.randn(600, 200).astype(np.float32))
    y = ops.gemm(a, w)
    check_table(ops.quantize_fp8(y), y)
    t = ops.fp8_table(700, 200, "cuda")
    ops.gemm_proj(a, [(w[:, :128], None, ops.ACT_NONE, t.block(0, 128)), (w[:, 128:], None, ops.ACT_NONE, t.block(128, 200))])
    check_table(t, y)


# ---- K1 --------------------------------------------------------------------------------------------------------------

def fp8_rows(n, d, seed):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    x = torch.randn((n, d), generator=g) * torch.exp2(torch.randint(-6, 6, (n, 1), generator=g).float())
    return ops.quantize_fp8(x.cuda())


@pytest.mark.parametrize("d", [1, 3, 16, 32, 47, 64, 100, 128, 200, 256, 264])
@pytest.mark.parametrize("reduce", ["sum", "mean", "max"])
@pytest.mark.parametrize("weighted", [False, True])
def test_spmm_fp8_is_fp32_over_the_dequantised_table(d, reduce, weighted):
    n = 1500
    ei = random_graph(n, 20000, seed=d, isolated=7)               # 7 empty rows
    csr = ops.csr_build(dev(ei[0]), dev(ei[1]), n)
    rs = np.random.RandomState(d + 1)
    w = dev(rs.rand(csr.nnz).astype(np.float32) - 0.3) if weighted else None
    t = fp8_rows(n, d, d)
    xh = padded_f32(deq(t))
    epi = {}
    if d % 2:
        epi = dict(alpha=0.5, addend=dev(rs.randn(n, d).astype(np.float32)), beta=-1.5,
                   bias=dev(rs.randn(d).astype(np.float32)), act=ops.ACT_RELU)
    got = ops.spmm(csr, w, t, reduce=reduce, **epi)
    same_bits(got, ops.spmm(csr, w, xh, reduce=reduce, **epi))
    same_bits(got, ops.spmm(csr, w, t, reduce=reduce, **epi))     # identical bits across runs


@pytest.mark.parametrize("d", [32, 47, 100, 128, 256])
def test_spmm_fp8_hub_row_through_the_plan(d):
    csr, w, n = hub_csr()
    t = fp8_rows(n, d, 7)
    xh = padded_f32(deq(t))
    for reduce in ("sum", "mean", "max"):
        got = ops.spmm(csr, w, t, reduce=reduce, bias=dev(np.ones(d, np.float32)), act=ops.ACT_RELU)
        same_bits(got, ops.spmm(csr, w, xh, reduce=reduce, bias=dev(np.ones(d, np.float32)), act=ops.ACT_RELU))


def test_spmm_fp8_refuses_a_column_block_of_a_wider_table():
    """gemm_proj writes into block views, whose exponents are a strided column: the gather refuses them instead of reading
    other rows' exponents."""
    n = 500
    ei = random_graph(n, 4000, seed=2)
    csr = ops.csr_build(dev(ei[0]), dev(ei[1]), n)
    x = dev(np.random.RandomState(3).randn(n, 16).astype(np.float32))
    w = dev(np.random.RandomState(4).randn(16, 200).astype(np.float32))
    t = ops.fp8_table(n, 200, "cuda")
    ops.gemm_proj(x, [(w[:, :128], None, ops.ACT_NONE, t.block(0, 128)), (w[:, 128:], None, ops.ACT_NONE, t.block(128, 200))])
    with pytest.raises(ValueError, match="dense"):
        ops.spmm(csr, None, t.block(0, 128))
    same_bits(ops.spmm(csr, None, t), ops.spmm(csr, None, padded_f32(deq(t))))


def test_spmm_fp8_column_override():
    n, d = 2000, 128
    ei = random_graph(n, 30000, seed=21)
    csr = ops.csr_build(dev(ei[0]), dev(ei[1]), n)
    t = fp8_rows(n, d, 3)
    col = dev(np.random.RandomState(4).randint(0, n, csr.nnz).astype(np.int32))
    xh = padded_f32(deq(t))
    want = ops.spmm(csr, None, xh, col=col)
    same_bits(ops.spmm(csr, None, t, col=col), want)


# ---- K3 --------------------------------------------------------------------------------------------------------------

def kv_table(n, a, seed):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    k = torch.randn((n, a), generator=g).cuda()
    v = (torch.randn((n, a), generator=g) * 4).cuda()
    t = ops.fp8_table(n, 2 * a, "cuda", groups=2)
    ops.quantize_fp8(k, out=t.block(0, a, group=0))
    ops.quantize_fp8(v, out=t.block(a, 2 * a, group=1))
    groups = torch.cat([torch.zeros(a, dtype=torch.long), torch.ones(a, dtype=torch.long)]).cuda()
    return t, deq(t, groups)


@pytest.mark.parametrize("heads", [1, 2, 4, 8])
@pytest.mark.parametrize("dqk", [4, 8, 16, 32])
def test_gat_fp8_against_float64_and_fp32_ring(heads, dqk):
    a = heads * dqk
    if a > 128:
        pytest.skip("A > 128 is outside the fp8 ring")
    n = 700
    csr = _gat_graph(n, 9000, heads * 100 + dqk)
    g = torch.Generator(device="cpu")
    g.manual_seed(a)
    q = torch.randn((n, a), generator=g).cuda()
    bias = torch.randn((a,), generator=g).cuda()
    t, kvh = kv_table(n, a, a + 1)
    got = ops.gat_fused(csr, q, t, None, heads, bias=bias, act=ops.ACT_RELU)
    want = gat_f64(csr.rowptr, csr.col, q, kvh[:, :a], kvh[:, a:], heads, True, bias=bias, relu=True)
    # the bound the fp32 K3 is held to (tests/test_gpu_gat.py): 2e-5 relative plus 2e-6 of the largest |entry|
    assert_close(host(got), want, rtol=2e-5, atol_scale=2e-6, what="gat fp8")
    same_bits(got, ops.gat_fused(csr, q, t, None, heads, bias=bias, act=ops.ACT_RELU))
    same_bits(got, ops.gat_fused(csr, q, kvh[:, :a], kvh[:, a:], heads, bias=bias, act=ops.ACT_RELU))


def test_gat_fp8_hub_row_matches_the_fp32_ring():
    n, heads, a = 3000, 8, 128
    csr = _gat_graph(n, 40000, 11, hub=(100, 9000))
    assert csr.plan is not None and csr.plan.n_hubs >= 1
    q = torch.randn((n, a), generator=torch.Generator().manual_seed(3)).cuda()
    t, kvh = kv_table(n, a, 5)
    got = ops.gat_fused(csr, q, t, None, heads)
    want = gat_f64(csr.rowptr, csr.col, q, kvh[:, :a], kvh[:, a:], heads, True)
    assert_close(host(got), want, rtol=2e-5, atol_scale=2e-6, what="gat fp8 hub")
    same_bits(got, ops.gat_fused(csr, q, kvh[:, :a], kvh[:, a:], heads))


def test_gat_fp8_unsupported_shapes_raise():
    n = 300
    csr = _gat_graph(n, 2000, 1)
    q = torch.randn((n, 96), device="cuda")
    t = ops.fp8_table(n, 192, "cuda", groups=2)
    t.exps.zero_()
    t.data.zero_()
    with pytest.raises(_ffi.TfgkError) as err:
        ops.gat_fused(csr, q, t, None, 4)                     # dqk = 24: dqk / 4 is not a power of two
    assert err.value.code == _ffi.ERR_UNSUPPORTED
    q = torch.randn((n, 256), device="cuda")
    t = ops.fp8_table(n, 512, "cuda", groups=2)
    with pytest.raises(_ffi.TfgkError) as err:
        ops.gat_fused(csr, q, t, None, 8)                     # A = 256
    assert err.value.code == _ffi.ERR_UNSUPPORTED
    with pytest.raises(NotImplementedError):
        ops.gat_fused(csr, q, t, None, 8, return_attention=True)


# ---- layers ----------------------------------------------------------------------------------------------------------

def test_gcn_layer_fp8_is_the_fp32_composition_and_within_bound():
    n, f, units = 4096, 100, 128
    ei = random_graph(n, 60000, seed=12)
    rs = np.random.RandomState(0)
    graph = tfg.Graph(rs.randn(n, f).astype(np.float32), ei).to_device()
    layer = tfg.layers.GCN(units, activation=tfg.nn.relu, seed=1)
    layer8 = tfg.layers.GCN(units, activation=tfg.nn.relu, seed=1, message_dtype=FP8)
    layer.build_cache_for_graph(graph)
    layer([graph.x, graph.edge_index], cache=graph.cache)
    layer8([graph.x, graph.edge_index], cache=graph.cache)
    layer8.kernel.data.copy_(layer.kernel.data)
    layer8.bias.data.copy_(torch.randn_like(layer.bias.data))
    layer.bias.data.copy_(layer8.bias.data)
    h8 = layer8([graph.x, graph.edge_index], cache=graph.cache)
    h32 = layer([graph.x, graph.edge_index], cache=graph.cache)
    normed = tfg.nn.conv.gcn.gcn_norm_adj(tfg.SparseMatrix(graph.edge_index, None, [n, n]), cache=graph.cache)
    xw = ops.gemm(graph.x, layer.kernel.data)                # the tensor-core kernel (K <= 184)
    t = ops.quantize_fp8(xw)
    xh = padded_f32(deq(t))
    same_bits(h8, normed.matmul(xh, bias=layer.bias.data, act=ops.ACT_RELU))
    # |relu(a) - relu(b)| <= sum_e |w_e| max(2^-4 |xw|, 2^(k-10)), up to the fp32 rounding of both sums
    k = t.exps.float()[:, :1]
    per = torch.maximum(xw.abs() * 2.0 ** -4, torch.exp2(k - 10))
    bound = normed.matmul(per) * (1 + 1e-5) + 1e-6 * normed.matmul(xw.abs())
    assert float(((h8 - h32).abs() - bound).max()) <= 0.0


def test_gat_layer_fp8_against_float64():
    n, f, units, heads = 2000, 100, 128, 8
    ei = random_graph(n, 30000, seed=13)
    rs = np.random.RandomState(1)
    x = dev(rs.randn(n, f).astype(np.float32))
    layer = tfg.layers.GAT(units, num_heads=heads, activation=tfg.nn.relu, seed=2, message_dtype=FP8)
    got = layer([x, dev(ei)])
    p = {k: v.data for k, v in layer.named_parameters()}
    q, k, v = ops.gemm_proj(x, [(p["query_kernel"], p["query_bias"], ops.ACT_RELU, None),
                                (p["key_kernel"], p["key_bias"], ops.ACT_RELU, None), (p["kernel"], None, ops.ACT_NONE, None)])
    kh, vh = deq(ops.quantize_fp8(k)), deq(ops.quantize_fp8(v))
    full = ops.self_loops(dev(ei), n)
    csr = ops.csr_build(full[0].contiguous(), full[1].contiguous(), n)
    want = gat_f64(csr.rowptr, csr.col, q, kh, vh, heads, True, bias=p["bias"], relu=True)
    assert_close(host(got), want, rtol=1e-4, atol_scale=1e-4, what="GAT fp8 layer")


@pytest.mark.parametrize("kind", ["gcn", "gat"])
def test_trained_models_keep_accuracy_in_fp8(kind):
    x, ei, y = _planted()
    n = len(y)
    perm = np.random.RandomState(1).permutation(n)
    train, test = perm[: n // 2], perm[n // 2:]
    graph = tfg.Graph(x, ei).to_device()
    torch.manual_seed(0)
    if kind == "gcn":
        l1 = tfg.layers.GCN(64, activation=tfg.nn.relu, seed=1, trainable=True)
        l1.build_cache_for_graph(graph)
    else:
        l1 = tfg.layers.GAT(64, num_heads=8, activation=tfg.nn.relu, seed=1, trainable=True)
    l2 = tfg.layers.GCN(4, seed=2, trainable=True)
    l2.build_cache_for_graph(graph)

    def forward(md=None):
        l1.message_dtype = l2.message_dtype = md
        h = l1([graph.x, graph.edge_index], cache=graph.cache)
        return l2([h, graph.edge_index], cache=graph.cache)
    forward()
    params = list(l1.parameters()) + list(l2.parameters())
    opt = torch.optim.Adam(params, lr=0.01)
    yt = torch.as_tensor(y, device="cuda").long()
    tr = torch.as_tensor(train, device="cuda").long()
    for _ in range(60):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(forward()[tr], yt[tr]).backward()
        opt.step()
    te = torch.as_tensor(test, device="cuda").long()
    with torch.no_grad():
        for p in params:
            p.requires_grad_(False)
        acc32 = float((forward()[te].argmax(1) == yt[te]).float().mean())
        acc8 = float((forward(FP8)[te].argmax(1) == yt[te]).float().mean())
    print("accuracy {}: fp32 {:.4f} fp8 {:.4f}".format(kind, acc32, acc8))
    assert acc32 > 0.6
    assert abs(acc32 - acc8) <= 0.02, (acc32, acc8)


def test_gcn_fp8_products_shape_sampled_rows():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    n = bench.PRODUCTS_NODES
    ei = bench.make_graph_device(n, bench.PRODUCTS_UNDIRECTED, 0, torch.device("cuda"))
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    x = torch.randn((n, bench.FEATURES), generator=g, device="cuda")
    graph = tfg.Graph(x, ei)
    layer = tfg.layers.GCN(bench.UNITS, activation=tfg.nn.relu, seed=1, message_dtype=FP8)
    layer.build_cache_for_graph(graph)
    got = layer([graph.x, graph.edge_index], cache=graph.cache)
    normed = tfg.nn.conv.gcn.gcn_norm_adj(tfg.SparseMatrix(graph.edge_index, None, [n, n]), cache=graph.cache)
    t = ops.fp8_table(n, bench.UNITS, "cuda")
    ops.gemm_proj(x, [(layer.kernel.data, None, ops.ACT_NONE, t)])
    want = ops.spmm(normed.csr, normed.value_csr, padded_f32(deq(t)), bias=layer.bias.data, act=ops.ACT_RELU)
    rows = torch.randint(0, n, (4096,), generator=g, device="cuda")
    same_bits(got[rows], want[rows])


# ---- refusals --------------------------------------------------------------------------------------------------------

def test_fp8_mode_refusals_on_the_device():
    n, f = 200, 16
    ei = dev(random_graph(n, 1500, seed=14))
    x = dev(np.random.RandomState(2).randn(n, f).astype(np.float32))
    gcn = tfg.layers.GCN(16, message_dtype=FP8, trainable=True)
    with pytest.raises(NotImplementedError):
        gcn([x, ei])                                          # trainable weights require grad
    gat = tfg.layers.GAT(16, num_heads=3, message_dtype=FP8)
    with pytest.raises(NotImplementedError, match="bfloat16 or float32"):
        gat([x, ei])
    gat = tfg.layers.GAT(16, num_heads=2, split_value_heads=False, message_dtype=FP8)
    with pytest.raises(NotImplementedError):
        gat([x, ei])
    with pytest.raises(ValueError):
        tfg.layers.GAT(16, message_dtype=torch.float8_e5m2)
    with pytest.raises(ValueError):
        tfg.layers.GIN(16, message_dtype=FP8)                 # the other convolutions keep refusing fp8
