# coding=utf-8
"""bf16 message rows for GCN and GAT inference (tfgk_spmm_bf16, tfgk_gemm_proj_mixed, tfgk_gat_fused_bf16).

Widening bf16 to fp32 is exact, so each bf16 kernel is defined as the fp32 kernel applied to the widened table:
K1 and K4 are checked bit for bit against the fp32 kernels, K3 against float64 over the widened K and V."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from conftest import random_graph, assert_close

pytestmark = pytest.mark.gpu


def dev(a, dtype=None):
    return ops.as_device(a, dtype)


def host(t):
    return t.detach().cpu().numpy()


def same_bits(a, b):
    """Equal bit patterns; NaNs only need to sit at the same places."""
    assert a.shape == b.shape and a.dtype == b.dtype
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), "NaN positions differ"
    view = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    ia, ib = a.contiguous().view(view), b.contiguous().view(view)
    diff = (ia != ib) & ~na
    assert not bool(diff.any()), "{} of {} entries differ".format(int(diff.sum()), a.numel())


_CSR = {}


def hub_csr():
    """3000 nodes, 11 without in-edges, and node 42 with an in-degree of 60 000: its row goes through the plan's slices."""
    if "hub" not in _CSR:
        n = 3000
        base = random_graph(n, 45000, seed=5, isolated=11)
        rs = np.random.RandomState(9)
        hub = np.stack([np.full(60000, 42), rs.randint(0, n, 60000)]).astype(np.int32)
        ei = np.concatenate([base, hub], axis=1)
        csr = ops.csr_build(dev(ei[0]), dev(ei[1]), n)
        assert csr.plan is not None and csr.plan.n_hubs == 1
        w = dev(rs.rand(csr.nnz).astype(np.float32) * 2 - 0.5)
        _CSR["hub"] = (csr, w, n)
    return _CSR["hub"]


def table(n, d, seed):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    return (torch.randn((n, d), generator=g) * 3).to(torch.bfloat16).cuda()


# ---- K1 --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [1, 3, 8, 32, 64, 100, 128, 132, 256, 264, 400, 600])
@pytest.mark.parametrize("reduce", ["sum", "mean", "max"])
@pytest.mark.parametrize("weighted", [False, True])
def test_spmm_bf16_is_fp32_over_the_widened_table(d, reduce, weighted):
    csr, w, n = hub_csr()
    w = w if weighted else None
    h = table(n, d, d)
    addend = torch.randn((n, d), device="cuda")
    bias = torch.randn((d,), device="cuda")
    for kw in ({}, dict(alpha=0.75, addend=addend, beta=-0.5, bias=bias, act=ops.ACT_RELU), dict(alpha=2.0, bias=bias)):
        got = ops.spmm(csr, w, h, reduce=reduce, **kw)
        want = ops.spmm(csr, w, h.float(), reduce=reduce, **kw)
        same_bits(got, want)
    same_bits(ops.spmm(csr, w, h, reduce=reduce), ops.spmm(csr, w, h, reduce=reduce))     # run to run


def test_spmm_bf16_empty_rows_and_hub_row():
    csr, w, n = hub_csr()
    h = table(n, 128, 1)
    got = ops.spmm(csr, w, h, reduce="mean")
    same_bits(got, ops.spmm(csr, w, h.float(), reduce="mean"))
    assert bool((got[:11] == 0).all())                                   # empty rows: mean of nothing is 0
    ref = (w.double()[:, None] * h.double()[csr.col.long()])
    deg = host(csr.degree_i64())
    r0, r1 = int(host(csr.rowptr)[42]), int(host(csr.rowptr)[43])
    want = ref[r0:r1].sum(0) / deg[42]
    assert torch.allclose(got[42].double(), want, rtol=1e-4, atol=1e-4 * float(want.abs().max()))


def test_spmm_bf16_column_override_and_odd_leading_dimension():
    csr, w, n = hub_csr()
    msg = table(csr.nnz, 64, 2)                                          # one message row per CSR slot, gathered via perm
    same_bits(ops.spmm(csr, None, msg, reduce="sum", col=csr.perm), ops.spmm(csr, None, msg.float(), reduce="sum", col=csr.perm))
    full = table(n, 135, 3)
    view = full[:, 3:103]                                                # leading dimension 135: not 8-byte aligned rows
    want = ops.spmm(csr, w, view.float(), reduce="sum")                  # dense widened table: hub row 42 via the plan
    same_bits(ops.spmm(csr, w, view, reduce="sum"), want)
    flat = table(n * 100 + 1, 1, 5).reshape(-1)
    shifted = flat[1:].view(n, 100)                                      # dense, but 2 bytes past an 8-byte boundary
    same_bits(ops.spmm(csr, w, shifted, reduce="sum"), ops.spmm(csr, w, shifted.float(), reduce="sum"))
    # read in place (SparseMatrix.matmul's column chunks): the fp32 product over a widened view of the same layout
    same_bits(ops.spmm(csr, w, view, reduce="sum", keep_layout=True),
              ops.spmm(csr, w, full.float()[:, 3:103], reduce="sum"))


def test_sparse_matrix_matmul_keeps_bf16():
    n = 2000
    ei = random_graph(n, 30000, seed=4)
    adj = tfg.SparseMatrix(ei, np.random.RandomState(0).rand(ei.shape[1]).astype(np.float32), [n, n])
    h = table(n, 128, 4)
    bias = torch.randn((128,), device="cuda")
    same_bits(adj.matmul(h, bias=bias, act=ops.ACT_RELU), adj.matmul(h.float(), bias=bias, act=ops.ACT_RELU))
    same_bits(adj.matmul(h, num_or_size_splits=[40, 88]), adj.matmul(h.float(), num_or_size_splits=[40, 88]))


def test_sparse_matrix_matmul_chunks_with_hub_row():
    n = 3000
    base = random_graph(n, 45000, seed=6)
    rs = np.random.RandomState(10)
    ei = np.concatenate([base, np.stack([np.full(9000, 7), rs.randint(0, n, 9000)]).astype(np.int32)], axis=1)
    adj = tfg.SparseMatrix(ei, rs.rand(ei.shape[1]).astype(np.float32), [n, n])
    assert adj.csr.plan is not None and adj.csr.plan.n_hubs == 1
    h = table(n, 130, 6)
    for splits in ([2, 128], [40, 90], None):                            # chunks at odd and at aligned column offsets
        same_bits(adj.matmul(h, num_or_size_splits=splits), adj.matmul(h.float(), num_or_size_splits=splits))


def test_sparse_matrix_matmul_bf16_with_trainable_values_trains_in_fp32():
    """A bf16 h with learnable edge weights takes the differentiable fp32 route: same output and gradients as h.float()."""
    n = 1500
    ei = random_graph(n, 20000, seed=8)
    value_np = np.random.RandomState(11).rand(ei.shape[1]).astype(np.float32)
    h = table(n, 64, 7)
    g = torch.randn((n, 64), device="cuda")
    results = []
    for hh in (h, h.float()):
        value = dev(value_np).requires_grad_(True)
        bias = torch.zeros((64,), device="cuda", requires_grad=True)
        y = tfg.SparseMatrix(ei, value, [n, n]).matmul(hh, bias=bias, act=ops.ACT_RELU)
        (y * g).sum().backward()
        results.append((y.detach(), value.grad.clone(), bias.grad.clone()))
    for a, b in zip(*results):
        same_bits(a, b)


def test_spmm_bf16_products_shape():
    import bench
    ei = bench.make_graph_device(bench.PRODUCTS_NODES, bench.PRODUCTS_UNDIRECTED, 0, torch.device("cuda"))
    n = bench.PRODUCTS_NODES
    csr = ops.csr_build(ei[0].contiguous(), ei[1].contiguous(), n)
    del ei
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    w = torch.rand((csr.nnz,), generator=g, device="cuda")
    h = torch.randn((n, 128), generator=g, device="cuda").to(torch.bfloat16)
    got = ops.spmm(csr, w, h, reduce="sum", act=ops.ACT_RELU)
    same_bits(got, ops.spmm(csr, w, h.float(), reduce="sum", act=ops.ACT_RELU))
    same_bits(got, ops.spmm(csr, w, h, reduce="sum", act=ops.ACT_RELU))


# ---- K4 --------------------------------------------------------------------------------------------------------------

def _proj_inputs(m, k, seed):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    x = torch.randn((m, k), generator=g).cuda()
    ws = [torch.randn((k, c), generator=g).cuda() * 0.3 for c in (128, 128, 100)]
    bs = [torch.randn((c,), generator=g).cuda() for c in (128, 128, 100)]
    return x, ws, bs


@pytest.mark.parametrize("k", [1, 8, 100, 128, 184, 185])
def test_gemm_proj_bf16_blocks_are_rounded_fp32(k):
    m = 1000
    x, ws, bs = _proj_inputs(m, k, k)
    ref = [torch.empty((m, w.shape[1]), device="cuda") for w in ws]
    ops.gemm_proj(x, [(ws[0], bs[0], ops.ACT_NONE, ref[0]), (ws[1], bs[1], ops.ACT_RELU, ref[1]),
                      (ws[2], None, ops.ACT_NONE, ref[2])])
    # fp32 Q next to bf16 K | V written into column slices of one buffer, all from one launch
    q = torch.empty((m, 128), device="cuda")
    kv = torch.empty((m, 228), dtype=torch.bfloat16, device="cuda")
    ops.gemm_proj(x, [(ws[0], bs[0], ops.ACT_NONE, q), (ws[1], bs[1], ops.ACT_RELU, kv[:, :128]),
                      (ws[2], None, ops.ACT_NONE, kv[:, 128:])])
    same_bits(q, ref[0])
    same_bits(kv[:, :128], ref[1].to(torch.bfloat16))
    same_bits(kv[:, 128:], ref[2].to(torch.bfloat16))


def test_gemm_proj_bf16_non_finite_and_beyond_bf16_range():
    m, k = 512, 8
    x, ws, _ = _proj_inputs(m, k, 7)
    x[0, 0], x[1, 3], x[2, 5] = float("inf"), float("-inf"), float("nan")
    x[3, :] = 0.0
    x[3, 0] = 3.3e38                                       # fp32-finite products above the bf16 maximum (3.39e38) ...
    w = ws[0].clone()
    w[0, :64] = 1.0305                                      # ... for these columns (3.40e38 rounds up to bf16 inf)
    ref = torch.empty((m, 128), device="cuda")
    ops.gemm_proj(x, [(w, None, ops.ACT_NONE, ref)])
    out = torch.empty((m, 128), dtype=torch.bfloat16, device="cuda")
    ops.gemm_proj(x, [(w, None, ops.ACT_NONE, out)])
    assert bool(torch.isinf(out[3, :64]).all()) and bool(torch.isfinite(ref[3, :64]).all())
    assert bool(torch.isnan(out).any()) and bool(torch.isinf(out[0]).any())
    same_bits(out, ref.to(torch.bfloat16))


def test_gemm_proj_mixed_refuses_several_parts():
    x = torch.randn((256, 16), device="cuda")
    w = torch.randn((16, 32), device="cuda")
    out = torch.empty((256, 32), dtype=torch.bfloat16, device="cuda")
    st = (_ffi.ProjBlockOut * 1)(_ffi.ProjBlockOut(w.data_ptr(), 32, 32, 0, None, 0, out.data_ptr(), 32, _ffi.DTYPE_BF16))
    import ctypes
    a = (ctypes.c_void_p * 2)(x.data_ptr(), x.data_ptr())
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_gemm_proj_mixed", a, 2, 128, 16, 256, 16, st, 1, 0, 0, None)
    assert err.value.code == _ffi.ERR_UNSUPPORTED


# ---- K3 --------------------------------------------------------------------------------------------------------------

def gat_f64(rowptr, col, q, k, v, heads, split, bias=None, relu=False):
    """float64 restatement of nn/conv/gat.py over the given (already widened) Q, K and V."""
    rowptr, col = host(rowptr), host(col)
    q, k, v = (t.double().cpu().numpy() for t in (q, k, v))
    n, a = q.shape
    dqk, dv = a // heads, v.shape[1] // heads
    out = np.zeros((n, v.shape[1] if split else dv))
    for r in range(n):
        c = col[rowptr[r]:rowptr[r + 1]]
        if len(c) == 0:
            continue
        heads_out = []
        for h in range(heads):
            s = k[c, h * dqk:(h + 1) * dqk] @ q[r, h * dqk:(h + 1) * dqk] / np.sqrt(np.float32(dqk))
            p = np.exp(s - s.max())
            att = p / (p.sum() + 1e-8)
            heads_out.append(att @ v[c, h * dv:(h + 1) * dv])
        out[r] = np.concatenate(heads_out) if split else np.mean(heads_out, axis=0)
    if bias is not None:
        out = out + host(bias)
    return np.maximum(out, 0) if relu else out


def _gat_graph(n, e, seed, hub=None):
    ei = random_graph(n, e, seed, hub=hub)
    full = ops.self_loops(dev(ei), n)
    return ops.csr_build(full[0].contiguous(), full[1].contiguous(), n)


@pytest.mark.parametrize("heads,dh", [(1, 4), (1, 128), (2, 16), (2, 64), (2, 128), (4, 8), (4, 32), (8, 4), (8, 16),
                                      (8, 64), (8, 12), (3, 20)])
@pytest.mark.parametrize("split", [True, False])
def test_gat_bf16_against_float64(heads, dh, split):
    n = 700
    csr = _gat_graph(n, 9000, heads * 100 + dh)
    a = heads * dh
    g = torch.Generator(device="cpu")
    g.manual_seed(a)
    q = torch.randn((n, a), generator=g).cuda()
    vw = a if split else a * 2
    kv = torch.randn((n, a + vw), generator=g).to(torch.bfloat16).cuda()     # K | V side by side, as the layer projects
    k, v = kv[:, :a], kv[:, a:]
    bias = torch.randn((vw if split else vw // heads,), generator=g).cuda()
    got = ops.gat_fused(csr, q, k, v, heads, split_value_heads=split, bias=bias, act=ops.ACT_RELU)
    want = gat_f64(csr.rowptr, csr.col, q, k, v, heads, split, bias=bias, relu=True)
    assert_close(host(got), want, rtol=2e-5, atol_scale=2e-6, what="gat bf16")
    same_bits(got, ops.gat_fused(csr, q, k, v, heads, split_value_heads=split, bias=bias, act=ops.ACT_RELU))


def test_gat_bf16_hub_row_and_tma_path_matches_fp32_kernel():
    n, heads, a = 3000, 8, 128
    csr = _gat_graph(n, 40000, 11, hub=(100, 9000))
    assert csr.plan is not None and csr.plan.n_hubs >= 1
    g = torch.Generator(device="cpu")
    g.manual_seed(3)
    q = torch.randn((n, a), generator=g).cuda()
    kv = torch.randn((n, 2 * a), generator=g).to(torch.bfloat16).cuda()
    k, v = kv[:, :a], kv[:, a:]
    got = ops.gat_fused(csr, q, k, v, heads)
    want = gat_f64(csr.rowptr, csr.col, q, k, v, heads, True)
    assert_close(host(got), want, rtol=2e-5, atol_scale=2e-6, what="gat bf16 hub")
    same_bits(got, ops.gat_fused(csr, q, k, v, heads))
    kvf = kv.float()                       # the TMA ring keeps the fp32 lane mapping: same bits as fp32 K3 over widened K | V
    same_bits(got, ops.gat_fused(csr, q, kvf[:, :a], kvf[:, a:], heads))


@pytest.mark.parametrize("a", [256, 512])
def test_gat_bf16_wide_heads_take_the_single_pass_kernel(a):
    """8 heads with A > 128: the register-staged single-pass kernel, the same bits as the fp32 kernel over widened K, V."""
    n, heads = 3000, 8
    csr = _gat_graph(n, 40000, a, hub=(100, 9000))
    g = torch.Generator(device="cpu")
    g.manual_seed(a)
    q = torch.randn((n, a), generator=g).cuda()
    kv = torch.randn((n, 2 * a), generator=g).to(torch.bfloat16).cuda()
    got = ops.gat_fused(csr, q, kv[:, :a], kv[:, a:], heads)
    kvf = kv.float()
    same_bits(got, ops.gat_fused(csr, q, kvf[:, :a], kvf[:, a:], heads))
    want = gat_f64(csr.rowptr, csr.col, q, kv[:, :a], kv[:, a:], heads, True)
    assert_close(host(got), want, rtol=2e-5, atol_scale=2e-6, what="gat bf16 wide")


# ---- layers ----------------------------------------------------------------------------------------------------------

def test_gcn_layer_bf16_is_the_fp32_composition_and_within_bound():
    n, f, units = 4096, 100, 128
    ei = random_graph(n, 60000, seed=12)
    rs = np.random.RandomState(0)
    graph = tfg.Graph(rs.randn(n, f).astype(np.float32), ei).to_device()
    layer = tfg.layers.GCN(units, activation=tfg.nn.relu, seed=1)
    layer16 = tfg.layers.GCN(units, activation=tfg.nn.relu, seed=1, message_dtype=torch.bfloat16)
    layer.build_cache_for_graph(graph)
    h32 = layer([graph.x, graph.edge_index], cache=graph.cache)
    layer16([graph.x, graph.edge_index], cache=graph.cache)                # builds its weights
    layer16.kernel.data.copy_(layer.kernel.data)
    layer16.bias.data.copy_(torch.randn_like(layer.bias.data))
    layer.bias.data.copy_(layer16.bias.data)
    h16 = layer16([graph.x, graph.edge_index], cache=graph.cache)
    h32 = layer([graph.x, graph.edge_index], cache=graph.cache)
    normed = tfg.nn.conv.gcn.gcn_norm_adj(tfg.SparseMatrix(graph.edge_index, None, [n, n]), cache=graph.cache)
    xw = ops.gemm(graph.x, layer.kernel.data)                              # M K >= 16384, K <= 184: the tensor-core kernel
    want = normed.matmul(xw.to(torch.bfloat16).float(), bias=layer.bias.data, act=ops.ACT_RELU)
    same_bits(h16, want)
    # |relu(a) - relu(b)| <= |a - b| <= sum_e |w_e| |xw - bf16(xw)| <= 2^-8 sum_e |w_e| |xw| (bf16's half ulp), up to
    # the fp32 rounding of both sums
    bound = 2.0 ** -8 * normed.matmul(xw.abs()) + 1e-30
    slack = ((h16 - h32).abs() - bound)
    assert float(slack.max()) <= 0.0


def test_gat_layer_bf16_against_float64():
    n, f, units, heads = 2000, 100, 128, 8
    ei = random_graph(n, 30000, seed=13)
    rs = np.random.RandomState(1)
    x = dev(rs.randn(n, f).astype(np.float32))
    layer = tfg.layers.GAT(units, num_heads=heads, activation=tfg.nn.relu, seed=2, message_dtype="bfloat16")
    got = layer([x, dev(ei)])
    p = {k: v.data for k, v in layer.named_parameters()}
    # the fp32 projections, K and V then rounded (what K4's bf16 blocks store, bit for bit)
    q, k, v = ops.gemm_proj(x, [(p["query_kernel"], p["query_bias"], ops.ACT_RELU, None),
                                (p["key_kernel"], p["key_bias"], ops.ACT_RELU, None), (p["kernel"], None, ops.ACT_NONE, None)])
    full = ops.self_loops(dev(ei), n)
    csr = ops.csr_build(full[0].contiguous(), full[1].contiguous(), n)
    want = gat_f64(csr.rowptr, csr.col, q, k.to(torch.bfloat16), v.to(torch.bfloat16), heads, True, bias=p["bias"], relu=True)
    assert_close(host(got), want, rtol=1e-4, atol_scale=1e-4, what="GAT bf16 layer")


def _planted(n=3000, classes=4, f=32, seed=0):
    rs = np.random.RandomState(seed)
    y = rs.randint(0, classes, n)
    src, dst = [], []
    for _ in range(12 * n):
        u = rs.randint(n)
        v = rs.choice(np.nonzero(y == y[u])[0]) if rs.rand() < 0.8 else rs.randint(n)
        src.append(u)
        dst.append(v)
    ei = np.array([src + dst, dst + src], dtype=np.int32)
    centers = rs.randn(classes, f)
    x = (centers[y] * 0.3 + rs.randn(n, f)).astype(np.float32)
    return x, ei, y


@pytest.mark.parametrize("kind", ["gcn", "gat"])
def test_trained_models_keep_accuracy_in_bf16(kind):
    x, ei, y = _planted()
    n = len(y)
    rs = np.random.RandomState(1)
    perm = rs.permutation(n)
    train, test = perm[: n // 2], perm[n // 2:]
    graph = tfg.Graph(x, ei).to_device()
    torch.manual_seed(0)
    if kind == "gcn":
        l1 = tfg.layers.GCN(64, activation=tfg.nn.relu, seed=1, trainable=True)
        l2 = tfg.layers.GCN(4, seed=2, trainable=True)
        l1.build_cache_for_graph(graph)

        def forward(md=None):
            l1.message_dtype = l2.message_dtype = md
            h = l1([graph.x, graph.edge_index], cache=graph.cache)
            return l2([h, graph.edge_index], cache=graph.cache)
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
        loss = torch.nn.functional.cross_entropy(forward()[tr], yt[tr])
        loss.backward()
        opt.step()
    te = torch.as_tensor(test, device="cuda").long()
    with torch.no_grad():
        for p in params:
            p.requires_grad_(False)
        acc32 = float((forward()[te].argmax(1) == yt[te]).float().mean())
        acc16 = float((forward(torch.bfloat16)[te].argmax(1) == yt[te]).float().mean())
    assert acc32 > 0.6
    assert abs(acc32 - acc16) <= 0.01, (acc32, acc16)


# ---- refusals --------------------------------------------------------------------------------------------------------

def test_bf16_mode_refuses_training_and_unsupported_inputs():
    n, f = 200, 16
    ei = random_graph(n, 1500, seed=14)
    x = dev(np.random.RandomState(2).randn(n, f).astype(np.float32))
    with pytest.raises(ValueError):
        tfg.layers.GCN(8, message_dtype=torch.float16)
    with pytest.raises(ValueError):
        tfg.layers.GAT(8, message_dtype="int8")
    kernel = torch.randn((f, 8), device="cuda")
    adj = tfg.SparseMatrix(ei, None, [n, n])
    with pytest.raises(NotImplementedError):
        tfg.nn.gcn(x, adj, kernel.clone().requires_grad_(True), message_dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        tfg.nn.gcn(x, adj, kernel, edge_drop_rate=0.5, training=True, message_dtype=torch.bfloat16)
    import scipy.sparse as sp
    xs = sp.random(n, f, density=0.1, format="csr", dtype=np.float32, random_state=0)
    with pytest.raises(NotImplementedError):
        tfg.nn.gcn(xs, adj, kernel, message_dtype=torch.bfloat16)
    w = [torch.randn((f, 8), device="cuda") for _ in range(3)]
    b = [torch.zeros((8,), device="cuda") for _ in range(2)]
    with pytest.raises(NotImplementedError):
        tfg.nn.gat(x.clone().requires_grad_(True), ei, w[0], b[0], None, w[1], b[1], None, w[2], num_heads=2,
                   message_dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        tfg.nn.gat(x, ei, w[0], b[0], None, w[1], b[1], None, w[2], num_heads=2, edge_drop_rate=0.2, training=True,
                   message_dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        tfg.nn.gat(xs, ei, w[0], b[0], None, w[1], b[1], None, w[2], num_heads=2, message_dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        tfg.nn.gcn(x, adj, kernel, message_dtype=torch.float64)

    class FakePartitioned(object):
        part = None

        def project_all_rows(self):
            raise AssertionError("must not be reached")
    for layer in (tfg.layers.GCN(8, message_dtype=torch.bfloat16), tfg.layers.GAT(8, message_dtype=torch.bfloat16)):
        with pytest.raises(NotImplementedError):
            layer([x, FakePartitioned()])
