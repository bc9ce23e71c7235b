# coding=utf-8
"""bf16 message rows for GraphSAGE, GIN, LEConv, APPNP, SGC, SSGC, TAGCN and ChebyNet inference, and the aggregation
entry that also stores its result in bf16 (tfgk_spmm_bf16_dual).

The kernel is checked bit for bit against tfgk_spmm_bf16, tfgk_spmm_f32 over the widened table and the rounding of that
result.  Each convolution is checked bit for bit against a composition of the fp32 kernels in which every gathered table
is replaced by its widened bf16 rounding, and against fp32 within the rounding bound, propagated hop by hop in float64."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from tf_geometric_b200.nn.conv import graph_sage as gs
from tf_geometric_b200.nn.conv.gcn import gcn_norm_adj
from conftest import random_graph

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def dev(a, dtype=None):
    return ops.as_device(a, dtype)


def same_bits(a, b):
    """Equal bit patterns; NaNs only need to sit at the same places."""
    assert a.shape == b.shape and a.dtype == b.dtype
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), "NaN positions differ"
    view = torch.int16 if a.dtype == BF16 else torch.int32
    diff = (a.contiguous().view(view) != b.contiguous().view(view)) & ~na
    assert not bool(diff.any()), "{} of {} entries differ".format(int(diff.sum()), a.numel())


def bf(t):
    """The widened bf16 rounding (nearest even) of an fp32 tensor."""
    return t.to(BF16).float()


_CSR = {}


def hub_csr():
    """3000 nodes, 11 without in-edges, and node 42 with an in-degree of 60 000: its row goes through the plan's slices."""
    if "hub" not in _CSR:
        n = 3000
        base = random_graph(n, 45000, seed=21, isolated=11)
        rs = np.random.RandomState(22)
        hub = np.stack([np.full(60000, 42), rs.randint(0, n, 60000)]).astype(np.int32)
        ei = np.concatenate([base, hub], axis=1)
        csr = ops.csr_build(dev(ei[0]), dev(ei[1]), n)
        assert csr.plan is not None and csr.plan.n_hubs == 1
        w = dev(rs.rand(csr.nnz).astype(np.float32) * 2 - 0.5)
        _CSR["hub"] = (csr, w, n)
    return _CSR["hub"]


def padded_table(n, d, seed):
    """A bf16 table as the library allocates it (rows padded to 8 elements), pad columns deliberately NaN."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    t = ops.bf16_table(n, d, "cuda")
    t.copy_((torch.randn((n, d), generator=g) * 3).to(BF16))
    pitch = t.stride(0)
    if pitch > d:
        t.as_strided((n, pitch), (pitch, 1))[:, d:] = float("nan")
    return t


def raw_spmm(name, csr, w, h, D, reduce, out=None, out_bf16=None, alpha=1.0, addend=None, beta=0.0, bias=None,
             act=ops.ACT_NONE):
    """One call of a K1 entry point with h's own layout (no copies)."""
    plan = csr.plan.struct(-(-D // 8) * 8, h.device) if csr.plan is not None else None
    args = [ops._p(csr.rowptr), ops._p(csr.col), ops._p(w), ops._p(h), h.stride(0), csr.n_rows, D,
            ops._REDUCE_CODES[reduce], float(alpha), ops._p(addend), 0 if addend is None else addend.stride(0),
            float(beta), ops._p(bias), act, ops._p(out), 0 if out is None else out.stride(0)]
    if name == "tfgk_spmm_bf16_dual":
        args += [ops._p(out_bf16), 0 if out_bf16 is None else out_bf16.stride(0)]
    _ffi.call(name, *(args + [ctypes.byref(plan) if plan is not None else None, None]))


# ---- kernel ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [1, 3, 7, 8, 16, 47, 64, 100, 128, 256, 264, 600])
@pytest.mark.parametrize("reduce", ["sum", "mean", "max"])
@pytest.mark.parametrize("weighted", [False, True])
def test_dual_store_is_spmm_bf16_and_its_rounding(d, reduce, weighted):
    csr, w, n = hub_csr()
    w = w if weighted else None
    h = padded_table(n, d, d)
    addend = torch.randn((n, d), device="cuda")
    bias = torch.randn((d,), device="cuda")
    for kw in ({}, dict(alpha=0.75, addend=addend, beta=-0.5, bias=bias, act=ops.ACT_RELU)):
        want = torch.empty((n, d), device="cuda")
        raw_spmm("tfgk_spmm_f32", csr, w, h.float(), d, reduce, out=want, **kw)       # dense widened table
        got_bf16_entry = torch.empty((n, d), device="cuda")
        raw_spmm("tfgk_spmm_bf16", csr, w, h, d, reduce, out=got_bf16_entry, **kw)
        same_bits(got_bf16_entry, want)
        want_b = ops.round_bf16(want)
        # both outputs, dense; then views with odd leading dimensions; then each output alone
        o, ob = torch.empty((n, d), device="cuda"), torch.empty((n, d), dtype=BF16, device="cuda")
        raw_spmm("tfgk_spmm_bf16_dual", csr, w, h, d, reduce, out=o, out_bf16=ob, **kw)
        same_bits(o, want)
        same_bits(ob, want_b)
        ov = torch.empty((n, d + 3), device="cuda")[:, 1:d + 1]
        obv = torch.empty((n, d + 1), dtype=BF16, device="cuda")[:, :d]
        raw_spmm("tfgk_spmm_bf16_dual", csr, w, h, d, reduce, out=ov, out_bf16=obv, **kw)
        # tfgk_spmm_bf16 into the same view (no plan for unaligned fp32 rows: hub rows summed in order), and its rounding
        want_v = torch.empty((n, d + 3), device="cuda")[:, 1:d + 1]
        raw_spmm("tfgk_spmm_bf16", csr, w, h, d, reduce, out=want_v, **kw)
        same_bits(ov, want_v)
        same_bits(obv, ops.round_bf16(want_v))
        ob_only = torch.empty((n, d), dtype=BF16, device="cuda")
        raw_spmm("tfgk_spmm_bf16_dual", csr, w, h, d, reduce, out_bf16=ob_only, **kw)
        same_bits(ob_only, want_b)
        o_only = torch.empty((n, d), device="cuda")
        raw_spmm("tfgk_spmm_bf16_dual", csr, w, h, d, reduce, out=o_only, **kw)
        same_bits(o_only, want)
        # the public route, twice: identical bits run to run
        for _ in range(2):
            o2 = torch.empty((n, d), device="cuda")
            ob2 = torch.empty((n, d), dtype=BF16, device="cuda")
            ops.spmm(csr, w, h, reduce=reduce, out=o2, out_bf16=ob2, **kw)
            same_bits(o2, want)
            same_bits(ob2, want_b)


def test_dual_store_empty_rows_hub_row_and_non_finite():
    csr, w, n = hub_csr()
    h = padded_table(n, 100, 1)
    h[5, 0], h[6, 1], h[7, 2] = float("inf"), float("-inf"), float("nan")
    h[8, 3] = 3.3e38
    o = torch.empty((n, 100), device="cuda")
    ob = torch.empty((n, 100), dtype=BF16, device="cuda")
    ops.spmm(csr, None, h, reduce="sum", alpha=1.03, out=o, out_bf16=ob)
    want = ops.spmm(csr, None, h.float(), reduce="sum", alpha=1.03)
    same_bits(o, want)
    same_bits(ob, ops.round_bf16(want))
    assert bool((o[:11] == 0).all()) and bool(torch.isinf(ob).any()) and bool(torch.isnan(ob).any())
    mean = ops.spmm(csr, w, h, reduce="mean", out_bf16=torch.empty((n, 100), dtype=BF16, device="cuda"))
    assert mean.dtype == BF16
    same_bits(mean, ops.round_bf16(ops.spmm(csr, w, h.float(), reduce="mean")))


def test_sparse_matrix_matmul_out_bf16():
    n = 3000
    base = random_graph(n, 45000, seed=23)
    rs = np.random.RandomState(24)
    ei = np.concatenate([base, np.stack([np.full(9000, 7), rs.randint(0, n, 9000)]).astype(np.int32)], axis=1)
    adj = tfg.SparseMatrix(ei, rs.rand(ei.shape[1]).astype(np.float32), [n, n])
    h = padded_table(n, 130, 6)
    for splits in ([2, 128], [40, 90], None):
        o = torch.empty((n, 130), device="cuda")
        ob = torch.empty((n, 130), dtype=BF16, device="cuda")
        assert adj.matmul(h, num_or_size_splits=splits, out=o, out_bf16=ob) is o
        want = adj.matmul(h, num_or_size_splits=splits)
        same_bits(o, want)
        same_bits(ob, ops.round_bf16(want))
    ob = torch.empty((n, 130), dtype=BF16, device="cuda")
    assert adj.matmul(h, out_bf16=ob) is ob                              # bf16 only
    same_bits(ob, ops.round_bf16(adj.matmul(h)))


# ---- compositions ----------------------------------------------------------------------------------------------------

def _graph(n=3000, e=40000, f=100, seed=30):
    rs = np.random.RandomState(seed)
    ei = random_graph(n, e, seed, hub=(5, 9000))
    x = dev(rs.randn(n, f).astype(np.float32))
    ew = dev(rs.rand(ei.shape[1]).astype(np.float32))
    return x, dev(ei), ew, rs


def _w(rs, *shape):
    return dev((rs.randn(*shape) * 0.2).astype(np.float32))


@pytest.mark.parametrize("reduce", ["mean", "sum"])
@pytest.mark.parametrize("concat", [True, False])
def test_plain_graph_sage_is_the_composition(reduce, concat):
    x, ei, ew, rs = _graph()
    ws, wn, b = _w(rs, 100, 64), _w(rs, 100, 64), _w(rs, 128 if concat else 64)
    fn = tfg.nn.mean_graph_sage if reduce == "mean" else tfg.nn.sum_graph_sage
    got = fn(x, ei, ew, ws, wn, b, activation=tfg.nn.relu, concat=concat, message_dtype=torch.bfloat16)
    csr, _ = tfg._structure.csr_for_edge_index(ei, x.shape[0])
    agg = ops.spmm(csr, tfg._structure.weights_in_csr_order(ew, csr), bf(x), reduce=reduce)
    same_bits(got, gs._project_pair(x, agg, ws, wn, b, tfg.nn.relu, concat, False))
    same_bits(fn(x, ei, ew, ws, wn, b, activation=tfg.nn.relu, concat=concat, message_dtype=None),
              fn(x, ei, ew, ws, wn, b, activation=tfg.nn.relu, concat=concat))
    same_bits(fn(x, ei, ew, ws, wn, b, activation=tfg.nn.relu, concat=concat, message_dtype=torch.float32),
              fn(x, ei, ew, ws, wn, b, activation=tfg.nn.relu, concat=concat))


def test_gcn_graph_sage_is_the_composition():
    x, ei, _, rs = _graph()
    k, b = _w(rs, 100, 128), _w(rs, 128)
    got = tfg.nn.gcn_graph_sage(x, ei, None, k, b, activation=tfg.nn.relu, message_dtype=torch.bfloat16)
    normed = tfg.SparseMatrix(*gs._norm_edge_as_matrix(ei, x.shape[0], None, renorm=False))
    same_bits(got, ops.gemm(normed.matmul(bf(x)), k, bias=b, act=ops.ACT_RELU))


@pytest.mark.parametrize("reduce", ["mean", "max"])
def test_pool_graph_sage_is_the_composition(reduce):
    x, ei, ew, rs = _graph()
    ws, wm, bm, wn, b = _w(rs, 100, 32), _w(rs, 100, 128), _w(rs, 128), _w(rs, 128, 32), _w(rs, 64)
    fn = tfg.nn.mean_pool_graph_sage if reduce == "mean" else tfg.nn.max_pool_graph_sage
    got = fn(x, ei, ew, ws, wm, wn, bm, b, activation=tfg.nn.relu, message_dtype=torch.bfloat16)
    csr, _ = tfg._structure.csr_for_edge_index(ei, x.shape[0])
    h_node = ops.gemm_proj(x, [(wm, bm, ops.ACT_RELU, None)])[0]         # the projection kernel of the bf16 path (K4)
    reduced = ops.spmm(csr, None, bf(h_node), reduce=reduce)
    same_bits(got, gs._project_pair(x, reduced, ws, wn, b, tfg.nn.relu, True, False))
    if reduce == "max":                                                   # rounding is monotone: max commutes with it
        same_bits(reduced.to(BF16), ops.spmm(csr, None, h_node, reduce="max").to(BF16))
    # an activation the epilogue does not fuse: rounded after it
    got = fn(x, ei, ew, ws, wm, wn, bm, b, activation=torch.tanh, message_dtype=torch.bfloat16)
    h_node = torch.tanh(ops.gemm(x, wm, bias=bm))
    reduced = ops.spmm(csr, None, bf(h_node), reduce=reduce)
    same_bits(got, gs._project_pair(x, reduced, ws, wn, b, torch.tanh, True, False))


def test_gin_and_le_conv_are_the_composition():
    x, ei, ew, rs = _graph()
    csr, _ = tfg._structure.csr_for_edge_index(ei, x.shape[0])
    got = tfg.nn.gin(x, ei, lambda h: h, eps=0.25, message_dtype=torch.bfloat16)
    same_bits(got, ops.spmm(csr, None, bf(x), reduce="sum", alpha=1.0, addend=x, beta=1.25))
    w = [_w(rs, 100, 64) for _ in range(3)]
    b = [_w(rs, 64) for _ in range(3)]
    got = tfg.nn.le_conv(x, ei, ew, w[0], b[0], w[1], b[1], w[2], b[2], activation=tfg.nn.relu,
                         message_dtype=torch.bfloat16)
    self_h = ops.gemm(x, w[0], bias=b[0])
    diff = ops.gemm(x, w[1], bias=b[1]) - ops.gemm(x, w[2], bias=b[2])
    want = ops.spmm(csr, tfg._structure.weights_in_csr_order(ew, csr), bf(diff), reduce="sum", alpha=1.0, addend=self_h,
                    beta=1.0, act=ops.ACT_RELU)
    same_bits(got, want)


def _appnp_composition(x, normed, kernels, biases, k, alpha, act):
    h = x
    for i, (kern, b) in enumerate(zip(kernels, biases)):
        h = ops.gemm(h, kern, bias=b, act=ops.ACT_RELU if i < len(kernels) - 1 else ops.ACT_NONE)
    cur = bf(h)
    for i in range(k):
        last = i == k - 1
        out = normed.matmul(cur, alpha=1.0 - alpha, addend=h, beta=alpha, act=act if last else ops.ACT_NONE)
        cur = bf(out)
    return out, h


@pytest.mark.parametrize("units", [47, 128])
def test_appnp_and_sgc_are_the_composition(units):
    x, ei, _, rs = _graph()
    n = x.shape[0]
    normed = gcn_norm_adj(tfg.SparseMatrix(ei, None, [n, n]))
    kernels, biases = [_w(rs, 100, 64), _w(rs, 64, units)], [_w(rs, 64), _w(rs, units)]
    got = tfg.nn.appnp(x, ei, None, kernels, biases, activation=tfg.nn.relu, k=10, alpha=0.1,
                       message_dtype=torch.bfloat16)
    same_bits(got, _appnp_composition(x, normed, kernels, biases, 10, 0.1, ops.ACT_RELU)[0])
    for k in (1, 3):
        kern, b = _w(rs, 100, units), _w(rs, units)
        got = tfg.nn.sgc(x, ei, None, k, kern, b, activation=tfg.nn.relu, message_dtype=torch.bfloat16)
        cur = bf(ops.gemm_proj(x, [(kern, None, ops.ACT_NONE, None)])[0])
        for i in range(k - 1):
            cur = bf(normed.matmul(cur))
        same_bits(got, normed.matmul(cur, bias=b, act=ops.ACT_RELU))


def test_ssgc_tagcn_chebynet_are_the_composition():
    x, ei, ew, rs = _graph()
    n = x.shape[0]
    normed = gcn_norm_adj(tfg.SparseMatrix(ei, ew, [n, n]))
    kernels, biases = [_w(rs, 100, 64)], [_w(rs, 64)]
    got = tfg.nn.ssgc(x, ei, ew, kernels, biases, k=10, alpha=0.1, message_dtype=torch.bfloat16)
    h = ops.gemm(x, kernels[0], bias=biases[0])
    output, cur = h * 0.1, h
    for _ in range(10):
        cur = normed.matmul(bf(cur))
        output = output + (1 - 0.1) * cur / 10
    same_bits(got, output)

    normed_t = gcn_norm_adj(tfg.SparseMatrix(ei, ew, [n, n]), renorm=False)
    kern, b = _w(rs, 100 * 4, 64), _w(rs, 64)
    got = tfg.nn.tagcn(x, ei, ew, 3, kern, b, activation=tfg.nn.relu, message_dtype=torch.bfloat16)
    hops = torch.empty((n, 400), device="cuda")
    hops[:, :100].copy_(x)
    for i in range(3):
        normed_t.matmul(bf(hops[:, i * 100:(i + 1) * 100]), out=hops[:, (i + 1) * 100:(i + 2) * 100])
    same_bits(got, ops.gemm(hops, kern, bias=b, act=ops.ACT_RELU))

    kernels = [_w(rs, 100, 32) for _ in range(4)]
    got = tfg.nn.chebynet(x, ei, ew, 4, kernels, b[:32].contiguous(), message_dtype=torch.bfloat16)
    idx, val = tfg.nn.conv.propagation.chebynet_norm_edge(ei, n, ew)
    adj = tfg.SparseMatrix(idx, val, [n, n])
    t0, t1 = x, adj.matmul(bf(x))
    out = ops.gemm(t0, kernels[0])
    ops.gemm(t1, kernels[1], beta=1.0, out=out)
    for i in range(2, 4):
        t2 = adj.matmul(bf(t1), alpha=2.0, addend=t0, beta=-1.0)
        ops.gemm(t2, kernels[i], beta=1.0, out=out)
        t0, t1 = t1, t2
    same_bits(got, out + b[:32])


def test_layers_match_the_functions():
    x, ei, ew, rs = _graph(n=2000, e=20000, f=32)
    kw = dict(message_dtype=torch.bfloat16)
    cases = [
        (tfg.layers.MeanGraphSage(32, seed=1, **kw), tfg.layers.MeanGraphSage(32, seed=1)),
        (tfg.layers.SumGraphSage(32, seed=1, **kw), tfg.layers.SumGraphSage(32, seed=1)),
        (tfg.layers.GCNGraphSage(32, seed=1, **kw), tfg.layers.GCNGraphSage(32, seed=1)),
        (tfg.layers.MeanPoolGraphSage(32, seed=1, **kw), tfg.layers.MeanPoolGraphSage(32, seed=1)),
        (tfg.layers.MaxPoolGraphSage(32, seed=1, **kw), tfg.layers.MaxPoolGraphSage(32, seed=1)),
        (tfg.layers.LEConv(32, seed=1, **kw), tfg.layers.LEConv(32, seed=1)),
        (tfg.layers.APPNP([32, 7], seed=1, **kw), tfg.layers.APPNP([32, 7], seed=1)),
        (tfg.layers.SGC(7, k=2, seed=1, **kw), tfg.layers.SGC(7, k=2, seed=1)),
        (tfg.layers.SSGC([16], seed=1, **kw), tfg.layers.SSGC([16], seed=1)),
        (tfg.layers.TAGCN(16, seed=1, **kw), tfg.layers.TAGCN(16, seed=1)),
        (tfg.layers.ChebyNet(16, 3, seed=1, **kw), tfg.layers.ChebyNet(16, 3, seed=1)),
        (tfg.layers.GIN(lambda h: h, **kw), tfg.layers.GIN(lambda h: h)),
    ]
    with torch.no_grad():
        for l16, l32 in cases:
            got = l16([x, ei, ew] if not isinstance(l16, tfg.layers.GIN) else [x, ei])
            want = l32([x, ei, ew] if not isinstance(l32, tfg.layers.GIN) else [x, ei])
            assert got.shape == want.shape and got.dtype == torch.float32
            # same seed, same weights: the bf16 layer stays within a few bf16 roundings of the fp32 one, run to run
            assert l16.message_dtype is torch.bfloat16 and l32.message_dtype is None
            scale = float(want.abs().max())
            assert float((got - want).abs().max()) <= 0.05 * scale + 1e-6, type(l16).__name__
            same_bits(got, l16([x, ei, ew] if not isinstance(l16, tfg.layers.GIN) else [x, ei]))


# ---- error bounds against fp32, in float64 -------------------------------------------------------------------------

def _abs_adj(idx, val, n):
    i, v = idx.cpu().numpy(), np.abs(val.double().cpu().numpy())
    return sp.csr_matrix((v, (i[0], i[1])), shape=(n, n))


def test_one_hop_error_bound():
    x, ei, ew, rs = _graph()
    n = x.shape[0]
    got = tfg.nn.gin(x, ei, lambda h: h, eps=0.0, message_dtype=torch.bfloat16).double().cpu().numpy()
    ref = tfg.nn.gin(x, ei, lambda h: h, eps=0.0).double().cpu().numpy()
    a = _abs_adj(ei, torch.ones(ei.shape[1], device="cuda"), n)
    xa = np.abs(x.double().cpu().numpy())
    s = a @ xa + xa                                                    # every term of both fp32 sums, in magnitude
    deg = np.asarray(a.sum(axis=1)).reshape(-1, 1) + 1
    bound = 2.0 ** -8 * (a @ xa) + 2 * deg * 2.0 ** -24 * s            # rounding of x, then fp32 rounding of both sums
    assert np.all(np.abs(got - ref) <= bound)


def test_k_hop_error_bound_appnp():
    x, ei, _, rs = _graph()
    n = x.shape[0]
    normed = gcn_norm_adj(tfg.SparseMatrix(ei, None, [n, n]))
    kernels, biases = [_w(rs, 100, 47)], [_w(rs, 47)]
    k, alpha = 10, 0.1
    got = tfg.nn.appnp(x, ei, None, kernels, biases, k=k, alpha=alpha, message_dtype=torch.bfloat16)
    ref = tfg.nn.appnp(x, ei, None, kernels, biases, k=k, alpha=alpha)
    a = _abs_adj(normed.index, normed.value, n)
    h = ops.gemm(x, kernels[0], bias=biases[0]).double().cpu().numpy()
    o, e = h.copy(), np.zeros_like(h)
    for _ in range(k):
        # |p' - o'| <= (1 - alpha) |A| (|bf(p) - p| + |p - o|) with |bf(p) - p| <= 2^-8 |p| <= 2^-8 (|o| + e)
        e = (1 - alpha) * (a @ (2.0 ** -8 * (np.abs(o) + e) + e))
        o = (1 - alpha) * (a @ o) + alpha * h
    diff = np.abs(got.double().cpu().numpy() - ref.double().cpu().numpy())
    assert np.all(diff <= 1.01 * e + 1e-5 * np.abs(o).max())


# ---- accuracy retention ------------------------------------------------------------------------------------------

def _planted(n=3000, classes=4, f=32, seed=0):
    rs = np.random.RandomState(seed)
    y = rs.randint(0, classes, n)
    src = rs.randint(0, n, 12 * n)
    same = rs.rand(12 * n) < 0.8
    by_class = [np.nonzero(y == c)[0] for c in range(classes)]
    dst = np.where(same, [rs.choice(by_class[y[u]]) for u in src], rs.randint(0, n, 12 * n))
    ei = np.array([np.concatenate([src, dst]), np.concatenate([dst, src])], dtype=np.int32)
    centers = rs.randn(classes, f)
    x = (centers[y] * 0.3 + rs.randn(n, f)).astype(np.float32)
    return x, ei, y


@pytest.mark.parametrize("kind", ["appnp", "sgc", "mean_sage", "gin"])
def test_trained_models_keep_accuracy_in_bf16(kind):
    x, ei, y = _planted()
    n = len(y)
    perm = np.random.RandomState(1).permutation(n)
    train, test = perm[: n // 2], perm[n // 2:]
    graph = tfg.Graph(x, ei).to_device()
    torch.manual_seed(0)
    if kind == "appnp":
        layer = tfg.layers.APPNP([64, 4], k=10, alpha=0.1, seed=1, trainable=True)
    elif kind == "sgc":
        layer = tfg.layers.SGC(4, k=2, seed=1, trainable=True)
    elif kind == "mean_sage":
        layer = tfg.layers.MeanGraphSage(4, activation=None, seed=1, trainable=True)
    else:
        mlp = torch.nn.Linear(32, 4).cuda()
        layer = tfg.layers.GIN(mlp)

    def forward(md=None):
        layer.message_dtype = md
        return layer([graph.x, graph.edge_index])
    forward()
    params = list(layer.parameters()) + (list(mlp.parameters()) if kind == "gin" else [])
    opt = torch.optim.Adam(params, lr=0.01)
    yt = torch.as_tensor(y, device="cuda").long()
    tr, te = (torch.as_tensor(i, device="cuda").long() for i in (train, test))
    for _ in range(60):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(forward()[tr], yt[tr]).backward()
        opt.step()
    with torch.no_grad():
        acc32 = float((forward()[te].argmax(1) == yt[te]).float().mean())
        acc16 = float((forward(torch.bfloat16)[te].argmax(1) == yt[te]).float().mean())
    assert acc32 > 0.6
    assert abs(acc32 - acc16) <= 0.01, (acc32, acc16)


# ---- refusals ------------------------------------------------------------------------------------------------------

def test_refusals():
    x, ei, ew, rs = _graph(n=300, e=2000, f=16)
    b16 = torch.bfloat16
    ws, wn = _w(rs, 16, 8), _w(rs, 16, 8)
    with pytest.raises(NotImplementedError):
        tfg.nn.mean_graph_sage(x, ei, None, ws.clone().requires_grad_(True), wn, message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.sgc(x.clone().requires_grad_(True), ei, None, 2, ws, message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.appnp(x, ei, None, [ws], [None], dense_drop_rate=0.0, last_dense_drop_rate=0.5, training=True,
                     message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.ssgc(x, ei, None, [ws], [None], edge_drop_rate=0.3, training=True, message_dtype=b16)
    xs = sp.random(300, 16, density=0.1, format="csr", dtype=np.float32, random_state=0)
    with pytest.raises(NotImplementedError):
        tfg.nn.gin(xs, ei, lambda h: h, message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.tagcn(xs, ei, None, 2, _w(rs, 48, 8), message_dtype=b16)
    with pytest.raises(ValueError):
        tfg.nn.chebynet(x, ei, None, 2, [ws, ws], message_dtype=torch.float16)
    with torch.no_grad():                       # inactive dropout (inference) is accepted
        tfg.nn.appnp(x, ei, None, [ws], [None], dense_drop_rate=0.5, training=False, message_dtype=b16)
