# coding=utf-8
"""The GAT training path without the [E, H] coefficient table, kernel by kernel: tfgk_gat_fused_stats_f32 (forward that
keeps (max, denominator) per (row, head)) and tfgk_gat_bwd_prepare/dst/src_f32 (backward that recomputes every
coefficient), against float64 torch autograd over oracle.torch_cpu_port.gat_attention and against the coefficient-table
backward (tfgk_gat_softmax_bwd_f32 + tfgk_spmm_heads_f32) on the same inputs.

Tolerance: assert_close(rtol=1e-4, atol_scale=1e-5), ten times tighter than the 1e-3 / 2e-4 of the whole-layer gradient
tests.  Both kernels accumulate in float32 (unit roundoff 6e-8): a row of d edges carries a relative error of about
sqrt(d) * 6e-8 in its sums and a few ulp in every coefficient, i.e. 1e-7 .. 1e-6 of the largest gradient even at the
5000-edge rows used here.  On an H100 the largest error of any comparison below is 0.27 of this tolerance (the large-bias
case, see next paragraph) and at most 0.17 elsewhere, while each of the errors these tests are meant to catch (a lost
1/scale in dK, the statistics of head 0 read for every head, delta without the bias removed) fails dozens of them.

What the precision of delta = <G, Y - bias> rests on: Y = fl(out + bias) is stored in float32, so out is recovered
only to 2^-24 |Y| (Y - bias itself is exact).  The aggregate keeps about 24 - log2(|bias| / |out|) bits: about 17 bits
with a bias 100 times the aggregate, where dQ and dK of the recompute path are off by about 3e-6 of their largest entry
(the coefficient-table path, which sums delta from the coefficients, by 2e-7).  That is well inside the tolerance, so the
kernel keeps this formulation; the error grows linearly with |bias| / |out| and would reach the tolerance at about
400 times.  test_large_bias checks the 100-times case.

Inputs are float32 values; the float64 reference starts from the same values.  Where the relu is used, the upstream
gradient is zeroed at the few elements whose pre-activation lies within float32 rounding of 0: there the float32 and the
float64 forwards can disagree on the relu mask, which says nothing about the backward kernels."""
import numpy as np
import pytest
import torch

from tf_geometric_b200 import ops, autograd
from oracle import torch_cpu_port as port
from conftest import assert_close

pytestmark = pytest.mark.gpu

RTOL, ATOL_SCALE = 1e-4, 1e-5
SHAPES = [(8, 16), (8, 8), (8, 4), (4, 4), (4, 32), (2, 64), (1, 128), (1, 4)]      # (H, dqk)


# ---- graphs: (row, col, n_dst, n_src), numpy int64 -------------------------------------------------------------------

def _with_self_loops(row, col, n):
    loops = np.arange(n)
    return np.concatenate([row, loops]), np.concatenate([col, loops])


def _main_graph():
    """3000 nodes, ~8 random in-edges each; nodes 0-39 have only their self loop, 500 edges are duplicated, and node 77
    has a self loop of its own before the self loops are appended (two in total)."""
    rs = np.random.RandomState(1)
    n, e = 3000, 24000
    row, col = rs.randint(40, n, e), rs.randint(0, n, e)
    dup = rs.randint(0, e, 500)
    row, col = np.concatenate([row, row[dup], [77]]), np.concatenate([col, col[dup], [77]])
    return _with_self_loops(row, col, n) + (n, n)


def _long_rows_graph():
    """Destination 7 has HUB_THRESHOLD - 1 edges (the longest row that is not cut into hub slices) and source 11 is
    gathered by 5000 destinations: the longest row of the transposed CSR, which the backward walks without a plan."""
    rs = np.random.RandomState(2)
    n = 6000
    row, col = rs.randint(0, n, 12000), rs.randint(0, n, 12000)
    keep = row != 7
    row, col = row[keep], col[keep]
    fan = rs.choice(np.setdiff1d(np.arange(n), [7]), 5000, replace=False)
    row = np.concatenate([row, np.full(ops.HUB_THRESHOLD - 2, 7), fan])
    col = np.concatenate([col, rs.randint(0, n, ops.HUB_THRESHOLD - 2), np.full(5000, 11)])
    return _with_self_loops(row, col, n) + (n, n)


def _hub_graph():
    """Node 5 has 3 * HUB_CHUNK + 100 in-edges: the forward cuts it into slices merged by the fixup kernel."""
    rs = np.random.RandomState(3)
    n = 2000
    deg = 3 * ops.HUB_CHUNK + 100
    row = np.concatenate([rs.randint(0, n, 10000), np.full(deg, 5)])
    col = np.concatenate([rs.randint(0, n, 10000), rs.randint(0, n, deg)])
    return _with_self_loops(row, col, n) + (n, n)


def _set2set_graph():
    """The set2set layout: 7 destination rows (graphs) over 3000 source rows (nodes); graph 3 is empty and nodes 0-9
    belong to no graph, so they receive zero dK and dV."""
    rs = np.random.RandomState(4)
    n_src = 3000
    graph_of = np.sort(rs.randint(0, 6, n_src - 10))
    graph_of[graph_of >= 3] += 1
    return graph_of, np.arange(10, n_src), 7, n_src


def _small_graph(n):
    rs = np.random.RandomState(n)
    return _with_self_loops(rs.randint(0, n, 3 * n), rs.randint(0, n, 3 * n), n) + (n, n)


# ---- one case ---------------------------------------------------------------------------------------------------------

def _device_graph(row, col, n_dst, n_src):
    ei = torch.from_numpy(np.stack([row, col]).astype(np.int32)).cuda()
    csr = ops.csr_build(ei[0].contiguous(), ei[1].contiguous(), n_dst, n_src)
    csr_t, emap = autograd._transposed_of_csr(csr, ei)
    return csr, csr_t, emap


def _segment_stats(score, row, n_dst):
    """float64 (max, sum exp(s - max) + 1e-8) per (row, head) of the scaled scores [E, H]."""
    m = port._segment_max(score, row, n_dst)
    den = port._segment_sum(torch.exp(score - m.index_select(0, row)), row, n_dst) + 1e-8
    return m.numpy(), den.numpy()


def _check(graph, H, dqk, relu, with_bias, scale=None, seed=0, score_span=None, bias_mult=None):
    row, col, n_dst, n_src = graph
    A = H * dqk
    rs = np.random.RandomState(seed + 97 * H + dqk)
    Q = rs.randn(n_dst, A).astype(np.float32)
    K = rs.randn(n_src, A).astype(np.float32)
    V = rs.randn(n_src, A).astype(np.float32)
    G = rs.randn(n_dst, A).astype(np.float32)
    scale = float(np.sqrt(np.float32(dqk))) if scale is None else float(scale)      # what GatAttention hands the kernels
    row_t, col_t = torch.from_numpy(row.astype(np.int64)), torch.from_numpy(col.astype(np.int64))
    t64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))                      # noqa: E731
    E = row.shape[0]

    def scores(q, k):
        return (q.index_select(0, row_t).reshape(E, H, dqk) * k.index_select(0, col_t).reshape(E, H, dqk)).sum(-1) / scale

    if score_span is not None:                      # scale Q and K so that the scores span about +-score_span
        f = np.sqrt(score_span / float(scores(t64(Q), t64(K)).abs().max()))
        Q, K = (Q * f).astype(np.float32), (K * f).astype(np.float32)
    bias = None
    if with_bias:
        bias = (rs.randn(A) * 0.5).astype(np.float32)
        if bias_mult is not None:                   # |bias| about bias_mult times the aggregate
            agg = port.gat_attention(t64(Q), t64(K), t64(V), row_t, col_t, n_dst, H, scale=scale)
            bias = (np.sign(rs.randn(A)) * bias_mult * float(agg.abs().mean()) * (1 + 0.1 * rs.rand(A))).astype(np.float32)
    if relu:
        pre = port.gat_attention(t64(Q), t64(K), t64(V), row_t, col_t, n_dst, H, scale=scale,
                                 bias=None if bias is None else t64(bias)).numpy()
        G[np.abs(pre) < 1e-5 * np.abs(pre).max()] = 0.0
    act = ops.ACT_RELU if relu else ops.ACT_NONE

    # float64 reference
    Q64, K64, V64 = (t64(a).requires_grad_(True) for a in (Q, K, V))
    y64 = port.gat_attention(Q64, K64, V64, row_t, col_t, n_dst, H, scale=scale,
                             bias=None if bias is None else t64(bias), relu=relu)
    (y64 * t64(G)).sum().backward()
    m_ref, den_ref = _segment_stats(scores(Q64.detach(), K64.detach()), row_t, n_dst)
    want = {"dQ": Q64.grad.numpy(), "dK": K64.grad.numpy(), "dV": V64.grad.numpy()}

    # recompute path: stats forward, prepare, dst pass, src pass
    csr, csr_t, emap = _device_graph(row, col, n_dst, n_src)
    Qd, Kd, Vd, Gd = (torch.from_numpy(a).cuda() for a in (Q, K, V, G))
    bd = None if bias is None else torch.from_numpy(bias).cuda()
    res = ops.gat_fused_stats(csr, Qd, Kd, Vd, H, bias=bd, act=act, scale=scale)
    assert res is not None, "the stats forward refused H={} dqk={}".format(H, dqk)
    y, stats = res
    grads = ops.gat_backward_recompute(csr, csr_t, Qd, Kd, Vd, Gd, y, bd, act, stats, H, scale)
    assert grads is not None, "the recompute backward refused H={} dqk={}".format(H, dqk)
    torch.cuda.synchronize()
    assert_close(y.cpu().numpy(), y64.detach().numpy(), RTOL, ATOL_SCALE, what="stats forward out")
    st = stats.cpu().numpy()
    has_edges = np.bincount(row, minlength=n_dst) > 0
    assert_close(st[has_edges, :H], m_ref[has_edges], RTOL, ATOL_SCALE, what="stats: row maximum")
    assert_close(st[has_edges, H:], den_ref[has_edges], RTOL, ATOL_SCALE, what="stats: denominator")
    got = dict(zip(("dQ", "dK", "dV"), (g.cpu().numpy() for g in grads)))
    # a one-node graph has only copies of the self loop: every coefficient of a row is the same, delta = da and the exact
    # dQ and dK are 0.  What is left in float32 is the rounding of da - delta, bounded here by 1e-5 of the largest term
    # of those sums instead of 1e-5 of a result that is zero
    zero = ("dQ", "dK") if n_dst == 1 and n_src == 1 else ()
    term = float(np.abs(G).max() * np.abs(V).max() * max(np.abs(Q).max(), np.abs(K).max())) * dqk / scale

    def compare(mine, ref, name, what):
        if name in zero:
            assert np.abs(mine).max() <= ATOL_SCALE * term, "{} {}: {} is not 0".format(what, name, np.abs(mine).max())
        else:
            assert_close(mine, ref, RTOL, ATOL_SCALE, what=what + " " + name)

    for name in want:
        compare(got[name], want[name], name, "recompute backward")

    # coefficient-table path on the same inputs
    yt, att = ops.gat_fused(csr, Qd, Kd, Vd, H, bias=bd, act=act, return_attention=True, scale=scale)
    gm = autograd._relu_grad(Gd, yt) if relu else Gd
    ds = ops.gat_softmax_bwd(csr, att, gm, Vd, H)
    table = {"dQ": ops.spmm_heads(csr, ds, Kd, H, alpha=1.0 / scale),
             "dK": ops.spmm_heads(csr_t, ds, Qd, H, emap=emap, alpha=1.0 / scale),
             "dV": ops.spmm_heads(csr_t, att, gm, H, emap=emap)}
    assert_close(yt.cpu().numpy(), y64.detach().numpy(), RTOL, ATOL_SCALE, what="table forward out")
    for name in want:
        tab = table[name].cpu().numpy()
        compare(tab, want[name], name, "table backward")
        compare(got[name], tab, name, "recompute vs table")
    return csr


_MAIN = {}


def _main():
    if "g" not in _MAIN:
        _MAIN["g"] = _main_graph()
    return _MAIN["g"]


# (relu, bias, scale): every combination of the epilogue, half of them at scale = 1 (set2set's raw dot products)
EPILOGUES = [(False, False, None), (True, True, None), (True, False, 1.0), (False, True, 1.0)]


@pytest.mark.parametrize("H,dqk", SHAPES)
@pytest.mark.parametrize("relu,with_bias,scale", EPILOGUES)
def test_main_graph(H, dqk, relu, with_bias, scale):
    csr = _check(_main(), H, dqk, relu, with_bias, scale)
    assert csr.plan is None


@pytest.mark.parametrize("n", [1, 33, 129])
@pytest.mark.parametrize("H,dqk", [(8, 16), (4, 4), (2, 64), (1, 4)])
def test_graph_sizes_around_the_row_blocks(n, H, dqk):
    """The backward kernels take 32 rows per warp and 128 per block: a single row, one row past a warp, one past a block."""
    _check(_small_graph(n), H, dqk, relu=True, with_bias=True)


@pytest.mark.parametrize("H,dqk", [(8, 16), (4, 32), (1, 4)])
def test_long_rows(H, dqk):
    graph = _long_rows_graph()
    assert np.sum(graph[0] == 7) == ops.HUB_THRESHOLD - 1 and np.sum(graph[1] == 11) >= 5000
    csr = _check(graph, H, dqk, relu=True, with_bias=True)
    assert csr.plan is None


@pytest.mark.parametrize("H,dqk", [(8, 16), (2, 64), (1, 4)])
def test_hub_rows(H, dqk):
    """Through ops the stats of the hub row come from the hub-slice and fixup kernels; _check compares them too."""
    csr = _check(_hub_graph(), H, dqk, relu=False, with_bias=True)
    assert csr.plan is not None and csr.plan.n_hubs > 0


@pytest.mark.parametrize("dqk,scale", [(32, 1.0), (4, None), (16, 1.0)])
def test_set2set_layout(dqk, scale):
    _check(_set2set_graph(), 4, dqk, relu=False, with_bias=False, scale=scale)


@pytest.mark.parametrize("H,dqk", [(8, 16), (1, 128), (4, 4)])
def test_large_scores(H, dqk):
    """Scores spanning about +-60: exp(s - max) underflows for most edges of a row and the maximum must be exact."""
    _check(_main(), H, dqk, relu=False, with_bias=False, score_span=60.0)


@pytest.mark.parametrize("H,dqk", [(8, 16), (2, 64)])
@pytest.mark.parametrize("relu", [False, True])
def test_large_bias(H, dqk, relu):
    """bias about 100 times the aggregate: delta = <G, Y - bias> keeps about 17 bits of the aggregate (module docstring)."""
    _check(_main(), H, dqk, relu=relu, with_bias=True, bias_mult=100.0)


# ---- the two forward rings give the same bits -------------------------------------------------------------------------

def _stats_forward(csr, Q, K, V, H, bias, act):
    out, stats = ops.gat_fused_stats(csr, Q, K, V, H, bias=bias, act=act)
    torch.cuda.synchronize()
    return out.cpu(), stats.cpu()


@pytest.mark.parametrize("graph", ["main", "hub"])
@pytest.mark.parametrize("H,dqk", [(8, 16), (8, 8), (4, 32), (1, 128), (1, 4)])
def test_rings_give_identical_out_and_stats(graph, H, dqk):
    """K|V in one [N, 2A] buffer takes the TMA ring; separate K and V buffers, which is what the training layer hands over,
    take the cp.async ring.  Same edge order, same online softmax: the same bits."""
    row, col, n, _ = _main() if graph == "main" else _hub_graph()
    A = H * dqk
    rs = np.random.RandomState(H + dqk)
    csr, _, _ = _device_graph(row, col, n, n)
    Q = torch.from_numpy(rs.randn(n, A).astype(np.float32)).cuda()
    kv = torch.from_numpy(rs.randn(n, 2 * A).astype(np.float32)).cuda()
    K, V = kv[:, :A], kv[:, A:]
    bias = torch.from_numpy(rs.randn(A).astype(np.float32)).cuda()
    want = _stats_forward(csr, Q, K.contiguous(), V.contiguous(), H, bias, ops.ACT_RELU)      # cp.async ring
    out, stats = _stats_forward(csr, Q, K, V, H, bias, ops.ACT_RELU)                           # TMA ring
    assert torch.equal(out, want[0]), "out differs"
    assert torch.equal(stats, want[1]), "stats differ"


def _kernel_names(fn):
    """The tfgk kernels fn launches, as recorded by torch.profiler.  A session opened after another one in the same process
    can come back without any kernel record (only the runtime calls); such a session says nothing about the kernels, so
    up to three sessions are opened and the first that recorded a kernel is used."""
    for _ in range(3):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if "tfgk::" in e.name]
        if names:
            return " ".join(names)
    raise AssertionError("three profiler sessions recorded no tfgk kernel")


def test_joint_and_separate_buffers_reach_the_named_rings():
    """The ring test above is only worth something if the joint buffer really reaches the TMA kernel and the separate
    buffers the cp.async kernel."""
    row, col, n, _ = _main()
    A = 128
    csr, _, _ = _device_graph(row, col, n, n)
    Q = torch.randn(n, A, device="cuda")
    kv = torch.randn(n, 2 * A, device="cuda")
    names = {}
    for label, K, V in (("joint", kv[:, :A], kv[:, A:]), ("separate", kv[:, :A].contiguous(), kv[:, A:].contiguous())):
        ops.gat_fused_stats(csr, Q, K, V, 8)
        names[label] = _kernel_names(lambda: ops.gat_fused_stats(csr, Q, K, V, 8))
    assert "gat_tma4_kernel" in names["joint"] and "gat_async_kernel" not in names["joint"], names["joint"]
    assert "gat_async_kernel" in names["separate"] and "gat_tma4_kernel" not in names["separate"], names["separate"]


# ---- the stats forward takes exactly the shapes the recompute backward takes -------------------------------------------

def test_stats_forward_only_takes_shapes_the_backward_takes():
    """A forward that keeps (max, denominator) for a shape the backward refuses would leave the layer without a backward
    (GatAttention raised on the first backward() for GAT(64, num_heads=16)).  Whenever ops.gat_fused_stats returns a
    result, ops.gat_backward_recompute must too; the accepted set is H in {1, 2, 4, 8}, dqk / 4 a power of two,
    H * dqk <= 128."""
    row, col, n, _ = _small_graph(40)
    csr, csr_t, _ = _device_graph(row, col, n, n)
    rs = np.random.RandomState(0)
    accepted = []
    for H in (1, 2, 3, 4, 8, 16, 32):
        for dqk in (1, 2, 4, 8, 12, 16, 32, 64, 128):
            A = H * dqk
            Q, K, V, G = (torch.from_numpy(rs.randn(n, A).astype(np.float32)).cuda() for _ in range(4))
            res = ops.gat_fused_stats(csr, Q, K, V, H)
            expected = H in (1, 2, 4, 8) and dqk % 4 == 0 and (dqk // 4) & (dqk // 4 - 1) == 0 and A <= 128
            assert (res is not None) == expected, (H, dqk)
            if res is not None:
                accepted.append((H, dqk))
                grads = ops.gat_backward_recompute(csr, csr_t, Q, K, V, G, res[0], None, ops.ACT_NONE, res[1], H,
                                                   float(np.sqrt(np.float32(dqk))))
                assert grads is not None, (H, dqk)
    torch.cuda.synchronize()
    assert (8, 16) in accepted and (16, 4) not in accepted and (32, 4) not in accepted
