# coding=utf-8
"""Training steps without a GPU.

1. A SparseMatrix whose values are a learnable parameter, updated in place between steps (what optimizer.step() does):
   the forward, dh, d value, segment_sum and segment_softmax of the next step must use the new values, over the CPU fake
   of the kernel layer.
2. The bound of the GPU training contract (tests/train_bound.py) is tight enough to see the faults it is meant to catch:
   each planted fault below falls outside it on the row it affects, while the same computation done right in float32
   stays inside."""
import numpy as np
import pytest
import torch

import edge_grad_fake_backend
import train_bound as tb
from conftest import assert_close, random_graph


@pytest.fixture
def fake(monkeypatch):
    edge_grad_fake_backend.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg


def _graph(n=30, e=120, seed=1):
    rs = np.random.RandomState(0)
    ei = random_graph(n, e, seed=seed)
    w = torch.nn.Parameter(torch.tensor(rs.rand(ei.shape[1]).astype(np.float32) + 0.5))
    return rs, ei, w


def _spmm64(ei, w, h, n):
    return torch.zeros(n, h.shape[1], dtype=torch.float64).index_add_(
        0, torch.tensor(ei[0]).long(), w.detach().double()[:, None] * h.detach().double()[torch.tensor(ei[1]).long()])


# ---- 1. values updated in place -----------------------------------------------------------------------------------

def test_sparse_matmul_after_in_place_update(fake):
    """Forward, dh and d value of A @ h after w.mul_(2): the permuted copies of the values are rebuilt."""
    rs, ei, w = _graph()
    n = 30
    A = fake.SparseMatrix(torch.tensor(ei), w, [n, n])
    assert A.value is w
    opt = torch.optim.SGD([w], lr=0.5)
    for step in range(3):
        h = torch.tensor(rs.randn(n, 4).astype(np.float32), requires_grad=True)
        g = rs.randn(n, 4)
        opt.zero_grad()
        y = A.matmul(h)
        (y * torch.tensor(g, dtype=torch.float32)).sum().backward()
        w64 = w.detach().double().requires_grad_(True)
        h64 = h.detach().double().requires_grad_(True)
        r, c = torch.tensor(ei[0]).long(), torch.tensor(ei[1]).long()
        y64 = torch.zeros(n, 4, dtype=torch.float64).index_add(0, r, w64[:, None] * h64[c])
        (y64 * torch.tensor(g)).sum().backward()
        what = "step {} ".format(step)
        assert_close(y.detach().numpy(), y64.detach().numpy(), what=what + "forward")
        assert_close(h.grad.numpy(), h64.grad.numpy(), what=what + "dh")
        assert_close(w.grad.numpy(), w64.grad.numpy(), what=what + "d value")
        opt.step()                                       # in place: the same tensor, a new version
        if step == 0:
            with torch.no_grad():
                w.mul_(2.0)                              # and a second in-place update before the next product


def test_segment_sum_and_softmax_after_in_place_update(fake):
    rs, ei, w = _graph(seed=2)
    n = 30
    A = fake.SparseMatrix(torch.tensor(ei), w, [n, n])
    A.segment_sum(), A.segment_softmax()                 # builds and keeps the CSR-ordered values
    with torch.no_grad():
        w.mul_(-1.5).add_(0.25)
    row = torch.tensor(ei[0]).long()
    v = w.detach().double()
    want = torch.zeros(n, dtype=torch.float64).index_add(0, row, v)
    assert_close(A.segment_sum().numpy(), want.numpy(), what="row sums after the update")
    col_sums = torch.zeros(n, dtype=torch.float64).index_add(0, torch.tensor(ei[1]).long(), v)
    assert_close(A.segment_sum(axis=0).numpy(), col_sums.numpy(), what="column sums after the update")
    m = torch.full((n,), -np.inf, dtype=torch.float64).scatter_reduce(0, row, v, "amax")
    ex = torch.exp(v - m[row])
    soft = ex / (torch.zeros(n, dtype=torch.float64).index_add(0, row, ex)[row] + 1e-8)
    assert_close(A.segment_softmax().value.numpy(), soft.numpy(), rtol=1e-5, atol_scale=1e-6,
                 what="segment softmax after the update")


def test_value_replaced_by_another_tensor(fake):
    """Assigning a new tensor to `value` (same shape, other storage) is seen too."""
    rs, ei, w = _graph(seed=3)
    n = 30
    A = fake.SparseMatrix(torch.tensor(ei), w.detach().clone(), [n, n])
    h = torch.tensor(rs.randn(n, 3).astype(np.float32))
    A.matmul(h)
    A.value = w.detach() * 3.0
    assert_close(A.matmul(h).numpy(), _spmm64(ei, A.value, h, n).numpy(), what="product with the new value tensor")


def test_unchanged_values_keep_one_permute(fake, monkeypatch):
    """Inference with values that never change permutes them once, however many products follow."""
    rs, ei, w = _graph(seed=4)
    n = 30
    A = fake.SparseMatrix(torch.tensor(ei), w.detach().clone(), [n, n])
    calls = _counting_permute(monkeypatch)
    h = torch.tensor(rs.randn(n, 3).astype(np.float32))
    first = A.matmul(h)
    for _ in range(4):
        np.testing.assert_array_equal(A.matmul(h).numpy(), first.numpy())
        A.segment_sum()
    assert len(calls) == 1


def test_prebuilt_csr_values_follow_their_source(fake):
    """A matrix built with its CSR-ordered values (segment_softmax's result) keeps them until its value changes."""
    rs, ei, w = _graph(seed=5)
    n = 30
    soft = fake.SparseMatrix(torch.tensor(ei), w.detach().clone(), [n, n]).segment_softmax()
    kept = soft.value_csr
    assert soft.value_csr is kept
    with torch.no_grad():
        soft.value.mul_(2.0)
    np.testing.assert_array_equal(soft.value_csr.numpy(), soft.value.numpy()[soft.csr.perm.numpy()])


def _counting_permute(monkeypatch):
    from tf_geometric_b200 import ops
    calls = []
    real = ops.permute

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(ops, "permute", counting)
    return calls


def test_inference_mode_values(fake, monkeypatch):
    """Values made under torch.inference_mode() have no version counter: GCN (whose self-loop weights and normalised
    values are made there), segment_softmax and A @ h work, give the products of the same values made outside inference
    mode, and permute each matrix's values once however many products follow."""
    rs, ei, w = _graph(seed=6)
    n = 30
    x = torch.tensor(rs.randn(n, 5).astype(np.float32))
    layer = fake.layers.GCN(4, seed=1)
    want_gcn = layer([x, torch.tensor(ei), w.detach()]).detach()
    want_soft = fake.SparseMatrix(torch.tensor(ei), w.detach() * 2, [n, n]).segment_softmax().value
    want_mm = fake.SparseMatrix(torch.tensor(ei), w.detach() * 2, [n, n]).matmul(x)
    with torch.inference_mode():
        np.testing.assert_array_equal(layer([x, torch.tensor(ei), w.detach()]).numpy(), want_gcn.numpy())
        A = fake.SparseMatrix(torch.tensor(ei), w.detach() * 2, [n, n])
        assert A.value.is_inference()
        calls = _counting_permute(monkeypatch)
        soft = A.segment_softmax()
        np.testing.assert_array_equal(soft.value.numpy(), want_soft.numpy())
        assert len(calls) == 2                     # A's values into the CSR, the softmax back into edge order
        for _ in range(3):
            np.testing.assert_array_equal(A.matmul(x).numpy(), want_mm.numpy())
            A.segment_sum()
            soft.matmul(x)                         # its CSR-ordered values came with it from the constructor
            soft.segment_sum()
        assert len(calls) == 2


def test_replaced_value_is_not_kept_alive(fake):
    """The stamp of the permuted copies holds the value it was made from by weak reference only."""
    import gc
    import weakref
    rs, ei, w = _graph(seed=7)
    n = 30
    A = fake.SparseMatrix(torch.tensor(ei), w.detach().clone(), [n, n])
    A.matmul(torch.tensor(rs.randn(n, 3).astype(np.float32)))
    old = weakref.ref(A.value)
    A.value = w.detach() * 3.0
    gc.collect()
    assert old() is None


# ---- 2. tightness of the contract's bound ---------------------------------------------------------------------------

def _hub_graph():
    """1500 nodes, 6 random in-edges each, and source 7 gathered by 2500 destinations (a hub of the transposed CSR only)."""
    rs = np.random.RandomState(11)
    n = 1500
    row, col = rs.randint(0, n, 6 * n), rs.randint(0, n, 6 * n)
    row = np.concatenate([row, rs.randint(0, n, 2500)])
    col = np.concatenate([col, np.full(2500, 7)])
    return rs, n, row.astype(np.int64), col.astype(np.int64)


def _transposed(row, col, n):
    """(rowptr, col, perm) of the reversed edges, stable by edge order (what csr_build gives)."""
    perm = np.argsort(col, kind="stable")
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(col, minlength=n))])
    return rowptr, row[perm], perm


def _dx_mean(row, col, w, g, n, magnitude=False):
    """dx of a mean aggregation, float64: sum over edges with col_e = c of (w_e / cnt[row_e]) g[row_e]."""
    R = tb.Replay(magnitude)
    cnt = torch.tensor(np.maximum(np.bincount(row, minlength=n), 1).astype(np.float64))
    wt = R.const(w) / cnt[torch.from_numpy(row)]
    return R.spmm(torch.from_numpy(col), torch.from_numpy(row), wt, R.upstream(g), n).numpy()


def _k1_f32(rowptr, cols, vals, g):
    """K1 as a float32 model: each row summed in CSR order."""
    out = np.zeros((len(rowptr) - 1, g.shape[1]), np.float32)
    for r in range(len(rowptr) - 1):
        acc = np.zeros(g.shape[1], np.float32)
        for p in range(rowptr[r], rowptr[r + 1]):
            acc = (acc + np.float32(vals[p]) * g[cols[p]]).astype(np.float32)
        out[r] = acc
    return out


@pytest.fixture(scope="module")
def dx_case():
    rs, n, row, col = _hub_graph()
    w = (rs.rand(len(row)) + 0.5).astype(np.float32)
    g = rs.randn(n, 16).astype(np.float32)
    cnt = np.maximum(np.bincount(row, minlength=n), 1).astype(np.float32)
    w_fwd_scaled = (w / cnt[row]).astype(np.float32)                     # in edge order
    rowptr, cols, perm = _transposed(row, col, n)
    ref = _dx_mean(row, col, w, g, n)
    S = _dx_mean(row, col, w, g, n, magnitude=True)
    e = tb.transposed_gather_eps(row, col, n)                           # SparseMatrix.matmul's dh in the GPU contract
    return dict(rs=rs, n=n, row=row, col=col, w=w, g=g, w_t=w_fwd_scaled[perm], rowptr=rowptr, cols=cols, perm=perm,
                ref=ref, S=S, e=e)


def test_bound_holds_for_the_float32_transposed_product(dx_case):
    c = dx_case
    got = _k1_f32(c["rowptr"], c["cols"], c["w_t"], c["g"])
    r = tb.ratio(got, c["ref"], c["S"], c["e"])
    assert r <= 1.0, r


def test_bound_catches_a_dropped_hub_edge(dx_case):
    """The hub source's last edge left out of the transposed product."""
    c = dx_case
    rowptr = c["rowptr"].copy()
    hub = 7
    keep = np.ones(len(c["cols"]), bool)
    keep[rowptr[hub + 1] - 1] = False
    rowptr[hub + 1:] -= 1
    got = _k1_f32(rowptr, c["cols"][keep], c["w_t"][keep], c["g"])
    assert tb.ratio(got[hub], c["ref"][hub], c["S"][hub], c["e"][hub]) > 1.0
    others = np.arange(c["n"]) != hub
    assert tb.ratio(got[others], c["ref"][others], c["S"][others], c["e"][others]) <= 1.0


def test_bound_catches_forward_ordered_weights(dx_case):
    """The scaled weights taken in the forward CSR's order instead of the transposed CSR's."""
    c = dx_case
    fwd_perm = np.argsort(c["row"], kind="stable")
    w_fwd = (c["w"] / np.maximum(np.bincount(c["row"], minlength=c["n"]), 1)[c["row"]]).astype(np.float32)[fwd_perm]
    got = _k1_f32(c["rowptr"], c["cols"], w_fwd, c["g"])
    assert tb.ratio(got[7], c["ref"][7], c["S"][7], c["e"][7]) > 1.0


def test_bound_catches_the_value_before_the_update(dx_case):
    """dh = A^T g with the values from before an SGD step w -= lr * dw."""
    c = dx_case
    step = (0.05 * c["rs"].randn(len(c["w"]))).astype(np.float32)
    new_w = (c["w"] - step).astype(np.float32)
    cnt = np.maximum(np.bincount(c["row"], minlength=c["n"]), 1).astype(np.float32)
    ref = _dx_mean(c["row"], c["col"], new_w, c["g"], c["n"])
    S = _dx_mean(c["row"], c["col"], new_w, c["g"], c["n"], magnitude=True)
    stale = _k1_f32(c["rowptr"], c["cols"], c["w_t"], c["g"])              # built from c["w"]
    fresh = _k1_f32(c["rowptr"], c["cols"], (new_w / cnt[c["row"]]).astype(np.float32)[c["perm"]], c["g"])
    assert tb.ratio(fresh, ref, S, c["e"]) <= 1.0
    assert tb.ratio(stale[7], ref[7], S[7], c["e"][7]) > 1.0


def _gcn_dx(row, col, w, g, k, n, magnitude=False, drop=None):
    """GCN's dx = (norm(A)^T g) K^T in float64 (self loops appended), or its magnitude replay; `drop` leaves that edge
    of the transposed product out."""
    R = tb.Replay(magnitude)
    r2, c2, v = R.gcn_norm(torch.from_numpy(row), torch.from_numpy(col), R.const(w), n)
    if drop is not None:
        keep = torch.ones(len(r2), dtype=torch.bool)
        keep[drop] = False
        r2, c2, v = r2[keep], c2[keep], v[keep]
    dh = R.spmm(c2, r2, v, R.upstream(g), n)
    return (dh @ R.const(k).T).numpy()


def _gcn_dx_f32(row, col, w, g, k, n, perm=None):
    """The same in float32: degree sums, rsqrt and the two scalings, the transposed product summed in CSR order (values
    taken through `perm`, the transposed CSR's permutation unless another is planted), then x K^T."""
    r2 = np.concatenate([row, np.arange(n)])
    c2 = np.concatenate([col, np.arange(n)])
    w2 = np.concatenate([w, np.ones(n, np.float32)]).astype(np.float32)
    deg = np.zeros(n, np.float32)
    for e_ in range(len(r2)):
        deg[r2[e_]] = np.float32(deg[r2[e_]] + w2[e_])
    dis = (np.float32(1) / np.sqrt(deg)).astype(np.float32)
    v = (dis[r2] * w2 * dis[c2]).astype(np.float32)
    rowptr, cols, tperm = _transposed(r2, c2, n)
    dh = _k1_f32(rowptr, cols, v[tperm if perm is None else perm], g)
    return (dh @ k.T.astype(np.float32)).astype(np.float32)


@pytest.fixture(scope="module")
def gcn_case():
    """GCN's dx on the hub graph, bounded by the GPU contract's own expression (tb.gcn_dx_eps) at U = 128."""
    rs, n, row, col = _hub_graph()
    w = (rs.rand(len(row)) + 0.5).astype(np.float32)
    g = rs.randn(n, 128).astype(np.float32)
    k = (rs.randn(16, 128) * 0.1).astype(np.float32)
    e = tb.gcn_dx_eps(row, col, n, 128)
    light = int(np.flatnonzero(np.bincount(col, minlength=n) == 6)[0])  # a source of out-degree 6
    return dict(rs=rs, n=n, row=row, col=col, w=w, g=g, k=k, e=e, light=light,
                ref=_gcn_dx(row, col, w, g, k, n), S=_gcn_dx(row, col, w, g, k, n, magnitude=True))


def test_gcn_dx_bound_holds_in_float32(gcn_case):
    c = gcn_case
    got = _gcn_dx_f32(c["row"], c["col"], c["w"], c["g"], c["k"], c["n"])
    assert tb.ratio(got, c["ref"], c["S"], c["e"]) <= 1.0


def test_gcn_dx_bound_catches_a_dropped_edge(gcn_case):
    """One edge of a light source row left out of the transposed product.  (At the hub source, one edge of 2 500 moves
    dx by less than that row's worst-case rounding after the 128-wide projection, which no rounding bound can tell
    apart; the sparse product's dh, which has no projection after the gather, catches it above.)"""
    c = gcn_case
    r = c["light"]
    drop = int(np.flatnonzero(c["col"] == r)[-1])
    got = _gcn_dx(c["row"], c["col"], c["w"], c["g"], c["k"], c["n"], drop=drop)
    assert tb.ratio(got[r], c["ref"][r], c["S"][r], c["e"][r]) > 1.0


def test_gcn_dx_bound_catches_forward_ordered_values(gcn_case):
    c = gcn_case
    n = c["n"]
    r2 = np.concatenate([c["row"], np.arange(n)])
    got = _gcn_dx_f32(c["row"], c["col"], c["w"], c["g"], c["k"], n, perm=np.argsort(r2, kind="stable"))
    assert tb.ratio(got[7], c["ref"][7], c["S"][7], c["e"][7]) > 1.0


def test_gcn_dx_bound_catches_the_value_before_the_update(gcn_case):
    c = gcn_case
    r = c["light"]
    new_w = (c["w"] - 0.05 * c["rs"].randn(len(c["w"]))).astype(np.float32)
    ref = _gcn_dx(c["row"], c["col"], new_w, c["g"], c["k"], c["n"])
    S = _gcn_dx(c["row"], c["col"], new_w, c["g"], c["k"], c["n"], magnitude=True)
    assert tb.ratio(c["ref"][r], ref[r], S[r], c["e"][r]) > 1.0            # dx computed from the old weights


def _split_k_dw(x, g, slice_rows, skip=None):
    """dW = x^T g as the split-K kernel computes it: float32 partial sums over slices of rows, then the slices added in
    order; `skip` leaves one slice out."""
    K = x.shape[0]
    acc = np.zeros((x.shape[1], g.shape[1]), np.float32)
    for i, k0 in enumerate(range(0, K, slice_rows)):
        if i == skip:
            continue
        part = np.zeros_like(acc)
        for k in range(k0, min(K, k0 + slice_rows)):
            part = (part + np.outer(x[k], g[k]).astype(np.float32)).astype(np.float32)
        acc = (acc + part).astype(np.float32)
    return acc


def test_bound_catches_an_omitted_split_k_slice():
    rs = np.random.RandomState(12)
    K, F, Uo = 8192, 6, 5
    x, g = rs.randn(K, F).astype(np.float32), rs.randn(K, Uo).astype(np.float32)
    ref = x.astype(np.float64).T @ g.astype(np.float64)
    S = np.abs(x.astype(np.float64)).T @ np.abs(g.astype(np.float64))
    e = tb.eps(K + 3)
    assert tb.ratio(_split_k_dw(x, g, 1024), ref, S, e) <= 1.0
    got = _split_k_dw(x, g, 1024, skip=3)
    for f in range(F):                                                     # every row of dW is affected
        assert tb.ratio(got[f], ref[f], S[f], e) > 1.0, f


def test_magnitude_replay_of_the_normalisation():
    """The magnitude mode of the GCN normalisation: same values, and a derivative that is the absolute value of the
    exact one, so that d w of a normalised product sums magnitudes."""
    rs = np.random.RandomState(13)
    n = 40
    row, col = torch.from_numpy(rs.randint(0, n, 200)), torch.from_numpy(rs.randint(0, n, 200))
    w = (rs.rand(200) + 0.1).astype(np.float32)
    outs = []
    for mag in (False, True):
        R = tb.Replay(mag)
        wt = R.leaf(w)
        _, _, v = R.gcn_norm(row, col, wt, n)
        v.sum().backward()
        outs.append((v.detach().numpy(), wt.grad.numpy()))
    np.testing.assert_allclose(outs[0][0], outs[1][0], rtol=1e-15)
    assert (outs[1][1] >= np.abs(outs[0][1]) * (1 - 1e-12)).all()
    assert (outs[1][1] > np.abs(outs[0][1]) * 1.01).any()                # the signed terms cancel, the magnitudes do not
