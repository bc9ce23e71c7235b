# coding=utf-8
"""K10 (the CSR x CSR product), cluster_pool and ASAP on the H100: K10 bit-exact against the numpy Gustavson restatement
and within 1e-5 of float64 scipy, independent of the workspace budget; cluster_pool and ASAP against the float64
restatement of the reference (forward and every gradient); a 200 000-node graph; and the demo_asap architecture trained
on graphs with 2 or 4 planted communities."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import asap_fake_backend as fake_k10
import asap_ref as ref
from conftest import assert_close

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _dev(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a), device=DEV)
    return t if dtype is None else t.to(dtype)


def _unsorted_csr(rs, n_rows, n_cols, nnz, dup=0, empty_rows=()):
    """CSR arrays with unsorted columns, `dup` repeated (row, col) pairs and the given rows empty."""
    row = rs.randint(0, n_rows, nnz)
    col = rs.randint(0, n_cols, nnz)
    if dup:
        row, col = np.concatenate([row, row[:dup]]), np.concatenate([col, col[:dup]])
    keep = ~np.isin(row, list(empty_rows))
    row, col = row[keep], col[keep]
    order = np.argsort(row, kind="stable")
    row, col = row[order], col[order]
    val = rs.uniform(-1, 1, len(row)).astype(np.float32)
    rowptr = np.zeros(n_rows + 1, np.int64)
    rowptr[1:] = np.cumsum(np.bincount(row, minlength=n_rows))
    return rowptr, col.astype(np.int32), val


def _spgemm_both(a, b, n_cols, budget=None):
    from tf_geometric_b200 import ops
    kw = {} if budget is None else {"budget": budget}
    got = ops.spgemm(*[_dev(v) for v in a], *[_dev(v) for v in b], n_cols, **kw)
    want = fake_k10.spgemm_reference(*a, *b, n_cols)
    return [g.cpu().numpy() for g in got], want


def _hub_case(rs):
    a = _unsorted_csr(rs, 400, 3000, 3000)
    rowptr, col, val = a
    hub_cols = rs.randint(0, 3000, 4500).astype(np.int32)                  # row 7 gets 4 500 more entries
    pos = rowptr[8]
    col = np.concatenate([col[:pos], hub_cols, col[pos:]])
    val = np.concatenate([val[:pos], rs.uniform(-1, 1, 4500).astype(np.float32), val[pos:]])
    rowptr = rowptr.copy()
    rowptr[8:] += 4500
    return (rowptr, col, val), _unsorted_csr(rs, 3000, 2000, 40000, dup=100), 2000


CASES = {
    # empty rows of A, an empty row of B, duplicates on both sides
    "small": lambda rs: (_unsorted_csr(rs, 300, 200, 2000, dup=40, empty_rows=(0, 17, 299)),
                         _unsorted_csr(rs, 200, 250, 1500, dup=30, empty_rows=(5, 6)), 250),
    # more than 2^16 columns
    "wide": lambda rs: (_unsorted_csr(rs, 500, 3000, 6000), _unsorted_csr(rs, 3000, 70000, 40000), 70000),
    # a hub row of A whose expansion (about 4 500 x 13 products) is far beyond the shared-memory tier
    "hub": _hub_case,
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_k10_bit_exact_against_gustavson(case):
    a, b, n_cols = CASES[case](np.random.RandomState(len(case)))
    got, want = _spgemm_both(a, b, n_cols)
    for g, w, name in zip(got, want, ("rowptr", "col", "val")):
        np.testing.assert_array_equal(g, w, err_msg=name)
    if case == "hub":
        prod = np.diff(b[0])[a[1][a[0][7]:a[0][8]]].sum()
        assert prod > 4 * 2048, prod
    # bits identical across runs and when every row is its own chunk
    again, _ = _spgemm_both(a, b, n_cols)
    tiny, _ = _spgemm_both(a, b, n_cols, budget=0)
    for g, h, t in zip(got, again, tiny):
        np.testing.assert_array_equal(g, h)
        np.testing.assert_array_equal(g, t)


def test_k10_stats_against_scipy_with_a_hub():
    """S^T A S for a graph with a node of in-degree 5 000 and an ASAP-like assignment (every edge whose target is selected
    assigns its source to that target's cluster), against float64 scipy."""
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(3)
    n = 20000
    row = np.concatenate([rs.randint(0, n, 10 * n), np.full(5000, 11)])
    col = rs.randint(0, n, len(row))
    w = rs.uniform(0.5, 1.5, len(row))
    A = sp.csr_matrix((w, (row, col)), shape=(n, n))
    sel = np.unique(np.concatenate([[11], rs.choice(n, n // 2, replace=False)]))
    cl = -np.ones(n, np.int64)
    cl[sel] = np.arange(len(sel))
    m = cl[row] >= 0
    S = sp.csr_matrix((rs.uniform(0.1, 1, m.sum()), (col[m], cl[row[m]])), shape=(n, len(sel)))
    St = S.T.tocsr()
    a = [_dev(v) for v in (A.indptr.astype(np.int64), A.indices.astype(np.int32), A.data.astype(np.float32))]
    s = [_dev(v) for v in (S.indptr.astype(np.int64), S.indices.astype(np.int32), S.data.astype(np.float32))]
    st = [_dev(v) for v in (St.indptr.astype(np.int64), St.indices.astype(np.int32), St.data.astype(np.float32))]
    t = ops.spgemm(*st, *a, n)
    p = ops.spgemm(*t, *s, len(sel))
    got = sp.csr_matrix((p[2].cpu().numpy().astype(np.float64), p[1].cpu().numpy(), p[0].cpu().numpy()),
                        shape=(len(sel), len(sel)))
    S64, A64 = S.astype(np.float32).astype(np.float64), A.astype(np.float32).astype(np.float64)
    want = (S64.T @ A64 @ S64).tocsr()
    want.sort_indices()
    np.testing.assert_array_equal(got.indptr, want.indptr)
    np.testing.assert_array_equal(got.indices, want.indices)
    err = np.abs(got.data - want.data)
    assert np.all(err <= 1e-5 * np.abs(want.data) + 1e-6 * np.abs(want.data).max()), err.max()
    tiny = ops.spgemm(*t, *s, len(sel), budget=0)
    assert torch.equal(tiny[2], p[2]) and torch.equal(tiny[1], p[1])


def test_k10_rejects_out_of_range_columns():
    from tf_geometric_b200 import ops, _ffi
    a = (np.array([0, 2], np.int64), np.array([0, 5], np.int32), np.ones(2, np.float32))
    b = (np.array([0, 1, 2], np.int64), np.array([0, 1], np.int32), np.ones(2, np.float32))
    with pytest.raises(_ffi.TfgkError) as err:
        ops.spgemm(*[_dev(v) for v in a], *[_dev(v) for v in b], 2)
    assert err.value.code == _ffi.ERR_INDEX_OUT_OF_RANGE
    a = (np.array([0, 1], np.int64), np.array([1], np.int32), np.ones(1, np.float32))
    with pytest.raises(_ffi.TfgkError) as err:
        ops.spgemm(*[_dev(v) for v in a], *[_dev(v) for v in b], 1)               # B's column 1 is outside [0, 1)
    assert err.value.code == _ffi.ERR_INDEX_OUT_OF_RANGE


# ---- cluster_pool ------------------------------------------------------------------------------------------------

def test_cluster_pool_against_float64():
    import tf_geometric_b200 as tfg
    x, ei, w, aei, aw, K, N = ref.cluster_case()
    for weight in (w, None):
        xt, awt = _dev(x).requires_grad_(), _dev(aw).requires_grad_()
        px, pei, pw = tfg.nn.cluster_pool(xt, _dev(ei), None if weight is None else _dev(weight), _dev(aei), awt, K)
        x64, aw64 = ref.t64(x, True), ref.t64(aw, True)
        want_x, want_ei, want_w = ref.cluster_pool(x64, ei, ref.t64(np.ones(ei.shape[1]) if weight is None else weight),
                                                   aei, aw64, K, N)
        np.testing.assert_array_equal(pei.cpu().numpy(), want_ei)
        assert_close(pw.detach().cpu().numpy(), want_w.detach().numpy(), what="pooled w")
        assert_close(px.detach().cpu().numpy(), want_x.detach().numpy(), what="pooled x")
        g = np.random.RandomState(2).randn(*px.shape)
        (px * _dev(g, torch.float32)).sum().backward()
        (want_x * torch.tensor(g)).sum().backward()
        assert_close(xt.grad.cpu().numpy(), x64.grad.numpy(), what="d x")
        assert_close(awt.grad.cpu().numpy(), aw64.grad.numpy(), what="d assign w")
    wt = _dev(w).requires_grad_()
    _, _, pw = tfg.nn.cluster_pool(None, _dev(ei), wt, _dev(aei), _dev(aw), K, num_nodes=N)
    with pytest.raises(RuntimeError, match="pooled edge weights"):
        pw.sum().backward()


# ---- ASAP --------------------------------------------------------------------------------------------------------

def _params(F, seed):
    return {k: _dev(v).requires_grad_() for k, v in ref.random_params(F, seed).items()}


def _asap(x, ei, w, ngi, p, **kw):
    import tf_geometric_b200 as tfg
    return tfg.nn.asap(x, ei, w, ngi, *[p[k] for k in ref.ORDER], None, **kw)


def _grads_close(pairs, rtol=1e-3, atol_scale=1e-4):
    scale = max(float(np.max(np.abs(w))) for _, _, w in pairs if np.size(w))
    for name, got, want in pairs:
        err = np.abs(np.asarray(got, np.float64) - want)
        assert np.all(err <= rtol * np.abs(want) + atol_scale * scale), "d {}: max err {:.3e} (scale {:.3e})".format(
            name, err.max(), scale)


@pytest.mark.parametrize("with_weight,drop,sel", [(False, 0.0, dict(ratio=0.5)), (True, 0.0, dict(k=3)),
                                                  (True, 0.3, dict(ratio=0.5)), (False, 0.3, dict(k=2))])
def test_asap_forward_and_gradients_against_float64(with_weight, drop, sel):
    from tf_geometric_b200 import ops
    F = 8
    x, ei, w, ngi = ref.batch([9, 1, 12, 6, 15], seed=5, F=F)
    p = _params(F, 4)
    xt = _dev(x).requires_grad_()
    wt = _dev(w).requires_grad_() if with_weight else None
    px, pei, pw, pngi = _asap(xt, _dev(ei), wt, _dev(ngi), p, drop_rate=drop, training=True, seed=77, **sel)
    mask = None
    if drop:
        n_sl = int((ei[0] != ei[1]).sum()) + x.shape[0]
        mask = torch.tensor(ops.dropout(torch.ones(n_sl, device=DEV), drop, 77).cpu().numpy(), dtype=torch.float64)
    x64, w64 = ref.t64(x, True), (ref.t64(w, True) if with_weight else None)
    p64 = {k: ref.t64(v.detach().cpu().numpy(), True) for k, v in p.items()}
    want_x, want_ei, want_w, want_ngi, _ = ref.asap(x64, ei, w64, ngi, p64, drop_mask=mask, **sel)
    np.testing.assert_array_equal(pei.cpu().numpy(), want_ei)
    np.testing.assert_array_equal(pngi.cpu().numpy(), want_ngi)
    assert_close(px.detach().cpu().numpy(), want_x.detach().numpy(), what="pooled x")
    assert_close(pw.detach().cpu().numpy(), want_w.detach().numpy(), what="pooled w")
    g = np.random.RandomState(6).randn(*px.shape)
    (px * _dev(g, torch.float32)).sum().backward()
    (want_x * torch.tensor(g)).sum().backward()
    pairs = [("x", xt.grad.cpu().numpy(), x64.grad.numpy())]
    pairs += [(k, p[k].grad.cpu().numpy(), p64[k].grad.numpy()) for k in ref.ORDER]
    if with_weight:
        pairs.append(("edge_weight", wt.grad.cpu().numpy(), w64.grad.numpy()))
    _grads_close(pairs)


def test_asap_bits_do_not_depend_on_requires_grad_and_backward_is_deterministic():
    F = 16
    x, ei, w, ngi = ref.batch([30, 25, 40, 2], seed=9, F=F)
    plain = _asap(_dev(x), _dev(ei), _dev(w), _dev(ngi), {k: v.detach() for k, v in _params(F, 1).items()}, ratio=0.5)
    grads = []
    for _ in range(2):
        p = _params(F, 1)
        xt = _dev(x).requires_grad_()
        out = _asap(xt, _dev(ei), _dev(w), _dev(ngi), p, ratio=0.5)
        for a, b in zip(plain, out):
            assert torch.equal(a, b.detach())
        (out[0] * out[0]).sum().backward()
        grads.append([xt.grad.clone()] + [p[k].grad.clone() for k in ref.ORDER])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def test_asap_layer_edgeless_graph_and_errors():
    import tf_geometric_b200 as tfg
    x, ei, _, ngi = ref.batch([6, 1, 5], seed=1, F=4)
    layer = tfg.layers.ASAP(ratio=0.5, trainable=True, seed=2)
    h, pei, pw, pngi = layer([_dev(x), _dev(ei), None, _dev(ngi)])
    assert h.shape == (3 + 1 + 3, 4) and pw.shape[0] == pei.shape[1]
    np.testing.assert_array_equal(np.sort(pngi.cpu().numpy()), [0, 0, 0, 1, 2, 2, 2])
    with pytest.raises(ValueError, match="attention_units"):
        tfg.layers.ASAP(ratio=0.5, attention_units=5)([_dev(x), _dev(ei), None, _dev(ngi)])


def test_asap_at_200k_nodes():
    """Forward and backward on a 200 000-node uniform graph (average in-degree 10, ratio 0.5); the pooled adjacency is
    checked against float64 scipy over the same assignment."""
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(0)
    n, F = 200000, 16
    ei = rs.randint(0, n, (2, 10 * n)).astype(np.int32)
    ngi = np.repeat(np.arange(200), n // 200).astype(np.int32)
    x = rs.randn(n, F).astype(np.float32)
    p = _params(F, 3)
    xt = _dev(x).requires_grad_()
    px, pei, pw, pngi = _asap(xt, _dev(ei), None, _dev(ngi), p, ratio=0.5)
    (px * px).sum().backward()
    assert px.shape == (n // 2, F) and torch.isfinite(xt.grad).all()
    assert all(torch.isfinite(p[k].grad).all() for k in ref.ORDER)
    # the pooled adjacency of an assignment with ASAP's structure (the self-looped edges whose target is selected)
    keep = ei[0] != ei[1]
    ei_sl = np.concatenate([ei[:, keep], np.stack([np.arange(n), np.arange(n)])], axis=1).astype(np.int32)
    sel = np.sort(rs.choice(n, n // 2, replace=False))
    cl = -np.ones(n, np.int64)
    cl[sel] = np.arange(len(sel))
    m = cl[ei_sl[0]] >= 0
    aei = np.stack([ei_sl[1][m], cl[ei_sl[0][m]]]).astype(np.int32)
    aw = rs.uniform(0.05, 1, m.sum()).astype(np.float32)
    _, got_ei, got_w = tfg.nn.cluster_pool(None, _dev(ei_sl), None, _dev(aei), _dev(aw), len(sel), num_nodes=n)
    A = sp.csr_matrix((np.ones(ei_sl.shape[1]), (ei_sl[0], ei_sl[1])), shape=(n, n))
    S = sp.csr_matrix((aw.astype(np.float64), (aei[0], aei[1])), shape=(n, len(sel)))
    want = (S.T @ A @ S).tocoo()
    order = np.lexsort((want.col, want.row))
    np.testing.assert_array_equal(got_ei.cpu().numpy(), np.stack([want.row[order], want.col[order]]))
    wv = want.data[order]
    err = np.abs(got_w.cpu().numpy().astype(np.float64) - wv)
    assert np.all(err <= 1e-5 * np.abs(wv) + 1e-7 * np.abs(wv).max()), err.max()


# ---- training ------------------------------------------------------------------------------------------------------

def _planted(rs, n, k, p_in, p_out):
    labels = np.repeat(np.arange(k), n // k)
    prob = np.where(labels[:, None] == labels[None, :], p_in, p_out)
    r, c = np.nonzero(np.triu(rs.rand(n, n) < prob, 1))
    return np.stack([np.concatenate([r, c]), np.concatenate([c, r])]).astype(np.int32)


def test_demo_asap_architecture_classifies_community_counts():
    """demo/demo_asap.py's model, 3 x (GCN -> ASAP(ratio 0.5, drop 0.1)) with a mean || max read-out per level, tells graphs
    with 2 planted communities from graphs with 4 (one-hot degree features)."""
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(0)
    graphs = []
    for i in range(240):
        k = 2 if i % 2 == 0 else 4
        ei = _planted(rs, 40, k, 0.5, 0.02)
        deg = np.minimum(np.bincount(ei[0], minlength=40), 15)
        x = np.zeros((40, 16), np.float32)
        x[np.arange(40), deg] = 1.0
        graphs.append((ei, x, k == 4))
    from tf_geometric_b200 import _rng
    torch.manual_seed(0)
    _rng.set_seed(0)
    gcns = [tfg.layers.GCN(32, activation=tfg.nn.relu, trainable=True, seed=i) for i in range(3)]
    asaps = [tfg.layers.ASAP(ratio=0.5, drop_rate=0.1, trainable=True, seed=10 + i) for i in range(3)]
    mlp = torch.nn.Sequential(torch.nn.Linear(64, 32), torch.nn.ReLU(), torch.nn.Dropout(0.5), torch.nn.Linear(32, 2)).to(DEV)

    def forward(batch, training):
        eis, ngis, xs, base = [], [], [], 0
        for j, (ei, x, _) in enumerate(batch):
            eis.append(ei + base)
            ngis.append(np.full(40, j, np.int32))
            xs.append(x)
            base += 40
        ei, ngi, h = _dev(np.concatenate(eis, 1)), _dev(np.concatenate(ngis)), _dev(np.concatenate(xs))
        w, outs = None, []
        for gcn, asap in zip(gcns, asaps):
            h = gcn([h, ei, w], training=training)
            h, ei, w, ngi = asap([h, ei, w, ngi], training=training)
            outs.append(torch.cat([tfg.nn.mean_pool(h, ngi), tfg.nn.max_pool(h, ngi)], -1))
        mlp.train(training)
        return mlp(torch.stack(outs, 1).sum(1))

    forward(graphs[:2], False)
    params = [q for m in gcns + asaps for q in m.parameters()] + list(mlp.parameters())
    opt = torch.optim.Adam(params, lr=0.01)
    train, test = graphs[:160], graphs[160:]
    for step in range(150):
        idx = np.random.RandomState(step).choice(len(train), 32, replace=False)
        batch = [train[i] for i in idx]
        y = torch.tensor([int(b[2]) for b in batch], device=DEV)
        loss = torch.nn.functional.cross_entropy(forward(batch, True), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
    with torch.no_grad():
        logits = forward(test, False)
    acc = float((logits.argmax(1).cpu().numpy() == np.array([int(b[2]) for b in test])).mean())
    print("held-out accuracy", acc)
    assert acc >= 0.8, acc


def test_golden_fixture_from_the_reference():
    import tf_geometric_b200 as tfg
    assert ref.check_golden(tfg, DEV) == 22
