# coding=utf-8
"""DiffPool / MinCutPool on the H100: K8a / K8b against float64, their bit-identity guarantees, the pooling API's
gradients against float64 torch autograd over dense per-graph blocks, and end-to-end training."""
import numpy as np
import pytest
import torch

import cluster_pool_ref as ref
import edge_grad_ref
from conftest import assert_close

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _dev(a, grad=False):
    t = torch.tensor(a, device=DEV)
    return t.requires_grad_(grad) if grad else t


def _graph_layout(sizes, rs, shuffle):
    ngi = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    if shuffle:
        ngi = ngi[rs.permutation(len(ngi))]
    order = np.argsort(ngi, kind="stable").astype(np.int32)
    gptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return ngi, gptr, order


def _tmm64(S, Y, gptr, order):
    out = np.zeros((len(gptr) - 1, S.shape[1], Y.shape[1]))
    for g in range(len(gptr) - 1):
        nodes = order[gptr[g]:gptr[g + 1]]
        out[g] = S[nodes].astype(np.float64).T @ Y[nodes].astype(np.float64)
    return out.reshape(-1, Y.shape[1])


@pytest.mark.parametrize("C", [1, 3, 5, 20, 64, 130, 256])
@pytest.mark.parametrize("D", [1, 3, 20, 100, 128, 256])
def test_k8a_against_float64(C, D):
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(C * 1000 + D)
    sizes = [7, 0, 33, 1, 64, 0, 5]
    shuffle = (C + D) % 2 == 1
    ngi, gptr, order = _graph_layout(sizes, rs, shuffle)
    N = len(ngi)
    S, Y = rs.rand(N, C).astype(np.float32), rs.randn(N, D).astype(np.float32)
    out = ops.graph_tmm(_dev(S), _dev(Y), _dev(gptr), len(sizes), gnodes=_dev(order) if shuffle else None)
    assert_close(out.cpu().numpy(), _tmm64(S, Y, gptr, order), what="K8a C={} D={}".format(C, D))


def test_k8a_column_slices_and_split_path():
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(1)
    sizes = [3, 2100, 0, 17]
    ngi, gptr, order = _graph_layout(sizes, rs, True)
    N = len(ngi)
    wide = rs.randn(N, 131).astype(np.float32)
    S, Y = wide[:, 2:9], wide[:, 11:120]                   # leading dimension 131, odd offsets
    out_wide = torch.zeros((len(sizes) * 7, 113), device=DEV)
    ops.graph_tmm(_dev(wide)[:, 2:9], _dev(wide)[:, 11:120], _dev(gptr), len(sizes), gnodes=_dev(order),
                  out=out_wide[:, 1:110])
    assert_close(out_wide[:, 1:110].cpu().numpy(), _tmm64(S, Y, gptr, order), what="K8a slices")


def test_k8a_one_large_graph():
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(2)
    N, C, D = 200000, 16, 128
    S, Y = rs.rand(N, C).astype(np.float32), rs.randn(N, D).astype(np.float32)
    gptr = np.array([0, N], np.int64)
    out = ops.graph_tmm(_dev(S), _dev(Y), _dev(gptr), 1)
    want = S.astype(np.float64).T @ Y.astype(np.float64)
    assert_close(out.cpu().numpy(), want, what="K8a 200000-node graph")


def test_k8a_bits_independent_of_the_batch():
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(3)
    sizes = [40, 3000, 0, 12, 5000]
    ngi, gptr, order = _graph_layout(sizes, rs, False)
    N, C, D = len(ngi), 20, 128
    S, Y = rs.rand(N, C).astype(np.float32), rs.randn(N, D).astype(np.float32)
    St, Yt = _dev(S), _dev(Y)
    a = ops.graph_tmm(St, Yt, _dev(gptr), len(sizes))
    b = ops.graph_tmm(St, Yt, _dev(gptr), len(sizes))
    assert torch.equal(a, b)
    for g in (1, 3, 4):                                     # the graph alone: G = 1, other offsets, other neighbours
        lo, hi = gptr[g], gptr[g + 1]
        alone = ops.graph_tmm(_dev(S[lo:hi]), _dev(Y[lo:hi]), _dev(np.array([0, hi - lo], np.int64)), 1)
        assert torch.equal(alone, a[g * C:(g + 1) * C]), "graph {}".format(g)


@pytest.mark.parametrize("with_nodes", [False, True])
def test_k8a_graph_past_the_node_count_is_nan(with_nodes):
    """A graph pointer that spans more positions than there are nodes gives that graph a NaN block (never reads past
    S, Y or the node list) and leaves the other graphs exact."""
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(6)
    N, C, D = 100, 4, 8
    S, Y = rs.rand(N, C).astype(np.float32), rs.randn(N, D).astype(np.float32)
    for gptr in ([0, 50, 3000], [0, 50, 600]):           # split path without workspace slots, and one chunk
        gp = np.array(gptr, np.int64)
        out = ops.graph_tmm(_dev(S), _dev(Y), _dev(gp), 2,
                            gnodes=_dev(np.arange(N, dtype=np.int32)) if with_nodes else None).cpu().numpy()
        assert_close(out[:C], S[:50].astype(np.float64).T @ Y[:50], what="graph 0")
        assert np.isnan(out[C:]).all()


@pytest.mark.parametrize("trans", [False, True])
@pytest.mark.parametrize("C,K", [(1, 1), (3, 20), (16, 128), (130, 7), (256, 33)])
def test_k8b_against_float64(trans, C, K):
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(C + K + int(trans))
    G, N = 6, 300
    ng = rs.randint(0, G, N).astype(np.int32)
    B = rs.randn(G * C, K).astype(np.float32)
    Y = rs.randn(N, K if trans else C).astype(np.float32)
    prev = rs.randn(N, C if trans else K).astype(np.float32)
    blocks = B.astype(np.float64).reshape(G, C, K)[ng]
    want = np.einsum("nk,nck->nc", Y, blocks) if trans else np.einsum("nc,nck->nk", Y, blocks)
    out = ops.graph_rmm(_dev(Y), _dev(B), _dev(ng), C, trans=trans)
    assert_close(out.cpu().numpy(), want, what="K8b")
    acc = _dev(prev)
    ops.graph_rmm(_dev(Y), _dev(B), _dev(ng), C, trans=trans, beta=1.0, out=acc)
    assert_close(acc.cpu().numpy(), want + prev, what="K8b beta")


# ---- the pooling API against float64 autograd ------------------------------------------------------------------

def _close_grad(mine, want, what):
    """assert_close, except that a gradient which is zero in exact arithmetic (C = 1: S is all ones and the losses are
    constant) only has to be zero up to fp32 rounding."""
    if np.abs(want).max() < 1e-6:
        assert np.abs(mine).max() < 1e-6, "{}: {} where 0 is exact".format(what, np.abs(mine).max())
    else:
        assert_close(mine, want, rtol=1e-3, atol_scale=1e-4, what=what)


def _case(sizes, seed, C, D, shuffle=True):
    ei, ngi, w = ref.batch(list(sizes), seed)
    rs = np.random.RandomState(seed + 100)
    N = len(ngi)
    if shuffle:
        p = rs.permutation(N)
        inv = np.empty_like(p)
        inv[p] = np.arange(N)
        ngi, ei = ngi[p], inv[ei].astype(np.int32)
    return ei, ngi, w, rs.randn(N, D).astype(np.float32), rs.randn(N, C).astype(np.float32)


def _run(tfg, kind, ei, ngi, w, x, logits, w_grad=True):
    xt, lt = _dev(x, True), _dev(logits, True)
    wt = _dev(w, w_grad)
    S = torch.softmax(lt, -1)
    eit, ngt = _dev(ei), _dev(ngi)
    if kind == "diff":
        px, pei, pw, _ = tfg.nn.diff_pool_coarsen(xt, eit, wt, ngt, S)
        extra = 0.0
    else:
        px, pei, pw, _ = tfg.nn.min_cut_pool_coarsen(xt, eit, wt, ngt, S)
        cut, orth = tfg.nn.min_cut_pool_compute_losses(eit, wt, ngt, S)
        extra = 0.7 * cut + 1.3 * orth
    rs = np.random.RandomState(11)
    gx, gw = _dev(rs.randn(*px.shape).astype(np.float32)), _dev(rs.randn(*pw.shape).astype(np.float32))
    ((px * gx).sum() + (pw * gw).sum() + extra).backward()
    return px, pei, pw, xt.grad, lt.grad, (wt.grad if w_grad else None), extra


@pytest.mark.parametrize("kind", ["diff", "min_cut"])
@pytest.mark.parametrize("C", [1, 4, 20])
def test_coarsen_gradients_against_float64(kind, C):
    import tf_geometric_b200 as tfg
    ei, ngi, w, x, logits = _case([12, 0, 30, 1, 25, 9], C + (kind == "diff"), C, 6)
    G, N = int(ngi.max()) + 1, len(ngi)
    px, pei, pw, dx, dl, dw, extra = _run(tfg, kind, ei, ngi, w, x, logits)
    x64, l64, w64 = ref.t64(x, True), ref.t64(logits, True), ref.t64(w, True)
    row, col = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    S64 = torch.softmax(l64, -1)
    wu = w64 if kind == "diff" else ref.adj_norm(row, col, w64, N)
    P, Q = ref.blocks(x64, S64, wu, row, col, ngi, G)
    want_ei, want_w = ref.pooled_edges(Q, C, drop_self_loops=kind != "diff")
    extra64 = 0.0
    if kind != "diff":
        cut, orth = ref.min_cut_losses(S64, wu, row, col, ngi, G)
        extra64 = 0.7 * cut + 1.3 * orth
        assert_close(float(extra), float(extra64), what="losses")
    np.testing.assert_array_equal(pei.cpu().numpy(), want_ei)
    assert_close(px.detach().cpu().numpy(), P.detach().numpy(), what="pooled x")
    assert_close(pw.detach().cpu().numpy(), want_w.detach().numpy(), what="pooled w")
    rs = np.random.RandomState(11)
    gx, gw = torch.tensor(rs.randn(*P.shape).astype(np.float32), dtype=torch.float64), \
        torch.tensor(rs.randn(*want_w.shape).astype(np.float32), dtype=torch.float64)
    ((P * gx).sum() + (want_w * gw).sum() + extra64).backward()
    for name, mine, want in (("x", dx, x64), ("logits", dl, l64), ("w", dw, w64)):
        _close_grad(mine.cpu().numpy(), want.grad.numpy(), "d " + name)


@pytest.mark.parametrize("kind", ["diff", "min_cut"])
def test_edge_weight_grad_changes_no_bit_and_backward_is_deterministic(kind):
    import tf_geometric_b200 as tfg
    ei, ngi, w, x, logits = _case([50, 2000, 7], 5, 8, 16)
    a = _run(tfg, kind, ei, ngi, w, x, logits, w_grad=True)
    b = _run(tfg, kind, ei, ngi, w, x, logits, w_grad=False)
    c = _run(tfg, kind, ei, ngi, w, x, logits, w_grad=True)
    for i in (0, 1, 2, 3, 4):
        assert torch.equal(a[i], b[i]) and torch.equal(a[i], c[i]), "output {}".format(i)
    assert torch.equal(a[5], c[5])


def test_two_stacked_levels_reach_level_one():
    """Level 1: MinCut with trainable logits; level 2: a GCN on level 1's pooled weights gives the assignment of a second
    MinCut, which normalises those weights with adj_norm_edge and adds its losses.  Gradients reach level 1's S and edge
    weights through K7 and the differentiable adj_norm_edge."""
    import tf_geometric_b200 as tfg
    from tf_geometric_b200.sparse import SparseMatrix
    C1, C2, D = 6, 3, 5
    ei, ngi, w, x, logits = _case([20, 31, 17], 9, C1, D, shuffle=False)
    G, N = int(ngi.max()) + 1, len(ngi)
    rs = np.random.RandomState(4)
    K = (rs.randn(D, C2) * 0.5).astype(np.float32)
    xt, lt, wt = _dev(x, True), _dev(logits, True), _dev(w, True)
    Kt = _dev(K, True)
    p1, e1, w1, g1 = tfg.nn.min_cut_pool_coarsen(xt, _dev(ei), wt, _dev(ngi), torch.softmax(lt, -1))
    n1 = G * C1
    s2 = torch.softmax(tfg.nn.gcn(p1, SparseMatrix(e1, w1, [n1, n1]), Kt, None, None), -1)
    p2, _, w2, _ = tfg.nn.min_cut_pool_coarsen(p1, e1, w1, g1, s2)
    cut, orth = tfg.nn.min_cut_pool_compute_losses(e1, w1, g1, s2)
    loss = (p2 * p2).sum() + w2.sum() + cut + orth
    loss.backward()

    x64, l64, w64, K64 = ref.t64(x, True), ref.t64(logits, True), ref.t64(w, True), ref.t64(K, True)
    row, col = torch.tensor(ei[0], dtype=torch.int64), torch.tensor(ei[1], dtype=torch.int64)
    P1, Q1 = ref.blocks(x64, torch.softmax(l64, -1), ref.adj_norm(row, col, w64, N), row, col, ngi, G)
    e1_64, w1_64 = ref.pooled_edges(Q1, C1, drop_self_loops=True)
    np.testing.assert_array_equal(e1.cpu().numpy(), e1_64)
    r1, c1 = torch.tensor(e1_64[0], dtype=torch.int64), torch.tensor(e1_64[1], dtype=torch.int64)
    nr, nc, nv = edge_grad_ref.gcn_norm(r1, c1, w1_64, [n1, n1])
    S2 = torch.softmax(edge_grad_ref.spmm(nr, nc, nv, P1 @ K64, n1), -1)
    g1_np = np.repeat(np.arange(G), C1).astype(np.int32)
    normed2 = ref.adj_norm(r1, c1, w1_64, n1)
    P2, Q2 = ref.blocks(P1, S2, normed2, r1, c1, g1_np, G)
    _, w2_64 = ref.pooled_edges(Q2, C2, drop_self_loops=True)
    cut64, orth64 = ref.min_cut_losses(S2, normed2, r1, c1, g1_np, G)
    loss64 = (P2 * P2).sum() + w2_64.sum() + cut64 + orth64
    loss64.backward()
    assert_close(float(loss), float(loss64), what="loss")
    for name, mine, want in (("x", xt, x64), ("logits", lt, l64), ("w", wt, w64), ("K", Kt, K64)):
        assert_close(mine.grad.cpu().numpy(), want.grad.numpy(), rtol=2e-3, atol_scale=2e-4, what="d " + name)


def test_golden_fixture_from_the_reference():
    """cluster_pool_exec.npz, the reference's own diff_pool / min_cut_pool / convert_dense_* executed over numpy stand-ins,
    replayed through the public API on the device: indices bit-exact, floats within rtol 1e-4, atol 1e-4 * max."""
    import tf_geometric_b200 as tfg
    assert ref.check_golden(tfg, DEV) == 44


def test_cross_graph_edges_raise():
    import tf_geometric_b200 as tfg
    ei, ngi, w, x, logits = _case([5, 6], 1, 2, 3, shuffle=False)
    bad = np.concatenate([ei, [[0], [10]]], axis=1).astype(np.int32)
    with pytest.raises(ValueError):
        tfg.nn.diff_pool_coarsen(_dev(x), _dev(bad), None, _dev(ngi), torch.softmax(_dev(logits), -1))
    with pytest.raises(Exception, match="cannot be set to True"):
        tfg.nn.min_cut_pool(_dev(x), _dev(ei), None, _dev(ngi), None, None, 2, return_loss_func=True, return_losses=True)


# ---- training ----------------------------------------------------------------------------------------------------

def _planted(rs, n, k, p_in, p_out):
    """Symmetric planted partition: k equal communities over n nodes; returns (edge_index int32, labels)."""
    labels = np.repeat(np.arange(k), n // k)
    same = labels[:, None] == labels[None, :]
    prob = np.where(same, p_in, p_out)
    upper = np.triu(rs.rand(n, n) < prob, 1)
    r, c = np.nonzero(upper)
    return np.stack([np.concatenate([r, c]), np.concatenate([c, r])]).astype(np.int32), labels


def test_demo_architectures_classify_community_counts():
    """Graphs with 2 planted communities against graphs with 4, one-hot degree features (the demos' one-hot node labels);
    both demo architectures (MeanGraphSage sub-GNNs, pooling, max_pool readout, dense head) learn to tell them apart."""
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(0)
    graphs = []
    for i in range(240):
        k = 2 if i % 2 == 0 else 4
        ei, _ = _planted(rs, 40, k, 0.5, 0.02)
        deg = np.minimum(np.bincount(ei[0], minlength=40), 15)
        x = np.zeros((40, 16), np.float32)
        x[np.arange(40), deg] = 1.0
        graphs.append((ei, x, k == 4))
    results = {}
    for kind in ("diff", "min_cut"):
        torch.manual_seed(0)
        feat = tfg.layers.MeanGraphSage(16, activation=tfg.nn.relu, trainable=True, seed=1)
        assign = tfg.layers.MeanGraphSage(4, trainable=True, seed=2)
        cls = tfg.layers.DiffPool if kind == "diff" else tfg.layers.MinCutPool
        pool = cls(feat, assign, 16, 4, activation=tfg.nn.relu, trainable=True)
        out_w = torch.nn.Parameter(torch.randn(16, 2, device=DEV) * 0.3)

        def forward(batch):
            eis, ngis, xs, base = [], [], [], 0
            for j, (ei, x, _) in enumerate(batch):
                eis.append(ei + base)
                ngis.append(np.full(40, j, np.int32))
                xs.append(x)
                base += 40
            ei, ngi, x = _dev(np.concatenate(eis, 1)), _dev(np.concatenate(ngis)), _dev(np.concatenate(xs))
            if kind == "min_cut":
                (h, _, _, pngi), (cut, orth) = pool([x, ei, None, ngi], return_losses=True)
                aux = cut + orth
            else:
                h, _, _, pngi = pool([x, ei, None, ngi])
                aux = 0.0
            return tfg.nn.max_pool(h, pngi) @ out_w, aux

        forward(graphs[:2])                                 # builds the lazily created weights
        opt = torch.optim.Adam(list(pool.parameters()) + [out_w], lr=0.01)
        train, test = graphs[:160], graphs[160:]
        for step in range(120):
            idx = np.random.RandomState(step).choice(len(train), 32, replace=False)
            batch = [train[i] for i in idx]
            logits, aux = forward(batch)
            y = torch.tensor([int(b[2]) for b in batch], device=DEV)
            loss = torch.nn.functional.cross_entropy(logits, y) + aux
            opt.zero_grad()
            loss.backward()
            opt.step()
        with torch.no_grad():
            logits, _ = forward(test)
        results[kind] = float((logits.argmax(1).cpu().numpy() == np.array([int(b[2]) for b in test])).mean())
    print("held-out accuracy", results)
    assert results["diff"] >= 0.8 and results["min_cut"] >= 0.8, results


def test_min_cut_recovers_planted_communities():
    import tf_geometric_b200 as tfg
    from scipy.optimize import linear_sum_assignment
    rs = np.random.RandomState(1)
    ei, labels = _planted(rs, 400, 4, 0.15, 0.005)
    n = len(labels)
    x = _dev(rs.randn(n, 16).astype(np.float32))
    eit, ngi = _dev(ei), _dev(np.zeros(n, np.int32))
    assign = tfg.layers.GCN(32, activation=tfg.nn.relu, trainable=True, seed=1)
    assign2 = tfg.layers.GCN(4, trainable=True, seed=2)
    feat = tfg.layers.GCN(8, trainable=True, seed=3)

    class Assign(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.a, self.b = assign, assign2

        def forward(self, inputs, training=None, cache=None):
            h = self.a(inputs, cache=cache)
            return self.b([h, inputs[1], inputs[2]], cache=cache)

    am = Assign()
    pool = tfg.layers.MinCutPool(feat, am, 8, 4, trainable=True)
    pool([x, eit, None, ngi])
    opt = torch.optim.Adam(list(pool.parameters()), lr=0.01)
    for step in range(300):
        _, (cut, orth) = pool([x, eit, None, ngi], return_losses=True)
        opt.zero_grad()
        (cut + orth).backward()
        opt.step()
    with torch.no_grad():
        from tf_geometric_b200.utils import adj_norm_edge
        _, nw = adj_norm_edge(eit, n, torch.ones(ei.shape[1], device=DEV))
        pred = am([x, eit, nw]).argmax(1).cpu().numpy()
    conf = np.zeros((4, 4))
    for p, t in zip(pred, labels):
        conf[p, t] += 1
    r, c = linear_sum_assignment(-conf)
    acc = conf[r, c].sum() / n
    print("planted-partition best-matching accuracy", acc)
    assert acc >= 0.8, acc
