# coding=utf-8
"""Float64 torch restatement of DiffPool / MinCutPool coarsening and the MinCut losses (TEST INFRASTRUCTURE), written
over padded per-graph dense blocks (bmm), differentiable in x, the assignment and the edge weights.  It restates the
reference's nn/pool/{cluster_pool,diff_pool,min_cut_pool}.py and utils/graph_utils.py adj_norm_edge /
convert_dense_adj_to_edge, and stands in for tf.GradientTape."""
import math

import numpy as np
import torch


def t64(a, grad=False):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=grad)


def _padded(ngi, G):
    ngi = torch.as_tensor(np.asarray(ngi), dtype=torch.int64)
    counts = torch.bincount(ngi, minlength=G)
    rank = torch.zeros_like(ngi)
    seen = torch.zeros(G, dtype=torch.int64)
    for i, g in enumerate(ngi.tolist()):                # position of every node within its graph, in input order
        rank[i] = seen[g]
        seen[g] += 1
    return ngi, rank, max(int(counts.max()) if G else 0, 1)


def blocks(x, S, w, row, col, ngi, G):
    """(P [G*C, D], Q [G*C, C]) = per graph S_g^T X_g and S_g^T A_g S_g, A[row, col] += w."""
    N, C = S.shape
    g, rank, m = _padded(ngi, G)
    Sp = torch.zeros((G, m, C), dtype=S.dtype).index_put((g, rank), S)
    A = torch.zeros((G, m, m), dtype=S.dtype).index_put((g[row], rank[row], rank[col]), w, accumulate=True)
    Q = torch.bmm(Sp.transpose(1, 2), torch.bmm(A, Sp)).reshape(G * C, C)
    P = None
    if x is not None:
        Xp = torch.zeros((G, m, x.shape[1]), dtype=x.dtype).index_put((g, rank), x)
        P = torch.bmm(Sp.transpose(1, 2), Xp).reshape(G * C, x.shape[1])
    return P, Q


def adj_norm(row, col, w, n):
    """utils/graph_utils.py:914-943 without self loops: row degrees on both sides, inf -> 0."""
    deg = torch.zeros(n, dtype=w.dtype).index_add(0, row, w)
    ok = deg > 0
    a = torch.where(ok, torch.where(ok, deg, torch.ones_like(deg)) ** -0.5, torch.zeros_like(deg))
    return a[row] * w * a[col]


def pooled_edges(Q, C, drop_self_loops=False):
    """convert_dense_adj_to_edge over the block-diagonal [G*C]^2 matrix (row-major, != 0), optionally without loops."""
    GC = Q.shape[0]
    big = torch.zeros((GC, GC), dtype=Q.dtype)
    for g in range(GC // C):
        big[g * C:(g + 1) * C, g * C:(g + 1) * C] = Q[g * C:(g + 1) * C]
    mask = big.detach() != 0
    row, col = torch.nonzero(mask, as_tuple=True)
    weight = big[row, col]
    if drop_self_loops:
        keep = row != col
        row, col, weight = row[keep], col[keep], weight[keep]
    return torch.stack([row, col]).numpy().astype(np.int32), weight


def min_cut_losses(S, normed, row, col, ngi, G):
    """(cut_loss, orth_loss) of min_cut_pool.py:19-93."""
    N, C = S.shape
    _, Q = blocks(None, S, normed, row, col, ngi, G)
    intra = Q.reshape(G, C, C).diagonal(dim1=1, dim2=2).sum(-1)
    deg = torch.zeros(N, dtype=S.dtype).index_add(0, row, normed)
    g = torch.as_tensor(np.asarray(ngi), dtype=torch.int64)
    all_edges = torch.zeros(G, dtype=S.dtype).index_add(0, g, deg * (S * S).sum(-1))
    cut = torch.mean(-intra / (all_edges + 1e-8))
    gi, rank, m = _padded(ngi, G)
    Sp = torch.zeros((G, m, C), dtype=S.dtype).index_put((gi, rank), S)
    STS = torch.bmm(Sp.transpose(1, 2), Sp)
    norm = torch.sqrt((STS * STS).sum((-2, -1), keepdim=True))
    dev = STS / (norm + 1e-8) - torch.eye(C, dtype=S.dtype) / math.sqrt(C)
    orth = torch.mean(torch.sqrt((dev * dev).sum((-2, -1))))
    return cut, orth


def batch(sizes, seed, edges_per_node=2.2, dup_loops=True):
    """A batch of random symmetric graphs (graph-major nodes): (edge_index int32, node_graph_index int32, weights)."""
    rs = np.random.RandomState(seed)
    rows, cols, ngi, base = [], [], [], 0
    for g, n in enumerate(sizes):
        ngi += [g] * n
        if n >= 2:
            half = max(1, int(edges_per_node * n / 2))
            u, v = rs.randint(0, n, half), rs.randint(0, n, half)
            keep = u != v
            u, v = u[keep], v[keep]
            rows += list(base + u) + list(base + v)
            cols += list(base + v) + list(base + u)
            if dup_loops:                                   # a duplicate edge and a self loop
                rows += [base + u[0], base]
                cols += [base + v[0], base]
        base += n
    ei = np.array([rows, cols], dtype=np.int32).reshape(2, -1)
    w = (rs.rand(ei.shape[1]) + 0.2).astype(np.float32)
    return ei, np.array(ngi, dtype=np.int32), w


# ---- tests/golden/cluster_pool_exec.npz: the reference's own diff_pool / min_cut_pool executed over numpy stand-ins ----

def golden_gnn(weight, mix, device):
    """The fixture's sub-GNN callable (tools/gen_golden_from_reference.py golden_gnn) on torch tensors:
    [x, edge_index, edge_weight] -> x W + sum_{e: row_e = r} w_e (x M)[col_e]."""
    W, M = torch.tensor(weight, device=device), torch.tensor(mix, device=device)

    def gnn(inputs, training=None, cache=None):
        x, ei, w = inputs
        ei = ei.long()
        m = x @ M
        return x @ W + torch.zeros_like(m).index_add(0, ei[0], w.unsqueeze(1) * m[ei[1]])
    return gnn


def golden_replay(tfg, device):
    """Replays every case of cluster_pool_exec.npz through the public API; yields (name, got numpy, want numpy, exact)."""
    import os
    f = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cluster_pool_exec.npz"))
    dev = torch.device(device)
    x, ei, w, gi = (torch.tensor(f[k], device=dev) for k in ("x", "ei", "w", "gi"))
    for c in (3, 1):
        feat = golden_gnn(f["wf_c%d" % c], f["mf_c%d" % c], dev)
        assign = golden_gnn(f["wa_c%d" % c], f["ma_c%d" % c], dev)
        bias = torch.tensor(f["bias_c%d" % c], device=dev)
        for tag, ew in (("w", w), ("none", None)):
            got = tfg.nn.diff_pool(x, ei, ew, gi, feat, assign, c, bias=bias, activation=tfg.nn.relu)
            for k, v in zip(("x", "ei", "w", "gi"), got):
                name = "diff_%s_c%d_%s" % (tag, c, k)
                yield name, v.detach().cpu().numpy(), f[name], k in ("ei", "gi")
        for tag, normed in (("normed", True), ("raw", False)):
            got, losses = tfg.nn.min_cut_pool(x, ei, w, gi, feat, assign, c, bias=bias, activation=tfg.nn.relu,
                                              gnn_use_normed_edge=normed, return_losses=True)
            for k, v in zip(("x", "ei", "w", "gi", "cut", "orth"), tuple(got) + tuple(losses)):
                name = "mincut_%s_c%d_%s" % (tag, c, k)
                yield name, v.detach().cpu().numpy(), f[name], k in ("ei", "gi")
    dense = torch.tensor(f["dense_adj"], device=dev)
    got_ei, got_w = tfg.utils.convert_dense_adj_to_edge(dense)
    yield "dense_adj_ei", got_ei.cpu().numpy(), f["dense_adj_ei"], True
    yield "dense_adj_w", got_w.cpu().numpy(), f["dense_adj_w"], True
    got_ei, got_w = tfg.utils.convert_dense_assign_to_edge(torch.tensor(f["dense_assign"], device=dev), gi)
    yield "dense_assign_ei", got_ei.cpu().numpy(), f["dense_assign_ei"], True
    yield "dense_assign_w", got_w.cpu().numpy(), f["dense_assign_w"], True


def check_golden(tfg, device):
    from conftest import assert_close
    seen = 0
    for name, got, want, exact in golden_replay(tfg, device):
        if exact:
            np.testing.assert_array_equal(got, want, err_msg=name)      # NaN == NaN for the dense converter
        else:
            assert_close(got, want, rtol=1e-4, atol_scale=1e-4, what=name)
        seen += 1
    return seen
