# coding=utf-8
"""Float64 torch restatement of the reference's nn/pool/asap.py and nn/pool/cluster_pool.py, op for op, with the two
adapters of DESIGN.md §5 (9): the attention GCN is the edge-list GCN, and the assignment goes to cluster_pool as
[node, cluster].  Dense adjacencies are fine at test sizes.  Differentiable in every float input."""
import numpy as np
import torch

F64 = torch.float64


def t64(a, grad=False):
    return torch.tensor(np.asarray(a), dtype=F64, requires_grad=grad)


def dense_adj(ei, w, n, m=None):
    """A[row_e, col_e] += w_e (row = aggregation target)."""
    a = torch.zeros((n, n if m is None else m), dtype=F64)
    return a.index_put((torch.as_tensor(ei[0]).long(), torch.as_tensor(ei[1]).long()), w, accumulate=True)


def gcn(x, ei, w, kernel, bias):
    """nn/conv/gcn.py defaults: D^-1/2 (A + I) D^-1/2 x W + b with row degrees."""
    n = x.shape[0]
    a = dense_adj(ei, w, n) + torch.eye(n, dtype=F64)
    deg = a.sum(1)
    dis = torch.where(deg > 0, deg.clamp(min=1e-300) ** -0.5, torch.zeros_like(deg))
    return (dis[:, None] * a * dis[None, :]) @ (x @ kernel) + bias


def segment_softmax(s, seg, n):
    m = torch.full((n,), -np.inf, dtype=F64).scatter_reduce(0, seg, s, "amax", include_self=True)
    e = torch.exp(s - m[seg])
    return e / (torch.zeros(n, dtype=F64).index_add(0, seg, e) + 1e-8)[seg]


def topk(ngi, score, k=None, ratio=None):
    """topk_pool: per graph in ascending graph order, the best scores first (ties by index)."""
    ngi, score = np.asarray(ngi), np.asarray(score, np.float64).reshape(-1)
    out = []
    for g in range(int(ngi.max()) + 1 if len(ngi) else 0):
        nodes = np.nonzero(ngi == g)[0]
        nodes = nodes[np.argsort(-score[nodes], kind="stable")]
        keep = min(k, len(nodes)) if k is not None else int(np.ceil(np.float32(len(nodes)) * np.float32(ratio)))
        out.append(nodes[:keep])
    return np.concatenate(out).astype(np.int64) if out else np.zeros(0, np.int64)


def cluster_pool(x, ei, w, aei, aw, num_clusters, num_nodes):
    """cluster_pool.py:9-44 with a dense [N, K] assignment from [node, cluster] pairs: (S^T x, edges, weights)."""
    s = dense_adj(aei, aw, num_nodes, num_clusters)
    p = s.t() @ dense_adj(ei, w, num_nodes) @ s
    nz = torch.nonzero(p != 0)
    return (None if x is None else s.t() @ x), nz.t().numpy().astype(np.int32), p[nz[:, 0], nz[:, 1]]


def asap(x, ei, w, ngi, p, k=None, ratio=None, act=torch.sigmoid, drop_mask=None, topk_index=None):
    """nn/pool/asap.py:46-145.  p: dict of the layer's weights (float64 tensors; le_conv_aggr_neighbor_bias absent).
    drop_mask: the kept-and-scaled dropout factor of every self-looped edge, or None.  topk_index: the selection to use
    (None: computed here)."""
    ei = np.asarray(ei)
    n = x.shape[0]
    keep = ei[0] != ei[1]
    ei = ei[:, keep]
    if w is not None:
        w = w[torch.as_tensor(keep)]
    diag = np.arange(n)
    ei_sl = np.concatenate([ei, np.stack([diag, diag])], axis=1)
    ones = torch.ones(ei.shape[1], dtype=F64)
    w_sl = None if w is None else torch.cat([w, torch.ones(n, dtype=F64)])
    row, col = torch.as_tensor(ei_sl[0]).long(), torch.as_tensor(ei_sl[1]).long()
    units = p["attention_gcn_kernel"].shape[1]

    h = gcn(x, ei, ones if w is None else w, p["attention_gcn_kernel"], p["attention_gcn_bias"])
    q = torch.full((n, units), -np.inf, dtype=F64).scatter_reduce(0, row[:, None].expand(-1, units), h[col], "amax")
    q = q @ p["attention_query_kernel"] + p["attention_query_bias"]
    s = torch.cat([q[row], h[col]], -1) @ p["attention_score_kernel"] + p["attention_score_bias"]
    s = torch.nn.functional.leaky_relu(s, 0.2).reshape(-1)
    normed = segment_softmax(s, row, n)
    if drop_mask is not None:
        normed = normed * drop_mask
    cluster_h = torch.zeros_like(x).index_add(0, row, normed[:, None] * x[col])

    a = dense_adj(ei, ones if w is None else w, n)
    diff = cluster_h @ p["le_conv_aggr_self_kernel"] + p.get("le_conv_aggr_self_bias", 0.0) \
        - cluster_h @ p["le_conv_aggr_neighbor_kernel"]
    node_score = cluster_h @ p["le_conv_self_kernel"] + p.get("le_conv_self_bias", 0.0) + a @ diff

    sel = topk(ngi, node_score.detach().numpy(), k, ratio) if topk_index is None else np.asarray(topk_index, np.int64)
    sel_t = torch.as_tensor(sel)
    score = node_score[sel_t]
    if act is not None:
        score = act(score)
    pooled_x = cluster_h[sel_t] * score

    K = len(sel)
    reverse = -np.ones(n, np.int64)
    reverse[sel] = np.arange(K)
    cl = reverse[ei_sl[0]]
    m = cl >= 0
    aei = np.stack([ei_sl[1][m], cl[m]])                           # adapter 2: [node, cluster]
    _, pei, pw = cluster_pool(None, ei_sl, torch.ones(ei_sl.shape[1], dtype=F64) if w_sl is None else w_sl, aei,
                              normed.detach()[torch.as_tensor(m)], K, n)
    loops = pei[0] == pei[1]
    pei, pw = pei[:, ~loops], pw[torch.as_tensor(~loops)]
    pei = np.concatenate([pei, np.stack([np.arange(K), np.arange(K)])], axis=1).astype(np.int32)
    pw = torch.cat([pw, torch.ones(K, dtype=F64)])
    return pooled_x, pei, pw, np.asarray(ngi)[sel].astype(np.int32), sel


PARAM_SHAPES = lambda F: {                                                           # noqa: E731
    "attention_gcn_kernel": (F, F), "attention_gcn_bias": (F,), "attention_query_kernel": (F, F),
    "attention_query_bias": (F,), "attention_score_kernel": (2 * F, 1), "attention_score_bias": (1,),
    "le_conv_self_kernel": (F, 1), "le_conv_self_bias": (1,), "le_conv_aggr_self_kernel": (F, 1),
    "le_conv_aggr_self_bias": (1,), "le_conv_aggr_neighbor_kernel": (F, 1)}
ORDER = list(PARAM_SHAPES(1))


def random_params(F, seed):
    rs = np.random.RandomState(seed)
    return {k: (rs.randn(*s) * (0.5 if len(s) == 2 else 0.2)).astype(np.float32) for k, s in PARAM_SHAPES(F).items()}


def batch(sizes, seed, F=6, self_loops=True, shuffle=True):
    """A batch of random graphs (edges inside graphs, duplicates and, optionally, self loops), unsorted graph ids."""
    rs = np.random.RandomState(seed)
    eis, ngi, base = [], [], 0
    for g, n in enumerate(sizes):
        ngi += [g] * n
        if n > 1:
            e = rs.randint(0, n, (2, 3 * n)) + base
            if not self_loops:
                e = e[:, e[0] != e[1]]
            eis.append(np.concatenate([e, e[:, :2]], axis=1))                   # two duplicates
        base += n
    ei = np.concatenate(eis, axis=1) if eis else np.zeros((2, 0), np.int64)
    ngi = np.array(ngi)
    N = len(ngi)
    if shuffle:
        perm = rs.permutation(N)
        inv = np.empty_like(perm)
        inv[perm] = np.arange(N)
        ngi, ei = ngi[perm], inv[ei]
    x = rs.randn(N, F).astype(np.float32)
    w = rs.uniform(0.5, 1.5, ei.shape[1]).astype(np.float32)
    return x, ei.astype(np.int32), w, ngi.astype(np.int32)


def cluster_case():
    """cluster_pool inputs with duplicate entries in S and A, a node in no cluster, an empty cluster, a self loop and a
    zero-weight edge that makes an exact-zero pooled entry."""
    ei = np.array([[0, 1, 2, 2, 3, 3, 4, 5, 1], [1, 2, 3, 3, 3, 5, 0, 4, 0]], np.int32)      # (3, 5) weighs 0
    w = np.array([1.0, 0.5, 2.0, 2.0, 1.5, 0.0, 0.75, 1.25, -1.0], np.float32)
    # [node, cluster]; node 6 in no cluster, cluster 3 empty, (2, 1) twice
    aei = np.array([[0, 1, 2, 2, 3, 4, 5, 0], [0, 0, 1, 1, 1, 2, 2, 2]], np.int32)
    aw = np.array([0.5, 1.0, 0.25, 0.25, 2.0, 1.0, 0.5, 0.3], np.float32)
    x = np.random.RandomState(3).randn(7, 3).astype(np.float32)
    return x, ei, w, aei, aw, 4, 7


def check_golden(tfg, device):
    """Replay tests/golden/asap_exec.npz (the reference's own cluster_pool.py and asap.py, the latter with the two
    adapters) through the public API on `device`: indices bit-exact, floats within assert_close.  Returns the number of
    arrays compared."""
    import os
    from conftest import assert_close
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "asap_exec.npz"))

    def dev(a):
        return torch.as_tensor(np.ascontiguousarray(a), device=device)

    def compare(got, key):
        want = g[key]
        got = got.detach().cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
        if want.dtype.kind in "iu":
            np.testing.assert_array_equal(got, want, err_msg=key)
        else:
            assert_close(got, want, what=key)
        return 1

    n = 0
    for tag, weighted in (("w", True), ("none", False)):
        res = tfg.nn.cluster_pool(dev(g["cp_x"]), dev(g["cp_ei"]), dev(g["cp_w"]) if weighted else None, dev(g["cp_aei"]),
                                  dev(g["cp_aw"]) if weighted else None, 4)
        n += sum(compare(v, "cp_%s_%s" % (tag, k)) for k, v in zip(("x", "ei", "w"), res))
    params = [dev(g["asap_p_" + k]) for k in ORDER]
    for tag, weighted, kw in (("r50_w", True, {"ratio": 0.5}), ("r50_none", False, {"ratio": 0.5}),
                              ("k2_w", True, {"k": 2}), ("k3_none", False, {"k": 3})):
        res = tfg.nn.asap(dev(g["asap_x"]), dev(g["asap_ei"]), dev(g["asap_w"]) if weighted else None, dev(g["asap_gi"]),
                          *params, None, training=False, **kw)
        n += sum(compare(v, "asap_%s_%s" % (tag, k)) for k, v in zip(("x", "ei", "w", "gi"), res))
    return n
