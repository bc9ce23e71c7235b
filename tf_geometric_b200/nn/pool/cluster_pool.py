# coding=utf-8
"""cluster_pool with a sparse assignment (reference nn/pool/cluster_pool.py:9-44), and the shared coarsening step of DiffPool
and MinCutPool, restricted to what both use: a dense [N, C] assignment in which every node belongs to the C clusters of
its own graph.

cluster_pool computes the reference's S^T A S without the dense N x N adjacency: T = S^T A, then P = T S, two launches of
K10 (csrc/spgemm.cu, the reference's left-to-right association).  Its pooled edges are P's entries != 0 in row-major
order, which is the order of the reference's tf.where over the dense [K, K] matrix.

The reference builds the [G*C, N] assignment as a sparse matrix, densifies the N x N adjacency and multiplies
S^T A S over [G*C]^2.  Here the pooled blocks are computed per graph by K8 (csrc/cluster_pool.cu): P = S_g^T X_g and
Q = S_g^T A_g S_g in block layout [G*C, *].  Every entry of the reference's [G*C]^2 matrix outside the diagonal blocks is
zero when no edge joins two graphs, so its non-zero entries in row-major order are exactly the non-zero entries of Q in
row-major order, with column g*C + c'.  An edge that joins two graphs raises ValueError (the reference would emit
off-block pooled edges for it; BatchGraph never produces one)."""
import weakref

import torch

from ... import ops, autograd, _structure
from ...sparse import SparseMatrix


def _weights(weight, n, dev):
    if weight is None:
        return torch.ones((n,), dtype=torch.float32, device=dev)
    return ops.as_device(weight, torch.float32, device=dev).reshape(-1)


def cluster_pool(x, edge_index, edge_weight, assign_edge_index, assign_edge_weight, num_clusters, num_nodes=None):
    """
    Coarsen a graph by a sparse assignment of nodes to clusters (reference nn/pool/cluster_pool.py:9-44).

    :param x: [num_nodes, num_features] or None
    :param edge_index: [2, num_edges]; edge_weight: [num_edges] or None (ones)
    :param assign_edge_index: [2, num_assignments] as [node, cluster]: entry e puts node assign_edge_index[0, e] in cluster
        assign_edge_index[1, e] with weight assign_edge_weight[e] (None: ones).  Duplicate entries, in the assignment or in
        the edges, add up.
    :param num_clusters: K
    :param num_nodes: required when x is None
    :return: [pooled_x (S^T x, or None), pooled_edge_index int32 [2, P], pooled_edge_weight [P]]: the entries != 0 of
        S^T A S (NaN kept) in row-major order.  pooled_x is differentiable in x and assign_edge_weight; the pooled edge
        weights have no gradient with respect to edge_weight or assign_edge_weight, and a backward that reaches them while
        either requires grad raises RuntimeError.
    """
    if num_nodes is None:
        if x is None:
            raise Exception("Please provide num_nodes if x is None")
        num_nodes = x.shape[0]
    N, K = int(num_nodes), int(num_clusters)
    ei = ops.as_device(edge_index, torch.int32).reshape(2, -1)
    dev = ei.device
    aei = ops.as_device(assign_edge_index, torch.int32, device=dev).reshape(2, -1)
    w = _weights(edge_weight, ei.shape[1], dev)
    aw = _weights(assign_edge_weight, aei.shape[1], dev)
    node, cluster = aei[0].contiguous(), aei[1].contiguous()
    a_csr, _ = _structure.csr_for_edge_index(ei, N)
    s_csr = ops.csr_build(node, cluster, N, K)                 # S by node, stable: the assignment order within a node
    st_csr = ops.csr_build(cluster, node, K, N)                # S^T by cluster
    awd = aw.detach()
    t = ops.spgemm(st_csr.rowptr, st_csr.col, ops.permute(awd, st_csr.perm), a_csr.rowptr, a_csr.col,
                   ops.permute(w.detach(), a_csr.perm), N)
    rowptr, col, val = ops.spgemm(*t, s_csr.rowptr, s_csr.col, ops.permute(awd, s_csr.perm), K)
    keep = ops.select_flagged((val != 0).to(torch.int32))      # != 0 keeps NaN, like convert_dense_adj_to_edge
    rows = torch.repeat_interleave(torch.arange(K, dtype=torch.int32, device=dev), rowptr[1:] - rowptr[:-1])
    pooled_edge_index = torch.stack([ops.gather_i32(rows, keep), ops.gather_i32(col, keep)])
    pooled_edge_weight = ops.permute(val, keep)
    if autograd.needs_grad(w, aw):
        pooled_edge_weight = autograd.RefusedPooledWeights.apply(pooled_edge_weight, w, aw)
    pooled_x = None
    if x is not None:
        st = SparseMatrix(torch.stack([cluster, node]), aw, [K, N], _csr=st_csr)
        pooled_x = st @ ops.as_device(x, torch.float32, device=dev)
    return pooled_x, pooled_edge_index, pooled_edge_weight


class ClusterLayout(object):
    """Everything K8 needs about a batch: the edge CSR, the graph pointer / node list of node_graph_index and the
    node -> graph ids (int32)."""

    __slots__ = ("edge_index", "csr", "gptr", "gnodes", "node_graph", "num_nodes", "num_graphs", "num_clusters")

    def __init__(self, edge_index, node_graph_index, num_nodes, num_clusters, num_graphs):
        self.edge_index = edge_index
        self.node_graph = node_graph_index
        self.num_nodes, self.num_clusters, self.num_graphs = int(num_nodes), int(num_clusters), int(num_graphs)
        if node_graph_index.numel() != self.num_nodes:
            raise ValueError("node_graph_index has {} entries for {} nodes".format(node_graph_index.numel(), num_nodes))
        # a stable CSR by graph id: rowptr delimits every graph's nodes, perm lists them in input order (any order is
        # accepted, like the reference)
        graphs = _structure.csr_for_segment_ids(node_graph_index, self.num_graphs)
        self.gptr, self.gnodes = graphs.rowptr, graphs.perm
        self.csr, _ = _structure.csr_for_edge_index(edge_index, self.num_nodes)
        _check_edges_within_graphs(edge_index, node_graph_index)


def _check_edges_within_graphs(edge_index, node_graph_index):
    """ValueError when an edge joins two graphs.  Memoised per (edge list, node_graph_index) tensor pair, so a warm call
    with the same int32 device tensors skips the two gathers and the synchronising any()."""
    tag = ("within_graphs",)
    hit = _structure._lookup(edge_index, tag)
    if hit is not None and hit() is node_graph_index:
        return
    if edge_index.shape[1]:
        g_row = ops.gather_i32(node_graph_index, edge_index[0].contiguous())
        g_col = ops.gather_i32(node_graph_index, edge_index[1].contiguous())
        if bool((g_row != g_col).any()):
            raise ValueError("an edge joins two graphs of the batch: DiffPool / MinCutPool pool every graph on its own")
    _structure._store(edge_index, tag, weakref.ref(node_graph_index))


def cluster_layout(edge_index, node_graph_index, num_nodes, num_clusters, num_graphs=None):
    """(edge_index int32, ClusterLayout); num_graphs defaults to max(node_graph_index) + 1 like the reference."""
    ei = ops.as_device(edge_index, torch.int32)
    ngi = ops.as_device(node_graph_index, torch.int32, device=ei.device)
    if ngi.dim() != 1:                   # a 1-D int32 device tensor is used as is: the per-tensor memos then hit
        ngi = ngi.reshape(-1)
    if ngi.numel():
        lo, hi = (int(v) for v in torch.aminmax(ngi))          # one synchronisation for both bounds
        if lo < 0:
            raise ValueError("node_graph_index holds a negative graph id")
        if num_graphs is None:
            num_graphs = hi + 1
    elif num_graphs is None:
        num_graphs = 0
    return ei, ClusterLayout(ei, ngi, num_nodes, num_clusters, num_graphs)


def coarsen(x, edge_weight, dense_assign, layout):
    """(pooled_x, Q, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index) of one coarsening step."""
    S = dense_assign if dense_assign.dtype == torch.float32 else dense_assign.to(torch.float32)
    if tuple(S.shape) != (layout.num_nodes, layout.num_clusters):
        raise ValueError("dense_assign is {}, expected [{}, {}]".format(tuple(S.shape), layout.num_nodes,
                                                                       layout.num_clusters))
    if x is not None and not torch.is_tensor(x):
        x = ops.as_device(x, torch.float32, device=S.device)
    pooled_x, Q = autograd.ClusterPool.apply(x, S, edge_weight, layout)
    pooled_edge_index, pooled_edge_weight = pooled_edges(Q, layout.num_clusters)
    dev = Q.device
    pooled_node_graph_index = torch.arange(layout.num_graphs, dtype=torch.int32, device=dev).repeat_interleave(
        layout.num_clusters)
    return (None if x is None else pooled_x), Q, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index


def pooled_edges(Q, num_clusters):
    """The non-zero entries of the block-diagonal [G*C]^2 matrix stored as Q [G*C, C], in the row-major order of the
    reference's convert_dense_adj_to_edge: entry (g*C + c, c') is edge (g*C + c, g*C + c'); the weights are a
    differentiable gather of Q."""
    C = int(num_clusters)
    flat = Q.reshape(-1)
    k = ops.select_flagged((flat != 0).to(torch.int32))          # != 0 keeps NaN, like tf.not_equal
    k64 = k.to(torch.int64)
    row = k64 // C
    col = (row // C) * C + k64 % C
    return torch.stack([row, col]).to(torch.int32), autograd.TakeRows.apply(flat, k)
