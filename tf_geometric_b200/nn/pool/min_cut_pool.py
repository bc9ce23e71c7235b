# coding=utf-8
"""MinCutPool, "Spectral Clustering with Graph Neural Networks for Graph Pooling" (reference nn/pool/min_cut_pool.py),
with the pooling step and the losses' S^T A S / S^T S on K8 instead of dense N x N and [G*C]^2 matrices."""
import math

import torch

from ... import ops, autograd
from ...utils.graph_utils import adj_norm_edge, remove_self_loop_edge
from . import cluster_pool as _cp
from .diff_pool import _call_gnn, _ones_like_edges


def _losses(Q, dense_assign, normed_edge_weight, layout):
    """(cut_loss, orth_loss) of min_cut_pool.py:19-93 from the pooled Q = S^T A S of the same normalised weights:
    trace(S^T A S) is the trace of every diagonal block of Q, trace(S^T D S) a per-graph sum of deg_n * |S[n]|^2, and
    S^T S is K8a.  Everything is differentiable."""
    G, C, N = layout.num_graphs, layout.num_clusters, layout.num_nodes
    S = dense_assign
    intra = Q.reshape(G, C, C).diagonal(dim1=1, dim2=2).sum(-1)
    row = layout.edge_index[0].contiguous()
    degree = autograd.SegmentReduce.apply(normed_edge_weight.reshape(-1, 1), row, N, "sum")
    per_node = (S * S).sum(-1, keepdim=True) * degree
    all_edges = autograd.SegmentReduce.apply(per_node, layout.node_graph, G, "sum").reshape(-1)
    cut_loss = torch.mean(-intra / (all_edges + 1e-8))

    STS = autograd.AssignGram.apply(S, layout).reshape(G, C, C)
    norm = torch.linalg.norm(STS, dim=(-2, -1), keepdim=True)
    eye = torch.eye(C, dtype=torch.float32, device=S.device) / math.sqrt(C)
    deviation = STS / (norm + 1e-8) - eye
    orth_loss = torch.mean(torch.linalg.norm(deviation, dim=(-2, -1)))
    return cut_loss, orth_loss


def _assign_probs(dense_assign):
    return dense_assign if dense_assign.dtype == torch.float32 else dense_assign.to(torch.float32)


def min_cut_pool_compute_losses(edge_index, edge_weight, node_graph_index, dense_assign, normed_edge_weight=None,
                                cache=None):
    """(cut_loss, orth_loss) of reference min_cut_pool.py:19-93, averaged over the graphs of the batch."""
    S = _assign_probs(dense_assign)
    num_nodes, num_clusters = S.shape
    if normed_edge_weight is None:
        _, normed_edge_weight = adj_norm_edge(edge_index, num_nodes, edge_weight, add_self_loop=False, cache=cache)
    ei, layout = _cp.cluster_layout(edge_index, node_graph_index, num_nodes, num_clusters)
    normed = ops.as_device(normed_edge_weight, torch.float32, device=ei.device)
    _, Q = autograd.ClusterPool.apply(None, S, normed, layout)
    return _losses(Q, S, normed, layout)


def _coarsen(x, edge_index, edge_weight, node_graph_index, dense_assign, num_nodes, num_clusters, num_graphs,
             normed_edge_weight, cache):
    S = _assign_probs(dense_assign)
    if num_nodes is None:
        num_nodes = S.shape[0]
    if num_clusters is None:
        num_clusters = S.shape[1]
    if edge_weight is None:
        edge_weight = _ones_like_edges(edge_index)
    if normed_edge_weight is None:
        _, normed_edge_weight = adj_norm_edge(edge_index, num_nodes, edge_weight, cache=cache)
    ei, layout = _cp.cluster_layout(edge_index, node_graph_index, num_nodes, num_clusters, num_graphs)
    normed = ops.as_device(normed_edge_weight, torch.float32, device=ei.device)
    pooled_x, Q, pooled_ei, pooled_w, pooled_ngi = _cp.coarsen(x, normed, S, layout)
    # the reference removes the pooled self loops and leaves the pooled weights unnormalised (min_cut_pool.py:136-138)
    pooled_ei, pooled_w = remove_self_loop_edge(pooled_ei, pooled_w)
    return (pooled_x, pooled_ei, pooled_w, pooled_ngi), (Q, S, normed, layout)


def min_cut_pool_coarsen(x, edge_index, edge_weight, node_graph_index, dense_assign,
                         num_nodes=None, num_clusters=None, num_graphs=None, normed_edge_weight=None, cache=None):
    """
    Coarsening method for MinCutPool (reference min_cut_pool.py:96-141): pools with the normalised edge weights
    (adj_norm_edge without self loops), then removes the pooled self loops.

    :return: [pooled_x, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index]
    """
    outputs, _ = _coarsen(x, edge_index, edge_weight, node_graph_index, dense_assign, num_nodes, num_clusters, num_graphs,
                          normed_edge_weight, cache)
    return outputs


def min_cut_pool(x, edge_index, edge_weight, node_graph_index,
                 feature_gnn, assign_gnn,
                 num_clusters, bias=None, activation=None,
                 gnn_use_normed_edge=True,
                 return_loss_func=False, return_losses=False,
                 cache=None, training=None):
    """
    Functional API for MinCutPool (reference min_cut_pool.py:144-224).

    :param gnn_use_normed_edge: feed the sub-GNNs the normalised edge weights instead of edge_weight
    :param return_loss_func: return (outputs, loss_func), loss_func() -> (cut_loss, orth_loss)
    :param return_losses: return (outputs, (cut_loss, orth_loss)); exclusive with return_loss_func
    :return: [pooled_x, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index] (and the losses as asked)
    """
    if return_loss_func and return_losses:
        raise Exception("return_loss_func and return_losses cannot be set to True at the same time")
    if edge_weight is None:
        edge_weight = _ones_like_edges(edge_index)
    num_nodes = x.shape[0]
    _, normed_edge_weight = adj_norm_edge(edge_index, num_nodes, edge_weight, add_self_loop=False, cache=cache)
    gnn_edge_weight = normed_edge_weight if gnn_use_normed_edge else edge_weight
    assign_logits = _call_gnn(assign_gnn, [x, edge_index, gnn_edge_weight], training, cache)
    h = _call_gnn(feature_gnn, [x, edge_index, gnn_edge_weight], training, cache)
    assign_probs = torch.softmax(assign_logits, dim=-1)
    (pooled_h, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index), state = _coarsen(
        h, edge_index, edge_weight, node_graph_index, assign_probs, num_nodes, num_clusters, None, normed_edge_weight,
        cache)
    if bias is not None:
        pooled_h = pooled_h + bias
    if activation is not None:
        pooled_h = activation(pooled_h)
    outputs = pooled_h, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index
    if not (return_loss_func or return_losses):
        return outputs

    def loss_func():
        return _losses(*state)

    if return_loss_func:
        return outputs, loss_func
    return outputs, loss_func()
