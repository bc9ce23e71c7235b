# coding=utf-8
"""ASAP: Adaptive Structure Aware Pooling (reference nn/pool/asap.py), composed of differentiable blocks whose backward
passes use no atomics.

The reference cannot be executed as written; two of its call sites are read the one way that runs (DESIGN.md §5 (9)):
  1. `gcn(x, edge_index, edge_weight, kernel, bias)` (asap.py:54) predates the SparseMatrix signature of gcn; it is the
     edge-list GCN, gcn(x, SparseMatrix(edge_index, edge_weight), kernel, bias), as layers/conv/gcn.py reads such inputs.
  2. The assignment is stacked as [cluster, node] (asap.py:107-115) while cluster_pool takes [node, cluster]; it is passed
     as [node, cluster], so S[n, i] = attention of member n for cluster i, the S^T x that cluster_h already is.
The edge score leaky_relu([q[row] || h[col]] W_s + b_s) is computed as q[row] W_s[:A] + h[col] W_s[A:] + b_s: the two
projections per node, then gathers, instead of an [E', 2A] concatenation (the same value up to rounding)."""
import torch

from ... import ops, autograd
from ...sparse import SparseMatrix
from ...utils.graph_utils import add_self_loop_edge, remove_self_loop_edge
from ..conv.gcn import gcn
from ..conv.propagation import le_conv
from .cluster_pool import cluster_pool
from .topk_pool import topk_pool


def _add_self_loops(edge_index, num_nodes, weight):
    """add_self_loop_edge, keeping the autograd history of weights that require grad (the appended ones are constants)."""
    index, weight_sl = add_self_loop_edge(edge_index, num_nodes, weight)
    if autograd.needs_grad(weight):
        weight_sl = torch.cat([weight, weight_sl[weight.shape[0]:]])
    return index, weight_sl


def asap(x, edge_index, edge_weight, node_graph_index,
         attention_gcn_kernel, attention_gcn_bias,
         attention_query_kernel, attention_query_bias,
         attention_score_kernel, attention_score_bias,
         le_conv_self_kernel, le_conv_self_bias,
         le_conv_aggr_self_kernel, le_conv_aggr_self_bias,
         le_conv_aggr_neighbor_kernel, le_conv_aggr_neighbor_bias,
         k=None, ratio=None,
         le_conv_activation=torch.sigmoid,
         drop_rate=0.0, training=None, cache=None, seed=None):
    """
    Functional API for ASAP (reference nn/pool/asap.py:19-145).

    :param x: [num_nodes, num_features]
    :param edge_index: [2, num_edges]; edge_weight: [num_edges] or None
    :param node_graph_index: [num_nodes] graph of every node (any order)
    :param k / ratio: keep the k best nodes, or ceil(ratio * n) of them, per graph (topk_pool)
    :param le_conv_activation: applied to the selected node scores before they scale the pooled features
    :param drop_rate: dropout on the attention coefficients when training
    :param cache: dict caching the normalised adjacency of the attention GCN
    :param seed: Philox key of the attention dropout (an extension; None draws a fresh one)
    :return: [pooled_x, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index]

    The attention units must equal num_features: the reference applies le_conv's [units, 1] kernels to the cluster
    features, which are num_features wide.  The assignment weights are detached, as in the reference, so the pooled edge
    weights need no gradient for any parameter; a caller whose edge_weight requires grad gets a RuntimeError if the
    backward reaches the pooled edge weights (cluster_pool).
    """
    ei = ops.as_device(edge_index, torch.int32).reshape(2, -1)
    dev = ei.device
    x = ops.as_device(x, torch.float32, device=dev)
    num_nodes, num_features = x.shape
    units = attention_gcn_kernel.shape[1]
    if units != num_features:
        raise ValueError("asap: attention_units ({}) must equal the number of features ({}): le_conv's [units, 1] kernels "
                         "are applied to the cluster features".format(units, num_features))
    weight = None if edge_weight is None else ops.as_device(edge_weight, torch.float32, device=dev).reshape(-1)
    ngi = ops.as_device(node_graph_index, torch.int32, device=dev).reshape(-1).contiguous()

    def f32(t):
        return None if t is None else ops.as_device(t, torch.float32, device=dev)

    ei, weight = remove_self_loop_edge(ei, weight)
    ei_sl, weight_sl = _add_self_loops(ei, num_nodes, weight)
    row_sl, col_sl = ei_sl[0].contiguous(), ei_sl[1].contiguous()

    attention_h = gcn(x, SparseMatrix(ei, weight, [num_nodes, num_nodes]), f32(attention_gcn_kernel),
                      f32(attention_gcn_bias), cache=cache)                                      # adapter 1

    # max aggregate over the self-looped edges (K11: tie counts forward, transposed-CSR backward, no per-edge messages)
    query = autograd.max_aggregate(attention_h, ei_sl, num_nodes)
    query = autograd.dense(query, f32(attention_query_kernel), f32(attention_query_bias))

    w_s = f32(attention_score_kernel)
    score = autograd.TakeRows.apply(autograd.dense(query, w_s[:units]), row_sl) \
        + autograd.TakeRows.apply(autograd.dense(attention_h, w_s[units:]), col_sl)
    if attention_score_bias is not None:
        score = score + f32(attention_score_bias)
    score = torch.nn.functional.leaky_relu(score, 0.2).reshape(-1)

    normed = autograd.SegmentSoftmax.apply(score, row_sl, num_nodes) if autograd.needs_grad(score) \
        else autograd.segment_softmax_forward(score, row_sl, num_nodes)
    if training and drop_rate > 0:
        normed = autograd.dropout(normed, drop_rate, True, seed=seed)

    cluster_h = autograd.NeighborAggregate.apply(x, ei_sl, normed, "sum", num_nodes)

    node_score = le_conv(cluster_h, ei, weight, f32(le_conv_self_kernel), f32(le_conv_self_bias),
                         f32(le_conv_aggr_self_kernel), f32(le_conv_aggr_self_bias), f32(le_conv_aggr_neighbor_kernel),
                         f32(le_conv_aggr_neighbor_bias), activation=None)

    topk = topk_pool(ngi, node_score, k=k, ratio=ratio)
    topk_score = autograd.TakeRows.apply(node_score, topk)
    if le_conv_activation is not None:
        topk_score = le_conv_activation(topk_score)
    pooled_x = autograd.TakeRows.apply(cluster_h, topk) * topk_score

    num_clusters = topk.numel()
    reverse = torch.full((num_nodes,), -1, dtype=torch.int32, device=dev)
    reverse[topk.long()] = torch.arange(num_clusters, dtype=torch.int32, device=dev)
    assign_cluster = ops.gather_i32(reverse, row_sl)
    selected = ops.select_flagged((assign_cluster >= 0).to(torch.int32))
    assign_edge_index = torch.stack([ops.gather_i32(col_sl, selected),
                                     ops.gather_i32(assign_cluster, selected)])                 # adapter 2: [node, cluster]
    assign_edge_weight = ops.permute(normed.detach().contiguous(), selected)

    _, pooled_edge_index, pooled_edge_weight = cluster_pool(None, ei_sl, weight_sl, assign_edge_index, assign_edge_weight,
                                                            num_clusters, num_nodes=num_nodes)
    pooled_edge_index, pooled_edge_weight = remove_self_loop_edge(pooled_edge_index, pooled_edge_weight)
    pooled_edge_index, pooled_edge_weight = _add_self_loops(pooled_edge_index, num_clusters, pooled_edge_weight)
    pooled_node_graph_index = ops.gather_i32(ngi, topk)
    return pooled_x, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index
