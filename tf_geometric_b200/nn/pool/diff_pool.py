# coding=utf-8
"""DiffPool, "Hierarchical graph representation learning with differentiable pooling" (reference nn/pool/diff_pool.py),
with the pooling step on K8 instead of the reference's dense N x N adjacency (nn/pool/cluster_pool.py)."""
import torch

from ... import ops
from . import cluster_pool as _cp


def _ones_like_edges(edge_index):
    ei = ops.as_device(edge_index, torch.int32)
    return torch.ones((ei.shape[1],), dtype=torch.float32, device=ei.device)


def diff_pool_coarsen(x, edge_index, edge_weight, node_graph_index, dense_assign,
                      num_nodes=None, num_clusters=None, num_graphs=None):
    """
    Coarsening method for DiffPool (reference diff_pool.py:8-53): every graph of the batch is pooled into the same
    number of clusters.

    :param x: Tensor [num_nodes, num_features] or None
    :param edge_index: [2, num_edges]; no edge may join two graphs (ValueError)
    :param edge_weight: [num_edges] or None (ones)
    :param node_graph_index: [num_nodes] graph of every node, in any order
    :param dense_assign: [num_nodes, num_clusters] cluster assignment of the nodes
    :return: [pooled_x, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index]
    """
    if num_nodes is None:
        num_nodes = dense_assign.shape[0]
    if num_clusters is None:
        num_clusters = dense_assign.shape[1]
    if edge_weight is None:
        edge_weight = _ones_like_edges(edge_index)
    ei, layout = _cp.cluster_layout(edge_index, node_graph_index, num_nodes, num_clusters, num_graphs)
    w = ops.as_device(edge_weight, torch.float32, device=ei.device)
    pooled_x, _, pooled_ei, pooled_w, pooled_ngi = _cp.coarsen(x, w, dense_assign, layout)
    return pooled_x, pooled_ei, pooled_w, pooled_ngi


def _call_gnn(gnn, inputs, training, cache):
    """The reference calls the sub-GNNs with `cache` only when one is given (diff_pool.py:88-93)."""
    if cache is None:
        return gnn(inputs, training=training)
    return gnn(inputs, training=training, cache=cache)


def diff_pool(x, edge_index, edge_weight, node_graph_index,
              feature_gnn, assign_gnn,
              num_clusters, bias=None, activation=None, cache=None, training=None):
    """
    Functional API for DiffPool (reference diff_pool.py:56-108).

    :param feature_gnn: [x, edge_index, edge_weight] => pooled features' source h
    :param assign_gnn: [x, edge_index, edge_weight] => assignment logits [num_nodes, num_clusters]
    :param num_clusters: clusters per graph
    :param bias: [num_output_features] added to the pooled features, then `activation`
    :return: [pooled_x, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index]
    """
    if edge_weight is None:
        edge_weight = _ones_like_edges(edge_index)
    num_nodes = x.shape[0]
    assign_logits = _call_gnn(assign_gnn, [x, edge_index, edge_weight], training, cache)
    h = _call_gnn(feature_gnn, [x, edge_index, edge_weight], training, cache)
    assign_probs = torch.softmax(assign_logits, dim=-1)
    pooled_h, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index = diff_pool_coarsen(
        h, edge_index, edge_weight, node_graph_index, assign_probs, num_nodes=num_nodes, num_clusters=num_clusters)
    if bias is not None:
        pooled_h = pooled_h + bias
    if activation is not None:
        pooled_h = activation(pooled_h)
    return pooled_h, pooled_edge_index, pooled_edge_weight, pooled_node_graph_index
