# coding=utf-8
"""The message-passing primitive of tf_geometric (nn/kernel/map_reduce.py) on the CUDA kernels.

`aggregate_neighbors` keeps the reference's mapper / reducer / updater protocol.  When the three callables are the
stock ones below, the whole gather -> map -> reduce -> update chain is ONE launch of tfgk_spmm_f32 (no [E, D]
temporaries); any other callable takes the generic route: rows are gathered, the user's mapper runs on them, and the
stock reducers - which are real segment reductions over arbitrary [E, D] messages - still run on the CSR kernel.
"""
import torch

from ... import ops, _structure, autograd


def identity_mapper(repeated_x, neighbor_x, edge_weight=None):
    return neighbor_x


def neighbor_count_mapper(repeated_x, neighbor_x, edge_weight=None):
    return torch.ones([neighbor_x.shape[0], 1], dtype=torch.float32, device=neighbor_x.device)


def gcn_mapper(repeated_x, neighbor_x, edge_weight=None):
    """neighbor_x * edge_weight[:, None] (reference nn/conv/gcn.py:221-222)."""
    return neighbor_x * edge_weight.unsqueeze(1)


def _segment_reduce(neighbor_msg, node_index, num_nodes, reduce):
    node_index = ops.as_device(node_index, torch.int32)
    msg = ops.as_device(neighbor_msg, torch.float32, device=node_index.device)
    squeeze = msg.dim() == 1
    if squeeze:
        msg = msg.unsqueeze(1)
    if num_nodes is None:
        num_nodes = int(node_index.max().item()) + 1
    if autograd.needs_grad(msg):      # trainable models pool / reduce through these (demo_mean_pool.py, demo_sag_pool_h.py)
        out = autograd.SegmentReduce.apply(msg.contiguous(), node_index, int(num_nodes), reduce)
        return out.squeeze(1) if squeeze else out
    csr = _structure.csr_for_segment_ids(node_index, int(num_nodes))
    # message e sits at row e of `msg`: gather through perm, no weights
    if reduce == "min":       # min(x) = -max(-x): weight -1 per message and epilogue scale -1, both exact
        minus = torch.full((csr.nnz,), -1.0, dtype=torch.float32, device=msg.device)
        out = ops.spmm(csr, minus, msg, reduce="max", alpha=-1.0, col=csr.perm)
    else:
        out = ops.spmm(csr, None, msg, reduce=reduce, col=csr.perm)
    return out.squeeze(1) if squeeze else out


def sum_reducer(neighbor_msg, node_index, num_nodes=None):
    """tf.math.unsorted_segment_sum (reference map_reduce.py:15-16)."""
    return _segment_reduce(neighbor_msg, node_index, num_nodes, "sum")


def mean_reducer(neighbor_msg, node_index, num_nodes=None):
    """tf.math.unsorted_segment_mean, empty segment -> 0 (reference map_reduce.py:27-28)."""
    return _segment_reduce(neighbor_msg, node_index, num_nodes, "mean")


def max_reducer(neighbor_msg, node_index, num_nodes=None):
    """tf.math.unsorted_segment_max, empty segment -> float32 lowest (reference map_reduce.py:38-42, TF2 branch)."""
    return _segment_reduce(neighbor_msg, node_index, num_nodes, "max")


def sum_updater(x, reduced_neighbor_msg):
    return x + reduced_neighbor_msg


def identity_updater(x, reduced_neighbor_msg):
    return reduced_neighbor_msg


_FUSED_REDUCERS = {sum_reducer: "sum", mean_reducer: "mean", max_reducer: "max"}


def aggregate_neighbors(x, edge_index, edge_weight=None, mapper=identity_mapper,
                        reducer=sum_reducer, updater=sum_updater, num_nodes=None):
    """
    :param x: [num_nodes, D] node features
    :param edge_index: [2, E]; edge_index[0] is the aggregation target, edge_index[1] the neighbour
    :param mapper: (features_of_node, features_of_neighbor_node, edge_weight) => neighbor_msg
    :param reducer: (neighbor_msg, node_index, num_nodes) => reduced_neighbor_msg
    :param updater: (features_of_node, reduced_neighbor_msg) => aggregated_node_features
    (reference map_reduce.py:45-73)
    """
    if len(edge_index) == 0:            # reference :57-58
        return x
    edge_index = ops.as_device(edge_index, torch.int32)
    x = ops.as_device(x, torch.float32, device=edge_index.device)
    if num_nodes is None:
        num_nodes = x.shape[0]
    num_nodes = int(num_nodes)

    fused = (reducer in _FUSED_REDUCERS and updater in (sum_updater, identity_updater)
             and (mapper is identity_mapper or (mapper is gcn_mapper and edge_weight is not None)))
    if fused and autograd.needs_grad(x, edge_weight):
        # differentiable route: sum / mean through NeighborAggregate, max through NeighborMax (both with a transposed-CSR
        # backward); differentiable edge weights (and max over host tensors) through the generic route below (gather +
        # SegmentReduce), which torch autograd can follow
        is_max = _FUSED_REDUCERS[reducer] == "max"
        max_ok = autograd._is_device(x) and num_nodes == x.shape[0]       # NeighborMax: device rows, one per node
        if not autograd.needs_grad(edge_weight) and (not is_max or max_ok):
            w = None
            if mapper is gcn_mapper:
                w = ops.as_device(edge_weight, torch.float32, device=x.device)
            if is_max:
                agg = autograd.NeighborMax.apply(x, edge_index, w, num_nodes)
            else:
                agg = autograd.NeighborAggregate.apply(x, edge_index, w, _FUSED_REDUCERS[reducer], num_nodes)
            return x + agg if updater is sum_updater else agg
        fused = False
    if fused:
        csr, _ = _structure.csr_for_edge_index(edge_index, num_nodes)
        w_csr = None
        if mapper is gcn_mapper:
            edge_weight = ops.as_device(edge_weight, torch.float32, device=x.device)
            w_csr = _structure.weights_in_csr_order(edge_weight, csr)
        if updater is sum_updater:
            return ops.spmm(csr, w_csr, x, reduce=_FUSED_REDUCERS[reducer], alpha=1.0, addend=x, beta=1.0)
        return ops.spmm(csr, w_csr, x, reduce=_FUSED_REDUCERS[reducer])

    # generic route for user callables (layers/kernel/map_reduce.py MapReduceGNN): correctness, not speed
    row, col = edge_index[0], edge_index[1]
    repeated_x = x.index_select(0, row.long())
    neighbor_x = x.index_select(0, col.long())
    if edge_weight is not None:
        edge_weight = ops.as_device(edge_weight, torch.float32, device=x.device)
    neighbor_msg = mapper(repeated_x, neighbor_x, edge_weight=edge_weight)
    reduced_msg = reducer(neighbor_msg, row, num_nodes=num_nodes)
    return updater(x, reduced_msg)
