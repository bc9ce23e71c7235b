# coding=utf-8
"""tfg.nn.drop_edge (reference nn/sampling/drop_edge.py:6-52) on the device: Bernoulli keep flags
(tfgk_edge_flags_i32), stable compaction (tfgk_select_flagged_i32) and gathers - no host round trip of the edge list.
The reference draws its mask from tf.nn.dropout; here it is the counter-based generator of csrc/rng.cuh."""
import numpy as np
import torch

from ... import ops, _rng


def _take_last_axis(attr, index):
    """attr[..., index] for device tensors: 4-byte types go through the gather kernel, anything else through torch."""
    if attr.dtype in (torch.float32, torch.int32) and attr.dim() <= 2 and attr.is_contiguous():
        view = attr if attr.dtype == torch.float32 else attr.view(torch.float32)
        if attr.dim() == 1:
            out = ops.permute(view, index)
        else:
            out = torch.stack([ops.permute(view[i].contiguous(), index) for i in range(attr.shape[0])])
        return out if attr.dtype == torch.float32 else out.view(torch.int32)
    return attr.index_select(-1, index.long())


def drop_edge(inputs, rate=0.5, force_undirected=False, training=None, seed=None):
    """
    :param inputs: [edge_index, edge_attr, ...]; attributes are gathered along their last axis
    :param rate: probability of dropping an edge
    :param force_undirected: decide once per undirected edge: only row < col edges are drawn, survivors are mirrored
    :param training: nothing happens unless truthy
    :param seed: optional 64-bit key pinning the mask (extension)
    :return: [dropped_edge_index, dropped_edge_attr, ...] in the container types of the inputs
    """
    if not training:
        return inputs
    if rate < 0.0 or rate > 1.0:
        raise ValueError('Dropout probability has to be between 0 and 1, '
                         'but got {}'.format(rate))
    edge_index, edge_attrs = inputs[0], list(inputs[1:])
    was_tensor = torch.is_tensor(edge_index)
    ei = ops.as_device(edge_index, torch.int32)
    dev = ei.device
    row, col = ei[0].contiguous(), ei[1].contiguous()
    flag = ops.edge_flags(row, col, row.numel(), mode=ops.FLAG_UPPER if force_undirected else ops.FLAG_ALL,
                          bernoulli=ops.BERNOULLI_DROPOUT, prob=float(rate), seed=_rng.resolve_host(seed))
    index = ops.select_flagged(flag)
    dropped = torch.stack([ops.gather_i32(row, index), ops.gather_i32(col, index)])
    if force_undirected:
        dropped = torch.cat([dropped, dropped.flip(0)], dim=-1)                     # drop_edge.py:38
        index = torch.cat([index, index])
    out = [dropped if was_tensor else dropped.cpu().numpy()]
    for attr in edge_attrs:
        if torch.is_tensor(attr):
            out.append(_take_last_axis(ops.as_device(attr, device=dev), index))
        else:
            out.append(np.take(attr, index.cpu().numpy(), axis=-1))                 # drop_edge.py:48
    return out
