# coding=utf-8
"""segment_softmax / segment_count with the signatures of tf_geometric/nn/kernel/segment.py, computed by the
CSR kernels (tfgk_segment_softmax_f32, tfgk_segment_count_i32)."""
import torch

from ... import ops, autograd


def segment_softmax(data, segment_ids, num_segments):
    """exp(d - max_seg) / (sum_seg + 1e-8) per segment (reference segment.py:26-33).  `data` is [E] or [E, C];
    differentiable w.r.t. `data` (autograd.SegmentSoftmax) with the same forward bits."""
    segment_ids = ops.as_device(segment_ids, torch.int32)
    data = ops.as_device(data, torch.float32, device=segment_ids.device)
    if autograd.needs_grad(data):
        return autograd.SegmentSoftmax.apply(data, segment_ids, int(num_segments))
    return autograd.segment_softmax_forward(data, segment_ids, num_segments)


def segment_count(index, num_segments=None):
    """int32 histogram of `index` (reference segment.py:36-40)."""
    index = ops.as_device(index, torch.int32)
    if num_segments is None:
        num_segments = int(index.max().item()) + 1
    return ops.segment_count(index, int(num_segments))
