# coding=utf-8
"""Per-source top-k selection (reference nn/pool/topk_pool.py:6-88).

The reference pads the scores into a dense [num_sources, max_targets] matrix and argsorts every row.  Here: one radix
argsort of order-preserving score keys (descending), one stable CSR build by source (tfgk_csr_build keeps the score
order inside every source), then the deterministic "first node_k entries of each row" rule of the fan-out sampler.
Ties keep their input order (the reference's tf.argsort leaves the order of equal scores unspecified)."""
import torch

from ... import ops, _ffi


def topk_pool(source_index, score, k=None, ratio=None):
    """
    :param source_index: [n] source (graph / node) of every target
    :param score: [n] or [n, 1] scores
    :param k: keep the k best targets of every source (all of them when it has fewer)
    :param ratio: keep ceil(num_targets * ratio) targets of every source
    :return: int32 [num_selected] indices into the inputs, grouped by ascending source, best score first
    """
    _ffi.refuse_capture("topk_pool", "it reads the number of sources and the selection size on the host")
    if k is None and ratio is None:
        raise Exception("you should provide either k or ratio for topk_pool")
    elif k is not None and ratio is not None:
        raise Exception("you should provide either k or ratio for topk_pool, not both of them")
    source_index = ops.as_device(source_index, torch.int32).reshape(-1)
    dev = source_index.device
    score = ops.as_device(score, torch.float32, device=dev).reshape(-1).contiguous()
    n = source_index.numel()
    if n == 0:
        return torch.empty((0,), dtype=torch.int32, device=dev)
    num_sources = int(source_index.max().item()) + 1
    by_score = ops.stable_argsort(ops.sort_keys_f32(score, descending=True))          # best score first, ties by index
    grouped = ops.csr_build(ops.gather_i32(source_index, by_score), by_score, num_sources, n)
    _, pos, _ = ops.neighbor_sample(grouped, k=k, ratio=ratio, padding=ops.SAMPLE_HEAD)
    return ops.gather_i32(grouped.col, pos)
