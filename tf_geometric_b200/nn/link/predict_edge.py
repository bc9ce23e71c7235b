# coding=utf-8
"""tfg.nn.predict_edge: the edge scorer of the reference's graph autoencoder demo (demo/demo_gae.py:53-60) as a library
op.  The demo gathers both endpoint rows ([E, D] each), multiplies and reduces; here one kernel reads the two rows and
writes one logit per edge (K6), and the gradient is one deterministic aggregation (autograd.EdgeDot)."""
import torch

from ... import ops
from ...autograd import EdgeDot


def predict_edge(embedded, edge_index):
    """
    :param embedded: float32 [N, D] node embeddings (a CUDA tensor, or anything ops.as_device accepts)
    :param edge_index: int [2, E] query pairs
    :return: float32 [E] logits, logits[e] = sum_d embedded[row_e, d] * embedded[col_e, d]; differentiable w.r.t.
        embedded.  Node ids outside [0, N) raise ValueError.
    """
    if not torch.is_tensor(embedded):
        embedded = ops.as_device(embedded, torch.float32)
    if embedded.dtype != torch.float32:
        embedded = embedded.to(torch.float32)
    ei = ops.as_device(edge_index, torch.int32, device=embedded.device)
    if ei.dim() != 2 or ei.shape[0] != 2:
        raise ValueError("edge_index must have shape [2, E]")
    if ei.numel():
        lo, hi = torch.aminmax(ei)
        if int(lo) < 0 or int(hi) >= embedded.shape[0]:
            raise ValueError("edge_index holds node ids outside [0, {})".format(embedded.shape[0]))
    return EdgeDot.apply(embedded, ei)
