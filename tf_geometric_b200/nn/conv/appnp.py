# coding=utf-8
"""APPNP with the reference's functional signature (tf_geometric/nn/conv/appnp.py:11-92):
an MLP followed by k steps of  out <- norm(A) out (1 - alpha) + h alpha, each step ONE tfgk_spmm_f32 launch with
the teleport term fused into the epilogue."""
import torch

from ... import ops, autograd
from ...sparse import SparseMatrix
from . import _bf16
from .gcn import gcn_norm_adj


def appnp(x, edge_index, edge_weight, kernels, biases,
          dense_activation=ops.relu, activation=None,
          k=10, alpha=0.1,
          dense_drop_rate=0.0, last_dense_drop_rate=0.0, edge_drop_rate=0.0,
          cache=None, training=False, message_dtype=None):
    """
    :param kernels/biases: weights of the dense layers; every layer but the last is followed by dense_activation
    :param k: number of propagation steps; alpha: teleport probability
    :param cache: dict memoising norm(A) (build it with gcn_build_cache_for_graph, like for GCN)
    :param message_dtype: None / torch.float32 (default), or torch.bfloat16: inference with the MLP output and every
        intermediate hop gathered from bf16 (hops 1 .. k-1 are stored only in bf16); the teleport term alpha h, the
        accumulators and the last hop stay fp32.  An extension of the reference API
    """
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        drop = training and max(dense_drop_rate, last_dense_drop_rate, edge_drop_rate) > 0.0
        _bf16.refuse_unsupported(x, [edge_weight] + [t for t in list(kernels) + list(biases) if t is not None], dropout=drop)
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = ops.as_device(x, torch.float32, device=dev)
    num_nodes = x.shape[0]
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [num_nodes, num_nodes]), cache=cache)
    normed = normed.dropout(edge_drop_rate, training=training)                          # appnp.py:54-55
    with_grad = autograd.needs_grad(x, normed.value, *[t for t in list(kernels) + list(biases) if t is not None])

    h = x
    num_dense = len(kernels)
    for i, (kern, b) in enumerate(zip(kernels, biases)):
        act_code, leftover = ops.activation_code(dense_activation if i < num_dense - 1 else None)
        kern = ops.as_device(kern, torch.float32, device=dev)
        b = None if b is None else ops.as_device(b, torch.float32, device=dev)
        h = autograd.Dense.apply(h, kern, b, act_code) if with_grad else ops.gemm(h, kern, bias=b, act=act_code)
        if leftover is not None:
            h = leftover(h)
        h = autograd.dropout(h, dense_drop_rate if i < num_dense - 1 else last_dense_drop_rate, training)   # :75-79

    act_code, leftover = ops.activation_code(activation)
    if with_grad:
        # training (demo/demo_appnp.py): every step is A @ out behind autograd (dOut = A^T g on the transposed CSR);
        # the teleport mix is elementwise
        out = h
        for _ in range(k):
            out = autograd.propagate(normed, out) * (1.0 - alpha) + h * alpha
        if act_code != ops.ACT_NONE:
            out = torch.relu(out)
        return leftover(out) if leftover is not None else out
    out = h
    if bf16 and k > 0:
        out = ops.round_bf16_table(h)
        bufs = [ops.bf16_table(num_nodes, h.shape[1], dev) for _ in range(min(k - 1, 2))]
        for i in range(k - 1):
            out = normed.matmul(out, alpha=1.0 - alpha, addend=h, beta=alpha, out_bf16=bufs[i % 2])
        out = normed.matmul(out, alpha=1.0 - alpha, addend=h, beta=alpha, act=act_code)
        return leftover(out) if leftover is not None else out
    bufs = [torch.empty_like(h), torch.empty_like(h)]
    for i in range(k):
        last = i == k - 1
        out = normed.matmul(out, alpha=1.0 - alpha, addend=h, beta=alpha, act=act_code if last else ops.ACT_NONE,
                            out=bufs[i % 2])
    if k == 0 and act_code != ops.ACT_NONE:
        out = torch.relu(out)
    if leftover is not None:
        out = leftover(out)
    return out
