# coding=utf-8
"""GraphSAGE aggregators with the reference's functional signatures (tf_geometric/nn/conv/graph_sage.py).

mean/sum aggregate the RAW features (D = num_features) with tfgk_spmm_f32, then project; the pooling variants apply
the neighbour MLP per NODE instead of per EDGE - relu(x[col] @ W + b) == relu(x @ W + b)[col], the same arithmetic
on E/N-times fewer rows - and reduce with the mean / max kernel.  Reference quirks are kept: a provided edge_weight
is replaced by ones in the gcn / pool variants (graph_sage.py:139-140,190-191,253-254), and gcn_graph_sage hands its
`cache` to gcn_norm_edge's `renorm` slot (graph_sage.py:142).
"""
import torch

from ... import ops, _structure, autograd
from . import _bf16
from .gat import project
from .gcn import gcn_norm_edge
from ...sparse import SparseMatrix
from ...utils.sampling import Block, SourceRows


def _project_pair(x, agg, self_kernel, neighbor_kernel, bias, activation, concat, normalize):
    """[x @ Ws || agg @ Wn] (+bias, act, l2) with both products written straight into the output columns."""
    dev = x.device
    ws = ops.as_device(self_kernel, torch.float32, device=dev)
    wn = ops.as_device(neighbor_kernel, torch.float32, device=dev)
    act_code, leftover = ops.activation_code(activation)
    b = None if bias is None else ops.as_device(bias, torch.float32, device=dev)
    if concat:
        u = ws.shape[1]
        out = torch.empty((x.shape[0], u + wn.shape[1]), dtype=torch.float32, device=dev)
        ops.gemm(x, ws, bias=None if b is None else b[:u].contiguous(), act=act_code, out=out[:, :u])
        ops.gemm(agg, wn, bias=None if b is None else b[u:].contiguous(), act=act_code, out=out[:, u:])
    else:
        out = ops.gemm(x, ws)
        ops.gemm(agg, wn, bias=b, act=act_code, beta=1.0, out=out)
    if leftover is not None:
        out = leftover(out)
    if normalize:
        out = ops.l2_normalize(out)
    return out


def _plain_sage_autograd(reduce, x, edge_index, edge_weight, ws, wn, bias, activation, concat, normalize):
    """Training path (any input requires grad): the same kernels wrapped in autograd Functions (autograd.py)."""
    act_code, leftover = ops.activation_code(activation)
    if leftover is None and not normalize and not autograd.needs_grad(edge_weight):
        return autograd.SagePair.apply(x, ws, wn, bias, edge_index, edge_weight, reduce, act_code, bool(concat))
    agg = autograd.NeighborAggregate.apply(x, edge_index, edge_weight, reduce, x.shape[0])
    return _project_pair_autograd(x, agg, ws, wn, bias, activation, concat, normalize)


def _project_pair_autograd(x, agg, ws, wn, bias, activation, concat, normalize):
    """Differentiable twin of _project_pair."""
    act_code, leftover = ops.activation_code(activation)
    if concat:
        u = ws.shape[1]
        left = autograd.Dense.apply(x, ws, None if bias is None else bias[:u], act_code)
        right = autograd.Dense.apply(agg, wn, None if bias is None else bias[u:], act_code)
        h = torch.cat([left, right], dim=1)
    else:
        h = autograd.Dense.apply(x, ws, None, ops.ACT_NONE) + autograd.Dense.apply(agg, wn, bias, ops.ACT_NONE)
        if act_code == ops.ACT_RELU:
            h = torch.relu(h)
    if leftover is not None:
        h = leftover(h)
    if normalize:
        h = h * torch.rsqrt(torch.clamp((h * h).sum(dim=-1, keepdim=True), min=1e-12))
    return h


def _block_input(x, block, edge_weight, message_dtype, gather_all):
    """(table, self_index) for a layer over a sampled block: the block's [num_src, F] input and None, or, for a SourceRows
    input that mean / sum can read in place, the global table and the node ids of the self rows.  Refuses what blocks do
    not support before any device work."""
    if _bf16.enabled(message_dtype):
        raise NotImplementedError("GraphSAGE on a sampled block takes fp32 messages only (message_dtype=None)")
    if edge_weight is not None:
        if torch.is_tensor(edge_weight) and edge_weight.requires_grad:
            raise NotImplementedError("GraphSAGE on a sampled block has no edge-weight gradient")
        raise ValueError("a sampled block carries its edge weights: pass [x, block]")
    if isinstance(x, SourceRows):
        if x.shape[0] != block.num_src:
            raise ValueError("the source rows ({}) are not this block's {} input rows".format(x.shape[0], block.num_src))
        if gather_all or (x.x.requires_grad and torch.is_grad_enabled()):
            return x.gather(), None
        return x.x, x.node_index[:block.num_dst]
    x = ops.as_device(x, torch.float32, device=block.edge_index.device)
    if x.dim() != 2 or x.shape[0] != block.num_src:
        raise ValueError("x has {} rows, the block has {} input rows".format(tuple(x.shape)[:1], block.num_src))
    return x, None


def _block_sage(reduce, x, block, edge_weight, self_kernel, neighbor_kernel, bias, activation, concat, normalize,
                message_dtype):
    """mean / sum GraphSAGE over a sampled block: num_dst output rows; the self term is the input's first num_dst rows."""
    table, self_index = _block_input(x, block, edge_weight, message_dtype, False)
    dev = table.device
    col = None if self_index is None else block.global_col
    if autograd.needs_grad(table, self_kernel, neighbor_kernel, bias):
        f32 = lambda t: None if t is None else ops.as_device(t, torch.float32, device=dev)   # noqa: E731
        act_code, leftover = ops.activation_code(activation)
        if leftover is None and not normalize:
            return autograd.BlockSagePair.apply(table, f32(self_kernel), f32(neighbor_kernel), f32(bias), block, reduce,
                                                act_code, bool(concat), self_index)
        agg = autograd.BlockAggregate.apply(table, block, reduce, True, col)
        x_self = table[:block.num_dst] if self_index is None else ops.permute(table, self_index)
        return _project_pair_autograd(x_self, agg, f32(self_kernel), f32(neighbor_kernel), f32(bias), activation, concat,
                                      normalize)
    agg = ops.spmm(block.csr, block.edge_weight, table, reduce=reduce, col=col)
    x_self = table[:block.num_dst] if self_index is None else ops.permute(table, self_index)
    return _project_pair(x_self, agg, self_kernel, neighbor_kernel, bias, activation, concat, normalize)


def _plain_sage(reduce, x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias, activation, concat, normalize,
                message_dtype=None):
    if isinstance(edge_index, Block):
        return _block_sage(reduce, x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias, activation, concat,
                           normalize, message_dtype)
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        _bf16.refuse_unsupported(x, (self_kernel, neighbor_kernel, bias, edge_weight))
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = ops.as_device(x, torch.float32, device=dev)
    num_nodes = x.shape[0]
    if autograd.needs_grad(x, self_kernel, neighbor_kernel, bias, edge_weight):
        ew = None if edge_weight is None else ops.as_device(edge_weight, torch.float32, device=dev)
        return _plain_sage_autograd(reduce, x, edge_index, ew, ops.as_device(self_kernel, torch.float32, device=dev),
                                    ops.as_device(neighbor_kernel, torch.float32, device=dev),
                                    None if bias is None else ops.as_device(bias, torch.float32, device=dev),
                                    activation, concat, normalize)
    csr, _ = _structure.csr_for_edge_index(edge_index, num_nodes)
    w_csr = None
    if edge_weight is not None:
        w_csr = _structure.weights_in_csr_order(ops.as_device(edge_weight, torch.float32, device=dev), csr)
    # bf16: the gathered copy of x is rounded, the self term x Ws reads the fp32 x
    agg = ops.spmm(csr, w_csr, ops.round_bf16_table(x) if bf16 else x, reduce=reduce)
    return _project_pair(x, agg, self_kernel, neighbor_kernel, bias, activation, concat, normalize)


def mean_graph_sage(x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias=None, activation=None,
                    concat=True, normalize=False, message_dtype=None):
    """h = act([x Ws || mean_{j in N(i)} (w_ij x_j) Wn] + b)  (reference graph_sage.py:9-60).
    message_dtype=torch.bfloat16: inference with the gathered x stored in bf16 (an extension of the reference API)."""
    return _plain_sage("mean", x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias, activation, concat,
                       normalize, message_dtype)


def sum_graph_sage(x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias=None, activation=None,
                   concat=True, normalize=False, message_dtype=None):
    """Sum aggregator (reference graph_sage.py:64-115).
    message_dtype=torch.bfloat16: inference with the gathered x stored in bf16 (an extension of the reference API)."""
    return _plain_sage("sum", x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias, activation, concat,
                       normalize, message_dtype)


def gcn_graph_sage(x, edge_index, edge_weight, kernel, bias=None, activation=None, normalize=False, cache=None,
                   message_dtype=None):
    """GCN aggregator (reference graph_sage.py:118-161): act((norm(A) x) W + b).  message_dtype=torch.bfloat16:
    inference with the gathered x stored in bf16 (an extension of the reference API)."""
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        _bf16.refuse_unsupported(x, (kernel, bias))
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = ops.as_device(x, torch.float32, device=dev)
    num_nodes = x.shape[0]
    if edge_weight is not None:
        edge_weight = torch.ones([edge_index.shape[1]], dtype=torch.float32, device=dev)
    # reference :142 passes `cache` positionally into gcn_norm_edge(edge_index, num_nodes, edge_weight, renorm=...)
    normed = SparseMatrix(*_norm_edge_as_matrix(edge_index, num_nodes, edge_weight, renorm=bool(cache)))
    if autograd.needs_grad(x, kernel, bias):
        h = autograd.dense(autograd.propagate(normed, x), ops.as_device(kernel, torch.float32, device=dev),
                           None if bias is None else ops.as_device(bias, torch.float32, device=dev), activation)
        if normalize:
            h = h * torch.rsqrt(torch.clamp((h * h).sum(dim=-1, keepdim=True), min=1e-12))
        return h
    reduced = normed.matmul(ops.round_bf16_table(x) if bf16 else x)
    act_code, leftover = ops.activation_code(activation)
    h = ops.gemm(reduced, ops.as_device(kernel, torch.float32, device=dev),
                 bias=None if bias is None else ops.as_device(bias, torch.float32, device=dev), act=act_code)
    if leftover is not None:
        h = leftover(h)
    if normalize:
        h = ops.l2_normalize(h)
    return h


def _norm_edge_as_matrix(edge_index, num_nodes, edge_weight, renorm):
    index, value = gcn_norm_edge(edge_index, num_nodes, edge_weight, renorm=renorm)
    return index, value, [num_nodes, num_nodes]


def _block_pool_sage(reduce, x, block, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel, neighbor_mlp_bias,
                     bias, activation, concat, normalize, message_dtype):
    """mean-pool / max-pool GraphSAGE over a sampled block: the neighbour MLP runs on every source row (so a SourceRows
    input is gathered), the reduction over the block's edges with unit weights (the reference's quirk), num_dst rows out."""
    x, _ = _block_input(x, block, edge_weight, message_dtype, True)
    dev = x.device
    f32 = lambda t: None if t is None else ops.as_device(t, torch.float32, device=dev)   # noqa: E731
    if autograd.needs_grad(x, self_kernel, neighbor_mlp_kernel, neighbor_kernel, neighbor_mlp_bias, bias):
        h_node = autograd.dense(x, f32(neighbor_mlp_kernel), f32(neighbor_mlp_bias), activation)
        if reduce == "mean":
            reduced = autograd.BlockAggregate.apply(h_node, block, "mean", False, None)
        else:
            reduced = autograd.BlockMax.apply(h_node, block)
        return _project_pair_autograd(x[:block.num_dst], reduced, f32(self_kernel), f32(neighbor_kernel), f32(bias),
                                      activation, concat, normalize)
    act_code, leftover = ops.activation_code(activation)
    h_node = ops.gemm(x, f32(neighbor_mlp_kernel), bias=f32(neighbor_mlp_bias), act=act_code)
    if leftover is not None:
        h_node = leftover(h_node)
    reduced = ops.spmm(block.csr, None, h_node, reduce=reduce)
    return _project_pair(x[:block.num_dst], reduced, self_kernel, neighbor_kernel, bias, activation, concat, normalize)


def _pool_sage(reduce, x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
               neighbor_mlp_bias, bias, activation, concat, normalize, message_dtype=None):
    if isinstance(edge_index, Block):
        return _block_pool_sage(reduce, x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                                neighbor_mlp_bias, bias, activation, concat, normalize, message_dtype)
    ops.refuse_sampled(edge_index)           # a SelfLoopBlock: the sampled-input refusal, not the edge_weight one
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        _bf16.refuse_unsupported(x, (self_kernel, neighbor_mlp_kernel, neighbor_kernel, neighbor_mlp_bias, bias))
    if edge_weight is None:
        # the reference multiplies by `edge_weight` unconditionally (gcn_mapper) and fails on None
        raise TypeError("edge_weight must not be None for the pooling GraphSAGE variants (reference behaviour)")
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = ops.as_device(x, torch.float32, device=dev)
    num_nodes = x.shape[0]
    if autograd.needs_grad(x, self_kernel, neighbor_mlp_kernel, neighbor_kernel, neighbor_mlp_bias, bias):
        f32 = lambda t: None if t is None else ops.as_device(t, torch.float32, device=dev)   # noqa: E731
        h_node = autograd.dense(x, f32(neighbor_mlp_kernel), f32(neighbor_mlp_bias), activation)
        if reduce == "mean":
            reduced = autograd.NeighborAggregate.apply(h_node, edge_index, None, "mean", num_nodes)
        else:
            # K11: the max keeps a tie count per output entry, and the backward routes the gradient to the selected
            # neighbours (ties share it, TF's UnsortedSegmentMax gradient) over the transposed CSR: no per-edge messages
            reduced = autograd.max_aggregate(h_node, edge_index, num_nodes)
        return _project_pair_autograd(x, reduced, f32(self_kernel), f32(neighbor_kernel), f32(bias), activation, concat,
                                      normalize)
    csr, _ = _structure.csr_for_edge_index(edge_index, num_nodes)
    act_code, leftover = ops.activation_code(activation)
    if bf16:
        reduced = ops.spmm(csr, None, _pool_mlp_bf16(x, neighbor_mlp_kernel, neighbor_mlp_bias, activation), reduce=reduce)
        return _project_pair(x, reduced, self_kernel, neighbor_kernel, bias, activation, concat, normalize)
    # per-node neighbour MLP (weights are all ones, so x[col] * w == x[col])
    h_node = ops.gemm(x, ops.as_device(neighbor_mlp_kernel, torch.float32, device=dev),
                      bias=None if neighbor_mlp_bias is None else ops.as_device(neighbor_mlp_bias, torch.float32, device=dev),
                      act=act_code)
    if leftover is not None:
        h_node = leftover(h_node)
    reduced = ops.spmm(csr, None, h_node, reduce=reduce)
    return _project_pair(x, reduced, self_kernel, neighbor_kernel, bias, activation, concat, normalize)


def _pool_mlp_bf16(x, kernel, bias, activation):
    """bf16(act(x W + b)) in a padded table: rounded by the projection's epilogue (K4) for relu / no activation, by
    tfgk_round_bf16 after any other activation."""
    dev = x.device
    kernel = ops.as_device(kernel, torch.float32, device=dev)
    bias = None if bias is None else ops.as_device(bias, torch.float32, device=dev)
    act_code, leftover = ops.activation_code(activation)
    if leftover is not None:
        return ops.round_bf16_table(leftover(ops.gemm(x, kernel, bias=bias, act=act_code)))
    h = ops.bf16_table(x.shape[0], kernel.shape[1], dev)
    project(x, [(kernel, bias, act_code, h)])
    return h


def mean_pool_graph_sage(x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                         neighbor_mlp_bias=None, bias=None, activation=None, concat=True, normalize=False,
                         message_dtype=None):
    """Mean-pooling aggregator (reference graph_sage.py:164-225).
    message_dtype=torch.bfloat16: inference with the neighbour MLP's output stored in bf16 (an extension of the
    reference API)."""
    return _pool_sage("mean", x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                      neighbor_mlp_bias, bias, activation, concat, normalize, message_dtype)


def max_pool_graph_sage(x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                        neighbor_mlp_bias=None, bias=None, activation=None, concat=True, normalize=False,
                        message_dtype=None):
    """Max-pooling aggregator (reference graph_sage.py:228-287); nodes without in-edges get float32 lowest.
    message_dtype=torch.bfloat16: inference with the neighbour MLP's output stored in bf16 (an extension of the
    reference API)."""
    return _pool_sage("max", x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                      neighbor_mlp_bias, bias, activation, concat, normalize, message_dtype)


def _lstm_sage(x, edge_index, reduce_steps, step_major, self_kernel, neighbor_kernel, bias, activation, concat,
               normalize):
    """Shared body of lstm_graph_sage and LSTMGraphSage: pad the neighbour rows (K9), `reduce_steps(padded)` -> [N, U]
    (the recurrence and the mean over all K steps), then the pair projection."""
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = ops.as_device(x, torch.float32, device=dev)
    num_nodes, num_edges = x.shape[0], edge_index.shape[1]
    if num_edges == 0:
        raise ValueError("lstm_graph_sage needs at least one edge (the reference would run the LSTM over zero steps)")
    csr, _ = _structure.csr_for_edge_index(edge_index, num_nodes)
    K = int(csr.degree_i64().max())                                  # graph_sage.py:325 reduce_max(degree)
    if K * num_nodes >= 2 ** 31:
        raise ValueError("lstm_graph_sage: max in-degree {} times {} nodes reaches 2^31 padded slots, beyond the int32 "
                         "slot index of the backward".format(K, num_nodes))
    padded = autograd.PadRows.apply(x, csr, K, step_major, edge_index)
    reduced = reduce_steps(padded)
    dev_f32 = lambda t: None if t is None else ops.as_device(t, torch.float32, device=dev)     # noqa: E731
    if autograd.needs_grad(x, self_kernel, neighbor_kernel, bias, reduced):
        return _project_pair_autograd(x, reduced, dev_f32(self_kernel), dev_f32(neighbor_kernel), dev_f32(bias),
                                      activation, concat, normalize)
    return _project_pair(x, reduced, self_kernel, neighbor_kernel, bias, activation, concat, normalize)


def lstm_graph_sage(x, edge_index, lstm, self_kernel, neighbor_kernel, bias=None, activation=None, concat=True,
                    normalize=False, training=False):
    """LSTM aggregator (reference graph_sage.py:290-356): every node's in-neighbours x[col], in edge order (stable by
    edge_index[0]), zero-padded to the maximum in-degree K, go through `lstm` - any callable with the Keras
    return_sequences=True convention, lstm([N, K, F], training=...) -> [N, K, U] - whose outputs are averaged over all K
    steps (padded steps included, divided by K, as the reference does); then [x Ws || mean Wn] (+ b, act, l2) with
    neighbor_kernel [U, U].  Differentiable in x, the kernels, the bias and the callable's parameters.  An edgeless graph
    raises ValueError; so does K * N >= 2^31."""
    return _lstm_sage(x, edge_index, lambda padded: lstm(padded, training=training).mean(dim=1), False, self_kernel,
                      neighbor_kernel, bias, activation, concat, normalize)
