# coding=utf-8
"""GCN normalisation and convolution with the reference's functional signatures (tf_geometric/nn/conv/gcn.py).

    gcn(x, A, W, b) = act( norm(A) @ (x @ W) + b )

norm(A) is computed once per graph by the integer/fp32 preprocessing kernels and memoised in `cache` (the reference
stores a numpy triple under the same key, gcn.py:125-128; here the cached object is a device SparseMatrix that also
carries the destination-sorted CSR, so a warm forward is exactly two launches: the dense projection and tfgk_spmm_f32
with bias + activation fused into its epilogue).  In inference, when the input is narrower than the output (ops.spmm_proj
takes the shapes), a warm forward is one launch instead: act((norm(A) x) W + b) by tfgk_spmm_proj_f32, which gathers the
narrower rows of x and projects each aggregate in its epilogue.
"""
import torch

from ... import ops, autograd
from ...sparse import SparseMatrix, as_sparse_features, project_features
from ...utils.sampling import GcnBlock, SourceRows, gcn_block_codes
from ..kernel.map_reduce import gcn_mapper  # noqa: F401  (re-exported like the reference)

CACHE_KEY_GCN_NORMED_ADJ_TEMPLATE = "gcn_normed_adj_{}_{}_{}_{}_{}"


def compute_cache_key(norm, add_self_loop, sym, renorm, improved):
    return CACHE_KEY_GCN_NORMED_ADJ_TEMPLATE.format(norm, add_self_loop, sym, renorm, improved)


def gcn_norm_adj(sparse_adj, norm="both", add_self_loop=True, sym=True, renorm=True, improved=False, cache=None):
    """
    Normalised adjacency for GCN (reference gcn.py:32-130).

    :param sparse_adj: SparseMatrix adjacency (row = aggregation target).
    :param norm: "both" (D^-1/2 A D^-1/2), "left" (D^-1 A) or "right" (A D^-1, with ROW sums - as the reference does).
    :param add_self_loop: add I * fill (fill = 2 if improved else 1); appended after the existing entries.
    :param sym: with norm="both", reuse the row degrees on the column side (valid for symmetric A).
    :param renorm: renormalisation trick: add the loops before normalising instead of after.
    :param cache: dict memoising the result under compute_cache_key(...).
    """
    if cache is not None:
        cache_key = compute_cache_key(norm, add_self_loop, sym, renorm, improved)
        cached = cache.get(cache_key, None)
        if cached is not None:
            if isinstance(cached, SparseMatrix):
                return cached
            return SparseMatrix(cached[0], cached[1], cached[2])      # a reference-style (index, value, shape) triple

    w = sparse_adj.value
    normed, aux = _normalize(sparse_adj, norm, add_self_loop, sym, renorm, improved)
    if cache is not None:
        normed.csr, normed.value_csr    # build the CSR now: cached objects are always warm
        cache[cache_key] = normed       # the cached matrix carries no gradient: a warm call returns it as is
    if autograd.needs_grad(w):
        # differentiable in the edge weights (tf.GradientTape sees through the reference's normalisation): same values,
        # same CSR, with a backward to w
        normed = normed.with_value(autograd.GcnNormValues.apply(w, normed.value, aux))
    return normed


def _normalize(sparse_adj, norm, add_self_loop, sym, renorm, improved):
    """(normed SparseMatrix, aux): the kernels of reference gcn.py:32-130, and what GcnNormValues' backward needs
    (kind, A' = the matrix whose sums are the degrees, its normalised values, the row and column factors)."""
    fill_weight = 2.0 if improved else 1.0
    if sparse_adj.shape[0] != sparse_adj.shape[1]:
        if add_self_loop:
            raise Exception("cannot set add_self_loop=True for GCN when sparse_adj.shape[0] != sparse_adj.shape[1]")
        if sym:
            raise Exception("cannot set sym=True for GCN when sparse_adj.shape[0] != sparse_adj.shape[1]")

    if add_self_loop and norm != "both":
        sparse_adj = sparse_adj.add_diag(fill_weight)

    if norm == "both":
        if add_self_loop and renorm:
            sparse_adj = sparse_adj.add_diag(fill_weight)
        row_dis = ops.deg_inv(sparse_adj.segment_sum(axis=-1), ops.POW_INV_SQRT)
        col_dis = row_dis if sym else ops.deg_inv(sparse_adj.segment_sum(axis=0), ops.POW_INV_SQRT)
        value = ops.scale_edges(sparse_adj.index[0].contiguous(), sparse_adj.index[1].contiguous(), sparse_adj.value,
                                dl=row_dis, dr=col_dis)
        normed = sparse_adj.with_value(value)
        aux = ("both_sym" if sym else "both", sparse_adj, value, row_dis, col_dis)
        if add_self_loop and not renorm:
            normed = normed.add_diag(fill_weight)
    elif norm == "left":
        row_inv = ops.deg_inv(sparse_adj.segment_sum(axis=-1), ops.POW_INV)
        normed = sparse_adj.with_value(ops.scale_edges(sparse_adj.index[0].contiguous(), None, sparse_adj.value,
                                                       dl=row_inv))
        aux = ("left", sparse_adj, normed.value, row_inv, None)
    elif norm == "right":
        col_inv = ops.deg_inv(sparse_adj.segment_sum(axis=-1), ops.POW_INV)     # row sums, literally as gcn.py:113
        normed = sparse_adj.with_value(ops.scale_edges(None, sparse_adj.index[1].contiguous(), sparse_adj.value,
                                                       dr=col_inv))
        aux = ("right", sparse_adj, normed.value, col_inv, None)
    else:
        raise Exception("wrong GCN norm type: {}".format(norm))
    return normed, aux


def gcn_build_cache_by_adj(sparse_adj, norm="both", add_self_loop=True, sym=True, renorm=True, improved=False,
                           override=False, cache=None):
    """Compute norm(A) for this configuration and store it in `cache` (reference gcn.py:133-152)."""
    if cache is None:
        cache = {}
    elif override:
        cache[compute_cache_key(norm, add_self_loop, sym, renorm, improved)] = None
    gcn_norm_adj(sparse_adj, norm, add_self_loop, sym, renorm, improved, cache)
    return cache


def gcn_build_cache_for_graph(graph, norm="both", add_self_loop=True, sym=True, renorm=True, improved=False,
                              override=False):
    """reference gcn.py:155-169."""
    graph.cache = gcn_build_cache_by_adj(graph.adj(), norm=norm, add_self_loop=add_self_loop, sym=sym, renorm=renorm,
                                         improved=improved, override=override, cache=graph.cache)
    return graph.cache


def gcn_norm_edge(edge_index, num_nodes, edge_weight=None, renorm=True, improved=False, cache=None):
    """Deprecated edge-list form (reference gcn.py:180-196)."""
    sparse_adj = SparseMatrix(edge_index, edge_weight, [num_nodes, num_nodes])
    normed = gcn_norm_adj(sparse_adj, renorm=renorm, improved=improved, cache=cache)
    return normed.index, normed.value


def gcn(x, sparse_adj, kernel, bias=None, activation=None,
        norm="both", add_self_loop=True, sym=True, renorm=True, improved=False, edge_drop_rate=0.0,
        num_or_size_splits=None, training=False, cache=None, message_dtype=None):
    """
    Functional GCN layer (reference gcn.py:225-290).

    :param x: [num_nodes, num_features] float32
    :param sparse_adj: SparseMatrix adjacency
    :param kernel: [num_features, units] or None (propagate x itself)
    :param bias: [units] or None
    :param activation: callable or None; relu is fused into the aggregation epilogue
    :param num_or_size_splits: column chunks of the propagation (gcn.py:274-280): one launch per chunk into slices of one
        output, same bits (the fused kernel has no [E, D] temporary to bound, so this is an API-parity feature)
    :param message_dtype: None / torch.float32 (default), or torch.bfloat16: inference with x W stored in bf16 (rounded
        once, to nearest even, by the projection) and aggregated from half the bytes in fp32; the output is fp32.  Or
        torch.float8_e4m3fn: x W stored as e4m3 bytes with a power-of-two scale per row (include/tfgk.h), a quarter of
        the bytes, aggregated in fp32.  An extension of the reference API
    :return: [num_nodes, units]

    On a sampled block (an extension of the reference API): sparse_adj is the GcnBlock of block.with_gcn_norm(), whose
    values for this call's norm / add_self_loop / sym / renorm / improved are the full graph's normalisation with each
    row's sampled edges rescaled by degree over fan-out (made on first use and kept on the GcnBlock; `cache` is not
    consulted).  x is the block's dense [num_src, F] input or a SourceRows (gathered: every source row is projected); the
    output has num_dst rows.  fp32 messages only, and not sym=False with norm="both".
    """
    if isinstance(sparse_adj, GcnBlock):
        return _gcn_block(x, sparse_adj, kernel, bias, activation, norm, add_self_loop, sym, renorm, improved,
                          edge_drop_rate, num_or_size_splits, training, message_dtype)
    mdt = ops.conv_message_dtype(message_dtype)
    if mdt is torch.float8_e4m3fn:
        return _gcn_fp8(x, sparse_adj, kernel, bias, activation, norm, add_self_loop, sym, renorm, improved, edge_drop_rate,
                        training, cache)
    if mdt is not None:
        return _gcn_bf16(x, sparse_adj, kernel, bias, activation, norm, add_self_loop, sym, renorm, improved, edge_drop_rate,
                         num_or_size_splits, training, cache)
    normed = gcn_norm_adj(sparse_adj, norm=norm, add_self_loop=add_self_loop, sym=sym, renorm=renorm,
                          improved=improved, cache=cache)
    return _gcn_normed(x, normed, kernel, bias, activation, edge_drop_rate, num_or_size_splits, training)


def _gcn_block(x, gcn_block, kernel, bias, activation, norm, add_self_loop, sym, renorm, improved, edge_drop_rate,
               num_or_size_splits, training, message_dtype):
    """gcn() over a GcnBlock: refuses what blocks do not support before any device work, then runs gcn()'s body over the
    block's [num_dst, num_src] normalised matrix."""
    if ops.conv_message_dtype(message_dtype) is not None:
        raise NotImplementedError("GCN on a sampled block takes fp32 messages only (message_dtype=None)")
    if not isinstance(x, SourceRows) and as_sparse_features(x) is not None:
        raise NotImplementedError("GCN on a sampled block takes a dense x")
    gcn_block_codes(norm, add_self_loop, sym, renorm, improved)
    rows = tuple(x.shape)[:1] if hasattr(x, "shape") and len(x.shape) == 2 else None
    if rows != (gcn_block.num_src,):
        raise ValueError("x has {} rows, the block has {} input rows".format(rows, gcn_block.num_src))
    if isinstance(x, SourceRows):
        x = x.gather()
    normed = gcn_block.normalized(norm, add_self_loop, sym, renorm, improved)
    return _gcn_normed(x, normed, kernel, bias, activation, edge_drop_rate, num_or_size_splits, training)


def _gcn_normed(x, normed, kernel, bias, activation, edge_drop_rate, num_or_size_splits, training):
    """gcn() after the normalisation: act(normed @ (x W) + b) over the normalised SparseMatrix `normed` (the full graph's
    square matrix, or a GcnBlock's [num_dst, num_src] one), with edge dropout on its values."""
    normed = normed.dropout(edge_drop_rate, training=training)
    dev = normed.index.device
    act_code, leftover = ops.activation_code(activation)
    bias = None if bias is None else ops.as_device(bias, torch.float32, device=dev)
    x_sparse = as_sparse_features(x)
    if x_sparse is not None:                   # tf.SparseTensor features (gcn.py:269-272): sparse x dense projection
        if kernel is None:
            raise ValueError("a sparse feature matrix needs a kernel (reference gcn.py:266-272)")
        if autograd.needs_grad(kernel, bias, x_sparse.value, normed.value):
            # training (demo/demo_gcn.py:60-75): dW = x^T dH is the same kernel over the transposed pattern of x; learnable
            # edge weights reach normed.value through the normalisation
            h = autograd.propagate(x_sparse, ops.as_device(kernel, torch.float32, device=dev))
            h = autograd.propagate(normed, h, bias, act_code)
            return leftover(h) if leftover is not None else h
        h = project_features(x_sparse, kernel)
        h = normed.matmul(h, num_or_size_splits=num_or_size_splits, bias=bias, act=act_code)
        return leftover(h) if leftover is not None else h
    x = ops.as_device(x, torch.float32, device=dev)
    if autograd.needs_grad(x, kernel, bias, normed.value):
        # training path (demo/demo_gcn.py:60-75 uses tf.GradientTape): same kernels behind autograd Functions
        h = x if kernel is None else autograd.Dense.apply(x, ops.as_device(kernel, torch.float32, device=dev), None,
                                                         ops.ACT_NONE)
        h = autograd.propagate(normed, h, bias, act_code)
        return leftover(h) if leftover is not None else h
    if kernel is not None:
        kernel = ops.as_device(kernel, torch.float32, device=dev)
        if num_or_size_splits is None and ops.spmm_proj_supported(x, kernel):
            # narrower input than output: gather the F-wide rows of x and project each aggregate in the kernel's epilogue
            h = ops.spmm_proj(normed.csr, normed.value_csr, x, kernel, bias=bias, act=act_code)
            return leftover(h) if leftover is not None else h
    h = x if kernel is None else ops.gemm(x, kernel)
    h = normed.matmul(h, num_or_size_splits=num_or_size_splits, bias=bias, act=act_code)
    if leftover is not None:
        h = leftover(h)
    return h


def _gcn_bf16(x, sparse_adj, kernel, bias, activation, norm, add_self_loop, sym, renorm, improved, edge_drop_rate,
              num_or_size_splits, training, cache):
    """gcn() with bf16 message rows: act(norm(A) @ bf16(x W) + b), the product over the widened rows in fp32."""
    from .gat import project
    if as_sparse_features(x) is not None:
        raise NotImplementedError("message_dtype=bfloat16 takes a dense x")
    if training and edge_drop_rate > 0.0:
        raise NotImplementedError("message_dtype=bfloat16 is for inference: edge dropout is not applied in bf16")
    normed = gcn_norm_adj(sparse_adj, norm=norm, add_self_loop=add_self_loop, sym=sym, renorm=renorm,
                          improved=improved, cache=cache)
    dev = normed.index.device
    x = ops.as_device(x, torch.float32, device=dev)
    if autograd.needs_grad(x, kernel, bias, normed.value):
        raise NotImplementedError("message_dtype=bfloat16 is for inference: no operand may require grad")
    act_code, leftover = ops.activation_code(activation)
    bias = None if bias is None else ops.as_device(bias, torch.float32, device=dev)
    if kernel is None:
        h = ops.round_bf16(x)
    else:
        kernel = ops.as_device(kernel, torch.float32, device=dev)
        h = torch.empty((x.shape[0], kernel.shape[1]), dtype=torch.bfloat16, device=dev)
        project(x, [(kernel, None, ops.ACT_NONE, h)])
    h = normed.matmul(h, num_or_size_splits=num_or_size_splits, bias=bias, act=act_code)
    return leftover(h) if leftover is not None else h


def _gcn_fp8(x, sparse_adj, kernel, bias, activation, norm, add_self_loop, sym, renorm, improved, edge_drop_rate, training,
             cache):
    """gcn() with fp8 message rows: act(norm(A) @ dequant(fp8(x W)) + b), the product over the dequantised rows in fp32.
    The projection writes the bytes and exponents in its epilogue; one aggregation launch reads them (column splits would
    give the same bits and are not applied)."""
    if as_sparse_features(x) is not None:
        raise NotImplementedError("message_dtype=float8_e4m3fn takes a dense x")
    if training and edge_drop_rate > 0.0:
        raise NotImplementedError("message_dtype=float8_e4m3fn is for inference: edge dropout is not applied in fp8")
    if autograd.needs_grad(x, kernel, bias, sparse_adj.value):
        raise NotImplementedError("message_dtype=float8_e4m3fn is for inference: no operand may require grad")
    normed = gcn_norm_adj(sparse_adj, norm=norm, add_self_loop=add_self_loop, sym=sym, renorm=renorm,
                          improved=improved, cache=cache)
    dev = normed.index.device
    x = ops.as_device(x, torch.float32, device=dev)
    act_code, leftover = ops.activation_code(activation)
    bias = None if bias is None else ops.as_device(bias, torch.float32, device=dev)
    if kernel is None:
        h = ops.quantize_fp8(x)
    else:
        kernel = ops.as_device(kernel, torch.float32, device=dev)
        units = kernel.shape[1]
        h = ops.fp8_table(x.shape[0], units, dev)
        pieces = [(kernel[:, c0:min(c0 + 128, units)], None, ops.ACT_NONE, h.block(c0, min(c0 + 128, units)))
                  for c0 in range(0, units, 128)]
        for i in range(0, len(pieces), 4):
            ops.gemm_proj(x, pieces[i:i + 4])
    h = ops.spmm(normed.csr, normed.value_csr, h, reduce="sum", bias=bias, act=act_code)
    return leftover(h) if leftover is not None else h
