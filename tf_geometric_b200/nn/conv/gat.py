# coding=utf-8
"""Multi-head graph attention with the reference's functional signature (tf_geometric/nn/conv/gat.py:13-122).

The reference materialises Q[row] and K[col] ([E', A] each), builds a virtual graph of H*N nodes, runs a 5-pass
segment_softmax over H*E' scores and finally a SpMM.  Here: three dense projections, then ONE fused kernel
(tfgk_gat_fused_f32) that streams K and V rows once per edge.
"""
import os

import torch

from ... import ops, _structure, _rng, autograd
from ...sparse import as_sparse_features, project_features
from ...utils.sampling import SelfLoopBlock, SourceRows


def project(x, blocks):
    """Dense projections of the same x: column blocks of at most 128 outputs, at most four per launch."""
    pieces = []
    for w, b, act, out in blocks:
        for c0 in range(0, w.shape[1], 128):
            c1 = min(c0 + 128, w.shape[1])
            pieces.append((w[:, c0:c1], None if b is None else b[c0:c1], act, out[:, c0:c1]))
    for i in range(0, len(pieces), 4):
        ops.gemm_proj(x, pieces[i:i + 4])


def _project_qkv(x, n_q, q_block, kv_blocks):
    """Q from x[:n_q] and K | V from every row of x: one launch that reads x once when Q takes every row, else Q from the
    view of the first n_q rows and K | V in a second launch."""
    if n_q == x.shape[0]:
        project(x, [q_block] + kv_blocks)
    else:
        project(x[:n_q], [q_block])
        project(x, kv_blocks)


def gat(x, edge_index,
        query_kernel, query_bias, query_activation,
        key_kernel, key_bias, key_activation,
        kernel, bias=None, activation=None, num_heads=1,
        split_value_heads=True, edge_drop_rate=0.0, training=False, cache=None, return_attention=False, seed=None,
        message_dtype=None):
    """
    :param x: [num_nodes, num_features]
    :param edge_index: [2, num_edges]; self loops are appended (never de-duplicated), reference gat.py:43
    :param query_kernel/key_kernel: [num_features, attention_units]; query_bias/key_bias: [attention_units]
    :param kernel: [num_features, units] (or [num_features, units * num_heads] when split_value_heads=False)
    :param num_heads: heads; attention_units (and units when splitting) must be divisible by it
    :param split_value_heads: True: heads own slices of V and are concatenated; False: every head sees a full V and
        the head outputs are averaged
    :param edge_drop_rate: dropout on the attention coefficients while training (gat.py:85)
    :param cache: optional dict (e.g. graph.cache) memoising the self-looped CSR; an extension of the reference API
    :param seed: optional 64-bit key pinning the dropout mask (extension; default: a fresh key per call)
    :param message_dtype: None / torch.float32 (default), or torch.bfloat16: inference with K and V stored in bf16 (rounded
        once, to nearest even, by the projection that also writes the fp32 Q) and read from half the bytes; scores,
        softmax, accumulation and output stay fp32.  Or torch.float8_e4m3fn: K | V stored as e4m3 bytes with a power-of-two
        scale per row (include/tfgk.h), a quarter of fp32's bytes; heads concatenated, units == attention_units = H * dqk
        <= 128 with dqk / 4 a power of two.  An extension of the reference API
    :return: [num_nodes, units]

    On a sampled block (an extension of the reference API): edge_index is the SelfLoopBlock of block.with_self_loops(),
    whose own self loops are the only ones; x is the block's [num_src, F] input or a SourceRows (gathered: every source
    row is read as a key and a value); the output has num_dst rows.  fp32 messages only.
    """
    if isinstance(edge_index, SelfLoopBlock):
        x = _block_input(x, edge_index, message_dtype, return_attention, training, edge_drop_rate,
                         (query_kernel, query_bias, key_kernel, key_bias, kernel, bias))
        return _gat_dense(x, edge_index.csr, edge_index, query_kernel, query_bias, query_activation, key_kernel,
                          key_bias, key_activation, kernel, bias, activation, num_heads, split_value_heads,
                          float(edge_drop_rate) if training else 0.0, False, return_attention, seed)
    mdt = ops.conv_message_dtype(message_dtype)
    if mdt is torch.float8_e4m3fn:
        return _gat_fp8(x, edge_index, query_kernel, query_bias, query_activation, key_kernel, key_bias, key_activation,
                        kernel, bias, activation, num_heads, split_value_heads, edge_drop_rate, training, cache,
                        return_attention)
    bf16 = mdt is not None
    if bf16:
        if as_sparse_features(x) is not None:
            raise NotImplementedError("message_dtype=bfloat16 takes a dense x")
        if training and edge_drop_rate > 0.0:
            raise NotImplementedError("message_dtype=bfloat16 is for inference: attention dropout is not applied in bf16")
        if return_attention:
            raise NotImplementedError("message_dtype=bfloat16 does not return attention coefficients")
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x_sparse = as_sparse_features(x)             # tf.SparseTensor features (reference gat.py:45-70)
    if x_sparse is None:
        x = ops.as_device(x, torch.float32, device=dev)
    num_nodes = len(x_sparse) if x_sparse is not None else x.shape[0]
    csr, edge_index_used = _structure.csr_for_edge_index(edge_index, num_nodes, add_self_loop=True, cache=cache)
    drop_rate = float(edge_drop_rate) if training else 0.0
    if x_sparse is not None:
        if drop_rate > 0.0 or autograd.needs_grad(query_kernel, query_bias, key_kernel, key_bias, kernel, bias):
            if return_attention:
                raise NotImplementedError("return_attention is an inference-path extension")
            return _gat_training(x_sparse, csr, edge_index_used, query_kernel, query_bias, query_activation, key_kernel,
                                 key_bias, key_activation, kernel, bias, activation, num_heads, split_value_heads, drop_rate,
                                 _rng.resolve(seed, dev) if drop_rate > 0.0 else 0)
        q_act, q_left = ops.activation_code(query_activation)
        k_act, k_left = ops.activation_code(key_activation)
        f32 = lambda t: None if t is None else ops.as_device(t, torch.float32, device=dev)     # noqa: E731
        Q = project_features(x_sparse, query_kernel, bias=f32(query_bias), act=q_act)
        K = project_features(x_sparse, key_kernel, bias=f32(key_bias), act=k_act)
        V = project_features(x_sparse, kernel)
        Q = q_left(Q) if q_left is not None else Q
        K = k_left(K) if k_left is not None else K
        act_code, leftover = ops.activation_code(activation)
        res = ops.gat_fused(csr, Q, K, V, num_heads, split_value_heads=split_value_heads, bias=f32(bias), act=act_code,
                            return_attention=return_attention)
        h, att = res if return_attention else (res, None)
        h = leftover(h) if leftover is not None else h
        return (h, ops.permute(att, csr.perm, inverse=True)) if return_attention else h
    return _gat_dense(x, csr, edge_index_used, query_kernel, query_bias, query_activation, key_kernel, key_bias,
                      key_activation, kernel, bias, activation, num_heads, split_value_heads, drop_rate, bf16,
                      return_attention, seed)


def _gat_dense(x, csr, edge_index_used, query_kernel, query_bias, query_activation, key_kernel, key_bias, key_activation,
               kernel, bias, activation, num_heads, split_value_heads, drop_rate, bf16, return_attention, seed):
    """gat() over a dense x on the device: csr.n_rows output rows, whose queries come from x[:csr.n_rows], over keys and
    values from all x.shape[0] rows (the same rows on a full graph; a SelfLoopBlock's num_dst and num_src)."""
    dev = x.device
    n_q, num_nodes = csr.n_rows, x.shape[0]
    if drop_rate > 0.0 or autograd.needs_grad(x, query_kernel, query_bias, key_kernel, key_bias, kernel, bias):
        if bf16:
            raise NotImplementedError("message_dtype=bfloat16 is for inference: no operand may require grad")
        if return_attention:
            raise NotImplementedError("return_attention is an inference-path extension")
        return _gat_training(x, csr, edge_index_used, query_kernel, query_bias, query_activation, key_kernel, key_bias,
                             key_activation, kernel, bias, activation, num_heads, split_value_heads, drop_rate,
                             _rng.resolve(seed, dev) if drop_rate > 0.0 else 0)

    q_act, q_left = ops.activation_code(query_activation)
    k_act, k_left = ops.activation_code(key_activation)
    wq = ops.as_device(query_kernel, torch.float32, device=dev)
    wk = ops.as_device(key_kernel, torch.float32, device=dev)
    wv = ops.as_device(kernel, torch.float32, device=dev)
    a_units = wk.shape[1]
    act_code, leftover = ops.activation_code(activation)
    bias = None if bias is None else ops.as_device(bias, torch.float32, device=dev)
    if not bf16 and not return_attention and k_act == ops.ACT_RELU and k_left is None and x.is_cuda and \
            _packed_keys_shape(wq, wk, wv, bias, num_heads, split_value_heads) and \
            os.environ.get("TFGK_GAT_KEYS", "packed") != "dense":
        # ReLU keys hold many exact zeros: K goes through a scratch buffer into a packed table whose slots hold V, a zero
        # mask and the non-zero keys, and the fused kernel gathers only those (same output bits as the dense route)
        Q = torch.empty((n_q, a_units), dtype=torch.float32, device=dev)
        K = torch.empty((num_nodes, a_units), dtype=torch.float32, device=dev)
        table, sizes = ops.packed_key_table(num_nodes, a_units, dev)
        _project_qkv(x, n_q, (wq, ops.as_device(query_bias, torch.float32, device=dev), q_act, Q),
                     [(wk, ops.as_device(key_bias, torch.float32, device=dev), k_act, K),
                      (wv, None, ops.ACT_NONE, table[:, :a_units])])
        if q_left is not None:
            Q = q_left(Q)
        ops.gat_pack_keys(K, table, sizes)
        del K
        h = ops.gat_fused_packed(csr, Q, table, sizes, num_heads, bias=bias, act=act_code)
        return leftover(h) if leftover is not None else h

    # Q, K and V come out of ONE launch that reads x once (tfgk_gemm_proj_f32).  K and V land in ONE [N, A + U]
    # buffer: the fused kernel then fetches a neighbour's key and value from the same DRAM burst
    Q = torch.empty((n_q, wq.shape[1]), dtype=torch.float32, device=dev)
    # bf16 messages: the projection rounds K | V in its epilogue; Q stays fp32
    kv = torch.empty((num_nodes, a_units + wv.shape[1]), dtype=torch.bfloat16 if bf16 else torch.float32, device=dev)
    K, V = kv[:, :a_units], kv[:, a_units:]
    # a key activation the projection cannot fuse is applied in fp32 before the keys are rounded
    K_f32 = torch.empty((num_nodes, a_units), dtype=torch.float32, device=dev) if bf16 and k_left is not None else K
    _project_qkv(x, n_q, (wq, ops.as_device(query_bias, torch.float32, device=dev), q_act, Q),
                 [(wk, ops.as_device(key_bias, torch.float32, device=dev), k_act, K_f32), (wv, None, ops.ACT_NONE, V)])
    if q_left is not None:
        Q = q_left(Q)
    if k_left is not None:
        if K_f32 is K:
            K.copy_(k_left(K))
        else:
            ops.round_bf16(k_left(K_f32), out=K)

    res = ops.gat_fused(csr, Q, K, V, num_heads, split_value_heads=split_value_heads, bias=bias, act=act_code,
                        return_attention=return_attention)
    h, att = res if return_attention else (res, None)
    if leftover is not None:
        h = leftover(h)
    if return_attention:
        return h, ops.permute(att, csr.perm, inverse=True)     # [E', H] in edge_index-with-self-loops order
    return h


def _block_input(x, block, message_dtype, return_attention, training, edge_drop_rate, weights):
    """The [num_src, F] device input of GAT over the SelfLoopBlock `block`; refuses what blocks do not support before any
    device work."""
    if ops.conv_message_dtype(message_dtype) is not None:
        raise NotImplementedError("GAT on a sampled block takes fp32 messages only (message_dtype=None)")
    rows = tuple(x.shape)[:1] if hasattr(x, "shape") and len(x.shape) == 2 else None
    if rows != (block.num_src,):
        raise ValueError("x has {} rows, the block has {} input rows".format(rows, block.num_src))
    if return_attention and ((training and edge_drop_rate > 0.0) or autograd.needs_grad(
            x.x if isinstance(x, SourceRows) else x, *weights)):
        raise NotImplementedError("return_attention is an inference-path extension")
    if isinstance(x, SourceRows):
        return x.gather()
    return ops.as_device(x, torch.float32, device=block.edge_index.device)


def _gat_fp8(x, edge_index, query_kernel, query_bias, query_activation, key_kernel, key_bias, key_activation, kernel, bias,
             activation, num_heads, split_value_heads, edge_drop_rate, training, cache, return_attention):
    """gat() with fp8 K | V: ONE projection launch writes the fp32 Q and the fp8 K | V (bytes and exponents) from one read
    of x, then tfgk_gat_fused_fp8 gathers 2A bytes per neighbour.  Every refusal comes before any device work."""
    if as_sparse_features(x) is not None:
        raise NotImplementedError("message_dtype=float8_e4m3fn takes a dense x")
    if training and edge_drop_rate > 0.0:
        raise NotImplementedError("message_dtype=float8_e4m3fn is for inference: attention dropout is not applied in fp8")
    if return_attention:
        raise NotImplementedError("message_dtype=float8_e4m3fn does not return attention coefficients; use bfloat16 or "
                                  "float32")
    if autograd.needs_grad(x, query_kernel, query_bias, key_kernel, key_bias, kernel, bias):
        raise NotImplementedError("message_dtype=float8_e4m3fn is for inference: no operand may require grad")
    H = int(num_heads)
    A = key_kernel.shape[1]
    dqk = A // H if H >= 1 and A % H == 0 else 0
    if not (split_value_heads and query_kernel.shape[1] == A and kernel.shape[1] == A and A <= 128 and 1 <= H <= 32 and
            not H & (H - 1) and dqk % 4 == 0 and dqk >= 4 and not (dqk // 4) & (dqk // 4 - 1)):
        raise NotImplementedError(
            "message_dtype=float8_e4m3fn takes concatenated heads with units == attention_units = num_heads * d <= 128, "
            "num_heads and d / 4 powers of two (got {} heads, {} attention units, {} units); use bfloat16 or float32".format(
                H, A, kernel.shape[1]))
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = ops.as_device(x, torch.float32, device=dev)
    num_nodes = x.shape[0]
    csr, _ = _structure.csr_for_edge_index(edge_index, num_nodes, add_self_loop=True, cache=cache)
    q_act, q_left = ops.activation_code(query_activation)
    k_act, k_left = ops.activation_code(key_activation)
    f32 = lambda t: None if t is None else ops.as_device(t, torch.float32, device=dev)     # noqa: E731
    Q = torch.empty((num_nodes, A), dtype=torch.float32, device=dev)
    kv = ops.fp8_table(num_nodes, 2 * A, dev, groups=2)
    K, V = kv.block(0, A, group=0), kv.block(A, 2 * A, group=1)
    # a key activation the projection cannot fuse is applied in fp32 before the keys are quantised
    K_f32 = torch.empty((num_nodes, A), dtype=torch.float32, device=dev) if k_left is not None else K
    ops.gemm_proj(x, [(f32(query_kernel), f32(query_bias), q_act, Q), (f32(key_kernel), f32(key_bias), k_act, K_f32),
                      (f32(kernel), None, ops.ACT_NONE, V)])
    if q_left is not None:
        Q = q_left(Q)
    if k_left is not None:
        ops.quantize_fp8(k_left(K_f32), out=K)
    act_code, leftover = ops.activation_code(activation)
    h = ops.gat_fused(csr, Q, kv, None, H, bias=f32(bias), act=act_code)
    return leftover(h) if leftover is not None else h


def _packed_keys_shape(wq, wk, wv, bias, num_heads, split_value_heads):
    """The shapes tfgk_gat_fused_packed_f32 takes: the TMA ring's (heads concatenated, Q, K and V of one width A = H * dqk
    <= 128, H a power of two <= 32, dqk / 4 a power of two) with a 16-byte aligned bias."""
    H, A = int(num_heads), wk.shape[1]
    if not split_value_heads or wq.shape[1] != A or wv.shape[1] != A or A > 128 or H < 1 or H > 32 or H & (H - 1) or A % H:
        return False
    d4 = (A // H) // 4
    return (A // H) % 4 == 0 and d4 >= 1 and d4 & (d4 - 1) == 0 and (bias is None or bias.data_ptr() % 16 == 0)


def _gat_training(x, csr, edge_index_used, query_kernel, query_bias, query_activation, key_kernel, key_bias,
                  key_activation, kernel, bias, activation, num_heads, split_value_heads, drop_rate, seed):
    """The same layer behind autograd Functions (demo/demo_gat.py trains through tf.GradientTape): dense projections
    with dX/dW/db GEMMs (sparse features: the aggregation kernel over x's pattern and its transpose), then GatAttention."""
    sparse_x = as_sparse_features(x)
    dev = csr.col.device

    def dense(x, w, b, act):
        code, left = ops.activation_code(act)
        w = ops.as_device(w, torch.float32, device=dev)
        b = None if b is None else ops.as_device(b, torch.float32, device=dev)
        y = autograd.Dense.apply(x, w, b, code) if sparse_x is None else autograd.SparseMatmul.apply(w, b, sparse_x, code)
        return left(y) if left is not None else y

    # a block's queries are its output rows, the first csr.n_rows input rows
    x_q = x if sparse_x is not None or x.shape[0] == csr.n_rows else x[:csr.n_rows]
    Q = dense(x_q, query_kernel, query_bias, query_activation)
    K = dense(x, key_kernel, key_bias, key_activation)
    V = dense(x, kernel, None, None)
    act_code, leftover = ops.activation_code(activation)
    bias = None if bias is None else ops.as_device(bias, torch.float32, device=dev)
    h = autograd.GatAttention.apply(Q, K, V, bias, csr, edge_index_used, int(num_heads), bool(split_value_heads),
                                    act_code, drop_rate, seed)
    return leftover(h) if leftover is not None else h
