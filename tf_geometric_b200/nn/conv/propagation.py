# coding=utf-8
"""The remaining `norm(A) @ H` convolutions of tf_geometric (SURVEY.md section 8f-1): sgc, ssgc, tagcn, gin, le_conv.
Each one is the K1 kernel (tfgk_spmm_f32) in a loop with the per-layer arithmetic fused into its epilogue where the
reference's rounding order allows it; signatures follow tf_geometric/nn/conv/{sgc,ssgc,tagcn,gin,le_conv}.py."""
import torch

from ... import ops, _structure, autograd, _ffi
from ...sparse import SparseMatrix
from . import _bf16
from .gat import project
from .gcn import gcn_norm_adj


def _f32(t, dev):
    return None if t is None else ops.as_device(t, torch.float32, device=dev)


def sgc(x, edge_index, edge_weight, k, kernel, bias=None, activation=None, renorm=True, improved=False, cache=None,
        message_dtype=None):
    """Simple Graph Convolution: act(norm(A)^k (x W) + b)   (reference sgc.py:10-61).  message_dtype=torch.bfloat16:
    inference with x W and the hops 1 .. k-1 stored in bf16 (an extension of the reference API)."""
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        _bf16.refuse_unsupported(x, (kernel, bias, edge_weight))
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = _f32(x, dev)
    n = x.shape[0]
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [n, n]), renorm=renorm, improved=improved, cache=cache)
    act_code, leftover = ops.activation_code(activation)
    b = _f32(bias, dev)
    with_grad = autograd.needs_grad(x, kernel, bias, normed.value)     # training: the same kernels behind autograd
    if bf16 and k > 0:
        kernel = _f32(kernel, dev)
        h = ops.bf16_table(n, kernel.shape[1], dev)
        project(x, [(kernel, None, ops.ACT_NONE, h)])                  # x W rounded by the projection's epilogue
        bufs = [ops.bf16_table(n, kernel.shape[1], dev) for _ in range(min(k - 1, 2))]
        for i in range(k - 1):
            h = normed.matmul(h, out_bf16=bufs[i % 2])                   # intermediate hops: bf16 only
        h = normed.matmul(h, bias=b, act=act_code)
        return leftover(h) if leftover is not None else h
    h = autograd.dense(x, _f32(kernel, dev)) if with_grad else ops.gemm(x, _f32(kernel, dev))
    for i in range(k):
        last = i == k - 1
        if with_grad:
            h = autograd.propagate(normed, h, b if last else None, act_code if last else ops.ACT_NONE)
        else:
            h = normed.matmul(h, bias=b if last else None, act=act_code if last else ops.ACT_NONE)
    if k == 0:
        if b is not None:
            h = h + b
        if act_code == ops.ACT_RELU:
            h = torch.relu(h)
    if leftover is not None:
        h = leftover(h)
    return h


def ssgc(x, edge_index, edge_weight, kernels=None, biases=None, k=10, alpha=0.1, dense_activation=ops.relu,
         activation=None, dense_drop_rate=0.0, last_dense_drop_rate=0.0, edge_drop_rate=0.0, cache=None, training=False,
         message_dtype=None):
    """Simple Spectral Graph Convolution: alpha * h + (1 - alpha)/k * sum_{i=1..k} norm(A)^i h   (reference ssgc.py:11-99).
    message_dtype=torch.bfloat16: inference with every gathered hop stored in bf16; the hops that are summed stay fp32 (an
    extension of the reference API)."""
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        drop = training and max(dense_drop_rate, last_dense_drop_rate, edge_drop_rate) > 0.0
        _bf16.refuse_unsupported(x, [edge_weight] + list(kernels or []) + list(biases or []), dropout=drop)
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    h = _f32(x, dev)
    n = h.shape[0]
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [n, n]), cache=cache)
    normed = normed.dropout(edge_drop_rate, training=training)                          # ssgc.py:60-61
    with_grad = autograd.needs_grad(h, normed.value, *[t for t in list(kernels or []) + list(biases or []) if t is not None])
    if kernels is not None:
        num_dense = len(kernels)
        for i, (kern, b) in enumerate(zip(kernels, biases)):
            act = dense_activation if i < num_dense - 1 else None
            if with_grad:
                h = autograd.dense(h, _f32(kern, dev), _f32(b, dev), act)
            else:
                act_code, leftover = ops.activation_code(act)
                h = ops.gemm(h, _f32(kern, dev), bias=_f32(b, dev), act=act_code)
                if leftover is not None:
                    h = leftover(h)
            h = autograd.dropout(h, dense_drop_rate if i < num_dense - 1 else last_dense_drop_rate, training)  # :84-88
    output = h * alpha                                    # elementwise glue in the reference's rounding order (:91-94)
    if bf16 and k > 0:
        # each hop in fp32 (it is summed) and, from the same launch, in bf16 for the next gather
        cur = ops.round_bf16_table(h)
        bufs = [ops.bf16_table(n, h.shape[1], dev) for _ in range(min(k - 1, 2))]
        for i in range(k):
            nxt = bufs[i % 2] if i < k - 1 else None
            h = normed.matmul(cur, out=torch.empty((n, h.shape[1]), dtype=torch.float32, device=dev), out_bf16=nxt)
            output = output + (1 - alpha) * h / k
            cur = nxt
        return activation(output) if activation is not None else output
    for _ in range(k):
        h = autograd.propagate(normed, h) if with_grad else normed.matmul(h)
        output = output + (1 - alpha) * h / k
    if activation is not None:
        output = activation(output)
    return output


def tagcn(x, edge_index, edge_weight, k, kernel, bias=None, activation=None, renorm=False, improved=False, cache=None,
          message_dtype=None):
    """Topology Adaptive GCN: act([x, Ax, ..., A^k x] W + b); the hops are written straight into the column blocks of
    the concatenated operand (reference tagcn.py:10-51).  message_dtype=torch.bfloat16: inference with x and the hops
    1 .. k-1 gathered from bf16 copies; the concatenated GEMM operand stays fp32 (an extension of the reference API)."""
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        _bf16.refuse_unsupported(x, (kernel, bias, edge_weight))
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = _f32(x, dev)
    n, f = x.shape
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [n, n]), renorm=renorm, improved=improved, cache=cache)
    if autograd.needs_grad(x, kernel, bias, normed.value):
        terms = [x]
        for _ in range(k):
            terms.append(autograd.propagate(normed, terms[-1]))
        return autograd.dense(torch.cat(terms, dim=1), _f32(kernel, dev), _f32(bias, dev), activation)
    hops = torch.empty((n, f * (k + 1)), dtype=torch.float32, device=dev)
    hops[:, :f].copy_(x)
    if bf16 and k > 0:
        # each hop fp32 into its column block and, from the same launch, bf16 for the next gather
        cur = ops.round_bf16_table(x)
        bufs = [ops.bf16_table(n, f, dev) for _ in range(min(k - 1, 2))]
        for i in range(k):
            nxt = bufs[i % 2] if i < k - 1 else None
            normed.matmul(cur, out=hops[:, (i + 1) * f:(i + 2) * f], out_bf16=nxt)
            cur = nxt
    for i in range(0 if bf16 else k):
        normed.matmul(hops[:, i * f:(i + 1) * f], out=hops[:, (i + 1) * f:(i + 2) * f])
    act_code, leftover = ops.activation_code(activation)
    out = ops.gemm(hops, _f32(kernel, dev), bias=_f32(bias, dev), act=act_code)
    return leftover(out) if leftover is not None else out


def gin_updater(x, reduced_neighbor_msg, eps):
    return x * (1.0 + eps) + reduced_neighbor_msg


def gin(x, edge_index, mlp_model, eps=0.0, training=None, message_dtype=None):
    """Graph Isomorphism Network: mlp((1 + eps) x + sum_{j in N(i)} x_j); the update is the aggregation kernel's axpby
    epilogue (reference gin.py:11-38).  message_dtype=torch.bfloat16: inference with the gathered x stored in bf16; the
    (1 + eps) x addend reads the fp32 x (an extension of the reference API)."""
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        params = list(mlp_model.parameters()) if hasattr(mlp_model, "parameters") else []
        _bf16.refuse_unsupported(x, [eps] + params)
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = _f32(x, dev)
    if autograd.needs_grad(x, eps):                        # trainable eps (layers/conv/gin.py train_eps) or upstream layers
        h = gin_updater(x, autograd.NeighborAggregate.apply(x, edge_index, None, "sum", x.shape[0]), eps)
    else:
        csr, _ = _structure.csr_for_edge_index(edge_index, x.shape[0])
        eps_value = float(eps.detach().item()) if torch.is_tensor(eps) else float(eps)
        h = ops.spmm(csr, None, ops.round_bf16_table(x) if bf16 else x, reduce="sum", alpha=1.0, addend=x,
                     beta=1.0 + eps_value)
    try:
        return mlp_model(h, training=training)
    except TypeError:
        return mlp_model(h)


def le_conv(x, edge_index, edge_weight, self_kernel, self_bias, aggr_self_kernel, aggr_self_bias,
            aggr_neighbor_kernel, aggr_neighbor_bias, activation=None, message_dtype=None):
    """LEConv (ASAP): act(x Ws + sum_j w_ij (x_j Wa - x_j Wn)).  Note the reference gathers BOTH aggregation terms by the
    neighbour index `col` (le_conv.py:40-43), so the per-edge difference is a per-node difference gathered once.
    message_dtype=torch.bfloat16: inference with that fp32 difference rounded once to bf16; the self term stays fp32 (an
    extension of the reference API)."""
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        _bf16.refuse_unsupported(x, (self_kernel, self_bias, aggr_self_kernel, aggr_self_bias, aggr_neighbor_kernel,
                                     aggr_neighbor_bias, edge_weight))
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = _f32(x, dev)
    n = x.shape[0]
    if autograd.needs_grad(x, self_kernel, self_bias, aggr_self_kernel, aggr_self_bias, aggr_neighbor_kernel,
                           aggr_neighbor_bias, edge_weight):
        self_h = autograd.dense(x, _f32(self_kernel, dev), _f32(self_bias, dev))
        diff = autograd.dense(x, _f32(aggr_self_kernel, dev), _f32(aggr_self_bias, dev)) \
            - autograd.dense(x, _f32(aggr_neighbor_kernel, dev), _f32(aggr_neighbor_bias, dev))
        h = autograd.NeighborAggregate.apply(diff, edge_index, _f32(edge_weight, dev), "sum", n) + self_h
        return activation(h) if activation is not None else h
    csr, _ = _structure.csr_for_edge_index(edge_index, n)
    w_csr = None
    if edge_weight is not None:
        w_csr = _structure.weights_in_csr_order(_f32(edge_weight, dev), csr)
    self_h = ops.gemm(x, _f32(self_kernel, dev), bias=_f32(self_bias, dev))
    diff = ops.gemm(x, _f32(aggr_self_kernel, dev), bias=_f32(aggr_self_bias, dev)) \
        - ops.gemm(x, _f32(aggr_neighbor_kernel, dev), bias=_f32(aggr_neighbor_bias, dev))
    act_code, leftover = ops.activation_code(activation)
    h = ops.spmm(csr, w_csr, ops.round_bf16_table(diff) if bf16 else diff, reduce="sum", alpha=1.0, addend=self_h, beta=1.0,
                 act=act_code)
    return leftover(h) if leftover is not None else h


# ---- ChebyNet (reference nn/conv/chebynet.py, utils/graph_utils.py:554-604,884-911) -------------------------------------

CACHE_KEY_CHEBYNET_NORMED_EDGE_TEMPLATE = "chebynet_normed_edge_{}"


def get_laplacian(edge_index, num_nodes, edge_weight, normalization_type, fill_weight=1.0):
    """The reference's `get_laplacian`, literally: for 'sym' it returns D^-1/2 A D^-1/2 with `fill_weight` self loops appended
    (positive off-diagonals - not I - D^-1/2 A D^-1/2), for 'rw' D^-1 A + loops, for None (deg[row] - w) with loops."""
    if normalization_type is not None:
        assert normalization_type in [None, 'sym', 'rw']
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    w = _f32(edge_weight, dev)
    adj = SparseMatrix(edge_index, w, [num_nodes, num_nodes])
    deg = adj.segment_sum(axis=-1)
    row, col = edge_index[0].contiguous(), edge_index[1].contiguous()
    if normalization_type is None:
        looped = adj.add_diag(fill_weight)
        deg_clean = torch.where(torch.isinf(deg) | torch.isnan(deg), torch.zeros_like(deg), deg)
        return looped.index, deg_clean[looped.index[0].long()] - looped.value
    if normalization_type == 'sym':
        dis = ops.deg_inv(deg, ops.POW_INV_SQRT)
        normed = ops.scale_edges(row, col, w, dl=dis, dr=dis)
    else:
        normed = ops.scale_edges(row, None, w, dl=ops.deg_inv(deg, ops.POW_INV))
    looped = SparseMatrix(edge_index, normed, [num_nodes, num_nodes]).add_diag(fill_weight)
    return looped.index, looped.value


def laplacian_max_eigenvalue(edge_index, num_nodes, edge_weight, normalization_type='sym', is_undirected=True):
    """LaplacianMaxEigenvalue(...)(normalization_type): host-side scipy eigs/eigsh, as in the reference (:884-911, including
    its quirk of building the operator from the edges WITH self loops while the weights had them removed)."""
    _ffi.refuse_capture("the dynamic lambda_max of ChebyNet", "scipy computes it on the host")
    import numpy as np
    import scipy.sparse
    from scipy.sparse.linalg import eigs, eigsh
    from ...utils.graph_utils import remove_self_loop_edge
    ei = edge_index.detach().cpu().numpy() if torch.is_tensor(edge_index) else np.asarray(edge_index)
    w = (edge_weight.detach().cpu().numpy() if torch.is_tensor(edge_weight) else
         (np.ones([ei.shape[1]], np.float32) if edge_weight is None else np.asarray(edge_weight)))
    _, w_nl = remove_self_loop_edge(ei, w)
    lap_index, lap_w = get_laplacian(ei, num_nodes, w_nl, normalization_type)
    li, lw = lap_index.cpu().numpy(), lap_w.cpu().numpy()
    L = scipy.sparse.coo_matrix((lw, (li[0], li[1])), shape=(num_nodes, num_nodes))
    fn = eigsh if (is_undirected and normalization_type) else eigs
    return float(np.real(fn(L, k=1, which='LM', return_eigenvectors=False))[0])


def chebynet_norm_edge(edge_index, num_nodes, edge_weight=None, normalization_type="sym", use_dynamic_lambda_max=False,
                       cache=None):
    """reference chebynet.py:17-43."""
    if cache is not None:
        cache_key = CACHE_KEY_CHEBYNET_NORMED_EDGE_TEMPLATE.format(normalization_type)
        if cache.get(cache_key, None) is not None:
            return cache[cache_key]
    from ...utils.graph_utils import remove_self_loop_edge
    edge_index = ops.as_device(edge_index, torch.int32)
    edge_weight = _f32(edge_weight, edge_index.device)
    ei_nl, w_nl = remove_self_loop_edge(edge_index, edge_weight)
    assert w_nl is not None
    upd_index, upd_w = get_laplacian(ei_nl, num_nodes, w_nl, normalization_type)
    lambda_max = laplacian_max_eigenvalue(ei_nl, num_nodes, w_nl, normalization_type) if use_dynamic_lambda_max else 2.0
    scaled = (2.0 * upd_w) / lambda_max
    if cache is not None:
        cache[cache_key] = upd_index, scaled
    return upd_index, scaled


def chebynet(x, edge_index, edge_weight, k, kernels, bias=None, activation=None, normalization_type="sym",
             use_dynamic_lambda_max=False, cache=None, message_dtype=None):
    """sum_i T_i(L~) x K_i with T_0 = x, T_1 = L~ x, T_i = 2 L~ T_{i-1} - T_{i-2}: the recurrence is the aggregation kernel's
    axpby epilogue, the projections accumulate into `out` through the GEMM's beta (reference chebynet.py:63-137).
    message_dtype=torch.bfloat16: inference with T_0 .. T_{k-2} gathered from bf16 copies; every T_i stays fp32 as GEMM
    operand and recurrence addend (an extension of the reference API)."""
    bf16 = _bf16.enabled(message_dtype)
    if bf16:
        _bf16.refuse_unsupported(x, [bias, edge_weight] + list(kernels))
    edge_index = ops.as_device(edge_index, torch.int32)
    dev = edge_index.device
    x = _f32(x, dev)
    n = x.shape[0]
    if edge_weight is None:
        edge_weight = torch.ones([edge_index.shape[1]], dtype=torch.float32, device=dev)
    n_index, n_weight = chebynet_norm_edge(edge_index, n, edge_weight, normalization_type,
                                           use_dynamic_lambda_max=use_dynamic_lambda_max, cache=cache)
    adj = SparseMatrix(n_index, n_weight, [n, n]) if cache is None else cache.setdefault(
        "tfgk_chebynet_adj_{}".format(normalization_type), SparseMatrix(n_index, n_weight, [n, n]))
    if autograd.needs_grad(x, bias, *kernels):
        t0 = x
        out = autograd.dense(t0, _f32(kernels[0], dev))
        if k > 1:
            t1 = autograd.propagate(adj, x)
            out = out + autograd.dense(t1, _f32(kernels[1], dev))
        for i in range(2, k):
            t2 = autograd.propagate(adj, t1) * 2.0 - t0
            out = out + autograd.dense(t2, _f32(kernels[i], dev))
            t0, t1 = t1, t2
        if bias is not None:
            out = out + _f32(bias, dev)
        return activation(out) if activation is not None else out
    t0 = x
    out = ops.gemm(t0, _f32(kernels[0], dev))
    # bf16: b1 is the bf16 copy of T1 for the next gather, written by the launch that writes T1 (none for T_{k-1})
    b1 = None
    if k > 1:
        if bf16:
            b1 = ops.bf16_table(n, x.shape[1], dev) if k > 2 else None
            t1 = adj.matmul(ops.round_bf16_table(x), out=torch.empty_like(x), out_bf16=b1)
        else:
            t1 = adj.matmul(x)
        ops.gemm(t1, _f32(kernels[1], dev), beta=1.0, out=out)
    if k > 2:
        for i in range(2, k):
            if bf16:
                b2 = ops.bf16_table(n, x.shape[1], dev) if i < k - 1 else None
                t2 = adj.matmul(b1, alpha=2.0, addend=t0, beta=-1.0, out=torch.empty_like(x), out_bf16=b2)
                b1 = b2
            else:
                t2 = adj.matmul(t1, alpha=2.0, addend=t0, beta=-1.0)          # (L~ @ T1) * 2.0 - T0
            ops.gemm(t2, _f32(kernels[i], dev), beta=1.0, out=out)
            t0, t1 = t1, t2
    if bias is not None:
        out = out + _f32(bias, dev)
    if activation is not None:
        out = activation(out)
    return out
