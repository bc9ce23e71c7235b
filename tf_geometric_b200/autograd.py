# coding=utf-8
"""Backward passes (SURVEY.md 8a10: mean/sum_graph_sage forward + backward; 8(f)4: GCN and GAT training); the reference
gets them from TensorFlow autodiff (demo/demo_graph_sage.py:100-106, demo/demo_gcn.py:60-75, demo/demo_gat.py).

    d(unsorted_segment_mean(x[col] * w, row)) / dx  =  scatter-add by col of  (w_e / max(cnt[row_e], 1)) * g[row_e]

i.e. the SAME gather - edge-apply - segment-reduce kernel (tfgk_spmm_f32) run on the TRANSPOSED structure (a CSC = the
destination-sorted CSR of the reversed edges) with rescaled weights; it is built once per edge list and memoised next
to the forward CSR.  Dense layers: dX = dY W^T and dW = X^T dY are tfgk_gemm_f32 with transposes (deterministic split-K
over the node dimension), db = 1^T dY through the same kernel.
"""
import weakref

import numpy as np
import torch

from . import ops, _structure


def _relu_grad(g, y):
    """dL/d(pre-activation) of y = relu(.): g where y > 0, else 0 - one elementwise pass (aten's relu backward) instead of
    compare + cast + multiply."""
    return torch.ops.aten.threshold_backward(g, y, 0.0)


def _transposed_structure(edge_index, num_nodes, edge_weight, mean, csr):
    """(csr_t, w_t): CSR of the reversed edges and w_e / max(cnt[row_e], 1) (or w_e for sum) in its order.
    The structure is memoised per edge list; the weights per (weight tensor, structure) with the weight tensor held by
    weak reference and checked by version (an id() recycled by a new tensor can never alias an old entry)."""
    tag = ("csc", int(num_nodes))
    csr_t = _structure._lookup(edge_index, tag)
    row, col = edge_index[0].contiguous(), edge_index[1].contiguous()
    if csr_t is None:
        csr_t = _structure._store(edge_index, tag, ops.csr_build(col, row, num_nodes, num_nodes))
    owner = edge_weight if edge_weight is not None else edge_index
    wtag = ("csc_w", bool(mean), edge_weight is None, id(csr_t), id(csr))
    hit = _structure._lookup(owner, wtag)
    if hit is not None and hit[0]() is csr_t and hit[1]() is csr:
        return csr_t, hit[2]
    w = edge_weight if edge_weight is not None else torch.ones((edge_index.shape[1],), dtype=torch.float32,
                                                               device=edge_index.device)
    if mean:
        cnt = (csr.rowptr[1:] - csr.rowptr[:-1]).clamp(min=1).to(torch.float32)
        w = ops.scale_edges(row, None, w, dl=torch.reciprocal(cnt))
    w_t = ops.permute(w.contiguous(), csr_t.perm)
    _structure._store(owner, wtag, (weakref.ref(csr_t), weakref.ref(csr), w_t))
    return csr_t, w_t


class NeighborAggregate(torch.autograd.Function):
    """agg = REDUCE_{e: row_e = r} w_e x[col_e]  (sum | mean), differentiable w.r.t. x and the edge weights.
    d w_e = <dagg[row_e], x[col_e]> (/ max(cnt[row_e], 1) for mean) is K7 over the forward CSR, written in edge order."""

    @staticmethod
    def forward(ctx, x, edge_index, edge_weight, reduce, num_nodes):
        csr, _ = _structure.csr_for_edge_index(edge_index, num_nodes)
        w_csr = None if edge_weight is None else _structure.weights_in_csr_order(edge_weight, csr)
        ctx.saved = (edge_index, edge_weight, reduce, num_nodes, csr)
        ctx.save_for_backward(x.detach() if edge_weight is not None and edge_weight.requires_grad else None)
        return ops.spmm(csr, w_csr, x.detach(), reduce=reduce)

    @staticmethod
    def backward(ctx, grad_out):
        edge_index, edge_weight, reduce, num_nodes, csr = ctx.saved
        (x,) = ctx.saved_tensors
        g = grad_out.contiguous()
        grad_x = grad_w = None
        if ctx.needs_input_grad[0]:
            csr_t, w_t = _transposed_structure(edge_index, num_nodes, edge_weight, reduce == "mean", csr)
            grad_x = ops.spmm(csr_t, w_t, g, reduce="sum")
        if ctx.needs_input_grad[2]:
            scale = None
            if reduce == "mean":
                scale = torch.reciprocal((csr.rowptr[1:] - csr.rowptr[:-1]).clamp(min=1).to(torch.float32))
            grad_w = ops.sddmm_csr(csr, g, x, row_scale=scale)
        return grad_x, None, grad_w, None, None


class NeighborMax(torch.autograd.Function):
    """agg = MAX_{e: row_e = r} w_e x[col_e] (-FLT_MAX for a node without in-edges), differentiable w.r.t. x; edge_weight
    (None = 1) is a constant.  Forward: K11a, which also counts the ties of every output entry; out, the counts and x are
    kept ([N, D] each, no per-edge tensor).  Backward: K11b over the transposed CSR (the one NeighborAggregate uses),
        dx[c] = sum_{e: col_e = c} ((g[row_e] / max(cnt[row_e], 1)) * (w_e x[c] == agg[row_e])) * w_e
    in edge order, without atomics: the gradient is shared equally among ties, as SegmentReduce's max backward does, and
    the bits are those of TakeRows + SegmentReduce("max") over the gathered messages."""

    @staticmethod
    def forward(ctx, x, edge_index, edge_weight, num_nodes):
        csr, _ = _structure.csr_for_edge_index(edge_index, num_nodes)
        w_csr = None if edge_weight is None else _structure.weights_in_csr_order(edge_weight.detach(), csr)
        xd = x.detach()
        out, cnt = ops.spmm_max(csr, w_csr, xd)
        ctx.saved = (edge_index, None if edge_weight is None else edge_weight.detach(), int(num_nodes))
        ctx.save_for_backward(xd, out, cnt)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        edge_index, edge_weight, num_nodes = ctx.saved
        x, out, cnt = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None, None, None
        csr_t, w_t = _max_transposed(edge_index, num_nodes, edge_weight)
        return ops.spmm_max_bwd(csr_t, w_t, x, out, cnt, grad_out.contiguous()), None, None, None


def _is_device(t):
    return torch.is_tensor(t) and t.is_cuda


def max_aggregate(x, edge_index, num_nodes):
    """Differentiable MAX_{e: row_e = r} x[col_e]: NeighborMax for device tensors (the operands of every public entry
    point, which as_device puts on the GPU).  Host tensors take the composition TakeRows + SegmentReduce("max") that
    NeighborMax replaces bit for bit, whose blocks any host stand-in of the kernel layer provides."""
    if _is_device(x):
        return NeighborMax.apply(x, edge_index, None, num_nodes)
    messages = TakeRows.apply(x, edge_index[1].contiguous())
    return SegmentReduce.apply(messages, edge_index[0].contiguous(), num_nodes, "max")


def _max_transposed(edge_index, num_nodes, edge_weight):
    """(csr_t, w_t) for NeighborMax's backward: the CSR of the reversed edges (its col = destination rows, stable by
    source, memoised under the tag _transposed_structure uses) and the weights in its order (None when unweighted)."""
    tag = ("csc", int(num_nodes))
    csr_t = _structure._lookup(edge_index, tag)
    if csr_t is None:
        row, col = edge_index[0].contiguous(), edge_index[1].contiguous()
        csr_t = _structure._store(edge_index, tag, ops.csr_build(col, row, num_nodes, num_nodes))
    if edge_weight is None:
        return csr_t, None
    return csr_t, _structure.weights_in_csr_order(edge_weight, csr_t)


class Dense(torch.autograd.Function):
    """y = act(x @ W + b) with act in {None, relu}; dX, dW, db through tfgk_gemm_f32."""

    @staticmethod
    def forward(ctx, x, weight, bias, act_code):
        y = ops.gemm(x.detach(), weight.detach(), bias=None if bias is None else bias.detach(), act=act_code)
        ctx.save_for_backward(x, weight, y if act_code == ops.ACT_RELU else None)
        ctx.has_bias = bias is not None
        ctx.act_code = act_code
        return y

    @staticmethod
    def backward(ctx, grad_y):
        x, weight, y = ctx.saved_tensors
        g = grad_y.contiguous()
        if ctx.act_code == ops.ACT_RELU:
            g = _relu_grad(g, y)                      # elementwise mask (torch: plumbing, not a hot op)
        grad_x = grad_w = grad_b = None
        if ctx.needs_input_grad[0]:
            grad_x = ops.gemm(g, weight.detach(), trans_b=True)
        if ctx.needs_input_grad[1]:
            grad_w = ops.gemm(x.detach(), g, trans_a=True)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            grad_b = ops.colsum(g)
        return grad_x, grad_w, grad_b, None


class SparseMatmul(torch.autograd.Function):
    """y = act(A @ h + b) for a cached SparseMatrix A (gcn.py:280-288), differentiable w.r.t. h, b and, when they are
    passed as the trailing input, the values of A (COO order; tf_sparse products are differentiable in their values).
    dz = dy * (y > 0) for relu; dh = A^T dz runs the same kernel on the transposed structure of A (built once per
    matrix, values permuted into it again after an in-place update, SparseMatrix.value_csc); d value_e =
    <dz[row_e], h[col_e]> is K7 over A's CSR, written in COO order."""

    @staticmethod
    def forward(ctx, h, bias, adj, act_code, value=None):
        y = ops.spmm(adj.csr, adj.value_csr, h.detach(), reduce="sum", bias=None if bias is None else bias.detach(),
                     act=act_code)
        ctx.adj = adj
        ctx.act_code = act_code
        ctx.has_bias = bias is not None
        ctx.save_for_backward(y if act_code == ops.ACT_RELU else None,
                              h.detach() if value is not None and value.requires_grad else None)
        return y

    @staticmethod
    def backward(ctx, grad_y):
        y, h = ctx.saved_tensors
        g = grad_y.contiguous()
        if ctx.act_code == ops.ACT_RELU:
            g = _relu_grad(g, y)
        adj = ctx.adj
        grad_h = grad_b = grad_value = None
        if ctx.needs_input_grad[0]:
            grad_h = ops.spmm(adj._transposed_csr(), adj.value_csc, g, reduce="sum")
        if ctx.has_bias and ctx.needs_input_grad[1]:
            grad_b = ops.colsum(g)
        if len(ctx.needs_input_grad) > 4 and ctx.needs_input_grad[4]:        # four-argument calls pass no values
            grad_value = ops.sddmm_csr(adj.csr, g, h)
        return grad_h, grad_b, None, None, grad_value


def _gather(values, index):
    """values[index] for a float32 per-node vector and an int32 index vector (tfgk_permute_f32)."""
    return ops.permute(values.contiguous(), index)


def _segment_sums(csr, per_edge):
    """Sum of a per-edge float32 vector (the order of the edge list `csr` was built from) over every CSR row:
    tfgk_spmm_f32 with D = 1 gathering through csr.perm; deterministic."""
    return ops.spmm(csr, None, per_edge.contiguous().unsqueeze(1), reduce="sum", col=csr.perm).squeeze(1)


class GcnNormValues(torch.autograd.Function):
    """The values of gcn_norm_adj(A) (nn/conv/gcn.py) as a function of A's values w, differentiable.

    The forward receives the values the normalisation kernels already produced (the caller runs exactly the kernels of the
    non-differentiable path, so requires_grad never changes a bit) and returns them.  `aux` holds what the backward needs:
    the matrix A' whose row / column sums are the degrees (A, plus the self loops appended before normalising), its
    normalised values v, and the degree factors.  With g = dL/dv and R_i = sum_{row_e = i} g_e v_e, C_j = sum_{col_e = j}
    g_e v_e over the entries of A' (two deterministic D = 1 segment sums, over A's CSR and CSC):
        both, sym   : v = a_r w a_c, a = deg^-1/2         dw = g a_r a_c - 1/2 a_r^2 (R_r + C_r)
        both, !sym  : v = a_r w b_c, b = coldeg^-1/2      dw = g a_r b_c - 1/2 a_r^2 R_r - 1/2 b_c^2 C_c
        left        : v = p_r w, p = 1/deg                dw = (g - R_r) p_r
        right       : v = w q_c, q = 1/rowdeg             dw = g q_c - q_r C_r
    A degree <= 0 has its factor forced to 0 (_remove_inf_and_nan), and so has its derivative.  Self loops (appended
    before or after normalising) carry constant fill weights: they enter the degrees and get no gradient.  Entries past
    A' (loops appended after normalising) are constants."""

    @staticmethod
    def forward(ctx, w, normed_value, aux):
        ctx.aux = aux
        ctx.n_w = w.shape[0]
        return normed_value

    @staticmethod
    def backward(ctx, grad_value):
        kind, adj, v, f_row, f_col = ctx.aux
        n_prime = v.shape[0]
        g = grad_value.contiguous()[:n_prime].contiguous()
        row, col = adj.index[0].contiguous(), adj.index[1].contiguous()
        gv = g * v
        if kind == "left":
            R = _segment_sums(adj.csr, gv)
            dw = (g - _gather(R, row)) * _gather(f_row, row)
        elif kind == "right":
            C = _segment_sums(adj._transposed_csr(), gv)
            if C.shape[0] < f_row.shape[0]:               # q is indexed by row ids, C by column ids
                C = torch.cat([C, C.new_zeros(f_row.shape[0] - C.shape[0])])
            dw = g * _gather(f_row, col) - _gather(f_row * C[:f_row.shape[0]], row)
        else:
            R = _segment_sums(adj.csr, gv)
            C = _segment_sums(adj._transposed_csr(), gv)
            a_r = _gather(f_row, row)
            if kind == "both_sym":
                dw = g * a_r * _gather(f_row, col) - _gather(0.5 * f_row * f_row * (R + C), row)
            else:
                dw = g * a_r * _gather(f_col, col) - _gather(0.5 * f_row * f_row * R, row) \
                    - _gather(0.5 * f_col * f_col * C, col)
        return dw[:ctx.n_w], None, None


def _transposed_of_csr(csr, edge_index_used):
    """(csr_t, emap) for a forward CSR: csr_t has one row per SOURCE node, its columns are the destination rows, and
    emap[p] is the forward-CSR position of transposed slot p (per-edge tables such as the attention coefficients are
    stored in forward-CSR order).  Built once per CSR object; a SelfLoopBlock (edge_index_used) keeps its own, built
    without re-checking its ids."""
    if isinstance(edge_index_used, ops.SampledInput):
        csr_t = edge_index_used.transposed()
        return csr_t, csr_t.perm
    hit = _structure._lookup(csr.col, ("csr_t",))
    if hit is not None and hit[0]() is csr:
        return hit[1], hit[2]
    row_of_pos = ops.gather_i32(edge_index_used[0].contiguous(), csr.perm)        # destination row of every CSR slot
    csr_t = ops.csr_build(csr.col, row_of_pos, csr.n_cols, csr.n_rows)
    _structure._store(csr.col, ("csr_t",), (weakref.ref(csr), csr_t, csr_t.perm))
    return csr_t, csr_t.perm


class GatAttention(torch.autograd.Function):
    """y = act(softmax-attention aggregate(Q, K, V) + b) (gat.py:73-120) with gradients for Q, K, V and b.

    Without attention dropout (the default path):
      forward : tfgk_gat_fused_stats_f32 keeps (max, denominator) per (row, head) - no [E', H] coefficient table;
      backward: tfgk_gat_bwd_prepare/dst/src_f32 recompute the coefficients from those two numbers (dQ over the forward
                CSR, dK and dV over the transposed CSR: gathers, never scatter-adds).
    With attention dropout (gat.py:85), averaged heads, hub-row plans or shapes the streaming kernel does not take:
      forward : tfgk_gat_fused_f32 with the coefficients kept; under dropout they are re-aggregated by
                tfgk_spmm_heads_f32 with a counter-based mask;
      backward: G = dy * act'(y);  ds = tfgk_gat_softmax_bwd_f32(att, G, V);
                dQ = sum_e ds K[col] / scale                       forward CSR
                dK = sum_e ds Q[row] / scale,  dV = sum_e a' G[row] transposed CSR
    The mask is regenerated from (seed, edge, head) in every kernel, never stored; `seed` is a host key or an
    _rng.DeviceKey, which the backward reuses as it is, so under CUDA-graph capture it reads the base its forward read."""

    @staticmethod
    def forward(ctx, Q, K, V, bias, csr, edge_index_used, num_heads, split, act_code, drop_rate, seed, scale=None):
        Qd, Kd, Vd = Q.detach(), K.detach(), V.detach()
        b = None if bias is None else bias.detach()
        H = int(num_heads)
        if scale is None:                                    # gat.py:78; set2set.py:37 passes 1 (raw dot products)
            scale = float(np.sqrt(np.float32(Q.shape[1] // H)))
        if drop_rate > 0.0:
            _, att = ops.gat_fused(csr, Qd, Kd, Vd, H, split_value_heads=split, return_attention=True, scale=scale)
            y = ops.spmm_heads(csr, att, Vd, H, mode=ops.HEADS_SPLIT if split else ops.HEADS_REDUCE,
                               drop_rate=drop_rate, seed=seed, alpha=1.0 if split else 1.0 / H, bias=b, act=act_code)
        else:
            # no dropout: keep (max, denominator) per (row, head) instead of the [E', H] coefficients and recompute them in
            # the backward pass; shapes the streaming kernel does not take, and hub-row plans, keep the coefficient table
            res = None
            plan = getattr(csr, "plan", None)
            if split and (plan is None or plan.n_hubs == 0) and csr.n_rows == Qd.shape[0]:
                res = ops.gat_fused_stats(csr, Qd, Kd, Vd, H, bias=b, act=act_code, scale=scale)
            if res is not None:
                y, stats = res
                ctx.save_for_backward(Qd, Kd, Vd, stats, y)
                ctx.meta = (csr, edge_index_used, H, bool(split), act_code, 0.0, seed, bias is not None, float(scale))
                ctx.recompute, ctx.bias = True, b
                return y
            y, att = ops.gat_fused(csr, Qd, Kd, Vd, H, split_value_heads=split, bias=b, act=act_code,
                                   return_attention=True, scale=scale)
        ctx.recompute = False
        ctx.save_for_backward(Qd, Kd, Vd, att, y if act_code == ops.ACT_RELU else None)
        ctx.meta = (csr, edge_index_used, H, bool(split), act_code, float(drop_rate), seed, bias is not None, float(scale))
        return y

    @staticmethod
    def backward(ctx, grad_y):
        Q, K, V, att, y = ctx.saved_tensors
        csr, edge_index_used, H, split, act_code, drop_rate, seed, has_bias, scale = ctx.meta
        g = grad_y.contiguous()
        if ctx.recompute:
            csr_t, _ = _transposed_of_csr(csr, edge_index_used)
            res = ops.gat_backward_recompute(csr, csr_t, Q, K, V, g, y, ctx.bias, act_code, att, H, scale)
            if res is None:
                raise RuntimeError("GatAttention: the recompute backward refused a shape its forward accepted")
            grad_b = None
            if has_bias and ctx.needs_input_grad[3]:
                gm = _relu_grad(g, y) if act_code == ops.ACT_RELU else g
                grad_b = ops.colsum(gm)
            return res[0], res[1], res[2], grad_b, None, None, None, None, None, None, None, None
        if act_code == ops.ACT_RELU:
            g = _relu_grad(g, y)
        inv_scale = 1.0 / scale
        ds = ops.gat_softmax_bwd(csr, att, g, V, H, split_value_heads=split, drop_rate=drop_rate, seed=seed)
        grad_q = grad_k = grad_v = grad_b = None
        if ctx.needs_input_grad[0]:
            grad_q = ops.spmm_heads(csr, ds, K, H, alpha=inv_scale)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            csr_t, emap = _transposed_of_csr(csr, edge_index_used)
            if ctx.needs_input_grad[1]:
                grad_k = ops.spmm_heads(csr_t, ds, Q, H, emap=emap, alpha=inv_scale)
            if ctx.needs_input_grad[2]:
                grad_v = ops.spmm_heads(csr_t, att, g, H, mode=ops.HEADS_SPLIT if split else ops.HEADS_BROADCAST,
                                        emap=emap, drop_rate=drop_rate, seed=seed, alpha=1.0 if split else 1.0 / H)
        if has_bias and ctx.needs_input_grad[3]:
            grad_b = ops.colsum(g)
        return grad_q, grad_k, grad_v, grad_b, None, None, None, None, None, None, None, None


class Dropout(torch.autograd.Function):
    """tf.nn.dropout on dense activations (appnp.py:75-79, ssgc.py:84-88); the backward re-applies the same
    counter-based mask to the incoming gradient."""

    @staticmethod
    def forward(ctx, x, rate, seed):
        ctx.rate, ctx.seed = float(rate), seed          # a host key or an _rng.DeviceKey
        return ops.dropout(x.detach().contiguous(), ctx.rate, ctx.seed)

    @staticmethod
    def backward(ctx, grad_y):
        return ops.dropout(grad_y.contiguous(), ctx.rate, ctx.seed), None, None


def dropout(x, rate, training, seed=None):
    """Functional helper: identity unless training and rate > 0."""
    if not training or rate <= 0.0:
        return x
    from . import _rng
    return Dropout.apply(x, float(rate), _rng.resolve(seed, x.device))


def dense(x, weight, bias=None, activation=None):
    """Differentiable act(x @ W + b): relu is fused into the GEMM epilogue, any other callable runs on the result."""
    code, leftover = ops.activation_code(activation)
    y = Dense.apply(x, weight, bias, code)
    return leftover(y) if leftover is not None else y


def propagate(adj, h, bias=None, act_code=ops.ACT_NONE):
    """Differentiable act(A @ h + b) for a SparseMatrix A (gradient w.r.t. h, b and A's values)."""
    return SparseMatmul.apply(h, bias, adj, act_code, adj.value)


class SegmentReduce(torch.autograd.Function):
    """out[s] = REDUCE_{i: ids_i = s} data[i] for sum | mean | max | min over a plain id vector (the stock reducers of
    nn/kernel/map_reduce.py:15-42 and the graph pooling of nn/pool/common_pool.py), differentiable w.r.t. data.
    Backward: sum/mean are a gather of the upstream rows by segment id (scaled by 1 / max(count, 1) for mean); max/min
    route the gradient to the selected entries, shared equally among ties like TensorFlow's UnsortedSegmentMax gradient."""

    @staticmethod
    def forward(ctx, data, ids, num_segments, reduce):
        csr = _structure.csr_for_segment_ids(ids, int(num_segments))
        d = data.detach()
        if reduce == "min":       # min(x) = -max(-x): weight -1 per message and epilogue scale -1, both exact
            minus = torch.full((csr.nnz,), -1.0, dtype=torch.float32, device=d.device)
            out = ops.spmm(csr, minus, d, reduce="max", alpha=-1.0, col=csr.perm)
        else:
            out = ops.spmm(csr, None, d, reduce=reduce, col=csr.perm)
        ctx.ids, ctx.csr, ctx.reduce = ids, csr, reduce
        ctx.save_for_backward(d if reduce in ("max", "min") else None, out if reduce in ("max", "min") else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        data, out = ctx.saved_tensors
        ids, csr, reduce = ctx.ids, ctx.csr, ctx.reduce
        g = grad_out.contiguous()
        if reduce == "mean":
            cnt = (csr.rowptr[1:] - csr.rowptr[:-1]).clamp(min=1).to(torch.float32)
            g = g / cnt.unsqueeze(1)
        if reduce in ("sum", "mean"):
            return ops.permute(g, ids), None, None, None
        selected = (data == ops.permute(out, ids)).to(torch.float32)
        n_selected = ops.spmm(csr, None, selected, reduce="sum", col=csr.perm).clamp(min=1.0)
        return ops.permute(g / n_selected, ids) * selected, None, None, None


def segment_softmax_forward(data, ids, num_segments):
    """exp(d - max_seg) / (sum_seg + 1e-8) per segment of a plain id vector, [E] or [E, C]: K3's segment softmax over the
    segment CSR, in and out of its order by permutation."""
    csr = _structure.csr_for_segment_ids(ids, int(num_segments))
    soft_csr = ops.segment_softmax_csr(csr, ops.permute(data.contiguous(), csr.perm))
    return ops.permute(soft_csr, csr.perm, inverse=True)


class SegmentSoftmax(torch.autograd.Function):
    """segment_softmax (nn/kernel/segment.py:26-33) differentiable w.r.t. the scores.  The forward is the kernel of the
    non-differentiable path (same bits).  Backward: ds = a * (g - segsum(a * g)[seg]), the segment sums through the
    segment CSR (K1 gathering by perm, no atomics).  Like tfgk_gat_softmax_bwd_f32 it drops the 1e-8 of the denominator,
    whose derivative is about 1e-8 relative."""

    @staticmethod
    def forward(ctx, data, ids, num_segments):
        a = segment_softmax_forward(data.detach(), ids, num_segments)
        ctx.ids, ctx.num_segments = ids, int(num_segments)
        ctx.save_for_backward(a)
        return a

    @staticmethod
    def backward(ctx, grad_a):
        (a,) = ctx.saved_tensors
        csr = _structure.csr_for_segment_ids(ctx.ids, ctx.num_segments)
        ag = a * grad_a
        flat = ag if ag.dim() == 2 else ag.unsqueeze(1)
        seg = ops.spmm(csr, None, flat.contiguous(), reduce="sum", col=csr.perm)
        back = ops.permute(seg, ctx.ids)
        return a * (grad_a - (back if ag.dim() == 2 else back.squeeze(1))), None, None


class TakeRows(torch.autograd.Function):
    """data[index] (tf.gather along axis 0) through the gather kernel; backward = segment sum of the upstream rows by
    index (a deterministic scatter-add on the CSR kernel)."""

    @staticmethod
    def forward(ctx, data, index):
        ctx.index, ctx.n = index, data.shape[0]
        return ops.permute(data.detach(), index)

    @staticmethod
    def backward(ctx, grad_out):
        g = grad_out.contiguous()
        if ctx.index.numel() == 0:                     # nothing was taken (e.g. a pooled graph without edges)
            return g.new_zeros((ctx.n,) + tuple(g.shape[1:])), None
        csr = _structure.csr_for_segment_ids(ctx.index, ctx.n)
        flat = g if g.dim() == 2 else g.unsqueeze(1)
        res = ops.spmm(csr, None, flat, reduce="sum", col=csr.perm)
        return (res if g.dim() == 2 else res.squeeze(1)), None


class PadRows(torch.autograd.Function):
    """out[r, j] = x[src[rowptr[r] + j]] zero-padded to K (K9; nn/conv/graph_sage.py:319-337, utils/graph_utils.py:215-249),
    differentiable w.r.t. x.
      edge_index None : src = csr.perm of a segment-id CSR (convert_x_to_3d), row-major; backward = unpad_rows (every
                        row of x is written once, truncated rows get 0).
      edge_index given: src = csr.col of that edge list's CSR (lstm_graph_sage); every padded slot comes from one edge,
                        so dx[c] = sum_{e: col_e = c} dout[slot(e)]: K1 over the transposed CSR whose column override is
                        the flat slot index of each edge (K9's slot output, permuted with gather_i32).  No atomics.
    The forward runs the same kernel whatever requires grad (the slot output does not change the padded values)."""

    @staticmethod
    def forward(ctx, x, csr, K, step_major, edge_index):
        xd = x.detach()
        by_col = edge_index is not None
        want_slots = by_col and ctx.needs_input_grad[0]
        res = ops.pad_rows(csr, xd, K, src=csr.col if by_col else csr.perm, step_major=step_major, slot_index=want_slots)
        out, slot = res if want_slots else (res, None)
        ctx.csr, ctx.edge_index, ctx.slot, ctx.n = csr, edge_index, slot, x.shape[0]
        return out

    @staticmethod
    def backward(ctx, grad_out):
        g = grad_out.contiguous()
        if ctx.edge_index is None:
            return ops.unpad_rows(ctx.csr, g), None, None, None, None
        D = g.shape[-1]
        csr_t, emap = _transposed_of_csr(ctx.csr, ctx.edge_index)
        slot_col = ops.gather_i32(ctx.slot, emap)
        return ops.spmm(csr_t, None, g.view(-1, D), reduce="sum", col=slot_col), None, None, None, None


class Fp32Recurrence(torch.autograd.Function):
    """seq = module(inputs)[0] for a torch.nn.LSTM with cuDNN's TF32 math off in the forward AND the backward: cuDNN
    reads `torch.backends.cudnn.allow_tf32` (default True) when it builds the RNN descriptor of each pass, so a context
    manager around the call alone would leave the backward on TF32.  The module's graph is built inside the forward and
    differentiated in the backward under the same setting; the parameters are passed as inputs so that they get their
    gradients through this node."""

    @staticmethod
    def forward(ctx, module, inputs, *params):
        with torch.enable_grad(), _cudnn_fp32():
            leaf = inputs.detach().requires_grad_(ctx.needs_input_grad[1])
            seq = module(leaf)[0]
        ctx.inner = (leaf, seq, params)
        return seq.detach()

    @staticmethod
    def backward(ctx, grad_seq):
        leaf, seq, params = ctx.inner
        wanted = [(i, t) for i, t in enumerate((leaf,) + tuple(params)) if ctx.needs_input_grad[i + 1]]
        grads = [None] * (1 + len(params))
        if wanted:
            with _cudnn_fp32():
                got = torch.autograd.grad(seq, [t for _, t in wanted], grad_seq, allow_unused=True)
            for (i, _), gi in zip(wanted, got):
                grads[i] = gi
        ctx.inner = None
        return (None,) + tuple(grads)


class _cudnn_fp32(object):
    """Context manager: cuDNN without TF32 (restores the caller's setting)."""

    def __enter__(self):
        self.prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32 = self.prev
        return False


def run_lstm_fp32(module, inputs):
    """Output sequence of a torch.nn.LSTM module with cuDNN's TF32 off in the forward and, when gradients flow, the
    backward (Fp32Recurrence)."""
    params = tuple(module.parameters())
    if needs_grad(inputs, *params):
        return Fp32Recurrence.apply(module, inputs, *params)
    with _cudnn_fp32():
        return module(inputs)[0]


def _pair_project(x, agg, ws, wn, b, act_code, concat):
    """act([x Ws || agg Wn] + b) or act(x Ws + agg Wn + b), both products written straight into the output."""
    u = ws.shape[1]
    if concat:
        out = torch.empty((x.shape[0], u + wn.shape[1]), dtype=torch.float32, device=x.device)
        ops.gemm(x, ws, bias=None if b is None else b[:u].contiguous(), act=act_code, out=out[:, :u])
        ops.gemm(agg, wn, bias=None if b is None else b[u:].contiguous(), act=act_code, out=out[:, u:])
    else:
        out = ops.gemm(x, ws)
        ops.gemm(agg, wn, bias=b, act=act_code, beta=1.0, out=out)
    return out


class SagePair(torch.autograd.Function):
    """mean / sum GraphSAGE (nn/conv/graph_sage.py:9-115) as ONE differentiable op:
        out = act([x Ws || agg Wn] + b)   (or x Ws + agg Wn + b),   agg = REDUCE_{e: row_e = r} w_e x[col_e].
    Compared with composing NeighborAggregate and two Dense Functions this writes both projections straight into the
    output (no concat copy), masks the upstream gradient once, and folds dX_self into the epilogue of the transposed
    aggregation (grad_x = A^T d_agg + dX_self in one pass, tfgk_spmm_f32's addend).  dX products run on the tensor-core
    projection kernel (transB), dW products are split-K over the node dimension."""

    @staticmethod
    def forward(ctx, x, ws, wn, bias, edge_index, edge_weight, reduce, act_code, concat):
        n = x.shape[0]
        csr, _ = _structure.csr_for_edge_index(edge_index, n)
        w_csr = None if edge_weight is None else _structure.weights_in_csr_order(edge_weight, csr)
        xd, wsd, wnd = x.detach(), ws.detach(), wn.detach()
        b = None if bias is None else bias.detach()
        agg = ops.spmm(csr, w_csr, xd, reduce=reduce)
        out = _pair_project(xd, agg, wsd, wnd, b, act_code, concat)
        ctx.save_for_backward(x, ws, wn, agg, out if act_code == ops.ACT_RELU else None)
        ctx.meta = (edge_index, edge_weight, reduce, act_code, concat, csr, bias is not None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x, ws, wn, agg, out = ctx.saved_tensors
        edge_index, edge_weight, reduce, act_code, concat, csr, has_bias = ctx.meta
        gm = grad_out.contiguous()
        if act_code == ops.ACT_RELU:
            gm = _relu_grad(gm, out)
        u = ws.shape[1]
        gs, gn = (gm[:, :u], gm[:, u:]) if concat else (gm, gm)
        xd, wsd, wnd = x.detach(), ws.detach(), wn.detach()
        grad_x = grad_ws = grad_wn = grad_b = None
        if ctx.needs_input_grad[0]:
            d_agg = ops.gemm(gn, wnd, trans_b=True)
            dx_self = ops.gemm(gs, wsd, trans_b=True)
            csr_t, w_t = _transposed_structure(edge_index, x.shape[0], edge_weight, reduce == "mean", csr)
            grad_x = ops.spmm(csr_t, w_t, d_agg, reduce="sum", alpha=1.0, addend=dx_self, beta=1.0)
        if ctx.needs_input_grad[1]:
            grad_ws = ops.gemm(xd, gs, trans_a=True)
        if ctx.needs_input_grad[2]:
            grad_wn = ops.gemm(agg, gn, trans_a=True)
        if has_bias and ctx.needs_input_grad[3]:
            grad_b = ops.colsum(gm)
        return grad_x, grad_ws, grad_wn, grad_b, None, None, None, None, None


class BlockSagePair(torch.autograd.Function):
    """SagePair over a sampled block (utils.sampling.Block): out = act([x_self Ws || agg Wn] + b) with num_dst rows, agg
    = REDUCE over block.csr of the block's weighted rows of x.  Without `self_index`, x is the block's [num_src, F] input
    and x_self its first num_dst rows (a view).  With `self_index` (the SourceRows route), x is the global feature table,
    the aggregate reads it through block.global_col, x_self = x[self_index] is gathered, and x gets no gradient.
    Backward: dX_src = K1 over the block's transposed CSR into num_src rows, plus dX_self added into the first num_dst
    rows by the GEMM's beta = 1 epilogue."""

    @staticmethod
    def forward(ctx, x, ws, wn, bias, block, reduce, act_code, concat, self_index):
        xd, wsd, wnd = x.detach(), ws.detach(), wn.detach()
        b = None if bias is None else bias.detach()
        if self_index is None:
            agg = ops.spmm(block.csr, block.edge_weight, xd, reduce=reduce)
            x_self = xd[:block.num_dst]
        else:
            agg = ops.spmm(block.csr, block.edge_weight, xd, reduce=reduce, col=block.global_col)
            x_self = ops.permute(xd, self_index)
        out = _pair_project(x_self, agg, wsd, wnd, b, act_code, concat)
        ctx.save_for_backward(x_self, ws, wn, agg, out if act_code == ops.ACT_RELU else None)
        ctx.meta = (block, reduce, act_code, concat, bias is not None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x_self, ws, wn, agg, out = ctx.saved_tensors
        block, reduce, act_code, concat, has_bias = ctx.meta
        gm = grad_out.contiguous()
        if act_code == ops.ACT_RELU:
            gm = _relu_grad(gm, out)
        u = ws.shape[1]
        gs, gn = (gm[:, :u], gm[:, u:]) if concat else (gm, gm)
        wsd, wnd = ws.detach(), wn.detach()
        grad_x = grad_ws = grad_wn = grad_b = None
        if ctx.needs_input_grad[0]:
            csr_t, w_t = block.transposed(reduce)
            grad_x = ops.spmm(csr_t, w_t, ops.gemm(gn, wnd, trans_b=True), reduce="sum")
            ops.gemm(gs, wsd, trans_b=True, beta=1.0, out=grad_x[:block.num_dst])
        if ctx.needs_input_grad[1]:
            grad_ws = ops.gemm(x_self, gs, trans_a=True)
        if ctx.needs_input_grad[2]:
            grad_wn = ops.gemm(agg, gn, trans_a=True)
        if has_bias and ctx.needs_input_grad[3]:
            grad_b = ops.colsum(gm)
        return grad_x, grad_ws, grad_wn, grad_b, None, None, None, None, None


class BlockAggregate(torch.autograd.Function):
    """NeighborAggregate over a sampled block: agg [num_dst, D] = REDUCE over block.csr (sum | mean) of x's rows, weighted
    by the block's edge weights or, with weighted=False, by ones; `col` overrides the block's local columns (the
    SourceRows route reads the global table through block.global_col and takes no gradient).  Backward: K1 over the
    block's transposed CSR into x's num_src rows."""

    @staticmethod
    def forward(ctx, x, block, reduce, weighted, col):
        ctx.meta = (block, reduce, weighted)
        return ops.spmm(block.csr, block.edge_weight if weighted else None, x.detach(), reduce=reduce, col=col)

    @staticmethod
    def backward(ctx, grad_out):
        block, reduce, weighted = ctx.meta
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None
        csr_t, w_t = block.transposed(reduce, weighted)
        return ops.spmm(csr_t, w_t, grad_out.contiguous(), reduce="sum"), None, None, None, None


class BlockMax(torch.autograd.Function):
    """NeighborMax over a sampled block, unweighted: K11a over block.csr into num_dst rows; K11b over the block's
    transposed CSR into x's num_src rows."""

    @staticmethod
    def forward(ctx, x, block):
        xd = x.detach()
        out, cnt = ops.spmm_max(block.csr, None, xd)
        ctx.block = block
        ctx.save_for_backward(xd, out, cnt)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x, out, cnt = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None
        csr_t, _ = ctx.block.transposed(None)
        return ops.spmm_max_bwd(csr_t, None, x, out, cnt, grad_out.contiguous()), None


def _half_edge_csr(edge_index, num_nodes, ids_in_range=False):
    """CSR of the 2E half-edges of a query edge list: keys [row || col], partners [col || row].  Memoised on the edge
    tensor.  ids_in_range=True (ids known to lie in [0, num_nodes)) skips the id check and the work plan, so the build
    makes no host synchronisation."""
    tag = ("half_edges", int(num_nodes))
    hit = _structure._lookup(edge_index, tag)
    if hit is None:
        row, col = edge_index[0].contiguous(), edge_index[1].contiguous()
        half = (torch.cat([row, col]), torch.cat([col, row]), num_nodes, num_nodes)
        csr = ops.csr_build(*half, ids_in_range=True, plan=False) if ids_in_range else ops.csr_build(*half)
        hit = _structure._store(edge_index, tag, csr)
    return hit


class EdgeDot(torch.autograd.Function):
    """logits[e] = <h[row_e], h[col_e]> (predict_edge of demo/demo_gae.py:53-60) through K6, differentiable w.r.t. h.
    Backward: dh[u] = sum_{e: row_e = u} g_e h[col_e] + sum_{e: col_e = u} g_e h[row_e], ONE tfgk_spmm_f32 over the CSR
    of the 2E half-edges with g permuted into its order: no atomics, run-to-run identical, hub rows through the work
    plan, and a self-loop query counted twice (as autodiff does)."""

    @staticmethod
    def forward(ctx, h, edge_index):
        hd = h.detach()
        ctx.save_for_backward(hd)
        ctx.edge_index = edge_index
        return ops.edge_dot(hd, edge_index[0].contiguous(), edge_index[1].contiguous())

    @staticmethod
    def backward(ctx, grad_logits):
        (h,) = ctx.saved_tensors
        csr = _half_edge_csr(ctx.edge_index, h.shape[0])
        g = grad_logits.to(torch.float32).reshape(-1)
        w = ops.permute(torch.cat([g, g]).contiguous(), csr.perm)
        return ops.spmm(csr, w, h, reduce="sum"), None


class ClusterPool(torch.autograd.Function):
    """DiffPool / MinCutPool coarsening (nn/pool/cluster_pool.py:32-44) per graph g, in block layout:
        P[g*C + c] = (S_g^T X_g)[c]          Q[g*C + c, c'] = (S_g^T A_g S_g)[c, c'],   A[row_e, col_e] += w_e
    without the dense [G*C, N] assignment or N x N adjacency of the reference.  `layout` (nn/pool/cluster_pool.py) holds
    the edge CSR, the graph pointer / node list and node -> graph ids.  x may be None (then P is [G*C, 0]).
    Forward: T = A S (K1), Q = K8a(S, T), P = K8a(S, X); T is kept for the backward (N * C floats).
    Backward, with U = A^T S (K1 over the transposed CSR):
        dX = S dP            dS = X dP^T + T dQ^T + U dQ          (K8b)
        dw_e = <(S dQ)[row_e], S[col_e]>                          (K8b, then K7)
    The forward runs the same kernels whatever requires grad, so gradients change no forward bit."""

    @staticmethod
    def forward(ctx, x, s, edge_weight, layout):
        sd = s.detach()
        xd = torch.empty((sd.shape[0], 0), dtype=torch.float32, device=sd.device) if x is None else x.detach()
        w_csr = _structure.weights_in_csr_order(edge_weight.detach(), layout.csr)
        t = ops.spmm(layout.csr, w_csr, sd, reduce="sum")
        q = ops.graph_tmm(sd, t, layout.gptr, layout.num_graphs, gnodes=layout.gnodes)
        p = ops.graph_tmm(sd, xd, layout.gptr, layout.num_graphs, gnodes=layout.gnodes)
        ctx.layout = layout
        ctx.edge_weight = edge_weight.detach()
        ctx.save_for_backward(xd, sd, t)
        return p, q

    @staticmethod
    def backward(ctx, grad_p, grad_q):
        x, s, t = ctx.saved_tensors
        lay = ctx.layout
        C, ng = lay.num_clusters, lay.node_graph
        dp, dq = grad_p.contiguous(), grad_q.contiguous()
        grad_x = grad_s = grad_w = None
        if ctx.needs_input_grad[0]:
            grad_x = ops.graph_rmm(s, dp, ng, C)
        if ctx.needs_input_grad[1]:
            grad_s = ops.graph_rmm(t, dq, ng, C, trans=True)
            if x.shape[1]:
                ops.graph_rmm(x, dp, ng, C, trans=True, beta=1.0, out=grad_s)
            csr_t, w_t = _transposed_structure(lay.edge_index, lay.num_nodes, ctx.edge_weight, False, lay.csr)
            u = ops.spmm(csr_t, w_t, s, reduce="sum")
            ops.graph_rmm(u, dq, ng, C, beta=1.0, out=grad_s)
        if ctx.needs_input_grad[2]:
            grad_w = ops.sddmm_csr(lay.csr, ops.graph_rmm(s, dq, ng, C), s)
        return grad_x, grad_s, grad_w, None


class AssignGram(torch.autograd.Function):
    """M[g*C + c, c'] = (S_g^T S_g)[c, c'] (the S^T S of min_cut_pool.py:85-93) through K8a; dS = S dM + S dM^T (K8b)."""

    @staticmethod
    def forward(ctx, s, layout):
        sd = s.detach()
        ctx.layout = layout
        ctx.save_for_backward(sd)
        return ops.graph_tmm(sd, sd, layout.gptr, layout.num_graphs, gnodes=layout.gnodes)

    @staticmethod
    def backward(ctx, grad_m):
        (s,) = ctx.saved_tensors
        lay = ctx.layout
        g = grad_m.contiguous()
        out = ops.graph_rmm(s, g, lay.node_graph, lay.num_clusters)
        return ops.graph_rmm(s, g, lay.node_graph, lay.num_clusters, trans=True, beta=1.0, out=out), None


class SparseProduct(torch.autograd.Function):
    """C = A B for two SparseMatrix operands, differentiable in both operands' values (COO order), as tf_sparse's
    product is under tf.GradientTape.  Forward: K10 over the operands' CSRs with the values permuted into CSR order,
    detached, so the bits are the same whatever requires grad; returns C's (values, rowptr, columns), ascending unique
    columns per row.  Backward, with g = dL/dC in C's value order (K12, written in each operand's COO order through its
    CSR perm):
        dA[(i, k)] = sum_{q in B.row(k)} B.val[q] g(i, B.col[q])           (left mode, over A's CSR and B's CSR)
        dB[(k, j)] = sum_{q in A^T.row(k)} A.val[q] g(A^T.col[q], j)       (right mode, over B's CSR and A's transposed CSR)
    Only the gradients asked for are computed."""

    @staticmethod
    def forward(ctx, a_value, b_value, a, b):
        a_coo = a_value.detach().contiguous()
        b_val = ops.permute(b_value.detach().contiguous(), b.csr.perm)
        a_val = ops.permute(a_coo, a.csr.perm)
        c_rowptr, c_col, c_val = ops.spgemm(a.csr.rowptr, a.csr.col, a_val, b.csr.rowptr, b.csr.col, b_val, b.shape[1])
        ctx.a, ctx.b = a, b
        ctx.save_for_backward(a_coo, b_val, c_rowptr, c_col)
        ctx.mark_non_differentiable(c_rowptr, c_col)
        return c_val, c_rowptr, c_col

    @staticmethod
    def backward(ctx, grad_c, grad_rowptr, grad_col):
        a, b = ctx.a, ctx.b
        a_coo, b_val, c_rowptr, c_col = ctx.saved_tensors
        g = grad_c.contiguous()
        m, k, n = a.shape[0], a.shape[1], b.shape[1]
        grad_a = grad_b = None
        if ctx.needs_input_grad[0]:
            grad_a = ops.spgemm_grad("left", a.csr.rowptr, a.csr.col, b.csr.rowptr, b.csr.col, b_val, c_rowptr, c_col, g,
                                     m, k, n, perm=a.csr.perm)
        if ctx.needs_input_grad[1]:
            at = a._transposed_csr()
            grad_b = ops.spgemm_grad("right", b.csr.rowptr, b.csr.col, at.rowptr, at.col, ops.permute(a_coo, at.perm),
                                     c_rowptr, c_col, g, m, k, n, perm=b.csr.perm)
        return grad_a, grad_b, None, None


class RefusedPooledWeights(torch.autograd.Function):
    """The pooled edge weights of cluster_pool (the entries of S^T A S) as a function of A's and S's values.  The forward
    returns the weights K10 computed; their backward is not built, so it raises instead of returning no gradient."""

    @staticmethod
    def forward(ctx, pooled_weight, edge_weight, assign_edge_weight):
        return pooled_weight

    @staticmethod
    def backward(ctx, grad):
        raise RuntimeError("cluster_pool: the gradient of the pooled edge weights with respect to edge_weight and "
                           "assign_edge_weight is not implemented; detach those weights (ASAP detaches its assignment) or "
                           "keep the pooled weights out of the loss")


def needs_grad(*tensors):
    return torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in tensors)
