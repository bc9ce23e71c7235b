# coding=utf-8
"""Op-for-op port of the reference's CPU path onto torch-CPU ops (TEST / BENCH INFRASTRUCTURE ONLY).

TensorFlow cannot be installed here, so the timed "reference arm" of bench.py is this restatement of the exact op
sequence the reference issues, using all host threads torch will take:
    tf.gather                      -> torch.index_select
    gcn_mapper (x * w[:, None])    -> torch mul                         (nn/conv/gcn.py:221-222)
    tf.math.unsorted_segment_sum   -> zeros(...).index_add_             (nn/kernel/map_reduce.py:15-16)
    tf.math.unsorted_segment_max   -> scatter_reduce_(amax)             (nn/kernel/segment.py:27)
    x @ kernel                     -> torch matmul
including the [E, D] temporaries the reference materialises (the thing the fused GPU kernels remove).
Numerically it is checked against tfg_oracle.py in tests/test_oracle.py."""
import torch


def _segment_sum(data, ids, n):
    out = torch.zeros((n,) + tuple(data.shape[1:]), dtype=data.dtype)
    return out.index_add_(0, ids, data)


def _segment_max(data, ids, n):
    out = torch.full((n,) + tuple(data.shape[1:]), torch.finfo(data.dtype).min, dtype=data.dtype)
    index = ids if data.dim() == 1 else ids.unsqueeze(1).expand_as(data)
    return out.scatter_reduce_(0, index, data, reduce="amax", include_self=True)


def segment_softmax(data, ids, n):                       # nn/kernel/segment.py:26-33
    mx = _segment_max(data, ids, n)
    e = torch.exp(data - mx.index_select(0, ids))
    den = _segment_sum(e, ids, n) + 1e-8
    return e / den.index_select(0, ids)


def spmm(row, col, value, h, n):                         # tf_sparse matmul = gather * value -> unsorted_segment_sum
    msg = h.index_select(0, col) * value.unsqueeze(1)
    return _segment_sum(msg, row, n)


def gcn_forward(x, row, col, normed_value, kernel, bias, relu=True):
    """nn/conv/gcn.py:260-288 with a warm cache (row/col/normed_value = cached normalised adjacency)."""
    h = x @ kernel
    h = spmm(row, col, normed_value, h, x.shape[0])
    h = h + bias
    return torch.relu(h) if relu else h


def gat_attention(Q, K, V, row, col, num_rows, num_heads, scale=None, bias=None, relu=False):
    """The attention core of nn/conv/gat.py:73-120 with the heads split and concatenated, on given Q [n_dst, A],
    K [n_src, A] and V [n_src, H * dv]: per head, a_e = segment_softmax(<Q[row_e], K[col_e]> / scale) over the edges of
    each destination row, out[r] = sum_e a_e V[col_e], then act(out + bias).  Rows without edges get act(bias).
    scale defaults to sqrt(A / H) (gat.py:78; set2set.py passes 1).  Differentiable w.r.t. Q, K, V and bias: in float64
    it is the reference the GAT backward kernels are checked against."""
    H = int(num_heads)
    E, A = row.shape[0], Q.shape[1]
    dqk, dv = A // H, V.shape[1] // H
    if scale is None:
        scale = dqk ** 0.5
    score = (Q.index_select(0, row).reshape(E, H, dqk) * K.index_select(0, col).reshape(E, H, dqk)).sum(-1) / scale
    att = segment_softmax(score, row, num_rows)                                          # [E, H]
    msg = (V.index_select(0, col).reshape(E, H, dv) * att.unsqueeze(-1)).reshape(E, H * dv)
    out = _segment_sum(msg, row, num_rows)
    if bias is not None:
        out = out + bias
    return torch.relu(out) if relu else out


def gat_forward(x, row, col, wq, bq, wk, bk, wv, bias, num_heads, relu=True, split_value_heads=True, att_scale=None):
    """nn/conv/gat.py:43-120; row/col already hold the appended self loops (gat.py:43).
    att_scale: optional [num_heads * E'] multiplier standing in for tf.nn.dropout on the attention values (gat.py:85),
    in the virtual-graph order the reference uses (head-major).  Differentiable: torch autograd over this function is
    the stand-in for TensorFlow autodiff over the reference in the backward-pass tests."""
    n = x.shape[0]
    Q = torch.relu(x @ wq + bq).index_select(0, row)
    K = torch.relu(x @ wk + bk).index_select(0, col)
    V = x @ wv
    Q_ = torch.cat(torch.split(Q, Q.shape[1] // num_heads, dim=-1), dim=0)
    K_ = torch.cat(torch.split(K, K.shape[1] // num_heads, dim=-1), dim=0)
    rows_ = torch.cat([row + i * n for i in range(num_heads)])
    cols_ = torch.cat([col + i * n for i in range(num_heads)])
    att = (Q_ * K_).sum(-1) / (Q_.shape[-1] ** 0.5)
    att = segment_softmax(att, rows_, n * num_heads)
    if att_scale is not None:
        att = att * att_scale
    V_ = torch.cat(torch.split(V, V.shape[1] // num_heads, dim=-1), dim=0)
    h_ = spmm(rows_, cols_, att, V_, n * num_heads)
    if split_value_heads:
        h = torch.cat(torch.split(h_, n, dim=0), dim=-1)                          # gat.py:112
    else:
        h = torch.stack(torch.split(h_, n, dim=0)).sum(0) / num_heads             # gat.py:114 (add_n / num_heads)
    if bias is not None:
        h = h + bias
    return torch.relu(h) if relu else h
