# coding=utf-8
"""Float64 torch restatements of the reference's op sequences that edge weights flow through (TEST INFRASTRUCTURE):
gcn_norm_adj (nn/conv/gcn.py:32-130, utils/graph_utils.py add_self_loop_edge) and the aggregations, differentiable in the
edge weights.  They stand in for tf.GradientTape.  One deliberate difference from TensorFlow: where a degree is <= 0,
_remove_inf_and_nan forces the factor to 0, and here its derivative is 0 as well (tf.where would propagate NaN)."""
import numpy as np
import torch


def t64(a, grad=False):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=grad)


def _inv(deg, power):
    """tf.pow(deg, power) followed by _remove_inf_and_nan, with a finite derivative where the factor is forced to 0."""
    ok = deg > 0 if power == -0.5 else deg != 0                   # pow(<0, -0.5) is NaN, pow(0, p) is inf
    safe = torch.where(ok, deg, torch.ones_like(deg))
    return torch.where(ok, safe ** power, torch.zeros_like(deg))


def gcn_norm(row, col, w, shape, norm="both", add_self_loop=True, sym=True, renorm=True, improved=False):
    """(row, col, value) of the normalised adjacency; row / col int64 tensors, w float64 (may require grad)."""
    fill = 2.0 if improved else 1.0
    n = min(shape)

    def add_diag(r, c, v):
        loops = torch.arange(n, dtype=torch.int64)
        return torch.cat([r, loops]), torch.cat([c, loops]), torch.cat([v, torch.full((n,), fill, dtype=v.dtype)])

    r, c, v = row, col, w
    if add_self_loop and norm != "both":
        r, c, v = add_diag(r, c, v)
    if norm == "both":
        if add_self_loop and renorm:
            r, c, v = add_diag(r, c, v)
        a = _inv(torch.zeros(shape[0], dtype=v.dtype).index_add(0, r, v), -0.5)
        b = a if sym else _inv(torch.zeros(shape[1], dtype=v.dtype).index_add(0, c, v), -0.5)
        v = a[r] * v * b[c]
        if add_self_loop and not renorm:
            r, c, v = add_diag(r, c, v)
    elif norm == "left":
        p = _inv(torch.zeros(shape[0], dtype=v.dtype).index_add(0, r, v), -1.0)
        v = p[r] * v
    else:
        q = _inv(torch.zeros(shape[0], dtype=v.dtype).index_add(0, r, v), -1.0)
        v = v * q[c]
    return r, c, v


def spmm(row, col, value, h, n):
    """sum_{e: row_e = i} value_e h[col_e] (tf_sparse matmul / unsorted_segment_sum of gathered messages)."""
    return torch.zeros((n, h.shape[1]), dtype=h.dtype).index_add(0, row, h[col] * value.unsqueeze(1))


def aggregate(row, col, w, h, n, reduce):
    """unsorted_segment_{sum,mean} of w_e h[col_e] by row (graph_sage.py:41, map_reduce.py:15-28)."""
    out = spmm(row, col, w, h, n)
    if reduce == "mean":
        cnt = torch.zeros(n, dtype=h.dtype).index_add(0, row, torch.ones_like(w)).clamp(min=1.0)
        out = out / cnt.unsqueeze(1)
    return out


# every (norm, add_self_loop, sym, renorm, improved) gcn_norm_adj accepts on a square matrix
NORM_COMBOS = [(norm, loop, sym, renorm, improved)
               for norm in ("both", "left", "right") for loop in (False, True)
               for sym in ((False, True) if norm == "both" else (True,))
               for renorm in ((False, True) if (norm == "both" and loop) else (True,))
               for improved in ((False, True) if loop else (False,))]
