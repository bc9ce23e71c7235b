# coding=utf-8
"""The per-entry error bound of the training contract (tests/test_gpu_train_contract.py, tests/test_train_steps_host.py).

A layer and its backward are compositions of float32 sums and products.  Every reference is written once, over the
operations of `Replay`, and run twice in float64 from the float32 values the kernels saw:

  exact     : the layer as written; autograd gives the reference forward and gradients;
  magnitude : every operand replaced by its absolute value (inputs, edge values, the upstream gradient), every
              subtraction by an addition, and every derivative of a nonlinear factor (the degree normalisation) by its
              absolute value.  Autograd then gives, per entry, S = the sum of the magnitudes of all the terms that entry
              is made of.

ReLU is multiplication by a fixed 0 / 1 mask in both runs.  The mask is the one the float32 path applied (its own output
> 0, as `autograd._relu_grad` reads it), so no entry whose pre-activation lies within rounding of 0 can flip.

Bound.  A float32 sum of k terms accumulated one after another (or in slices whose partial sums are then added) carries
at most (k + 1) roundings, each of relative size u = 2^-24, on its longest chain; an elementwise product or epilogue
(bias, alpha, the addend) one more.  An error of relative size e·S_mid introduced at an intermediate entry reaches an
output through sums and products with non-negative magnitudes, so it contributes at most e·S_out there: the errors of
successive stages add up.  Each output of a case therefore gets

    |got - ref| <= (c · u + sum over K4 stages of (K · 2^-23 + 2^-19)) · S

with c the sum of the longest reductions of the stages on its chain (in-degree for K1 over the forward CSR, out-degree
over the transposed CSR, n for the column sums and the split-K weight gradients, whose slices and partials add at most
one rounding per row) and the second term the documented bound of the 3xTF32 tensor-core projection (K4, DESIGN.md §5),
counted wherever a dense product of depth K <= 184 may run on it.  The first-order bound neglects u^2 terms."""
import numpy as np
import torch

U = 2.0 ** -24


def k4_term(K):
    """Relative bound of one K4 product of depth K (DESIGN.md §5)."""
    return K * 2.0 ** -23 + 2.0 ** -19


def eps(c, *k4_depths):
    """Relative bound of a chain of c float32 roundings plus one K4 product per depth given."""
    return c * U + sum(k4_term(K) for K in k4_depths)


def _per_entry(e, got):
    """e as given (a scalar) or per row (a vector over the first axis of got), broadcast over got's other axes."""
    e = np.asarray(e, np.float64)
    return e.reshape(e.shape + (1,) * (got.ndim - e.ndim)) if e.ndim else e


def ratio(got, ref, S, e):
    """Worst |got - ref| / (e · S) over the entries; an entry with S = 0 must match exactly (ratio inf otherwise).
    e is one relative bound, or one per row of got."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    err = np.abs(got - ref)
    bound = _per_entry(e, got) * np.asarray(S, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def worst_entry(got, ref, S, e):
    """(flat index, got, ref, bound) of the entry with the largest err / bound, for failure messages."""
    got = np.asarray(got, np.float64)
    bound = (_per_entry(e, got) * np.asarray(S, np.float64)).ravel()
    got = got.ravel()
    ref = np.asarray(ref, np.float64).ravel()
    err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    i = int(np.argmax(r))
    return i, got[i], ref[i], bound[i]


# ---- per-row chains ----------------------------------------------------------------------------------------------
# The longest chain of an entry is that of its own row: the reduction of the last stage over that row's edges, plus the
# longest chain among the rows it gathers from (an input error reaches the row through its neighbours only).

def degrees(row, col, n, loops=0):
    """(in-degree, out-degree) per node, each plus `loops` (the self loops a layer appends)."""
    return np.bincount(row, minlength=n) + loops, np.bincount(col, minlength=n) + loops


def neighbour_max(row, col, c):
    """Per row r: the largest of c[r] and c[col_e] over the edges e with row_e = r."""
    out = np.array(c, np.int64, copy=True)
    np.maximum.at(out, row, np.asarray(c, np.int64)[col])
    return out


def transposed_gather_eps(row, col, n):
    """dh = A^T g (SparseMatrix.matmul's dh, an unnormalised aggregation's dx): per source node, its out-degree of
    fused multiply-adds and the epilogue."""
    _, dout = degrees(row, col, n)
    return eps(dout + 3)


def gcn_dx_eps(row, col, n, units):
    """GCN's dx = (norm(A)^T g) W^T per source node c: c's out-degree in the transposed product, the degree sums behind
    the normalised values it gathers (deg of c and of every destination of c; self loops appended), rsqrt and two
    scalings, then K4 of depth `units`."""
    din, dout = degrees(row, col, n, loops=1)
    return eps(dout + neighbour_max(col, row, din) + 12, units)


class Replay(object):
    """The float64 operations of a reference, in the exact or the magnitude mode (module docstring)."""

    def __init__(self, magnitude):
        self.magnitude = bool(magnitude)

    def leaf(self, a, grad=True):
        t = torch.tensor(np.asarray(a, np.float64))
        if self.magnitude:
            t = t.abs()
        return t.requires_grad_(grad)

    def const(self, a):
        return self.leaf(a, grad=False)

    def upstream(self, g):
        g = torch.as_tensor(np.asarray(g, np.float64))
        return g.abs() if self.magnitude else g

    @staticmethod
    def relu(z, mask):
        """ReLU with the mask of the float32 path (a float64 0 / 1 tensor)."""
        return z * mask

    def sub(self, a, b):
        return a + b if self.magnitude else a - b

    def spmm(self, row, col, val, h, n):
        """out[r] = sum_{e: row_e = r} val_e h[col_e] in edge order; row / col int64 tensors."""
        if self.magnitude:
            val = val.abs()
        return torch.zeros((n, h.shape[1]), dtype=torch.float64).index_add(0, row, val.unsqueeze(1) * h[col])

    def inv_sqrt(self, deg):
        """deg^-1/2, 0 where deg <= 0 (gcn.py's _remove_inf_and_nan); the magnitude mode keeps the value and makes the
        derivative |d deg^-1/2 / d deg|.  That value is the exact one only when the magnitude degree (the sum of |w|)
        equals the degree, i.e. for non-negative weights; with weights of both signs a degree near 0 amplifies the
        rounding of its sum beyond what this replay accounts for."""
        pos = deg > 0
        safe = torch.where(pos, deg, torch.ones_like(deg))
        f = torch.where(pos, safe ** -0.5, torch.zeros_like(deg))
        if not self.magnitude:
            return f
        fp = torch.where(pos, 0.5 * safe ** -1.5, torch.zeros_like(deg))
        return f.detach() + fp.detach() * (deg - deg.detach())

    def gcn_norm(self, row, col, w, n, fill=1.0):
        """gcn_norm_adj(norm="both", sym=True, renorm=True): self loops of weight `fill` appended, then
        deg^-1/2[row] w deg^-1/2[col] with deg the row sums.  Returns (row', col', values)."""
        loops = torch.arange(n, dtype=torch.int64)
        r2, c2 = torch.cat([row, loops]), torch.cat([col, loops])
        w2 = torch.cat([w, torch.full((n,), float(fill), dtype=torch.float64)])
        deg = torch.zeros(n, dtype=torch.float64).index_add(0, r2, w2)
        dis = self.inv_sqrt(deg)
        return r2, c2, dis[r2] * w2 * dis[c2]
