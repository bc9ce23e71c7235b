# coding=utf-8
"""SparseMatrix: the subset of tf_sparse.SparseMatrix that tf_geometric's hot path calls
(nn/conv/gcn.py:56,72-119,262,280; gat.py:83-89; appnp.py:51-55,86; data/graph.py:208-210), backed by the
destination-sorted CSR + sm_90a kernels instead of tf.gather / tf.math.unsorted_segment_sum.

COO semantics are kept on the outside: `index` int32 [2, nnz] (row = aggregation target), `value` float32 [nnz]
in the caller's edge order, no sorting or merging is visible.  The CSR (stable sort by row) is built lazily, once per
object, and reused by every product - this is what `graph.cache` memoises.  The values permuted into the CSR (and into
the transposed CSR) are kept too, for as long as `value` is the same tensor with the same version and storage: an
in-place update of learnable values (optimizer.step()) makes the next product permute them again.
"""
import weakref

import torch

from . import ops, _rng


class SparseMatrix(object):

    def __init__(self, index, value=None, shape=None, _csr=None, _value_csr=None):
        index = ops.as_device(index, torch.int32)
        if index.dim() != 2:
            index = index.reshape(2, -1)
        self.index = index
        nnz = index.shape[1]
        if value is None:
            self.value = torch.ones((nnz,), dtype=torch.float32, device=index.device)
        else:
            self.value = ops.as_device(value, torch.float32, device=index.device)
        if shape is None:
            n = int(index.max().item()) + 1 if nnz else 0
            shape = [n, n]
        self._shape = [int(shape[0]), int(shape[1])]
        self._csr = _csr
        self._value_csr = _value_csr
        self._value_csr_of = None if _value_csr is None else self._value_stamp()    # derived from the value as given
        self._csc = None
        self._value_csc = None
        self._value_csc_of = None
        self._pattern_of = None           # matrix with the same pattern whose transposed CSR is shared (dropout)

    # ---- structure ----
    @property
    def shape(self):
        return self._shape

    @property
    def row(self):
        return self.index[0]

    @property
    def col(self):
        return self.index[1]

    @property
    def nnz(self):
        return self.index.shape[1]

    @property
    def csr(self):
        if self._csr is None:
            self._csr = ops.csr_build(self.index[0].contiguous(), self.index[1].contiguous(), self._shape[0],
                                      self._shape[1])
        return self._csr

    def _value_stamp(self):
        """What a permuted copy of `value` is valid for: the same tensor (held by weak reference, as _structure._lookup
        holds its keys), unmodified in place (its version counter) and over the same storage.  An inference tensor
        (made under torch.inference_mode()) has no version counter: it can only be modified in place inside inference
        mode, where nothing is learned, so identity and storage are its whole stamp."""
        v = self.value
        return weakref.ref(v), None if v.is_inference() else v._version, v.data_ptr()

    def _stamp_current(self, stamp):
        return stamp is not None and stamp[0]() is self.value and stamp[1:] == self._value_stamp()[1:]

    @property
    def value_csr(self):
        if self._value_csr is None or not self._stamp_current(self._value_csr_of):
            self._value_csr = ops.permute(self.value, self.csr.perm)
            self._value_csr_of = self._value_stamp()
        return self._value_csr

    @property
    def value_csc(self):
        """`value` (detached) in the order of the transposed CSR, rebuilt under value_csr's rule."""
        if self._value_csc is None or not self._stamp_current(self._value_csc_of):
            self._value_csc = ops.permute(self.value.detach(), self._transposed_csr().perm)
            self._value_csc_of = self._value_stamp()
        return self._value_csc

    def _transposed_csr(self):
        if self._csc is None and self._pattern_of is not None:
            self._csc = self._pattern_of._transposed_csr()
        if self._csc is None:
            self._csc = ops.csr_build(self.index[1].contiguous(), self.index[0].contiguous(), self._shape[1],
                                      self._shape[0])
        return self._csc

    def with_value(self, value):
        """Same sparsity pattern (and cached CSR), new values in COO order."""
        return SparseMatrix(self.index, value, self._shape, _csr=self._csr)

    # ---- tf_sparse API subset ----
    def segment_sum(self, axis=-1):
        """Row sums (axis=-1/1) or column sums (axis=0/-2), sequential fp32 in edge order."""
        if axis in (-1, 1):
            return ops.csr_rowsum(self.csr, self.value_csr)
        csc = self._transposed_csr()
        return ops.csr_rowsum(csc, ops.permute(self.value, csc.perm))

    def segment_softmax(self, axis=-1):
        if axis not in (-1, 1):
            raise NotImplementedError("segment_softmax is only used with axis=-1 on this path (gat.py:84)")
        soft_csr = ops.segment_softmax_csr(self.csr, self.value_csr)
        out = SparseMatrix(self.index, ops.permute(soft_csr, self.csr.perm, inverse=True), self._shape, _csr=self._csr,
                           _value_csr=soft_csr)
        return out

    def add_diag(self, diag_value):
        """A + diag(diag_value): the diagonal is appended after the existing entries, no merge
        (same order as utils/graph_utils.py:350-366 add_self_loop_edge)."""
        n = min(self._shape)
        index = ops.self_loops(self.index, n)
        value = ops.self_loop_weights(self.value, self.nnz, n, diag_value, self.index.device)
        return SparseMatrix(index, value, self._shape)

    def dropout(self, rate, training=False, seed=None):
        """tf.nn.dropout on the stored values (gcn.py:262, appnp.py:84): the pattern is unchanged, dropped entries
        become explicit zeros and the kept ones are scaled by 1/(1-rate).  `seed` (an extension) pins the mask."""
        if not training or rate <= 0.0:
            return self
        from . import autograd
        seed = _rng.resolve(seed, self.value.device)
        # differentiable values (learnable edge weights) take the gradient through the same regenerated mask
        value = autograd.Dropout.apply(self.value, rate, seed) if autograd.needs_grad(self.value) else \
            ops.dropout(self.value, rate, seed)
        out = SparseMatrix(self.index, value, self._shape, _csr=self._csr)
        out._pattern_of = self            # the transposed structure (backward) is built once, on the cached parent
        return out

    def matmul(self, h, num_or_size_splits=None, **epilogue):
        """A @ h (gcn.py:280).  With a SparseMatrix h, the sparse x sparse product A @ B (see `_sparse_product`), which
        takes neither `num_or_size_splits` nor epilogue keywords.  `num_or_size_splits` (tf.split semantics: a count of equal column chunks or a list of
        chunk widths, utils/tf_sparse_utils.py:71-90) runs one launch per column chunk into slices of one output, like the
        reference's split -> matmul -> concat; the fused kernel has no [E, D] temporary to bound, so the results are the
        same bits with or without it.  A bfloat16 h stays bfloat16 and is gathered as such (tfgk_spmm_bf16) when no operand
        (h, bias, the values) needs a gradient: the float32 result is bit-identical to the product over h.float(), from
        half the row bytes.  With a bfloat16 h, `out_bf16=` (see ops.spmm) also stores the result rounded to bf16, or only
        that when no `out` is given."""
        from . import autograd
        if isinstance(h, SparseMatrix):
            if num_or_size_splits is not None or epilogue:
                raise TypeError("SparseMatrix.matmul: a sparse right operand takes no num_or_size_splits or epilogue "
                                "keywords")
            return self._sparse_product(h)
        # the differentiable route below works in fp32 (its backward products take fp32 operands): a bf16 h is widened
        # for it, as it always was
        keep_bf16 = torch.is_tensor(h) and h.dtype == torch.bfloat16 and \
            not autograd.needs_grad(h, epilogue.get("bias"), self.value)
        h = ops.as_device(h, torch.bfloat16 if keep_bf16 else torch.float32, device=self.index.device)
        if autograd.needs_grad(h, epilogue.get("bias"), self.value):
            # `A @ h` inside a user's training loop (tf_sparse products are differentiable under tf.GradientTape, in h and
            # in A's values): the same kernel behind autograd (dh = A^T g over the transposed structure, d value by K7);
            # column chunks change no bit, so none here
            if h.dim() != 2 or set(epilogue) - {"bias", "act"}:
                raise NotImplementedError("SparseMatrix.matmul: gradients are built for act(A @ h + bias) with a 2-D h")
            return autograd.propagate(self, h, epilogue.get("bias"), epilogue.get("act", ops.ACT_NONE))
        if num_or_size_splits is None or h.dim() != 2:
            return ops.spmm(self.csr, self.value_csr, h, reduce="sum", **epilogue)
        d = h.shape[1]
        if isinstance(num_or_size_splits, int):
            if num_or_size_splits <= 0 or d % num_or_size_splits:
                raise ValueError("num_or_size_splits={} does not evenly divide {} columns".format(num_or_size_splits, d))
            sizes = [d // num_or_size_splits] * num_or_size_splits
        else:
            sizes = [int(v) for v in num_or_size_splits]
            if sum(sizes) != d:
                raise ValueError("split sizes {} do not add up to {} columns".format(sizes, d))
        out = epilogue.pop("out", None)
        out_bf16 = epilogue.pop("out_bf16", None)
        if out is None and out_bf16 is None:
            out = torch.empty((self._shape[0], d), dtype=torch.float32, device=h.device)
        bias, addend = epilogue.pop("bias", None), epilogue.pop("addend", None)
        if h.dtype == torch.bfloat16:
            # each chunk is read in place, so it matches the fp32 chunk of h.float() (same layout, same use of the plan)
            epilogue["keep_layout"] = True
        c0 = 0
        for width in sizes:
            c1 = c0 + width
            if width:
                if out_bf16 is not None:
                    epilogue["out_bf16"] = out_bf16[:, c0:c1]
                ops.spmm(self.csr, self.value_csr, h[:, c0:c1], reduce="sum", out=None if out is None else out[:, c0:c1],
                         bias=None if bias is None else bias[c0:c1].contiguous(),
                         addend=None if addend is None else addend[:, c0:c1], **epilogue)
            c0 = c1
        return out if out is not None else out_bf16

    def _sparse_product(self, other):
        """C = A @ B for two SparseMatrix operands (tf_sparse's sparse x sparse product, as in gcn.py:83-94's
        diags(d) @ A @ diags(d) and cluster_pool.py:32-36's S^T A S): K10 on the device, differentiable in both operands'
        values (autograd.SparseProduct, K12).
        The result has shape [A.shape[0], B.shape[1]] and an int32 index in row-major order: ascending, unique columns
        in every row, duplicates of the operands merged (their products summed in Gustavson order: A's row left to right,
        then B's row left to right), exact zeros kept.  tf_sparse's own order for this product cannot be checked (tf_sparse
        is not available to compare against), so row-major is the order here.  The CSR is prebuilt with the identity
        permutation and its work plan, so a following C @ h does no sort."""
        from . import autograd
        if self._shape[1] != other._shape[0]:
            raise ValueError("SparseMatrix @ SparseMatrix: inner dimensions differ ({} x {} @ {} x {})".format(
                self._shape[0], self._shape[1], other._shape[0], other._shape[1]))
        if self.index.device != other.index.device:
            raise ValueError("SparseMatrix @ SparseMatrix: operands on {} and {}".format(self.index.device,
                                                                                        other.index.device))
        value, rowptr, col = autograd.SparseProduct.apply(self.value, other.value, self, other)
        nnz = col.shape[0]
        if nnz >= 2 ** 31:
            raise ValueError("SparseMatrix @ SparseMatrix: the product has {} entries, more than an int32 index "
                             "addresses".format(nnz))
        m, n = self._shape[0], other._shape[1]
        dev = rowptr.device
        row = torch.repeat_interleave(torch.arange(m, dtype=torch.int32, device=dev), rowptr[1:] - rowptr[:-1],
                                      output_size=nnz)
        csr = ops.CSR(rowptr, col, torch.arange(nnz, dtype=torch.int32, device=dev), m, n)
        csr.plan = ops.build_plan(csr)
        return SparseMatrix(torch.stack([row, col]), value, [m, n], _csr=csr, _value_csr=value.detach())

    def __matmul__(self, h):
        return self.matmul(h)

    def transpose(self):
        return SparseMatrix(torch.stack([self.index[1], self.index[0]]), self.value, [self._shape[1], self._shape[0]])

    def to_dense(self):
        out = torch.zeros(self._shape, dtype=torch.float32, device=self.index.device)
        out.index_put_((self.index[0].long(), self.index[1].long()), self.value, accumulate=True)
        return out

    def __len__(self):
        return self._shape[0]

    def __repr__(self):
        return "SparseMatrix(shape={}, nnz={})".format(self._shape, self.nnz)


def diags(values):
    """tf_sparse's diags: the n x n diagonal SparseMatrix whose values are `values` (a 1-D tensor; gradients flow through
    them), so the reference's normalisation diags(d) @ A @ diags(d) (gcn.py:83-94) can be written as it is there."""
    values = ops.as_device(values, torch.float32)
    if values.dim() != 1:
        raise ValueError("diags: values must be 1-D (got shape {})".format(tuple(values.shape)))
    n = values.shape[0]
    ids = torch.arange(n, dtype=torch.int32, device=values.device)
    return SparseMatrix(torch.stack([ids, ids]), values, [n, n])


def as_sparse_features(x):
    """A sparse FEATURE matrix (the tf.SparseTensor `x` of nn/conv/gcn.py:269-272, gat.py:45-70; Cora's bag of words) as
    a SparseMatrix, or None when x is dense.  Accepts SparseMatrix, torch sparse COO / CSR tensors and scipy sparse
    matrices; entries keep their order (canonical row-major for TF's SparseTensor), which is the summation order."""
    if isinstance(x, SparseMatrix):
        return x
    if torch.is_tensor(x):
        if x.layout == torch.sparse_coo:
            x = x.coalesce()
            return SparseMatrix(x.indices().to(torch.int32), x.values().to(torch.float32), list(x.shape))
        if x.layout == torch.sparse_csr:
            return as_sparse_features(x.to_sparse_coo())
        return None
    if hasattr(x, "tocoo") and hasattr(x, "nnz"):          # scipy.sparse
        import numpy as np
        coo = x.tocsr().tocoo()                            # row-major order
        return SparseMatrix(np.stack([coo.row, coo.col]).astype(np.int32), coo.data.astype(np.float32), list(coo.shape))
    return None


def project_features(x, kernel, bias=None, act=0):
    """act(x @ kernel + bias) for a dense or sparse x: the sparse product gathers rows of the kernel by the column ids of
    x's non-zeros - the same gather / edge-apply / segment-reduce kernel as the aggregation (tf.sparse.sparse_dense_matmul
    at gcn.py:272)."""
    sp = as_sparse_features(x)
    if sp is None:
        return None
    kernel = ops.as_device(kernel, torch.float32, device=sp.index.device)
    return sp.matmul(kernel, bias=bias, act=act)
