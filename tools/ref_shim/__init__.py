# coding=utf-8
"""numpy stand-ins for `tensorflow` and `tf_sparse`, just large enough to EXECUTE the reference's own Python files
for the message-passing hot path (nn/kernel/*.py, nn/conv/{gcn,gat,graph_sage,appnp}.py, utils/graph_utils.py)
and the cluster pooling (nn/pool/{cluster_pool,diff_pool,min_cut_pool}.py)
in a container that has neither package.  Used ONLY by tools/gen_golden_from_reference.py to produce
tests/golden/ref_exec_*.npz.  What this pins: the reference's control flow, call order, quirks and in-repo arithmetic.
What it cannot pin: TensorFlow's / tf_sparse's own kernels - their semantics are restated here from the public docs
(and, for tf_sparse, from the commented-out legacy code in the reference; SURVEY.md section 8c)."""
import sys
import types

import numpy as np

# NOTE: this module deliberately imports nothing from the repository (in particular not its CPU checker).  The TensorFlow /
# tf_sparse ops the reference calls are restated a SECOND time here, independently and in the most literal form (explicit
# per-element loops in input order), so that a fixture produced through this shim can disagree with the checker under tests/
# if either restatement of the documented TF semantics is wrong.  (Round-1 review: a shim that delegated to the checker made
# fixture == checker by construction.)


def _seg_loop(data, ids, num_segments, init, combine):
    """out[ids[i]] = combine(out[ids[i]], data[i]) for i = 0, 1, ... in input order, in data's dtype (TF's CPU kernels)."""
    data = np.asarray(data)
    ids = np.asarray(ids).reshape(-1)
    out = np.full((int(num_segments),) + data.shape[1:], init, dtype=data.dtype)
    for i in range(ids.shape[0]):
        s = int(ids[i])
        if s < 0:
            continue                              # tf.math.unsorted_segment_*: negative ids are dropped
        if s >= num_segments:
            raise IndexError("segment id {} out of range [0, {})".format(s, num_segments))
        out[s] = combine(out[s], data[i])
    return out


def _segment_sum(data, ids, n):
    data = np.asarray(data)
    return _seg_loop(data, ids, n, data.dtype.type(0), lambda a, b: (a + b).astype(data.dtype))


def _segment_mean(data, ids, n):
    data = np.asarray(data)
    total = _segment_sum(data, ids, n)
    count = _segment_sum(np.ones(np.asarray(ids).reshape(-1).shape[0], dtype=data.dtype), ids, n)
    count = np.maximum(count, data.dtype.type(1))
    return (total / count.reshape((-1,) + (1,) * (data.ndim - 1))).astype(data.dtype)


def _lowest(dtype):
    return np.finfo(dtype).min if np.dtype(dtype).kind == "f" else np.iinfo(dtype).min


def _highest(dtype):
    return np.finfo(dtype).max if np.dtype(dtype).kind == "f" else np.iinfo(dtype).max


def _segment_max(data, ids, n):
    data = np.asarray(data)
    return _seg_loop(data, ids, n, _lowest(data.dtype), np.maximum)      # empty segment: numeric_limits<T>::lowest()


def _segment_min(data, ids, n):
    data = np.asarray(data)
    return _seg_loop(data, ids, n, _highest(data.dtype), np.minimum)


def _gather0(params, indices):
    params, indices = np.asarray(params), np.asarray(indices)
    if indices.size and (indices.min() < 0 or indices.max() >= params.shape[0]):
        raise IndexError("tf.gather: index out of range (the CPU kernel raises InvalidArgument)")
    return np.take(params, indices, axis=0)


def _unique_first_occurrence(x):
    """tf.unique: distinct values in order of first appearance, and for every element the position of its value there."""
    seen, values, index = {}, [], []
    for v in np.asarray(x).reshape(-1).tolist():
        if v not in seen:
            seen[v] = len(values)
            values.append(v)
        index.append(seen[v])
    return np.asarray(values, dtype=np.asarray(x).dtype), np.asarray(index, dtype=np.int32)


def _l2_normalize_last_axis(x, eps=1e-12):
    x = np.asarray(x, dtype=np.float32)
    sq = np.sum(x * x, axis=-1, keepdims=True, dtype=np.float32)
    return (x * (np.float32(1) / np.sqrt(np.maximum(sq, np.float32(eps))))).astype(np.float32)


class Tensor(np.ndarray):
    """An eager tensor: an ndarray that also answers .numpy()."""

    def numpy(self):
        return np.asarray(self)


def T(a, dtype=None):
    return np.asarray(a, dtype=dtype).view(Tensor)


def _unsupported(name):
    def fn(*a, **k):
        raise NotImplementedError("tensorflow shim: {} is not implemented".format(name))
    return fn


def build_tensorflow():
    tf = types.ModuleType("tensorflow")
    tf.__version__ = "2.15.0"
    tf.float32, tf.float64, tf.int32, tf.int64, tf.bool = np.float32, np.float64, np.int32, np.int64, np.bool_
    tf.is_tensor = lambda x: isinstance(x, Tensor)
    tf.executing_eagerly = lambda: True
    tf.function = lambda f=None, **k: (f if f is not None else (lambda g: g))
    tf.convert_to_tensor = lambda x, dtype=None: T(x, dtype)
    tf.cast = lambda x, dtype: (T(np.asarray(x).astype(dtype)) if np.ndim(x) else dtype(x))
    tf.shape = lambda x: T(np.array(np.shape(x), dtype=np.int32))
    tf.range = lambda *a, dtype=np.int32: T(np.arange(*[int(v) for v in a], dtype=dtype))
    tf.ones = lambda shape, dtype=np.float32: T(np.ones([int(s) for s in shape], dtype=dtype))
    tf.zeros = lambda shape, dtype=np.float32: T(np.zeros([int(s) for s in shape], dtype=dtype))
    tf.fill = lambda shape, v: T(np.full([int(s) for s in shape], v))
    tf.ones_like = lambda x: T(np.ones_like(np.asarray(x)))
    tf.zeros_like = lambda x: T(np.zeros_like(np.asarray(x)))
    tf.stack = lambda xs, axis=0: T(np.stack([np.asarray(x) for x in xs], axis=axis))
    tf.concat = lambda xs, axis=0: T(np.concatenate([np.asarray(x) for x in xs], axis=axis))
    tf.split = lambda x, n, axis=0: [T(p) for p in np.split(np.asarray(x), n, axis=axis)]
    tf.reshape = lambda x, shape: T(np.reshape(np.asarray(x), shape))
    tf.expand_dims = lambda x, axis: T(np.expand_dims(np.asarray(x), axis))
    tf.where = lambda c, a, b: T(np.where(np.asarray(c), np.asarray(a), np.asarray(b)))
    tf.boolean_mask = lambda t, m, axis=None: T(np.compress(np.asarray(m), np.asarray(t), axis=0 if axis is None else axis))
    tf.not_equal = lambda a, b: T(np.not_equal(np.asarray(a), np.asarray(b)))
    tf.less = lambda a, b: T(np.less(np.asarray(a), np.asarray(b)))
    tf.maximum = lambda a, b: T(np.maximum(np.asarray(a), np.asarray(b)))
    tf.pow = lambda x, p: T(_pow(np.asarray(x), p))
    tf.exp = lambda x: T(np.exp(np.asarray(x)))
    tf.stop_gradient = lambda x: x
    tf.add_n = lambda xs: T(_add_n(xs))
    tf.reduce_sum = lambda x, axis=None: _red(np.sum, x, axis)
    tf.reduce_mean = lambda x, axis=None: _red(np.mean, x, axis)
    tf.reduce_max = lambda x, axis=None: _red(np.max, x, axis)
    tf.reduce_any = lambda x, axis=None: bool(np.any(np.asarray(x)))
    tf.reduce_min = lambda x, axis=None: _red(np.min, x, axis)
    tf.TensorSpec = lambda shape=None, dtype=None, name=None: (shape, dtype)
    tf.cond = lambda pred, true_fn, false_fn: true_fn() if bool(pred) else false_fn()
    tf.squeeze = lambda x, axis=None: T(np.squeeze(np.asarray(x), axis=axis))
    tf.minimum = lambda a, b: T(np.minimum(np.asarray(a), np.asarray(b)))
    tf.greater_equal = lambda a, b: T(np.greater_equal(np.asarray(a), np.asarray(b)))
    tf.logical_and = lambda a, b: T(np.logical_and(np.asarray(a), np.asarray(b)))
    tf.gather_nd = lambda params, indices: T(np.asarray(params)[tuple(np.asarray(indices).T)])

    def reduce_sum(x, axis=None, keepdims=False):
        r = np.sum(np.asarray(x), axis=axis, keepdims=keepdims)
        return T(r) if np.ndim(r) else r
    tf.reduce_sum = reduce_sum

    def argsort(values, axis=-1, direction="ASCENDING", stable=False):
        v = np.asarray(values)
        return T(np.argsort(-v if direction == "DESCENDING" else v, axis=axis, kind="stable").astype(np.int32))
    tf.argsort = argsort

    def tensor_scatter_nd_update(tensor, indices, updates):
        out = np.array(np.asarray(tensor), copy=True)
        out[tuple(np.asarray(indices).T)] = np.asarray(updates)
        return T(out)
    tf.tensor_scatter_nd_update = tensor_scatter_nd_update

    def scatter_nd(indices, updates, shape):
        out = np.zeros([int(s) for s in shape], dtype=np.asarray(updates).dtype)
        np.add.at(out, tuple(np.asarray(indices).T), np.asarray(updates))
        return T(out)
    tf.scatter_nd = scatter_nd

    def meshgrid(*xs, indexing="xy"):
        return [T(a) for a in np.meshgrid(*[np.asarray(x) for x in xs], indexing=indexing)]
    tf.meshgrid = meshgrid

    def gather(params, indices, axis=0):
        return T(_gather0(params, indices))
    tf.gather = gather

    def unique(x):
        vals, idx = _unique_first_occurrence(x)
        return T(vals), T(idx)
    tf.unique = unique

    math = types.ModuleType("tensorflow.math")
    math.unsorted_segment_sum = lambda d, i, num_segments: T(_segment_sum(d, i, int(num_segments)))
    math.unsorted_segment_mean = lambda d, i, num_segments: T(_segment_mean(d, i, int(num_segments)))
    math.unsorted_segment_max = lambda d, i, num_segments: T(_segment_max(d, i, int(num_segments)))
    math.unsorted_segment_min = lambda d, i, num_segments: T(_segment_min(d, i, int(num_segments)))
    math.logical_or = lambda a, b: T(np.logical_or(np.asarray(a), np.asarray(b)))
    math.logical_and = lambda a, b: T(np.logical_and(np.asarray(a), np.asarray(b)))
    math.is_inf = lambda x: T(np.isinf(np.asarray(x)))
    math.is_nan = lambda x: T(np.isnan(np.asarray(x)))
    math.sqrt = lambda x: (T(np.sqrt(np.asarray(x))) if np.ndim(x) else np.sqrt(np.float32(x)))
    math.floordiv = lambda a, b: T(np.asarray(a) // np.asarray(b))
    math.floormod = lambda a, b: T(np.asarray(a) % np.asarray(b))
    math.segment_sum = lambda d, i: T(_segment_sum(d, i, int(np.max(np.asarray(i))) + 1))
    math.cumsum = lambda x, axis=0: T(np.cumsum(np.asarray(x), axis=axis))
    math.minimum = lambda a, b: T(np.minimum(np.asarray(a), np.asarray(b)))
    math.ceil = lambda x: T(np.ceil(np.asarray(x)))
    math.reduce_min = lambda x, axis=None: _red(np.min, x, axis)
    math.reduce_max = lambda x, axis=None: _red(np.max, x, axis)
    math.__getattr__ = lambda name: _unsupported("tf.math." + name)
    tf.math = math

    nn = types.ModuleType("tensorflow.nn")
    nn.relu = lambda x: T(np.maximum(np.asarray(x), np.float32(0)))
    nn.l2_normalize = lambda x, axis=-1: T(_l2_normalize_last_axis(x))

    def softmax(logits, axis=-1):
        x = np.asarray(logits, dtype=np.float32)
        e = np.exp(x - np.max(x, axis=axis, keepdims=True)).astype(np.float32)
        return T((e / np.sum(e, axis=axis, keepdims=True, dtype=np.float32)).astype(np.float32))
    nn.softmax = softmax
    nn.leaky_relu = lambda x, alpha=0.2: T(np.where(np.asarray(x) > 0, np.asarray(x),
                                                    np.float32(alpha) * np.asarray(x)).astype(np.float32))
    nn.sigmoid = lambda x: T((1 / (1 + np.exp(-np.asarray(x, np.float32)))).astype(np.float32))
    nn.__getattr__ = lambda name: _unsupported("tf.nn." + name)
    tf.nn = nn

    tf.sqrt = lambda x: (T(np.sqrt(np.asarray(x))) if np.ndim(x) else np.sqrt(np.float32(x)))
    tf.transpose = lambda x, perm=None: T(np.transpose(np.asarray(x), perm))
    tf.tile = lambda x, multiples: T(np.tile(np.asarray(x), [int(m) for m in multiples]))

    def eye(num_rows, num_columns=None, batch_shape=None, dtype=np.float32):
        m = np.eye(int(num_rows), int(num_rows if num_columns is None else num_columns), dtype=dtype)
        if batch_shape is not None:
            m = np.tile(m, [int(b) for b in batch_shape] + [1, 1])
        return T(m)
    tf.eye = eye

    def norm(x, ord="euclidean", axis=None, keepdims=False):
        # tf.norm(ord="euclidean", axis=[-2, -1]): the Frobenius norm of every matrix, sqrt of the sum of squares in float32
        assert ord == "euclidean" and axis is not None and [int(a) for a in axis] == [-2, -1]
        x = np.asarray(x, dtype=np.float32)
        out = np.zeros(x.shape[:-2], dtype=np.float32)
        for b in np.ndindex(*x.shape[:-2]):
            acc = np.float32(0)
            for v in x[b].reshape(-1):
                acc = np.float32(acc + v * v)
            out[b] = np.sqrt(acc)
        return T(out.reshape(x.shape[:-2] + (1, 1)) if keepdims else out)
    tf.norm = norm

    sparse = types.ModuleType("tensorflow.sparse")

    class SparseTensor(object):
        """tf.SparseTensor of rank 2: indices [nnz, 2] int64, values [nnz], dense_shape; no implicit ordering."""

        def __init__(self, indices, values, dense_shape):
            self.indices = np.asarray(indices, dtype=np.int64).reshape(-1, 2)
            self.values = np.asarray(values)
            self.dense_shape = [int(d) for d in np.asarray([int(v) for v in dense_shape])]

        def __mul__(self, other):
            # SparseTensor * dense: the dense operand is read at the stored positions only (sparse_dense_cwise_mul)
            d = np.asarray(other)
            vals = np.empty_like(self.values)
            for k in range(self.indices.shape[0]):
                i, j = self.indices[k]
                vals[k] = self.values[k] * d[i, j]
            return SparseTensor(self.indices, vals, self.dense_shape)

    def reorder(sp):
        """tf.sparse.reorder: canonical row-major order of the indices (stable for repeated indices)."""
        order = sorted(range(sp.indices.shape[0]), key=lambda k: (int(sp.indices[k, 0]), int(sp.indices[k, 1])))
        return SparseTensor(sp.indices[order], sp.values[order], sp.dense_shape)

    def to_dense(sp):
        # repeated indices add up here, like tf_sparse's SparseMatrix.to_dense (scatter-add); tf.sparse.to_dense's default
        # validate_indices would reject them instead, so an adjacency with duplicate edges pins the summing semantics
        out = np.zeros(sp.dense_shape, dtype=sp.values.dtype)
        for k in range(sp.indices.shape[0]):
            i, j = sp.indices[k]
            out[i, j] = out[i, j] + sp.values[k]
        return T(out)

    def transpose(sp, perm=None):
        assert perm is None or [int(p) for p in perm] == [1, 0]
        return reorder(SparseTensor(sp.indices[:, ::-1], sp.values, sp.dense_shape[::-1]))

    def sparse_dense_matmul(sp, dense):
        d = np.asarray(dense)
        out = np.zeros((sp.dense_shape[0], d.shape[1]), dtype=np.result_type(sp.values.dtype, d.dtype))
        for k in range(sp.indices.shape[0]):              # accumulated entry by entry in index order
            i, j = sp.indices[k]
            out[i] = out[i] + sp.values[k] * d[j]
        return T(out)

    def sparse_reduce_sum(sp, axis=None):
        assert axis is not None and int(axis) in (-1, 1), "only the row sums are restated"
        out = np.zeros(sp.dense_shape[0], dtype=sp.values.dtype)
        for k in range(sp.indices.shape[0]):
            out[sp.indices[k, 0]] = out[sp.indices[k, 0]] + sp.values[k]
        return T(out)

    sparse.SparseTensor = SparseTensor
    tf.SparseTensor = SparseTensor
    sparse.reorder = reorder
    sparse.to_dense = to_dense
    sparse.transpose = transpose
    sparse.sparse_dense_matmul = sparse_dense_matmul
    sparse.reduce_sum = sparse_reduce_sum

    class Variable(object):
        pass
    tf.Variable = Variable
    sparse.__getattr__ = lambda name: _unsupported("tf.sparse." + name)
    tf.sparse = sparse
    tf.__getattr__ = lambda name: _unsupported("tf." + name)
    return tf


def _pow(x, p):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.power(x, x.dtype.type(p))


def _add_n(xs):
    acc = np.asarray(xs[0])
    for x in xs[1:]:
        acc = acc + np.asarray(x)
    return acc


def _red(fn, x, axis):
    r = fn(np.asarray(x), axis=axis)
    return T(r) if np.ndim(r) else r


def build_tf_sparse():
    """tf_sparse >= 0.0.17 [UNVERIFIED restatement]: COO, no sort, no merge; add_diag appends the diagonal."""
    tfs = types.ModuleType("tf_sparse")

    class DiagMatrix(object):
        def __init__(self, d):
            self.d = np.asarray(d)

        def __matmul__(self, other):                      # diags(d) @ A : scale rows
            return SparseMatrix(other.index, T(self.d[np.asarray(other.index[0])] * np.asarray(other.value)), other.shape)

    class SparseMatrix(object):
        def __init__(self, index, value=None, shape=None, merge=False):
            self.index = T(np.asarray(index, dtype=np.int32).reshape(2, -1))
            nnz = self.index.shape[1]
            self.value = T(np.ones([nnz], np.float32)) if value is None else T(np.asarray(value, dtype=np.float32))
            if shape is None:
                n = int(np.max(self.index)) + 1
                shape = [n, n]
            self._shape = T(np.array([int(s) for s in np.asarray(shape)], dtype=np.int64))

        @property
        def shape(self):
            return [int(s) for s in self._shape]

        def add_diag(self, w):
            # [UNVERIFIED, SURVEY.md 8c] self + diags(w * ones): the diagonal entries are APPENDED after the existing ones,
            # in node order, without merging duplicates (the order utils/graph_utils.py:350-366 add_self_loop_edge uses)
            n = min(self.shape)
            d = np.arange(n, dtype=np.int32)
            index = np.concatenate([np.asarray(self.index), np.stack([d, d])], axis=1)
            value = np.concatenate([np.asarray(self.value), np.full([n], w, dtype=np.float32)])
            return SparseMatrix(index, value, self.shape)

        def _segment_ids(self, axis):
            if axis in (-1, 1):
                return np.asarray(self.index[0]), self.shape[0]      # reduce over columns: one value per row
            return np.asarray(self.index[1]), self.shape[1]

        def segment_sum(self, axis=-1):
            ids, n = self._segment_ids(axis)
            return T(_segment_sum(np.asarray(self.value), ids, n))

        def segment_softmax(self, axis=-1):
            # nn/kernel/segment.py:26-33 applied to the values: max, exp(v - max), sum + 1e-8, divide
            ids, n = self._segment_ids(axis)
            v = np.asarray(self.value)
            mx = _segment_max(v, ids, n)
            e = np.exp(v - mx[ids]).astype(np.float32)
            den = (_segment_sum(e, ids, n) + np.float32(1e-8)).astype(np.float32)
            return SparseMatrix(self.index, (e / den[ids]).astype(np.float32), self.shape)

        def dropout(self, rate, training=False):
            assert not (training and rate > 0.0)
            return self

        def matmul(self, h, num_or_size_splits=None):
            # [UNVERIFIED] gather(h, col) * value[:, None] -> unsorted_segment_sum by row (the legacy path kept as comments in
            # the reference: nn/conv/gcn.py:175-176, gat.py:91-109)
            h = np.asarray(h, dtype=np.float32)
            msg = (_gather0(h, np.asarray(self.index[1])) * np.asarray(self.value)[:, None]).astype(np.float32)
            return T(_segment_sum(msg, np.asarray(self.index[0]), self.shape[0]))

        __array_ufunc__ = None                            # dense @ SparseMatrix must reach __rmatmul__

        def to_dense(self):
            # scatter-add of the entries: duplicates add up
            out = np.zeros(self.shape, dtype=np.float32)
            idx, val = np.asarray(self.index), np.asarray(self.value)
            for k in range(idx.shape[1]):
                out[idx[0, k], idx[1, k]] = out[idx[0, k], idx[1, k]] + val[k]
            return T(out)

        def transpose(self):
            return SparseMatrix(np.asarray(self.index)[::-1], self.value, self.shape[::-1])

        def __matmul__(self, other):
            if isinstance(other, DiagMatrix):             # A @ diags(d) : scale columns
                return SparseMatrix(self.index, T(np.asarray(self.value) * other.d[np.asarray(self.index[1])]), self.shape)
            if isinstance(other, SparseMatrix):           # sparse @ sparse: the non-zero entries of the product, row-major
                prod = np.asarray(self.matmul(other.to_dense()))
                r, c = np.nonzero(prod)
                return SparseMatrix(np.stack([r, c]), prod[r, c], [self.shape[0], other.shape[1]])
            return self.matmul(other)

        def __rmatmul__(self, other):
            # dense @ sparse: out[:, j] += dense[:, i] * v for every entry (i, j, v) in stored order
            d = np.asarray(other, dtype=np.float32)
            out = np.zeros((d.shape[0], self.shape[1]), dtype=np.float32)
            idx, val = np.asarray(self.index), np.asarray(self.value)
            for k in range(idx.shape[1]):
                out[:, idx[1, k]] = out[:, idx[1, k]] + d[:, idx[0, k]] * val[k]
            return T(out)

    tfs.SparseMatrix = SparseMatrix
    tfs.diags = lambda d: DiagMatrix(d)
    tfs.shape = lambda x: list(np.shape(x)) if not isinstance(x, SparseMatrix) else x.shape
    tfs.__getattr__ = lambda name: _unsupported("tf_sparse." + name)
    return tfs


def install(reference_root):
    """Put the shims and stub packages into sys.modules so individual reference files can be imported without
    running tf_geometric/__init__.py (which pulls in keras layers, datasets and downloads)."""
    import os
    sys.modules["tensorflow"] = build_tensorflow()
    sys.modules["tf_sparse"] = build_tf_sparse()
    pkg_root = os.path.join(reference_root, "tf_geometric")
    for name, sub in (("tf_geometric", ""), ("tf_geometric.nn", "nn"), ("tf_geometric.nn.kernel", "nn/kernel"),
                      ("tf_geometric.nn.conv", "nn/conv"), ("tf_geometric.utils", "utils")):
        mod = types.ModuleType(name)
        mod.__path__ = [os.path.join(pkg_root, sub)]
        sys.modules[name] = mod
    import importlib
    mr = importlib.import_module("tf_geometric.nn.kernel.map_reduce")
    for n in ("mean_reducer", "max_reducer", "sum_reducer", "identity_mapper", "neighbor_count_mapper", "sum_updater",
              "identity_updater", "aggregate_neighbors"):
        setattr(sys.modules["tf_geometric.nn"], n, getattr(mr, n))
    return T
