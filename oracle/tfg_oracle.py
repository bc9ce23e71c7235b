# coding=utf-8
"""
CPU ORACLE (numpy) for the tf_geometric message-passing hot path.

  *** TEST INFRASTRUCTURE ONLY. ***  Nothing under ``tf_geometric_b200/`` may import this module.
  Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference`` legs of
  ``bench.py`` use it, and only as the checker / the timed CPU arm.

PARITY PINNING STATUS
  The reference (CrawlScript/tf_geometric @4539f11) ships *no* tests and no golden vectors for
  this path, and neither TensorFlow nor the un-vendored dependency ``tf_sparse`` (setup.py:25, ">= 0.0.17") can be
  imported here.  The oracle is pinned two ways (see tests/golden/README.md):
    (1) tests/golden/ref_exec_*.npz - the reference's OWN Python functions (nn/kernel/*.py, nn/conv/{gcn,gat,
        graph_sage,appnp}.py, utils/graph_utils.py) executed here over a numpy shim of the TF ops they call
        (tools/gen_golden_from_reference.py).  That pins call order, quirks and the in-repo arithmetic; it does
        NOT pin TensorFlow's kernels or tf_sparse themselves, whose semantics are restated from their public
        documentation:  => "parity unpinned" for the TF/tf_sparse half.
    (2) the tiny hard-coded fixtures of the reference's README/demos (SURVEY.md section 4) and the derived KAT of
        SURVEY.md section 8c.

TF op semantics restated here (TensorFlow 2.x CPU kernels):
  * tf.gather(params, ids)                      -> params[ids]  (out-of-range raises on CPU)
  * tf.math.unsorted_segment_sum(d, ids, n)     -> sequential float32 adds in input order, empty segment = 0,
                                                   negative ids are dropped.
  * tf.math.unsorted_segment_mean               -> unsorted_segment_sum / maximum(count, 1)
  * tf.math.unsorted_segment_max / _min         -> empty segment = lowest()/max() of the dtype
  * tf.unique                                   -> first-occurrence order, plus inverse index

All floating point arithmetic is float32, indices int32 (data/graph.py:22-23,58-66).
Every function cites the reference file:line it restates (paths relative to tf_geometric/ of the reference, CrawlScript/tf_geometric).
"""
import numpy as np

F32 = np.float32
I32 = np.int32
FLT_LOWEST = np.finfo(np.float32).min
FLT_MAX = np.finfo(np.float32).max


# --------------------------------------------------------------------------------------------------------------
# TensorFlow op semantics
# --------------------------------------------------------------------------------------------------------------

def _as_f32(a):
    return np.ascontiguousarray(a, dtype=F32)


def gather(params, ids):
    """tf.gather on axis 0."""
    ids = np.asarray(ids)
    if ids.size and (ids.min() < 0 or ids.max() >= params.shape[0]):
        raise IndexError("gather index out of range (TF-CPU raises InvalidArgument)")
    return params[ids]


def unsorted_segment_sum(data, segment_ids, num_segments):
    """tf.math.unsorted_segment_sum, CPU kernel: out[ids[i]] += data[i] for i = 0..n-1 in order, fp32."""
    data = np.asarray(data)
    segment_ids = np.asarray(segment_ids)
    out = np.zeros((int(num_segments),) + data.shape[1:], dtype=data.dtype)
    keep = segment_ids >= 0
    if not keep.all():
        data, segment_ids = data[keep], segment_ids[keep]
    if segment_ids.size and segment_ids.max() >= num_segments:
        raise IndexError("segment id out of range")
    np.add.at(out, segment_ids, data)  # unbuffered, applied in index order -> sequential fp32 rounding
    return out


def unsorted_segment_mean(data, segment_ids, num_segments):
    """tf.math.unsorted_segment_mean = segment_sum(data) / maximum(segment_sum(ones), 1)."""
    data = np.asarray(data)
    s = unsorted_segment_sum(data, segment_ids, num_segments)
    cnt = unsorted_segment_sum(np.ones(len(segment_ids), dtype=data.dtype), segment_ids, num_segments)
    cnt = np.maximum(cnt, data.dtype.type(1))
    return (s / cnt.reshape((-1,) + (1,) * (data.ndim - 1))).astype(data.dtype)


def unsorted_segment_max(data, segment_ids, num_segments):
    """tf.math.unsorted_segment_max: empty segment -> numeric_limits<T>::lowest()."""
    data = np.asarray(data)
    low = np.finfo(data.dtype).min if data.dtype.kind == "f" else np.iinfo(data.dtype).min
    out = np.full((int(num_segments),) + data.shape[1:], low, dtype=data.dtype)
    np.maximum.at(out, np.asarray(segment_ids), data)
    return out


def unsorted_segment_min(data, segment_ids, num_segments):
    data = np.asarray(data)
    high = np.finfo(data.dtype).max if data.dtype.kind == "f" else np.iinfo(data.dtype).max
    out = np.full((int(num_segments),) + data.shape[1:], high, dtype=data.dtype)
    np.minimum.at(out, np.asarray(segment_ids), data)
    return out


def tf_unique(x):
    """tf.unique: values in first-occurrence order + index of each input element into them."""
    x = np.asarray(x)
    uniq_sorted, first_pos, inverse_sorted = np.unique(x, return_index=True, return_inverse=True)
    order = np.argsort(first_pos, kind="stable")          # sorted-unique slot -> first-occurrence rank
    rank_of_sorted_slot = np.empty_like(order)
    rank_of_sorted_slot[order] = np.arange(len(order))
    return uniq_sorted[order], rank_of_sorted_slot[inverse_sorted].astype(I32)


def relu(x):
    return np.maximum(x, F32(0))


def l2_normalize(x, eps=1e-12):
    """tf.nn.l2_normalize(x, axis=-1): x * rsqrt(max(sum(x^2), eps))."""
    sq = np.sum(x * x, axis=-1, keepdims=True, dtype=F32)
    return (x * (F32(1) / np.sqrt(np.maximum(sq, F32(eps))))).astype(F32)


# --------------------------------------------------------------------------------------------------------------
# nn/kernel/map_reduce.py
# --------------------------------------------------------------------------------------------------------------

def identity_mapper(repeated_x, neighbor_x, edge_weight=None):          # map_reduce.py:7-8
    return neighbor_x


def neighbor_count_mapper(repeated_x, neighbor_x, edge_weight=None):    # map_reduce.py:11-12
    return np.ones([neighbor_x.shape[0], 1], dtype=F32)


def gcn_mapper(repeated_x, neighbor_x, edge_weight=None):               # nn/conv/gcn.py:221-222
    return (neighbor_x * np.asarray(edge_weight, dtype=F32)[:, None]).astype(F32)


def sum_reducer(neighbor_msg, node_index, num_nodes=None):              # map_reduce.py:15-16
    return unsorted_segment_sum(neighbor_msg, node_index, num_nodes)


def mean_reducer(neighbor_msg, node_index, num_nodes=None):             # map_reduce.py:27-28
    return unsorted_segment_mean(neighbor_msg, node_index, num_nodes)


def max_reducer(neighbor_msg, node_index, num_nodes=None):              # map_reduce.py:38-42 (TF2 branch)
    if num_nodes is None:
        num_nodes = int(np.max(node_index)) + 1
    return unsorted_segment_max(neighbor_msg, node_index, num_nodes)


def sum_updater(x, reduced_neighbor_msg):                               # map_reduce.py:19-20
    return x + reduced_neighbor_msg


def identity_updater(x, reduced_neighbor_msg):                          # map_reduce.py:23-24
    return reduced_neighbor_msg


def aggregate_neighbors(x, edge_index, edge_weight=None, mapper=identity_mapper,
                        reducer=sum_reducer, updater=sum_updater, num_nodes=None):
    """map_reduce.py:45-73.  Note `tf.shape(edge_index)[0] == 0` only triggers for a rank-1 empty tensor."""
    edge_index = np.asarray(edge_index)
    if edge_index.shape[0] == 0:                                        # :57-58
        return x
    row, col = edge_index[0], edge_index[1]                             # :60
    repeated_x = gather(x, row)                                         # :62
    neighbor_x = gather(x, col)                                         # :63
    neighbor_msg = mapper(repeated_x, neighbor_x, edge_weight=edge_weight)  # :65
    if num_nodes is None:
        num_nodes = x.shape[0]                                          # :67-68
    reduced_msg = reducer(neighbor_msg, row, num_nodes=num_nodes)       # :70
    return updater(x, reduced_msg)                                      # :71


# --------------------------------------------------------------------------------------------------------------
# nn/kernel/segment.py
# --------------------------------------------------------------------------------------------------------------

def segment_softmax(data, segment_ids, num_segments):
    """segment.py:26-33: max -> gather -> exp -> sum (+1e-8) -> gather -> divide."""
    data = _as_f32(data)
    max_values = unsorted_segment_max(data, segment_ids, num_segments)
    e = np.exp(data - max_values[segment_ids]).astype(F32)
    denominator = unsorted_segment_sum(e, segment_ids, num_segments) + F32(1e-8)
    return (e / denominator[segment_ids]).astype(F32)


def segment_count(index, num_segments=None):
    """segment.py:36-40: histogram in the dtype of `index`."""
    index = np.asarray(index)
    if num_segments is None:
        num_segments = int(index.max()) + 1
    return unsorted_segment_sum(np.ones_like(index), index, num_segments)


# --------------------------------------------------------------------------------------------------------------
# utils/graph_utils.py (integer edge preprocessing)
# --------------------------------------------------------------------------------------------------------------

def convert_edge_index_to_edge_hash(edge_index, num_nodes=None):
    """graph_utils.py:14-43: hash = num_nodes * row + col in int64; num_nodes defaults to max id + 1."""
    ei = np.asarray(edge_index).astype(np.int64)
    if num_nodes is None:
        num_nodes = int(ei.max()) + 1
    return np.int64(num_nodes) * ei[0] + ei[1], int(num_nodes)


def convert_edge_hash_to_edge_index(edge_hash, num_nodes):
    """graph_utils.py:46-64."""
    edge_hash = np.asarray(edge_hash, dtype=np.int64)
    return np.stack([edge_hash // num_nodes, edge_hash % num_nodes], axis=0).astype(I32)


def merge_duplicated_edge(edge_index, edge_props=None, merge_modes=None):
    """graph_utils.py:67-125: tf.unique on the hash (first-occurrence order), props merged per unique slot."""
    if edge_props is not None and len(edge_props) > 0 and merge_modes is None:
        merge_modes = ["sum"] * len(edge_props)
    edge_index = np.asarray(edge_index, dtype=I32)
    edge_hash, hash_n = convert_edge_index_to_edge_hash(edge_index)
    uniq_hash, uniq_idx = tf_unique(edge_hash)
    uniq_edge_index = convert_edge_hash_to_edge_index(uniq_hash, hash_n)
    if edge_props is None:
        return uniq_edge_index, None
    fn = {"min": unsorted_segment_min, "max": unsorted_segment_max,
          "mean": unsorted_segment_mean, "sum": unsorted_segment_sum}
    out = []
    for prop, mode in zip(edge_props, merge_modes):
        if prop is None:
            out.append(None)
        else:
            if mode not in fn:
                raise Exception("wrong merge mode: {}".format(mode))
            out.append(fn[mode](np.asarray(prop), uniq_idx, len(uniq_hash)))
    return uniq_edge_index, out


def convert_edge_to_upper(edge_index, edge_props=None, merge_modes=None):
    """graph_utils.py:128-151: (min(u,v), max(u,v)) then merge duplicates."""
    edge_index = np.asarray(edge_index, dtype=I32)
    upper = np.stack([edge_index.min(axis=0), edge_index.max(axis=0)], axis=0)
    return merge_duplicated_edge(upper, edge_props, merge_modes)


def convert_edge_to_directed(edge_index, edge_props=None, merge_modes=None):
    """graph_utils.py:155-212: upper edges followed by the mirrored non-self-loop upper edges."""
    edge_index = np.asarray(edge_index, dtype=I32)
    if edge_props is not None and len(edge_props) > 0 and merge_modes is None:
        merge_modes = ["sum"] * len(edge_props)
    upper, upper_props = convert_edge_to_upper(edge_index, edge_props, merge_modes)
    mask = upper[0] != upper[1]
    if not mask.any():                                                  # :205-207
        return edge_index, edge_props
    lower = np.stack([upper[1][mask], upper[0][mask]], axis=0)
    out_index = np.concatenate([upper, lower], axis=1)
    if edge_props is None:
        return out_index, None
    out_props = []
    for prop, up in zip(edge_props, upper_props):
        out_props.append(None if prop is None else np.concatenate([up, up[mask]], axis=0))
    return out_index, out_props


def remove_self_loop_edge(edge_index, edge_weight=None):
    """graph_utils.py:252-269."""
    edge_index = np.asarray(edge_index)
    mask = edge_index[0] != edge_index[1]
    return edge_index[:, mask], (None if edge_weight is None else np.asarray(edge_weight)[mask])


def add_self_loop_edge(edge_index, num_nodes, edge_weight=None, fill_weight=1.0):
    """graph_utils.py:350-366: diagonal appended AFTER the existing edges, no dedup."""
    edge_index = np.asarray(edge_index, dtype=I32).reshape(2, -1)
    diag = np.arange(num_nodes, dtype=I32)
    out_index = np.concatenate([edge_index, np.stack([diag, diag])], axis=1)
    if edge_weight is None:
        return out_index, None
    out_w = np.concatenate([_as_f32(edge_weight), np.full([num_nodes], fill_weight, dtype=F32)])
    return out_index, out_w


def _remove_inf_and_nan(x):                                             # nn/conv/gcn.py:23-29
    return np.where(np.isinf(x) | np.isnan(x), F32(0), x).astype(F32)


def adj_norm_edge(edge_index, num_nodes, edge_weight=None, add_self_loop=False):
    """graph_utils.py:914-943 (live, tf_sparse-free twin of gcn_norm_adj's default path)."""
    edge_index = np.asarray(edge_index, dtype=I32)
    if edge_weight is None:
        edge_weight = np.ones([edge_index.shape[1]], dtype=F32)
    if add_self_loop:
        edge_index, edge_weight = add_self_loop_edge(edge_index, num_nodes, edge_weight, 1.0)
    row, col = edge_index
    deg = unsorted_segment_sum(_as_f32(edge_weight), row, num_nodes)
    with np.errstate(divide="ignore", invalid="ignore"):
        dis = _remove_inf_and_nan(np.power(deg, F32(-0.5)))
    return edge_index, (dis[row] * _as_f32(edge_weight) * dis[col]).astype(F32)


def csr_build(row, col, num_rows):
    """Integer oracle for the destination-sorted CSR the backend caches: a STABLE sort by row.
    Returns rowptr[int64, N+1], col_sorted[int32], perm[int32] with row[perm] non-decreasing and ties in input
    order - so a per-row left-to-right sum reproduces unsorted_segment_sum's sequential rounding."""
    row = np.asarray(row, dtype=I32)
    perm = np.argsort(row, kind="stable").astype(I32)
    counts = np.bincount(row, minlength=num_rows).astype(np.int64)
    rowptr = np.zeros(num_rows + 1, dtype=np.int64)
    np.cumsum(counts, out=rowptr[1:])
    return rowptr, np.asarray(col, dtype=I32)[perm], perm


# --------------------------------------------------------------------------------------------------------------
# tf_sparse.SparseMatrix  [UNVERIFIED restatement - the package is not part of the reference]
# --------------------------------------------------------------------------------------------------------------

class SparseMatrix(object):
    """COO matrix with the subset of tf_sparse.SparseMatrix the reference calls (SURVEY.md section 8c).
    index int32 [2, nnz] (row = aggregation target), value float32 [nnz] (ones if None), no sort, no merge."""

    def __init__(self, index, value=None, shape=None):
        self.index = np.asarray(index, dtype=I32).reshape(2, -1)
        nnz = self.index.shape[1]
        self.value = np.ones([nnz], dtype=F32) if value is None else _as_f32(value)
        if shape is None:
            n = int(self.index.max()) + 1 if nnz else 0
            shape = [n, n]
        self.shape = [int(shape[0]), int(shape[1])]

    @property
    def row(self):
        return self.index[0]

    @property
    def col(self):
        return self.index[1]

    def segment_sum(self, axis=-1):
        if axis in (-1, 1):
            return unsorted_segment_sum(self.value, self.row, self.shape[0])
        return unsorted_segment_sum(self.value, self.col, self.shape[1])

    def segment_softmax(self, axis=-1):
        ids, n = (self.row, self.shape[0]) if axis in (-1, 1) else (self.col, self.shape[1])
        return SparseMatrix(self.index, segment_softmax(self.value, ids, n), self.shape)

    def add_diag(self, w):
        """A + diag(w): diagonal entries appended after the existing ones (same convention as
        graph_utils.add_self_loop_edge, and as the commented-out legacy `add_self_loop` at gcn.py:78)."""
        n = min(self.shape)
        index, value = add_self_loop_edge(self.index, n, self.value, fill_weight=w)
        return SparseMatrix(index, value, self.shape)

    def scale_rows(self, d):      # diags(d) @ A
        return SparseMatrix(self.index, (d[self.row] * self.value).astype(F32), self.shape)

    def scale_cols(self, d):      # A @ diags(d)
        return SparseMatrix(self.index, (self.value * d[self.col]).astype(F32), self.shape)

    def dropout(self, rate, training=False):
        if training and rate > 0.0:
            raise NotImplementedError("edge dropout uses the TF RNG stream; parity is defined for inference only")
        return self

    def matmul(self, h, num_or_size_splits=None):
        """A @ h = unsorted_segment_sum(gather(h, col) * value[:, None], row)  (legacy code kept in comments at
        gat.py:91-109, gcn.py:175-176).  Column splitting does not change any output element."""
        h = _as_f32(h)
        msg = (h[self.col] * self.value[:, None]).astype(F32)
        return unsorted_segment_sum(msg, self.row, self.shape[0])

    def __matmul__(self, h):
        return self.matmul(h)

    def to_dense(self):
        out = np.zeros(self.shape, dtype=F32)
        np.add.at(out, (self.row, self.col), self.value)
        return out


# --------------------------------------------------------------------------------------------------------------
# nn/conv/gcn.py
# --------------------------------------------------------------------------------------------------------------

def gcn_norm_adj(sparse_adj, norm="both", add_self_loop=True, sym=True, renorm=True, improved=False):
    """nn/conv/gcn.py:32-130 (cache handling omitted: it only memoises the returned triple)."""
    fill_weight = 2.0 if improved else 1.0                               # :62
    if sparse_adj.shape[0] != sparse_adj.shape[1]:                       # :65-69
        if add_self_loop:
            raise Exception("cannot set add_self_loop=True for GCN when sparse_adj.shape[0] != sparse_adj.shape[1]")
        if sym:
            raise Exception("cannot set sym=True for GCN when sparse_adj.shape[0] != sparse_adj.shape[1]")
    if add_self_loop and norm != "both":                                 # :71-72
        sparse_adj = sparse_adj.add_diag(fill_weight)
    with np.errstate(divide="ignore", invalid="ignore"):
        if norm == "both":                                               # :75-98
            if add_self_loop and renorm:
                sparse_adj = sparse_adj.add_diag(fill_weight)
            row_dis = _remove_inf_and_nan(np.power(sparse_adj.segment_sum(axis=-1), F32(-0.5)))
            if sym:
                col_dis = row_dis
            else:
                col_dis = _remove_inf_and_nan(np.power(sparse_adj.segment_sum(axis=0), F32(-0.5)))
            normed = sparse_adj.scale_rows(row_dis).scale_cols(col_dis)  # (D^-1/2 A) D^-1/2, :94
            if add_self_loop and not renorm:
                normed = normed.add_diag(fill_weight)                    # :97-98
        elif norm == "left":                                             # :101-109
            row_inv = _remove_inf_and_nan(np.power(sparse_adj.segment_sum(axis=-1), F32(-1)))
            normed = sparse_adj.scale_rows(row_inv)
        elif norm == "right":                                            # :112-119 (row sums, sic)
            col_inv = _remove_inf_and_nan(np.power(sparse_adj.segment_sum(axis=-1), F32(-1)))
            normed = sparse_adj.scale_cols(col_inv)
        else:
            raise Exception("wrong GCN norm type: {}".format(norm))
    return normed


def gcn_norm_edge(edge_index, num_nodes, edge_weight=None, renorm=True, improved=False):
    """nn/conv/gcn.py:180-196 (deprecated wrapper still used by gcn_graph_sage)."""
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [num_nodes, num_nodes]),
                          renorm=renorm, improved=improved)
    return normed.index, normed.value


def gcn(x, sparse_adj, kernel, bias=None, activation=None, norm="both", add_self_loop=True, sym=True,
        renorm=True, improved=False):
    """nn/conv/gcn.py:225-290 at inference (edge dropout inactive)."""
    normed = gcn_norm_adj(sparse_adj, norm, add_self_loop, sym, renorm, improved)
    h = _as_f32(x) if kernel is None else (_as_f32(x) @ _as_f32(kernel)).astype(F32)   # :266-272
    h = normed.matmul(h)                                                 # :280
    if bias is not None:
        h = h + _as_f32(bias)
    if activation is not None:
        h = activation(h)
    return h.astype(F32)


# --------------------------------------------------------------------------------------------------------------
# nn/conv/gat.py
# --------------------------------------------------------------------------------------------------------------

def gat(x, edge_index, query_kernel, query_bias, query_activation, key_kernel, key_bias, key_activation,
        kernel, bias=None, activation=None, num_heads=1, split_value_heads=True, return_attention=False):
    """nn/conv/gat.py:13-122 at inference, op for op (including the H*N-node virtual graph)."""
    x = _as_f32(x)
    num_nodes = x.shape[0]
    edge_index, _ = add_self_loop_edge(edge_index, num_nodes)            # :43
    row, col = edge_index
    Q = (x @ _as_f32(query_kernel)).astype(F32) + _as_f32(query_bias)    # :52-53
    if query_activation is not None:
        Q = query_activation(Q)
    Q = Q[row]                                                           # :56
    K = (x @ _as_f32(key_kernel)).astype(F32) + _as_f32(key_bias)        # :61-62
    if key_activation is not None:
        K = key_activation(K)
    K = K[col]                                                           # :65
    V = (x @ _as_f32(kernel)).astype(F32)                                # :70
    Q_ = np.concatenate(np.split(Q, num_heads, axis=-1), axis=0)         # :73
    K_ = np.concatenate(np.split(K, num_heads, axis=-1), axis=0)         # :74
    qk_edge_index_ = np.concatenate([edge_index.astype(np.int64) + i * num_nodes for i in range(num_heads)], axis=1)
    scale = np.sqrt(F32(Q_.shape[-1]))                                   # :78
    att_score_ = (np.sum(Q_ * K_, axis=-1, dtype=F32) / scale).astype(F32)   # :79
    num_nodes_ = num_nodes * num_heads
    att = segment_softmax(att_score_, qk_edge_index_[0], num_nodes_)     # :83-84
    V_ = np.concatenate(np.split(V, num_heads, axis=-1), axis=0)         # :87
    msg = (V_[qk_edge_index_[1]] * att[:, None]).astype(F32)
    h_ = unsorted_segment_sum(msg, qk_edge_index_[0], num_nodes_)        # :89
    if split_value_heads:
        h = np.concatenate(np.split(h_, num_heads, axis=0), axis=-1)     # :112
    else:
        parts = np.split(h_, num_heads, axis=0)
        acc = parts[0]
        for p in parts[1:]:                                              # tf.add_n, :114
            acc = acc + p
        h = acc / F32(num_heads)
    if bias is not None:
        h = h + _as_f32(bias)
    if activation is not None:
        h = activation(h)
    h = h.astype(F32)
    if return_attention:
        return h, att.reshape(num_heads, -1).T.copy()                    # [E', H]
    return h


# --------------------------------------------------------------------------------------------------------------
# nn/conv/graph_sage.py
# --------------------------------------------------------------------------------------------------------------

def _sage_tail(x_self, neighbor_msg, bias, activation, concat, normalize):
    h = np.concatenate([x_self, neighbor_msg], axis=1) if concat else x_self + neighbor_msg
    if bias is not None:
        h = h + _as_f32(bias)
    if activation is not None:
        h = activation(h)
    if normalize:
        h = l2_normalize(h)
    return h.astype(F32)


def _sage_plain(reducer, x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias, activation, concat,
                normalize):
    x = _as_f32(x)
    num_nodes = x.shape[0]
    row, col = np.asarray(edge_index, dtype=I32)
    neighbor_x = x[col]                                                  # graph_sage.py:36
    if edge_weight is not None:
        neighbor_x = gcn_mapper(None, neighbor_x, edge_weight)           # :38-39
    reduced = reducer(neighbor_x, row, num_nodes=num_nodes)              # :41 / :96
    neighbor_msg = (reduced @ _as_f32(neighbor_kernel)).astype(F32)      # :43
    x_self = (x @ _as_f32(self_kernel)).astype(F32)                      # :44
    return _sage_tail(x_self, neighbor_msg, bias, activation, concat, normalize)


def mean_graph_sage(x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias=None, activation=None,
                    concat=True, normalize=False):
    """nn/conv/graph_sage.py:9-60."""
    return _sage_plain(mean_reducer, x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias, activation,
                       concat, normalize)


def sum_graph_sage(x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias=None, activation=None,
                   concat=True, normalize=False):
    """nn/conv/graph_sage.py:64-115."""
    return _sage_plain(sum_reducer, x, edge_index, edge_weight, self_kernel, neighbor_kernel, bias, activation,
                       concat, normalize)


def gcn_graph_sage(x, edge_index, edge_weight, kernel, bias=None, activation=None, normalize=False, cache=None):
    """nn/conv/graph_sage.py:118-161.  Quirks restated literally: a provided edge_weight is replaced by ones
    (:139-140) and `cache` is passed POSITIONALLY into gcn_norm_edge's `renorm` slot (:142), so
    renorm = bool(cache): None or {} -> D^-1/2 A D^-1/2 + I ; non-empty dict -> renormalisation trick."""
    x = _as_f32(x)
    num_nodes = x.shape[0]
    edge_index = np.asarray(edge_index, dtype=I32)
    if edge_weight is not None:
        edge_weight = np.ones([edge_index.shape[1]], dtype=F32)
    upd_index, normed_w = gcn_norm_edge(edge_index, num_nodes, edge_weight, renorm=bool(cache))
    row, col = upd_index
    reduced = sum_reducer(gcn_mapper(None, x[col], normed_w), row, num_nodes=num_nodes)
    h = (reduced @ _as_f32(kernel)).astype(F32)
    if bias is not None:
        h = h + _as_f32(bias)
    if activation is not None:
        h = activation(h)
    if normalize:
        h = l2_normalize(h)
    return h.astype(F32)


def _sage_pool(reducer, x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
               neighbor_mlp_bias, bias, activation, concat, normalize):
    x = _as_f32(x)
    num_nodes = x.shape[0]
    edge_index = np.asarray(edge_index, dtype=I32)
    if edge_weight is not None:                                          # :190-191 / :253-254
        edge_weight = np.ones([edge_index.shape[1]], dtype=F32)
    row, col = edge_index
    neighbor_x = gcn_mapper(None, x[col], edge_weight)                   # crashes for None, like the reference
    h = (neighbor_x @ _as_f32(neighbor_mlp_kernel)).astype(F32)          # per-EDGE dense layer
    if neighbor_mlp_bias is not None:
        h = h + _as_f32(neighbor_mlp_bias)
    if activation is not None:
        h = activation(h)
    reduced = reducer(h.astype(F32), row, num_nodes=num_nodes)
    from_neighbor = (reduced @ _as_f32(neighbor_kernel)).astype(F32)
    from_x = (x @ _as_f32(self_kernel)).astype(F32)
    return _sage_tail(from_x, from_neighbor, bias, activation, concat, normalize)


def mean_pool_graph_sage(x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                         neighbor_mlp_bias=None, bias=None, activation=None, concat=True, normalize=False):
    """nn/conv/graph_sage.py:164-225."""
    return _sage_pool(mean_reducer, x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                      neighbor_mlp_bias, bias, activation, concat, normalize)


def max_pool_graph_sage(x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                        neighbor_mlp_bias=None, bias=None, activation=None, concat=True, normalize=False):
    """nn/conv/graph_sage.py:228-287."""
    return _sage_pool(max_reducer, x, edge_index, edge_weight, self_kernel, neighbor_mlp_kernel, neighbor_kernel,
                      neighbor_mlp_bias, bias, activation, concat, normalize)


# --------------------------------------------------------------------------------------------------------------
# nn/conv/appnp.py
# --------------------------------------------------------------------------------------------------------------

def appnp(x, edge_index, edge_weight, kernels, biases, dense_activation=relu, activation=None, k=10, alpha=0.1):
    """nn/conv/appnp.py:11-92 at inference."""
    x = _as_f32(x)
    num_nodes = x.shape[0]
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [num_nodes, num_nodes]))   # :51-53
    h = x
    n_dense = len(kernels)
    for i, (kern, b) in enumerate(zip(kernels, biases)):                 # :64-81
        h = (h @ _as_f32(kern)).astype(F32)
        if b is not None:
            h = h + _as_f32(b)
        if i < n_dense - 1 and dense_activation is not None:
            h = dense_activation(h)
    h = h.astype(F32)
    out = h
    for _ in range(k):                                                   # :85-87
        out = normed.matmul(out)
        out = (out * F32(1.0 - alpha) + h * F32(alpha)).astype(F32)
    if activation is not None:
        out = activation(out)
    return out.astype(F32)


# --------------------------------------------------------------------------------------------------------------
# nn/conv/{sgc,ssgc,tagcn,gin,le_conv}.py  (SURVEY.md section 8f-1)
# --------------------------------------------------------------------------------------------------------------

def sgc(x, edge_index, edge_weight, k, kernel, bias=None, activation=None, renorm=True, improved=False):
    """nn/conv/sgc.py:10-61."""
    x = _as_f32(x)
    n = x.shape[0]
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [n, n]), renorm=renorm, improved=improved)
    h = (x @ _as_f32(kernel)).astype(F32)
    for _ in range(k):
        h = normed.matmul(h)
    if bias is not None:
        h = h + _as_f32(bias)
    if activation is not None:
        h = activation(h)
    return h.astype(F32)


def ssgc(x, edge_index, edge_weight, kernels=None, biases=None, k=10, alpha=0.1, dense_activation=relu, activation=None):
    """nn/conv/ssgc.py:11-99 at inference."""
    h = _as_f32(x)
    n = h.shape[0]
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [n, n]))
    if kernels is not None:
        nd = len(kernels)
        for i, (kern, b) in enumerate(zip(kernels, biases)):
            h = (h @ _as_f32(kern)).astype(F32)
            if b is not None:
                h = h + _as_f32(b)
            if i < nd - 1 and dense_activation is not None:
                h = dense_activation(h)
    h = h.astype(F32)
    output = (h * F32(alpha)).astype(F32)
    for _ in range(k):
        h = normed.matmul(h)
        output = (output + (F32(1 - alpha) * h / F32(k)).astype(F32)).astype(F32)
    if activation is not None:
        output = activation(output)
    return output.astype(F32)


def tagcn(x, edge_index, edge_weight, k, kernel, bias=None, activation=None, renorm=False, improved=False):
    """nn/conv/tagcn.py:10-51."""
    x = _as_f32(x)
    n = x.shape[0]
    normed = gcn_norm_adj(SparseMatrix(edge_index, edge_weight, [n, n]), renorm=renorm, improved=improved)
    xs = [x]
    for _ in range(k):
        xs.append(normed.matmul(xs[-1]))
    out = (np.concatenate(xs, axis=-1) @ _as_f32(kernel)).astype(F32)
    if bias is not None:
        out = out + _as_f32(bias)
    if activation is not None:
        out = activation(out)
    return out.astype(F32)


def gin(x, edge_index, mlp_model, eps=0.0):
    """nn/conv/gin.py:11-38."""
    x = _as_f32(x)
    n = x.shape[0]
    neighbor_h = SparseMatrix(edge_index, None, [n, n]).matmul(x)
    h = (x * F32(1.0 + eps) + neighbor_h).astype(F32)
    return mlp_model(h)


def le_conv(x, edge_index, edge_weight, self_kernel, self_bias, aggr_self_kernel, aggr_self_bias,
            aggr_neighbor_kernel, aggr_neighbor_bias, activation=None):
    """nn/conv/le_conv.py:5-52 - both aggregation terms are gathered by `col` (:40-41), literally."""
    x = _as_f32(x)
    edge_index = np.asarray(edge_index, dtype=I32)
    if edge_weight is None:
        edge_weight = np.ones([edge_index.shape[1]], dtype=F32)
    n = x.shape[0]
    self_h = (x @ _as_f32(self_kernel)).astype(F32)
    if self_bias is not None:
        self_h = self_h + _as_f32(self_bias)
    aggr_self_h = (x @ _as_f32(aggr_self_kernel)).astype(F32)
    if aggr_self_bias is not None:
        aggr_self_h = aggr_self_h + _as_f32(aggr_self_bias)
    aggr_neighbor_h = (x @ _as_f32(aggr_neighbor_kernel)).astype(F32)
    if aggr_neighbor_bias is not None:
        aggr_neighbor_h = aggr_neighbor_h + _as_f32(aggr_neighbor_bias)
    row, col = edge_index
    rep = ((aggr_self_h[col] - aggr_neighbor_h[col]) * _as_f32(edge_weight)[:, None]).astype(F32)
    h = self_h + unsorted_segment_sum(rep, row, n)
    if activation is not None:
        h = activation(h)
    return h.astype(F32)


def get_laplacian(edge_index, num_nodes, edge_weight, normalization_type, fill_weight=1.0):
    """utils/graph_utils.py:554-604, literally (for 'sym' it is D^-1/2 A D^-1/2 with self loops appended)."""
    edge_index = np.asarray(edge_index, dtype=I32)
    edge_weight = _as_f32(edge_weight)
    row, col = edge_index
    deg = unsorted_segment_sum(edge_weight, row, num_nodes)
    with np.errstate(divide="ignore", invalid="ignore"):
        if normalization_type is None:
            edge_index, edge_weight = add_self_loop_edge(edge_index, num_nodes, edge_weight, fill_weight=fill_weight)
            return edge_index, (_remove_inf_and_nan(deg)[edge_index[0]] - edge_weight).astype(F32)
        if normalization_type == 'sym':
            dis = _remove_inf_and_nan(np.power(deg, F32(-0.5)))
            normed = (dis[row] * edge_weight * dis[col]).astype(F32)
        else:
            inv = _remove_inf_and_nan((F32(1.0) / deg).astype(F32))
            normed = (inv[row] * edge_weight).astype(F32)
    return add_self_loop_edge(edge_index, num_nodes, normed, fill_weight=fill_weight)


def chebynet_norm_edge(edge_index, num_nodes, edge_weight, normalization_type="sym", lambda_max=2.0):
    """nn/conv/chebynet.py:17-43 (lambda_max passed in: 2.0 unless the caller computed the dynamic one)."""
    ei, w = remove_self_loop_edge(np.asarray(edge_index, dtype=I32), _as_f32(edge_weight))
    upd_index, upd_w = get_laplacian(ei, num_nodes, w, normalization_type)
    return upd_index, ((F32(2.0) * upd_w) / F32(lambda_max)).astype(F32)


def chebynet(x, edge_index, edge_weight, k, kernels, bias=None, activation=None, normalization_type="sym", lambda_max=2.0):
    """nn/conv/chebynet.py:63-137."""
    x = _as_f32(x)
    n = x.shape[0]
    if edge_weight is None:
        edge_weight = np.ones([np.asarray(edge_index).shape[1]], dtype=F32)
    ni, nw = chebynet_norm_edge(edge_index, n, edge_weight, normalization_type, lambda_max)
    adj = SparseMatrix(ni, nw, [n, n])
    t0 = x
    out = (t0 @ _as_f32(kernels[0])).astype(F32)
    if k > 1:
        t1 = adj.matmul(x)
        out = out + (t1 @ _as_f32(kernels[1])).astype(F32)
    if k > 2:
        for i in range(2, k):
            t2 = (adj.matmul(t1) * F32(2.0) - t0).astype(F32)
            out = out + (t2 @ _as_f32(kernels[i])).astype(F32)
            t0, t1 = t1, t2
    if bias is not None:
        out = out + _as_f32(bias)
    if activation is not None:
        out = activation(out)
    return out.astype(F32)


# --------------------------------------------------------------------------------------------------------------
# nn/pool/common_pool.py  (SURVEY.md section 8f-2)
# --------------------------------------------------------------------------------------------------------------

def _num_graphs(node_graph_index, num_graphs):
    return int(np.max(node_graph_index)) + 1 if num_graphs is None else int(num_graphs)


def mean_pool(x, node_graph_index, num_graphs=None):
    """common_pool.py:7-12: segment_sum / (float(segment_count) + 1e-8)."""
    n = _num_graphs(node_graph_index, num_graphs)
    cnt = segment_count(np.asarray(node_graph_index, dtype=I32), n)
    s = unsorted_segment_sum(_as_f32(x), node_graph_index, n)
    return (s / (cnt.astype(F32)[:, None] + F32(1e-8))).astype(F32)


def sum_pool(x, node_graph_index, num_graphs=None):
    return unsorted_segment_sum(_as_f32(x), node_graph_index, _num_graphs(node_graph_index, num_graphs))


def max_pool(x, node_graph_index, num_graphs=None):
    return unsorted_segment_max(_as_f32(x), node_graph_index, _num_graphs(node_graph_index, num_graphs))


def min_pool(x, node_graph_index, num_graphs=None):
    return unsorted_segment_min(_as_f32(x), node_graph_index, _num_graphs(node_graph_index, num_graphs))


# --------------------------------------------------------------------------------------------------------------
# float64 dense model used by property tests (NOT a restatement: an independent cross-check of the oracle)
# --------------------------------------------------------------------------------------------------------------

def dense_spmm_f64(index, value, shape, h):
    a = np.zeros(shape, dtype=np.float64)
    np.add.at(a, (index[0], index[1]), np.asarray(value, dtype=np.float64))
    return a @ np.asarray(h, dtype=np.float64)


# --------------------------------------------------------------------------------------------------------------
# Training-mode extras and samplers (SURVEY.md 8(f)3-4).
# The reference draws from TensorFlow's / numpy's global generators (tf.nn.dropout, tf.random.uniform,
# np.random.choice), which cannot be reproduced; the product uses the counter-based Philox4x32-10 generator instead
# and this section restates it, so that masks and samples are bit-exact oracle <-> kernels while the parity with the
# reference is about SEMANTICS (which elements may be kept, scaling, with/without replacement, output layout).
# Philox is pinned by the Random123 known-answer vectors in tests/test_oracle.py.
# --------------------------------------------------------------------------------------------------------------

_PHILOX_M0, _PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_PHILOX_W0, _PHILOX_W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32(counter, key, rounds=10):
    """Philox4x32 (Salmon et al., SC'11).  counter: uint32 [..., 4], key: uint32 [..., 2] -> uint32 [..., 4]."""
    c = [np.asarray(counter[..., i], dtype=np.uint32).copy() for i in range(4)]
    k0 = np.asarray(key[..., 0], dtype=np.uint32).copy()
    k1 = np.asarray(key[..., 1], dtype=np.uint32).copy()
    with np.errstate(over="ignore"):
        for _ in range(rounds):
            p0 = _PHILOX_M0 * c[0].astype(np.uint64)
            p1 = _PHILOX_M1 * c[2].astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _MASK32).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _MASK32).astype(np.uint32)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
            k0 = (k0 + _PHILOX_W0).astype(np.uint32)
            k1 = (k1 + _PHILOX_W1).astype(np.uint32)
    return np.stack(c, axis=-1)


def random_u32(seed, stream, idx):
    """Draw `idx` (uint64 array) of (seed, stream): counter = (idx >> 2 [lo, hi], stream, 0), lane idx & 3
    (tf_geometric_b200/csrc/rng.cuh random_u32)."""
    idx = np.asarray(idx, dtype=np.uint64)
    blk = idx >> np.uint64(2)
    counter = np.stack([(blk & _MASK32).astype(np.uint32), (blk >> np.uint64(32)).astype(np.uint32),
                        np.full(idx.shape, stream, np.uint32), np.zeros(idx.shape, np.uint32)], axis=-1)
    seed = int(seed)
    key = np.empty(idx.shape + (2,), np.uint32)
    key[..., 0] = seed & 0xFFFFFFFF
    key[..., 1] = (seed >> 32) & 0xFFFFFFFF
    out = philox4x32(counter, key)
    lane = (idx & np.uint64(3)).astype(np.int64)
    return np.take_along_axis(out, lane[..., None], axis=-1)[..., 0]


def random_uniform(seed, stream, idx):
    """uniform [0, 1) with 24 random bits, exactly representable in float32."""
    return (random_u32(seed, stream, idx) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def random_below(seed, stream, idx, n):
    return ((random_u32(seed, stream, idx).astype(np.uint64) * np.asarray(n, dtype=np.uint64)) >> np.uint64(32)).astype(np.int64)


RNG_STREAM_DROPOUT, RNG_STREAM_SAMPLER = 0, 1


def dropout_scale(n, rate, seed, stream=RNG_STREAM_DROPOUT):
    """tf.nn.dropout's multiplier per element: 1/(1-rate) where u >= rate, else 0."""
    if rate <= 0.0:
        return np.ones(n, F32)
    scale = F32(1.0) / (F32(1.0) - F32(rate))
    u = random_uniform(seed, stream, np.arange(n, dtype=np.uint64))
    return np.where(u >= F32(rate), scale, F32(0.0)).astype(F32)


def dropout(x, rate, seed, stream=RNG_STREAM_DROPOUT):
    """tf.nn.dropout(x, rate) (gcn.py:262 through tf_sparse's SparseMatrix.dropout, gat.py:85)."""
    x = _as_f32(x)
    return (x.reshape(-1) * dropout_scale(x.size, rate, seed, stream)).reshape(x.shape).astype(F32)


def drop_edge(inputs, rate=0.5, force_undirected=False, training=None, seed=0):
    """nn/sampling/drop_edge.py:6-52 with the counter-based mask: edge e survives iff u(seed, e) >= rate."""
    if not training:
        return inputs
    if rate < 0.0 or rate > 1.0:
        raise ValueError("Dropout probability has to be between 0 and 1, but got {}".format(rate))
    edge_index, edge_attrs = np.asarray(inputs[0]), [np.asarray(a) for a in inputs[1:]]
    row, col = edge_index[0], edge_index[1]
    E = row.shape[0]
    keep = random_uniform(seed, RNG_STREAM_SAMPLER, np.arange(E, dtype=np.uint64)) >= F32(rate)
    if force_undirected:
        index = np.nonzero((row < col) & keep)[0]                       # drop_edge.py:35-36
        dropped = edge_index[:, index]
        dropped = np.concatenate([dropped, dropped[[1, 0]]], axis=-1)    # drop_edge.py:38
        index = np.concatenate([index, index])
    else:
        index = np.nonzero(keep)[0]                                      # drop_edge.py:41-43
        dropped = edge_index[:, index]
    return [dropped] + [np.take(a, index, axis=-1) for a in edge_attrs]


def uniform_neighbor_sample(edge_index, edge_weight, prob, sampled_node_index=None, seed=0):
    """UniformNeighborSampler.sample (utils/graph_utils.py:801-846): keep edge e iff u(seed, e) <= prob, after the
    optional restriction to (and relabelling into) the virtual node set."""
    edge_index = np.asarray(edge_index, I32)
    E = edge_index.shape[1]
    w = np.ones(E, F32) if edge_weight is None else _as_f32(edge_weight)
    keep = random_uniform(seed, RNG_STREAM_SAMPLER, np.arange(E, dtype=np.uint64)) <= F32(prob)
    if sampled_node_index is None:
        return edge_index[:, keep], w[keep]
    virtual, vw, mask = _virtual_edges(edge_index, w, sampled_node_index)
    sel = keep[mask]                                  # the draw of an edge is indexed by its ORIGINAL position
    return virtual[:, sel], vw[sel]


def _virtual_edges(edge_index, w, sampled_node_index):
    """Restriction to / relabelling into a sampled node set (graph_utils.py:690-733): virtual id = position in the
    sampled list; edges with an end outside the set are dropped, edge order is kept."""
    if isinstance(sampled_node_index, tuple):
        rows, cols = sampled_node_index
    else:
        rows = cols = sampled_node_index
    n_row, n_col = int(edge_index[0].max()) + 1, int(edge_index[1].max()) + 1
    row_map = -np.ones(n_row, np.int64)
    row_map[np.asarray(rows)] = np.arange(len(rows))
    if isinstance(sampled_node_index, tuple) or n_col != n_row:
        col_map = -np.ones(n_col, np.int64)
        cols = np.asarray(cols)
        ok = cols < n_col
        col_map[cols[ok]] = np.arange(len(cols))[ok]
    else:
        col_map = row_map
    vr, vc = row_map[edge_index[0]], col_map[edge_index[1]]
    mask = (vr >= 0) & (vc >= 0)
    return np.stack([vr[mask], vc[mask]]).astype(I32), w[mask], mask


def random_neighbor_sample(edge_index, edge_weight=None, k=None, ratio=None, padding=False, seed=0,
                           sampled_node_index=None):
    """RandomNeighborSampler(edge_index, edge_weight).sample(k, ratio, sampled_node_index, padding)
    (utils/graph_utils.py:631-776): rows in ascending (virtual) order, neighbours in edge order; per row either all
    neighbours, k draws with replacement (padding and k >= degree), or a reservoir sample without replacement.
    Returns (sampled_edge_index [2, S], sampled_edge_weight [S]) or (None, None) when nothing is sampled."""
    if k is not None and ratio is not None:
        raise Exception("k and ratio cannot be provided simultaneously")
    edge_index = np.asarray(edge_index, I32)
    E = edge_index.shape[1]
    w = np.ones(E, F32) if edge_weight is None else _as_f32(edge_weight)
    if sampled_node_index is not None:
        edge_index, w, _ = _virtual_edges(edge_index, w, sampled_node_index)
        E = edge_index.shape[1]
    n_rows = int(edge_index[0].max()) + 1 if E else 0
    rowptr, col_sorted, perm = csr_build(edge_index[0], edge_index[1], n_rows)
    out_row, pos, _ = neighbor_sample_csr(rowptr, k, ratio, padding, seed)
    if len(pos) == 0:
        return None, None
    return np.stack([out_row, col_sorted[pos]]).astype(I32), w[perm[pos]]


def neighbor_sample_csr(rowptr, k=None, ratio=None, padding=False, seed=0, stream=RNG_STREAM_SAMPLER):
    """Restatement of tfgk_neighbor_sample_count/_fill: (row int32 [S], CSR position int64 [S], offsets int64 [n+1])."""
    rowptr = np.asarray(rowptr, np.int64)
    n_rows = len(rowptr) - 1
    out_row, out_pos, counts = [], [], np.zeros(n_rows, np.int64)
    for r in range(n_rows):
        start, deg = int(rowptr[r]), int(rowptr[r + 1] - rowptr[r])
        if deg == 0:
            continue
        base = np.uint64(r) << np.uint64(32)
        if padding == "head":                                   # topk_pool.py:59-82: the first node_k entries, in order
            num = min(int(k), deg) if ratio is None else int(np.ceil(F32(deg) * F32(ratio)))
            pos = start + np.arange(max(min(num, deg), 0))
        elif (k is None and ratio is None) or (ratio is None and not padding and k >= deg):
            pos = start + np.arange(deg)
        elif ratio is None and padding and k >= deg:
            pos = start + random_below(seed, stream, base + np.arange(k, dtype=np.uint64), deg)
        else:
            num = k if ratio is None else int(np.ceil(deg * ratio).astype(np.int32))
            res = start + np.arange(num)
            if deg > num:
                i = np.arange(num, deg, dtype=np.uint64)
                j = random_below(seed, stream, base + i, i + np.uint64(1))
                for ii, jj in zip(i.astype(np.int64), j):
                    if jj < num:
                        res[jj] = start + ii
            pos = res
        counts[r] = len(pos)
        out_row.append(np.full(len(pos), r, I32))
        out_pos.append(np.asarray(pos, np.int64))
    out_rowptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    if not out_row:
        return np.zeros(0, I32), np.zeros(0, np.int64), out_rowptr
    return np.concatenate(out_row), np.concatenate(out_pos), out_rowptr


def _row_ids(rowptr):
    rowptr = np.asarray(rowptr, np.int64)
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))


def spmm_heads(rowptr, col, w, src, num_heads, mode="split", emap=None, drop_rate=0.0, seed=0, alpha=1.0, bias=None,
               act=None):
    """Restatement of tfgk_spmm_heads_f32 (include/tfgk.h): per row, fp32 products added in CSR order.
    mode 'split': out[r, h*dh+u] = alpha sum_e W(e,h) src[col_e, h*dh+u]; 'broadcast': src has dh columns;
    'reduce': out[r, u] = alpha sum_h sum_e W(e,h) src[col_e, h*dh+u] (heads added in order, tf.add_n, gat.py:114).
    W(e,h) = w[pos, h] * dropout multiplier of element pos*H+h, pos = emap[e] if given."""
    rowptr, col = np.asarray(rowptr, np.int64), np.asarray(col, np.int64)
    w, src = _as_f32(w), _as_f32(src)
    H = int(num_heads)
    n = len(rowptr) - 1
    pos = np.arange(len(col)) if emap is None else np.asarray(emap, np.int64)
    mult = dropout_scale(w.size, drop_rate, seed).reshape(w.shape)
    W = np.where(mult[pos] == 0, F32(0), (w[pos] * mult[pos]) if drop_rate > 0 else w[pos]).astype(F32)   # [E, H]
    dh = src.shape[1] if mode == "broadcast" else src.shape[1] // H
    out_w = dh if mode == "reduce" else H * dh
    out = np.zeros((n, out_w), F32)
    for r in range(n):
        if mode == "reduce":
            tot = None
            for h in range(H):
                acc = np.zeros(dh, F32)
                for e in range(rowptr[r], rowptr[r + 1]):
                    acc = acc + src[col[e], h * dh:(h + 1) * dh] * W[e, h]
                tot = acc if tot is None else tot + acc
            out[r] = tot * F32(alpha)
        else:
            acc = np.zeros(H * dh, F32)
            for e in range(rowptr[r], rowptr[r + 1]):
                row = np.tile(src[col[e]], H) if mode == "broadcast" else src[col[e]]
                acc = acc + row * np.repeat(W[e], dh)
            out[r] = acc * F32(alpha)
    if bias is not None:
        out = out + _as_f32(bias)
    if act == "relu":
        out = np.maximum(out, F32(0))
    return out.astype(F32)


def gat_softmax_bwd(rowptr, col, att, G, V, num_heads, split_value_heads=True, drop_rate=0.0, seed=0):
    """Restatement of tfgk_gat_softmax_bwd_f32: gradient of gat.py:83-114 w.r.t. the scaled scores, [E, H] CSR order.
    (float64 accumulation here: the kernel's dot products are compared with a tolerance, not bit for bit.)"""
    rowptr, col = np.asarray(rowptr, np.int64), np.asarray(col, np.int64)
    H = int(num_heads)
    att64, G64, V64 = np.asarray(att, np.float64), np.asarray(G, np.float64), np.asarray(V, np.float64)
    E = len(col)
    dv = V64.shape[1] // H
    rows = _row_ids(rowptr)
    Vh = V64[col].reshape(E, H, dv)
    if split_value_heads:
        da = np.einsum("ehd,ehd->eh", G64[rows].reshape(E, H, dv), Vh)
    else:
        da = np.einsum("ed,ehd->eh", G64[rows], Vh) / H
    da = da * dropout_scale(E * H, drop_rate, seed).reshape(E, H).astype(np.float64)
    delta = np.zeros((len(rowptr) - 1, H))
    np.add.at(delta, rows, att64 * da)
    return (att64 * (da - delta[rows])).astype(F32)


# --------------------------------------------------------------------------------------------------------------
# Pooling beyond the plain segment reductions (SURVEY.md 8(f)2): set2set, topk_pool, sag_pool, induced subgraphs
# --------------------------------------------------------------------------------------------------------------

def set2set(x, node_graph_index, lstm, num_iterations, training=None):
    """nn/pool/set2set.py:8-44.  `lstm` keeps the Keras calling convention (inputs [1, G, 2F], initial_state=[h, c]) ->
    (sequence [1, G, F], h, c); it is an argument of the reference too."""
    x = _as_f32(x)
    gi = np.asarray(node_graph_index, I32)
    num_graphs = int(gi.max()) + 1
    units = x.shape[-1]
    h = np.zeros((num_graphs, units * 2), F32)
    state = [np.zeros((1, units), F32), np.zeros((1, units), F32)]
    for _ in range(num_iterations):
        h, state_h, state_c = lstm(h[None], initial_state=state, training=training)       # :30-33
        state = [state_h, state_c]
        h = np.asarray(h, F32)[0]
        repeated_h = gather(h, gi)                                                         # :35
        att_score = np.sum(x * repeated_h, axis=-1, keepdims=True).astype(F32)             # :37
        normed = segment_softmax(att_score, gi, num_graphs)                                # :38
        att_h = unsorted_segment_sum((x * normed).astype(F32), gi, num_graphs)             # :39
        h = np.concatenate([h, att_h], axis=-1).astype(F32)                                # :40
    return h


def topk_pool(source_index, score, k=None, ratio=None):
    """nn/pool/topk_pool.py:6-88: indices of the node_k best-scored targets of every source, sources ascending, best
    first.  tf.argsort is restated as a STABLE sort (equal keys keep their order; TF leaves it unspecified)."""
    if k is None and ratio is None:
        raise Exception("you should provide either k or ratio for topk_pool")
    elif k is not None and ratio is not None:
        raise Exception("you should provide either k or ratio for topk_pool, not both of them")
    source_index = np.asarray(source_index, np.int64).reshape(-1)
    score = _as_f32(score).reshape(-1)
    perm = np.argsort(source_index, kind="stable")                                         # :31-33
    sorted_source, sorted_score = source_index[perm], score[perm]
    counts = np.bincount(sorted_source)                                                    # :38 segment_sum(ones)
    before = np.concatenate([[0], np.cumsum(counts)[:-1]])                                 # :46-49
    out = []
    for s in range(len(counts)):
        cnt = int(counts[s])
        seg = sorted_score[before[s]:before[s] + cnt]
        order = np.argsort(-seg, kind="stable")                                            # :58 DESCENDING
        node_k = min(int(k), cnt) if k is not None else int(np.ceil(F32(cnt) * F32(ratio)))  # :60-68 (float32)
        out.append(before[s] + order[:node_k])
    topk = np.concatenate(out).astype(np.int64) if out else np.zeros(0, np.int64)
    return perm[topk].astype(I32)                                                          # :87


def sample_new_graph_by_node_index(x, edge_index, edge_weight, sampled_node_index, node_graph_index=None, y=None):
    """data/graph.py:276-359: (x, edge_index, edge_weight, node_graph_index, y) of the induced subgraph; nodes are
    relabelled by their position in sampled_node_index, edges keep their order."""
    idx = np.asarray(sampled_node_index, np.int64).reshape(-1)
    edge_index = np.asarray(edge_index, I32)
    n_ids = max(int(edge_index.max()) if edge_index.size else 0, int(idx.max()) if idx.size else 0) + 1
    reverse = -np.ones(n_ids, np.int64)
    reverse[idx] = np.arange(len(idx))
    mask = (reverse[edge_index[0]] >= 0) & (reverse[edge_index[1]] >= 0)
    new_ei = np.stack([reverse[edge_index[0][mask]], reverse[edge_index[1][mask]]]).astype(I32)
    return (np.asarray(x)[idx], new_ei, None if edge_weight is None else np.asarray(edge_weight)[mask],
            None if node_graph_index is None else np.asarray(node_graph_index)[idx], None if y is None else np.asarray(y)[idx])


def sag_pool(x, edge_index, edge_weight, node_graph_index, score_gnn, k=None, ratio=None, score_activation=None):
    """nn/pool/sag_pool.py:7-47."""
    x = _as_f32(x)
    node_score = _as_f32(score_gnn([x, edge_index, edge_weight]))
    topk_node_index = topk_pool(node_graph_index, node_score, k=k, ratio=ratio)
    if score_activation is not None:
        node_score = score_activation(node_score)
    px, pei, pw, pgi, _ = sample_new_graph_by_node_index((x * node_score).astype(F32), edge_index, edge_weight, topk_node_index,
                                                         node_graph_index)
    return px, pei, pw, pgi


def numpy_lstm(kernel, recurrent_kernel, bias):
    """A plain LSTM (gate order i, f, c, o; sigmoid gates, tanh cell - tf.keras.layers.LSTM's defaults) with the Keras
    calling convention, used as the `lstm` ARGUMENT of set2set in the tests and the golden generator."""
    kernel, recurrent_kernel, bias = _as_f32(kernel), _as_f32(recurrent_kernel), _as_f32(bias)
    units = recurrent_kernel.shape[0]

    def sigmoid(v):
        return (F32(1) / (F32(1) + np.exp(-v))).astype(F32)

    def lstm(inputs, initial_state=None, training=None):
        inputs = _as_f32(inputs)
        h, c = _as_f32(initial_state[0]), _as_f32(initial_state[1])
        seq = []
        for t in range(inputs.shape[1]):
            z = (inputs[:, t] @ kernel + h @ recurrent_kernel + bias).astype(F32)
            i, f, g, o = (z[:, j * units:(j + 1) * units] for j in range(4))
            c = (sigmoid(f) * c + sigmoid(i) * np.tanh(g)).astype(F32)
            h = (sigmoid(o) * np.tanh(c)).astype(F32)
            seq.append(h)
        return np.stack(seq, axis=1).astype(F32), h, c
    return lstm


def sort_pool(x, edge_index, edge_weight, node_graph_index, k=None, ratio=None, sort_index=-1):
    """nn/pool/sort_pool.py:7-37."""
    x = _as_f32(x)
    topk_node_index = topk_pool(node_graph_index, x[:, sort_index], k=k, ratio=ratio)
    px, pei, pw, pgi, _ = sample_new_graph_by_node_index(x, edge_index, edge_weight, topk_node_index, node_graph_index)
    return px, pei, pw, pgi


def batch_graphs(parts):
    """BatchGraph.from_graphs (data/graph.py:463-560) for parts = [(x, edge_index, edge_weight, y), ...]:
    returns (x, edge_index, edge_weight, y, node_graph_index, edge_graph_index)."""
    xs, eis, ws, ys, ngi, egi, before = [], [], [], [], [], [], 0
    for i, (x, ei, w, y) in enumerate(parts):
        xs.append(np.asarray(x)); ws.append(np.asarray(w)); ys.append(np.asarray(y))
        eis.append(np.asarray(ei, I32) + before)
        ngi.append(np.full(len(x), i, I32)); egi.append(np.full(np.asarray(ei).shape[1], i, I32))
        before += len(x)
    return (np.concatenate(xs), np.concatenate(eis, axis=1).astype(I32), np.concatenate(ws), np.concatenate(ys),
            np.concatenate(ngi), np.concatenate(egi))
