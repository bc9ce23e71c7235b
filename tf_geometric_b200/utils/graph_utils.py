# coding=utf-8
"""Edge-index integer preprocessing with the reference's semantics (utils/graph_utils.py of tf_geometric).

Device inputs (torch CUDA tensors) run on the GPU kernels - including the hash/unique based helpers
(merge_duplicated_edge, convert_edge_to_upper, convert_edge_to_directed: tfgk_edge_unique / tfgk_directed_edges, bit-exact
with tf.unique's first-occurrence order) - and return device tensors.  numpy / list inputs are processed with numpy and
return numpy, exactly like the reference does for non-tensor inputs (its eager host path).
"""
import math
import warnings

import numpy as np
import torch

from .. import ops, _rng, _structure, autograd


def _is_device(x):
    return torch.is_tensor(x) and x.is_cuda


def _to_numpy(x):
    if x is None:
        return None
    if torch.is_tensor(x):
        return x.detach().cpu().numpy()
    return np.asarray(x)


def _like(result, template, dtype):
    """Return `result` (numpy) in the container type of `template`."""
    if torch.is_tensor(template):
        return torch.from_numpy(np.ascontiguousarray(result)).to(device=template.device, dtype=dtype)
    return result


def convert_edge_index_to_edge_hash(edge_index, num_nodes=None):
    """hash = num_nodes * row + col in int64; num_nodes defaults to max id + 1 (reference :14-43)."""
    ei = _to_numpy(edge_index).astype(np.int64)
    if num_nodes is None:
        num_nodes = int(ei.max()) + 1
    edge_hash = np.int64(num_nodes) * ei[0] + ei[1]
    return _like(edge_hash, edge_index, torch.int64), int(num_nodes)


def convert_edge_hash_to_edge_index(edge_hash, num_nodes):
    """reference :46-64."""
    h = _to_numpy(edge_hash).astype(np.int64)
    ei = np.stack([h // num_nodes, h % num_nodes], axis=0).astype(np.int32)
    return _like(ei, edge_hash, torch.int32)


def _first_occurrence_unique(values):
    uniq, first, inverse = np.unique(values, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return uniq[order], rank[inverse]


def _segment_merge(prop, ids, n, mode):
    prop = np.asarray(prop)
    if mode == "sum":
        out = np.zeros((n,) + prop.shape[1:], dtype=prop.dtype)
        np.add.at(out, ids, prop)
    elif mode == "mean":
        out = np.zeros((n,) + prop.shape[1:], dtype=prop.dtype)
        np.add.at(out, ids, prop)
        cnt = np.maximum(np.bincount(ids, minlength=n), 1).astype(prop.dtype)
        out = (out / cnt.reshape((-1,) + (1,) * (prop.ndim - 1))).astype(prop.dtype)
    elif mode == "max":
        out = np.full((n,) + prop.shape[1:], np.finfo(prop.dtype).min if prop.dtype.kind == "f" else np.iinfo(prop.dtype).min,
                      dtype=prop.dtype)
        np.maximum.at(out, ids, prop)
    elif mode == "min":
        out = np.full((n,) + prop.shape[1:], np.finfo(prop.dtype).max if prop.dtype.kind == "f" else np.iinfo(prop.dtype).max,
                      dtype=prop.dtype)
        np.minimum.at(out, ids, prop)
    else:
        raise Exception("wrong merge mode: {}".format(mode))
    return out


def merge_duplicated_edge(edge_index, edge_props=None, merge_modes=None):
    """Duplicates collapse onto their first occurrence; props merged with sum|min|max|mean (reference :67-125)."""
    if edge_props is not None and len(edge_props) > 0:
        if merge_modes is None:
            merge_modes = ["sum"] * len(edge_props)
        elif type(merge_modes) is not list:
            raise Exception("type error: merge_modes should be a list of strings")
    if _is_device(edge_index):
        return _merge_duplicated_edge_device(edge_index, edge_props, merge_modes)
    ei = _to_numpy(edge_index).astype(np.int32)
    edge_hash, hash_n = convert_edge_index_to_edge_hash(ei)
    uniq_hash, uniq_idx = _first_occurrence_unique(edge_hash)
    uniq_ei = convert_edge_hash_to_edge_index(uniq_hash, hash_n)
    out_index = _like(uniq_ei, edge_index, torch.int32)
    if edge_props is None:
        return out_index, None
    out_props = []
    for prop, mode in zip(edge_props, merge_modes):
        if prop is None:
            out_props.append(None)
        else:
            merged = _segment_merge(_to_numpy(prop), uniq_idx, len(uniq_hash), mode)
            out_props.append(_like(merged, prop, prop.dtype if torch.is_tensor(prop) else None))
    return out_index, out_props


def _merge_duplicated_edge_device(edge_index, edge_props, merge_modes):
    from ..nn.kernel.map_reduce import _segment_reduce
    ei = edge_index if edge_index.dtype == torch.int32 else edge_index.to(torch.int32)
    ei = ei.contiguous()
    if ei.shape[1] == 0:
        return ei, (None if edge_props is None else list(edge_props))
    hash_n = int(ei.max().item()) + 1                                 # reference: num_nodes = reduce_max(edge_index) + 1
    uniq_index, of_edge = ops.edge_unique(ei[0].contiguous(), ei[1].contiguous(), hash_n)
    if edge_props is None:
        return uniq_index, None
    out = []
    for prop, mode in zip(edge_props, merge_modes):
        if prop is None:
            out.append(None)
            continue
        if mode not in ("sum", "min", "max", "mean"):
            raise Exception("wrong merge mode: {}".format(mode))
        p = ops.as_device(prop, torch.float32, device=ei.device)
        out.append(_segment_reduce(p, of_edge, uniq_index.shape[1], mode))
    return uniq_index, out


def convert_edge_to_upper(edge_index, edge_props=None, merge_modes=None):
    """(min(u,v), max(u,v)) for every edge, then merge duplicates (reference :128-151)."""
    if _is_device(edge_index):
        ei = edge_index.to(torch.int32)
        upper = torch.stack([torch.minimum(ei[0], ei[1]), torch.maximum(ei[0], ei[1])]).contiguous()
        return merge_duplicated_edge(upper, edge_props, merge_modes)
    ei = _to_numpy(edge_index).astype(np.int32)
    upper = np.stack([ei.min(axis=0), ei.max(axis=0)], axis=0)
    upper_index, upper_props = merge_duplicated_edge(_like(upper, edge_index, torch.int32), edge_props, merge_modes)
    return upper_index, upper_props


def convert_edge_to_directed(edge_index, edge_props=None, merge_modes=None):
    """Undirected -> both directions: upper edges followed by the mirrored non-loop upper edges (reference :155-212)."""
    if edge_props is not None and len(edge_props) > 0 and merge_modes is None:
        merge_modes = ["sum"] * len(edge_props)
    upper_index, upper_props = convert_edge_to_upper(edge_index, edge_props, merge_modes)
    if _is_device(edge_index):
        if upper_index.shape[1] == 0:
            return edge_index, edge_props
        out_index, lower_src = ops.directed_edges(upper_index.contiguous())
        if lower_src.numel() == 0:                                     # only self loops: reference returns the inputs
            return edge_index, edge_props
        if edge_props is None:
            return out_index, None
        out_props = []
        for prop, up_prop in zip(edge_props, upper_props):
            if prop is None:
                out_props.append(None)
            else:
                out_props.append(torch.cat([up_prop, ops.permute(up_prop.contiguous(), lower_src)]))
        return out_index, out_props
    up = _to_numpy(upper_index)
    mask = up[0] != up[1]
    if not mask.any():
        return edge_index, edge_props
    lower = np.stack([up[1][mask], up[0][mask]], axis=0)
    out_index = _like(np.concatenate([up, lower], axis=1), edge_index, torch.int32)
    if edge_props is None:
        return out_index, None
    out_props = []
    for prop, up_prop in zip(edge_props, upper_props):
        if prop is None:
            out_props.append(None)
        else:
            upn = _to_numpy(up_prop)
            out_props.append(_like(np.concatenate([upn, upn[mask]], axis=0), prop,
                                   prop.dtype if torch.is_tensor(prop) else None))
    return out_index, out_props


def remove_self_loop_edge(edge_index, edge_weight=None):
    """reference :252-269.  Device tensors stay on the device: the kept positions come from tfgk_select_flagged_i32 and
    the kept weights are a differentiable gather (the same bits as the host path, and the weights' autograd graph is
    kept, which MinCutPool's pooled weights need)."""
    if _is_device(edge_index):
        from .. import autograd
        ei = (edge_index if edge_index.dtype == torch.int32 else edge_index.to(torch.int32)).contiguous()
        row, col = ei[0].contiguous(), ei[1].contiguous()
        keep = ops.select_flagged((row != col).to(torch.int32))
        out_index = torch.stack([ops.gather_i32(row, keep), ops.gather_i32(col, keep)])
        out_w = None
        if edge_weight is not None:
            out_w = autograd.TakeRows.apply(ops.as_device(edge_weight, torch.float32, device=ei.device).reshape(-1), keep)
        return out_index, out_w
    ei = _to_numpy(edge_index)
    mask = ei[0] != ei[1]
    out_w = None
    if edge_weight is not None:
        out_w = _like(_to_numpy(edge_weight)[mask], edge_weight, torch.float32)
    return _like(ei[:, mask], edge_index, torch.int32), out_w


def add_self_loop_edge(edge_index, num_nodes, edge_weight=None, fill_weight=1.0):
    """Append [[0..N-1],[0..N-1]] AFTER the existing edges; weights get `fill_weight`; no dedup (reference :350-366).
    Device tensors run tfgk_self_loops_i32 / tfgk_self_loop_weights_f32 (bit-exact integers)."""
    num_nodes = int(num_nodes)
    if _is_device(edge_index):
        ei = edge_index if edge_index.dtype == torch.int32 else edge_index.to(torch.int32)
        out_index = ops.self_loops(ei.contiguous(), num_nodes)
        out_w = None
        if edge_weight is not None:
            w = ops.as_device(edge_weight, torch.float32, device=ei.device)
            out_w = ops.self_loop_weights(w, ei.shape[1], num_nodes, fill_weight, ei.device)
        return out_index, out_w
    ei = np.asarray(_to_numpy(edge_index), dtype=np.int32).reshape(2, -1)
    diag = np.arange(num_nodes, dtype=np.int32)
    out_index = _like(np.concatenate([ei, np.stack([diag, diag])], axis=1), edge_index, torch.int32)
    out_w = None
    if edge_weight is not None:
        w = np.concatenate([_to_numpy(edge_weight).astype(np.float32), np.full([num_nodes], fill_weight, dtype=np.float32)])
        out_w = _like(w, edge_weight, torch.float32)
    return out_index, out_w


def adj_norm_edge(edge_index, num_nodes, edge_weight=None, add_self_loop=False, cache=None):
    """D^-1/2 A D^-1/2 on the edge list with ROW degrees on both sides (reference :914-943).  Differentiable in
    edge_weight (GcnNormValues, kind "both_sym"); the forward runs the same kernels either way.  A warm cache hit returns
    the cached constant, as gcn_norm_adj does."""
    cache_key = "adj_normed_edge"
    if cache is not None and cache.get(cache_key) is not None:
        return cache[cache_key]
    from .. import autograd
    from ..sparse import SparseMatrix
    ei = ops.as_device(edge_index, torch.int32)
    adj = SparseMatrix(ei, edge_weight, [num_nodes, num_nodes])
    w = adj.value
    if add_self_loop:
        adj = adj.add_diag(1.0)
    dis = ops.deg_inv(adj.segment_sum(axis=-1), ops.POW_INV_SQRT)
    normed = ops.scale_edges(adj.index[0].contiguous(), adj.index[1].contiguous(), adj.value.detach(), dl=dis, dr=dis)
    if cache is not None:
        cache[cache_key] = adj.index, normed
    if autograd.needs_grad(w):
        normed = autograd.GcnNormValues.apply(w, normed, ("both_sym", adj, normed, dis, dis))
    return adj.index, normed


def convert_dense_adj_to_edge(dense_adj):
    """The non-zero entries of a dense [M, M] matrix as an edge list, row-major (reference :272-285): entries != 0 are
    kept, so NaN is.  Device tensors: positions from tfgk_select_flagged_i32, weights a differentiable gather."""
    if _is_device(dense_adj):
        from .. import autograd
        m = dense_adj.shape[0]
        flat = dense_adj.reshape(-1)
        if flat.dtype != torch.float32:
            flat = flat.to(torch.float32)
        k = ops.select_flagged((flat != 0).to(torch.int32))
        k64 = k.to(torch.int64)
        edge_index = torch.stack([k64 // m, k64 % m]).to(torch.int32)
        return edge_index, autograd.TakeRows.apply(flat.contiguous(), k)
    a = _to_numpy(dense_adj)
    row, col = np.nonzero(a != 0)
    return np.stack([row, col]).astype(np.int32), a[row, col]


def convert_dense_assign_to_edge(dense_assign, node_graph_index=None, num_nodes=None, num_clusters=None):
    """Assignment matrix [N, C] -> (edge_index [2, N*C], edge_weight [N*C]) with edge (n, C * graph(n) + c) for entry
    (n, c), row-major (reference :288-322).  Device tensors stay on the device and the weights are a differentiable
    view of the matrix."""
    if _is_device(dense_assign):
        n = int(dense_assign.shape[0] if num_nodes is None else num_nodes)
        c = int(dense_assign.shape[1] if num_clusters is None else num_clusters)
        dev = dense_assign.device
        row = torch.arange(n, dtype=torch.int32, device=dev).repeat_interleave(c)
        col = torch.arange(c, dtype=torch.int32, device=dev).repeat(n)
        if node_graph_index is not None:
            ngi = ops.as_device(node_graph_index, torch.int32, device=dev)
            col = col + ngi.repeat_interleave(c) * c
        return torch.stack([row, col]), dense_assign.reshape(-1)
    a = _to_numpy(dense_assign)
    n = a.shape[0] if num_nodes is None else int(num_nodes)
    c = a.shape[1] if num_clusters is None else int(num_clusters)
    row = np.repeat(np.arange(n, dtype=np.int32), c)
    col = np.tile(np.arange(c, dtype=np.int32), n)
    if node_graph_index is not None:
        col = col + np.repeat(_to_numpy(node_graph_index).astype(np.int32), c) * c
    return np.stack([row, col]).astype(np.int32), a.reshape(-1)


def compute_num_or_size_splits(num_h_features, num_splits):
    """utils/tf_sparse_utils.py:71-90 - how GCN(num_splits=...) chunks the feature columns of XW."""
    if num_splits is None or num_splits == 1:
        return None
    if num_h_features % num_splits == 0:
        return num_splits
    split_size = int(np.ceil(num_h_features / num_splits))
    num_pre_splits = int(np.floor(num_h_features / split_size))
    last_split_size = num_h_features % split_size
    sizes = [split_size] * num_pre_splits + ([last_split_size] if last_split_size > 0 else [])
    if len(sizes) != num_splits:
        raise Exception("cannot split H of shape [None, {}] into {} matrices, please provide a valid num_splits"
                        .format(num_h_features, num_splits))
    return sizes


# ---- link prediction: negative sampling and the edge split (reference :369-452, :488-535) ---------------------------
# One implementation for every container: numpy inputs are copied to the device and the results back (the draws come
# from the counter-based generator of csrc/rng.cuh, so they cannot follow numpy's global generator anyway).

_MASK64 = (1 << 64) - 1


def _batch_seed(seed, b):
    """Key of draw b of a batch: independent Philox keys for the same base seed."""
    return (seed + b * 0x9E3779B97F4A7C15) & _MASK64


def _check_ids(ids, num_nodes, what):
    if ids.numel():
        lo, hi = torch.aminmax(ids)
        if int(lo) < 0 or int(hi) >= num_nodes:
            raise ValueError("{} holds node ids outside [0, {})".format(what, num_nodes))


def _excluded_structure(edge_index, num_nodes, mode):
    """(csr, offsets, C): row i of csr holds the sorted distinct columns row i may not pair with (tfgk.h tfgk_neg_*):
    NEG_UPPER - the upper neighbours j > i of the undirected edge set (self loops are never candidates anyway);
    NEG_START - the out-neighbours of i and i itself.  Memoised on the edge tensor."""
    tag = ("neg", int(num_nodes), int(mode))
    hit = _structure._lookup(edge_index, tag)
    if hit is not None:
        return hit
    row, col = edge_index[0].contiguous(), edge_index[1].contiguous()
    if mode == ops.NEG_UPPER:
        lo, hi = torch.minimum(row, col).contiguous(), torch.maximum(row, col).contiguous()
        keep = ops.select_flagged(ops.edge_flags(lo, hi, lo.numel(), mode=ops.FLAG_UPPER))
        lo, hi = ops.gather_i32(lo, keep), ops.gather_i32(hi, keep)
    else:
        loops = torch.arange(num_nodes, dtype=torch.int32, device=row.device)
        lo, hi = torch.cat([row, loops]), torch.cat([col, loops])
    if lo.numel():
        uniq, _ = ops.edge_unique(lo, hi, num_nodes)
        lo, hi = uniq[0].contiguous(), uniq[1].contiguous()
        by_col = ops.stable_argsort(hi, key_bits=max(1, (num_nodes - 1).bit_length()))
        lo, hi = ops.gather_i32(lo, by_col), ops.gather_i32(hi, by_col)
    csr = ops.csr_build(lo, hi, num_nodes, num_nodes)           # stable by row: columns stay ascending within a row
    offsets, C = ops.neg_offsets(csr, mode)
    return _structure._store(edge_index, tag, (csr, offsets, C))


def _words(k):
    """(low, high) 32-bit halves of an int64 vector, as int32 vectors."""
    halves = k.view(torch.int32).view(-1, 2)
    return halves[:, 0].contiguous(), halves[:, 1].contiguous()


def _random_keys(n, seed, device):
    """n independent 32-bit keys (the high word of a 64-bit draw below 2^32 is zero)."""
    return _words(ops.neg_draw(1 << 32, n, seed, device=device))[0]


def _argsort_i64(k, C):
    """Stable argsort of int64 values in [0, C): LSD passes over the low, then the high 32-bit word."""
    bits = max(1, (C - 1).bit_length())
    lo, hi = _words(k)
    order = ops.stable_argsort(lo, key_bits=min(bits, 32))
    if bits > 32:
        order = ops.gather_i32(order, ops.stable_argsort(ops.gather_i32(hi, order), key_bits=bits - 32))
    return order


def _draw_candidates(C, S, replace, seed, device):
    """S candidate indices in [0, C) as int64: independent draws, or S distinct ones."""
    if replace:
        return ops.neg_draw(C, S, seed, device=device)
    if 2 * S > C:               # dense: shuffle the whole range and take a prefix (work O(C) <= O(2 S))
        # The keys are 32-bit, so equal keys keep index order: about C^2 / 2^33 ties (0.1 at C = 10^4, 116 at C = 10^6),
        # a bias below what any test of reasonable size can see.
        perm = ops.stable_argsort(_random_keys(C, seed, device))
        return perm[:S].to(torch.int64)
    k = ops.neg_draw(C, S, seed, device=device)
    rnd = 0
    while True:                 # redraw the later duplicates; draw s of round r has the counter (s, r)
        dup = ops.select_flagged(ops.neg_dup_flags(k, _argsort_i64(k, C)))
        if dup.numel() == 0:
            return k
        rnd += 1
        ops.neg_draw(C, S, seed, round=rnd, index=dup, out=k)


def negative_sampling(num_samples, num_nodes, edge_index=None, replace=True, mode="undirected", batch_size=None,
                      seed=None):
    """Node pairs that are not edges (reference :369-412), drawn exactly from the implicit candidate list.

    :param num_samples: pairs per draw
    :param num_nodes: number of nodes
    :param edge_index: optional positive edges.  Given: the candidates are the pairs i < j that are not in
        convert_edge_to_upper(edge_index), in the reference's row-major order, and no dense N x N matrix is built.
        None: both ends are uniform in [0, num_nodes) (self loops and positives included, like np.random.randint).
    :param replace: with edge_index, whether the same pair may be drawn twice
    :param mode: only "undirected" (the reference raises NotImplementedError otherwise)
    :param batch_size: None -> one int32 [2, num_samples] edge index; else a list of batch_size independent draws
    :param seed: optional 64-bit key pinning the draws
    :return: device tensors for device (and for absent) edge_index, numpy arrays for numpy edge_index
    """
    seed = _rng.resolve_host(seed)
    num_samples, num_nodes = int(num_samples), int(num_nodes)
    n_batches = 1 if batch_size is None else int(batch_size)
    if num_samples < 0 or num_nodes < 0:
        raise ValueError("num_samples and num_nodes must be non-negative")
    if edge_index is None:
        if num_samples and num_nodes == 0:
            raise ValueError("cannot sample node pairs from an empty graph")
        dev = ops.default_device()
        out = [ops.random_pairs(num_nodes, num_samples, _batch_seed(seed, b), dev) for b in range(n_batches)]
        return out[0] if batch_size is None else out
    if mode != "undirected":
        raise NotImplementedError()
    on_device = _is_device(edge_index)
    ei = ops.as_device(edge_index, torch.int32)
    _check_ids(ei, num_nodes, "edge_index")
    csr, offsets, C = _excluded_structure(ei, num_nodes, ops.NEG_UPPER)
    if num_samples and C == 0:
        raise ValueError("no candidate pair: every pair i < j of the {} nodes is an edge".format(num_nodes))
    if not replace and num_samples > C:
        raise ValueError("cannot draw {} distinct pairs without replacement from {} candidates".format(num_samples, C))
    out = []
    for b in range(n_batches):
        k = _draw_candidates(C, num_samples, replace, _batch_seed(seed, b), ei.device) if num_samples else \
            torch.empty((0,), dtype=torch.int64, device=ei.device)
        pairs = ops.neg_decode(csr, offsets, ops.NEG_UPPER, k)
        out.append(pairs if on_device else pairs.cpu().numpy())
    return out[0] if batch_size is None else out


def negative_sampling_with_start_node(start_node_index, num_nodes, edge_index=None, seed=None):
    """One negative partner per start node (reference :415-452): b != a with (a, b) not in edge_index (directed),
    uniform over the candidates.  A start node adjacent to every other node raises ValueError (the reference loops
    forever).  Without edge_index b is uniform in [0, num_nodes).  Returns int32 [2, S] in the container of
    start_node_index."""
    seed = _rng.resolve_host(seed)
    num_nodes = int(num_nodes)
    on_device = _is_device(start_node_index)
    dev = edge_index.device if _is_device(edge_index) else None
    start = ops.as_device(start_node_index, torch.int32, device=dev).reshape(-1).contiguous()
    _check_ids(start, num_nodes, "start_node_index")
    if edge_index is None:
        end = ops.random_pairs(num_nodes, start.numel(), seed, start.device)[1]
    else:
        ei = ops.as_device(edge_index, torch.int32, device=start.device)
        _check_ids(ei, num_nodes, "edge_index")
        csr, offsets, _ = _excluded_structure(ei, num_nodes, ops.NEG_START)
        if start.numel():
            s = start.to(torch.int64)
            if bool(((offsets[s + 1] - offsets[s]) == 0).any()):
                raise ValueError("a start node is adjacent to every other node: it has no negative partner")
        end = ops.neg_sample_start(csr, start, seed)
    out = torch.stack([start, end])
    return out if on_device else out.cpu().numpy()


def edge_train_test_split(edge_index, test_size, edge_weight=None, mode="undirected", seed=None, **kwargs):
    """Split the undirected edges into train and test sets (reference :488-535).

    The edges are merged into convert_edge_to_upper(edge_index, [edge_weight], merge_modes=["max"]) and permuted by
    random keys; with n merged edges, n_test = ceil(test_size * n) for a float test_size and test_size for an int
    (sklearn's sizes), test = the first n_test of the permutation and train = the rest.  Weights follow their edges.
    :return: (train_edge_index, test_edge_index, train_edge_weight, test_edge_weight), each in the container of its
        input (weights None without edge_weight)
    """
    if "num_nodes" in kwargs:
        warnings.warn("argument \"num_nodes\" is deprecated for the method \"edge_train_test_split\", you can remove it")
    if mode != "undirected":
        raise NotImplementedError()
    seed = _rng.resolve_host(seed)
    ei = ops.as_device(edge_index, torch.int32)
    w = None if edge_weight is None else ops.as_device(edge_weight, torch.float32, device=ei.device).reshape(-1)
    upper, props = convert_edge_to_upper(ei, None if w is None else [w], None if w is None else ["max"])
    n = upper.shape[1]
    if isinstance(test_size, (float, np.floating)):
        if not 0.0 < test_size < 1.0:
            raise ValueError("test_size={} should be in (0, 1) as a fraction".format(test_size))
        n_test = int(math.ceil(test_size * n))
    else:
        n_test = int(test_size)
    n_train = n - n_test
    if n_test <= 0 or n_train <= 0:
        raise ValueError("with n_samples={} and test_size={} the train or the test set would be empty".format(n, test_size))
    perm = ops.stable_argsort(_random_keys(n, seed, ei.device))
    row, col = upper[0].contiguous(), upper[1].contiguous()
    parts = []
    for idx in (perm[n_test:].contiguous(), perm[:n_test].contiguous()):
        part = torch.stack([ops.gather_i32(row, idx), ops.gather_i32(col, idx)])
        parts.append(part if _is_device(edge_index) else part.cpu().numpy())
    weights = [None, None]
    if w is not None:
        upw = props[0].contiguous()
        weights = [ops.permute(upw, idx) for idx in (perm[n_test:].contiguous(), perm[:n_test].contiguous())]
        if not _is_device(edge_weight):
            weights = [x.cpu().numpy() for x in weights]
    return parts[0], parts[1], weights[0], weights[1]


def convert_x_to_3d(x, source_index, k=None, pad=True):
    """Group the rows of x by source_index into a zero-padded [num_sources, k, D] tensor (reference :215-249): row j of
    group s is the j-th row of x with id s, in input order (stable); num_sources = max(source_index) + 1, so ids that do
    not appear give all-zero groups.  k=None takes the largest group; a k above it keeps its width with pad=True and
    shrinks to it with pad=False; a k below it keeps each group's first k rows.  One K9 launch (pad_rows over the
    segment-id CSR); differentiable in x.  Tensors or numpy in, a device tensor out.  A length mismatch between x and
    source_index, a negative id or an empty input raises ValueError."""
    sid = ops.as_device(source_index, torch.int32).reshape(-1)
    dev = sid.device
    x = ops.as_device(x, torch.float32, device=dev)
    if x.dim() != 2:
        raise ValueError("convert_x_to_3d: x must be 2-D, got shape {}".format(tuple(x.shape)))
    if x.shape[0] != sid.numel():
        raise ValueError("convert_x_to_3d: x has {} rows but source_index {} entries".format(x.shape[0], sid.numel()))
    if sid.numel() == 0:
        raise ValueError("convert_x_to_3d: empty input")
    lo, hi = (int(v) for v in torch.stack([sid.min(), sid.max()]).cpu())
    if lo < 0:
        raise ValueError("convert_x_to_3d: negative source id {}".format(lo))
    csr = _structure.csr_for_segment_ids(sid, hi + 1)
    largest = int(csr.degree_i64().max())
    if k is None or (int(k) > largest and not pad):
        k = largest
    return autograd.PadRows.apply(x, csr, int(k), False, None)


# ---- sampled-subgraph helpers (reference :455-485, :538-551, :946-975) --------------------------------------------

def reindex_sampled_edge_index(sampled_edge_index, sampled_node_index):
    """Every id of sampled_edge_index replaced by its position in sampled_node_index, -1 for ids not in it (the
    reference's StaticHashTable with default_value=-1).  Duplicate ids in sampled_node_index raise ValueError, as TF's
    table refuses duplicate keys.  Device tensors run tfgk_reindex_i32; the int32 result is in the container of
    sampled_edge_index."""
    if _is_device(sampled_edge_index):
        ei = sampled_edge_index.to(torch.int32).contiguous()
        nodes = ops.as_device(sampled_node_index, torch.int32, device=ei.device).reshape(-1).contiguous()
        if nodes.numel() and int(nodes.min()) < 0:
            raise ValueError("sampled_node_index holds negative ids")
        top = torch.cat([ei.reshape(-1), nodes]).max() if ei.numel() + nodes.numel() else None
        N = 0 if top is None else max(int(top) + 1, 0)
        node_map = torch.full((N,), -1, dtype=torch.int32, device=ei.device)
        out, n_dup = ops.reindex(nodes, ei.reshape(-1), node_map)
        if n_dup:
            raise ValueError("sampled_node_index holds {} duplicate ids".format(n_dup))
        return out.reshape(ei.shape)
    ei = np.asarray(_to_numpy(sampled_edge_index)).astype(np.int64)
    nodes = np.asarray(_to_numpy(sampled_node_index)).astype(np.int64).reshape(-1)
    order = np.argsort(nodes, kind="stable")
    ordered = nodes[order]
    if len(ordered) > 1 and np.any(ordered[1:] == ordered[:-1]):
        raise ValueError("sampled_node_index holds duplicate ids")
    at = np.clip(np.searchsorted(ordered, ei), 0, max(len(ordered) - 1, 0))
    found = (ordered[at] == ei) if len(ordered) else np.zeros(ei.shape, bool)
    out = np.where(found, order[at] if len(ordered) else -1, -1).astype(np.int32)
    return _like(out, sampled_edge_index, torch.int32)


def compute_edge_mask_by_node_index(edge_index, node_index):
    """bool [E]: both ends of the edge are in node_index (reference :538-551).  Device tensors: the node set becomes an
    [N] map and tfgk_edge_flags_i32 tests both ends."""
    if _is_device(edge_index):
        ei = edge_index.to(torch.int32).contiguous()
        nodes = ops.as_device(node_index, torch.int32, device=ei.device).reshape(-1)
        E = ei.shape[1]
        N = int(torch.cat([ei.reshape(-1), nodes]).max()) + 1 if E + nodes.numel() else 0
        node_map, _ = _sampling._virtual_mapping(nodes, N, ei.device)
        flag = ops.edge_flags(ei[0].contiguous(), ei[1].contiguous(), E, mode=ops.FLAG_MAPPED, row_map=node_map,
                              col_map=node_map)
        return flag.to(torch.bool)
    ei = np.asarray(_to_numpy(edge_index)).astype(np.int64)
    nodes = np.asarray(_to_numpy(node_index)).astype(np.int64).reshape(-1)
    n = int(max(ei.max(initial=-1), nodes.max(initial=-1))) + 1
    node_mask = np.zeros(n, bool)
    node_mask[nodes] = True
    return node_mask[ei[0]] & node_mask[ei[1]]


def extract_unique_edge(edge_index, edge_weight=None, mode="undirected"):
    """The first occurrence of every edge, in edge order, with its weight (reference :455-485); mode "undirected"
    compares the ends as a sorted pair, any other mode as an ordered one.  Kept edges keep their orientation.  Device
    tensors: tfgk_edge_unique over the (sorted) pairs; each container follows its input."""
    if _is_device(edge_index):
        ei = edge_index.to(torch.int32).contiguous()
        row, col = ei[0].contiguous(), ei[1].contiguous()
        E = row.numel()
        keep = torch.empty((0,), dtype=torch.int32, device=ei.device)
        if E:
            if mode == "undirected":
                row, col = torch.minimum(row, col).contiguous(), torch.maximum(row, col).contiguous()
            uniq, of_edge = ops.edge_unique(row, col, int(ei.max()) + 1)
            first = torch.full((uniq.shape[1],), E, dtype=torch.int64, device=ei.device)
            first.scatter_reduce_(0, of_edge.long(), torch.arange(E, device=ei.device), reduce="amin")
            keep = first.to(torch.int32)
        out_index = torch.stack([ops.gather_i32(ei[0].contiguous(), keep), ops.gather_i32(ei[1].contiguous(), keep)])
    else:
        ei = np.asarray(_to_numpy(edge_index)).astype(np.int32).reshape(2, -1)
        pairs = np.sort(ei, axis=0) if mode == "undirected" else ei
        h = pairs[0].astype(np.int64) * (int(ei.max(initial=0)) + 1) + pairs[1]
        _, keep = np.unique(h, return_index=True)
        keep = np.sort(keep)
        out_index = _like(ei[:, keep], edge_index, torch.int32)
    if edge_weight is None:
        return out_index, None
    if _is_device(edge_index):
        out_w = ops.permute(ops.as_device(edge_weight, torch.float32, device=keep.device).reshape(-1), keep)
        return out_index, (out_w if _is_device(edge_weight) else out_w.cpu().numpy())
    return out_index, _like(np.asarray(_to_numpy(edge_weight), np.float32).reshape(-1)[keep], edge_weight, torch.float32)


# samplers live in utils/sampling.py; re-exported here because the reference defines them in this module (:630-846)
from . import sampling as _sampling  # noqa: E402
from .sampling import RandomNeighborSampler, UniformNeighborSampler, SampledNeighborhood  # noqa: E402,F401
