# coding=utf-8
"""Test-side restatement of the link-prediction path (SURVEY.md 8(f)5, demo/demo_gae.py): predict_edge, exact negative
sampling over the implicit candidate list, start-node sampling and the edge train/test split.  It restates
tf_geometric_b200/csrc/link_ops.cu and the host logic of tf_geometric_b200/utils/graph_utils.py on top of the oracle's
Philox generator (oracle.tfg_oracle.random_u32); integer outputs are bit-exact against the kernels.  It is pinned
against the reference's own functions by tests/golden/link_exec.npz (tools/gen_golden_from_reference.py).
TEST INFRASTRUCTURE ONLY: nothing under tf_geometric_b200/ imports it."""
import numpy as np

from oracle import tfg_oracle as o

RNG_STREAM_LINK = 2
_M32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def _mulhi64(u, n):
    """High 64 bits of the 128-bit product of two uint64 arrays (schoolbook on 32-bit halves)."""
    u, n = np.asarray(u, np.uint64), np.asarray(n, np.uint64)
    ul, uh, nl, nh = u & _M32, u >> _S32, n & _M32, n >> _S32
    with np.errstate(over="ignore"):
        ll, lh, hl, hh = ul * nl, ul * nh, uh * nl, uh * nh
        mid = (ll >> _S32) + (lh & _M32) + (hl & _M32)
        return hh + (lh >> _S32) + (hl >> _S32) + (mid >> _S32)


def random_below64(seed, stream, idx, n):
    """rng.cuh random_below64: u = random_u32(2 idx) | random_u32(2 idx + 1) << 32, k = (u * n) >> 64."""
    idx = np.asarray(idx, np.uint64)
    lo = o.random_u32(seed, stream, idx * np.uint64(2)).astype(np.uint64)
    hi = o.random_u32(seed, stream, idx * np.uint64(2) + np.uint64(1)).astype(np.uint64)
    return _mulhi64(lo | (hi << _S32), n).astype(np.int64)


def predict_edge(embedded, edge_index):
    """demo/demo_gae.py:53-60 in float64: sum_d h[row_e, d] * h[col_e, d]."""
    h = np.asarray(embedded, np.float64)
    ei = np.asarray(edge_index, np.int64)
    return (h[ei[0]] * h[ei[1]]).sum(-1)


def link_batch_seed(seed, b):
    return (int(seed) + b * 0x9E3779B97F4A7C15) & ((1 << 64) - 1)


def negative_structure(edge_index, num_nodes, start=False):
    """(rowptr, col, offsets): row i of the CSR holds X_i, the sorted distinct columns row i may not pair with -
    the upper neighbours j > i of the undirected edge set, or (start=True) the out-neighbours of i and i itself;
    offsets[i] = number of candidates before row i, candidates of row i = [base_i, N) minus X_i (base_i = i + 1 | 0)."""
    ei = np.asarray(edge_index, np.int64).reshape(2, -1)
    n = int(num_nodes)
    if start:
        r, c = np.concatenate([ei[0], np.arange(n)]), np.concatenate([ei[1], np.arange(n)])
    else:
        r, c = ei.min(axis=0), ei.max(axis=0)
        keep = r < c
        r, c = r[keep], c[keep]
    h = np.unique(r * n + c)
    r, c = h // n, h % n
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=n))]).astype(np.int64)
    base = np.zeros(n, np.int64) if start else np.arange(1, n + 1, dtype=np.int64)
    counts = np.maximum((n - base) - np.diff(rowptr), 0)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return rowptr, c.astype(np.int32), offsets


def _decode_in_row(x, base, r):
    """the r-th value of [base, N) not in the sorted distinct x: base + r + #{m : x[m] - base - m <= r}."""
    x = np.asarray(x, np.int64)
    return int(base + r + np.searchsorted(x - base - np.arange(len(x)), r, side="right"))


def negative_decode(rowptr, col, offsets, k, start=False):
    """Candidate indices k -> int32 [2, S] pairs (tfgk_neg_decode)."""
    k = np.asarray(k, np.int64)
    rows = np.searchsorted(offsets, k, side="right") - 1
    out = np.empty((2, len(k)), np.int32)
    for s, (kk, i) in enumerate(zip(k, rows)):
        base = 0 if start else i + 1
        out[0, s] = i
        out[1, s] = _decode_in_row(col[rowptr[i]:rowptr[i + 1]], base, kk - offsets[i])
    return out


def negative_candidates(edge_index, num_nodes):
    """The whole candidate list in order: np.nonzero(np.triu(adj, 1)) of graph_utils.py:391-396 without the matrix."""
    rowptr, col, offsets = negative_structure(edge_index, num_nodes)
    return negative_decode(rowptr, col, offsets, np.arange(offsets[-1]))


def _random_keys(n, seed, stream=RNG_STREAM_LINK):
    return random_below64(seed, stream, np.arange(n, dtype=np.uint64), 1 << 32).astype(np.uint32)


def draw_candidates(C, S, replace, seed, stream=RNG_STREAM_LINK):
    """S indices in [0, C): independent draws; or distinct - a shuffle of the whole range when 2 S > C, otherwise
    rounds in which the later duplicates (stable sort order) are redrawn with counter (sample, round)."""
    if replace:
        return random_below64(seed, stream, np.arange(S, dtype=np.uint64), C)
    if 2 * S > C:
        return np.argsort(_random_keys(C, seed, stream), kind="stable")[:S].astype(np.int64)
    k = random_below64(seed, stream, np.arange(S, dtype=np.uint64), C)
    rnd = 0
    while True:
        order = np.argsort(k, kind="stable")
        dup = np.zeros(S, bool)
        dup[order[1:]] = k[order[1:]] == k[order[:-1]]
        idx = np.nonzero(dup)[0]
        if len(idx) == 0:
            return k
        rnd += 1
        k[idx] = random_below64(seed, stream, (np.uint64(rnd) << _S32) | idx.astype(np.uint64), C)


def negative_sampling(num_samples, num_nodes, edge_index=None, replace=True, batch_size=None, seed=0):
    """utils/graph_utils.py:369-412 with the counter-based draws (tfgk_neg_* / tfgk_random_pairs_i32)."""
    out = []
    for b in range(1 if batch_size is None else batch_size):
        sb = link_batch_seed(seed, b)
        if edge_index is None:
            s2 = np.arange(num_samples, dtype=np.uint64) * np.uint64(2)
            out.append(np.stack([random_below64(sb, RNG_STREAM_LINK, s2, num_nodes),
                                 random_below64(sb, RNG_STREAM_LINK, s2 + np.uint64(1), num_nodes)]).astype(np.int32))
            continue
        rowptr, col, offsets = negative_structure(edge_index, num_nodes)
        C = int(offsets[-1])
        if num_samples and C == 0:
            raise ValueError("no candidate pair")
        if not replace and num_samples > C:
            raise ValueError("more samples than candidates")
        k = draw_candidates(C, num_samples, replace, sb) if num_samples else np.zeros(0, np.int64)
        out.append(negative_decode(rowptr, col, offsets, k))
    return out[0] if batch_size is None else out


def negative_sampling_with_start_node(start_node_index, num_nodes, edge_index=None, seed=0):
    """utils/graph_utils.py:415-452 without the retry loop: b uniform over [0, N) minus (out-neighbours of a and a)."""
    start = np.asarray(start_node_index, np.int64).reshape(-1)
    S = len(start)
    if edge_index is None:
        end = random_below64(seed, RNG_STREAM_LINK, np.arange(S, dtype=np.uint64) * np.uint64(2) + np.uint64(1), num_nodes)
        return np.stack([start, end]).astype(np.int32)
    rowptr, col, offsets = negative_structure(edge_index, num_nodes, start=True)
    end = np.empty(S, np.int64)
    for s, a in enumerate(start):
        cnt = int(offsets[a + 1] - offsets[a])
        if cnt == 0:
            raise ValueError("start node {} has no negative partner".format(a))
        r = int(random_below64(seed, RNG_STREAM_LINK, np.array([s], np.uint64), cnt)[0])
        end[s] = _decode_in_row(col[rowptr[a]:rowptr[a + 1]], 0, r)
    return np.stack([start, end]).astype(np.int32)


def edge_train_test_split(edge_index, test_size, edge_weight=None, seed=0):
    """utils/graph_utils.py:488-535: merged upper edges (max weights), permuted by Philox keys; sklearn's sizes,
    test = the first n_test of the permutation.  Returns (train_index, test_index, train_w, test_w)."""
    props = None if edge_weight is None else [o._as_f32(edge_weight)]
    upper, up_props = o.convert_edge_to_upper(edge_index, props, None if props is None else ["max"])
    n = upper.shape[1]
    n_test = int(np.ceil(test_size * n)) if isinstance(test_size, float) else int(test_size)
    perm = np.argsort(_random_keys(n, seed), kind="stable")
    test, train = perm[:n_test], perm[n_test:]
    if up_props is None:
        return upper[:, train], upper[:, test], None, None
    return upper[:, train], upper[:, test], up_props[0][train], up_props[0][test]


def predict_edge_torch(embedded, edge_index):
    """demo/demo_gae.py:53-60 on torch ops (tf.gather both endpoints, multiply, reduce_sum over the last axis).
    Differentiable w.r.t. embedded: in float64 it is the reference the edge-scoring kernel and its backward are checked
    against."""
    row, col = edge_index[0], edge_index[1]
    return (embedded.index_select(0, row) * embedded.index_select(0, col)).sum(-1)
