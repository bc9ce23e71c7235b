# coding=utf-8
"""Numpy restatement of the layer-neighbour (LABOR-0) rule (include/tfgk.h, "LABOR block sampler"): one Philox variate
per column node id under the hop key, the per-row integer test u * d < k 2^32, and the LABOR neighbourhood of
sample_blocks / sample_link_blocks hop by hop with a dict, optionally with excluded CSR positions and layer dependency."""
import numpy as np

from oracle import tfg_oracle as o
from weighted_ref import hop_seed

RNG_STREAM_LABOR = 4


def variates(cols, key, stream=RNG_STREAM_LABOR):
    """u_c (uint32) of the columns `cols` under the hop key: lane 0 of the Philox block with counter (c, 0, stream, 0)."""
    c = np.asarray(cols, np.int64).astype(np.uint32)
    shape = c.shape
    counter = np.stack([c, np.zeros(shape, np.uint32), np.full(shape, stream, np.uint32), np.zeros(shape, np.uint32)],
                       axis=-1)
    k = np.empty(shape + (2,), np.uint32)
    k[..., 0] = key & 0xFFFFFFFF
    k[..., 1] = (key >> 32) & 0xFFFFFFFF
    return o.philox4x32(counter, k)[..., 0]


def keep_mask(u, d, k):
    """The row rule on variates u (uint32) of a row of d candidates and integer fan-out k >= 0."""
    u = np.asarray(u, np.uint32)
    if k == 0:
        return np.zeros(u.shape, bool)
    if d <= k:
        return np.ones(u.shape, bool)
    return u.astype(np.uint64) * np.uint64(d) < np.uint64(k) << np.uint64(32)


def pi(k, d):
    """P(a candidate is kept) for integer fan-out k and d candidates: ceil(k 2^32 / d) / 2^32, or 1 for d <= k."""
    if k == 0:
        return 0.0
    if d <= k:
        return 1.0
    return float(-(-(k << 32) // d)) / 2.0 ** 32


def row_positions(rowptr, col, r, k, key, excluded=()):
    """Real CSR positions kept for global row r (fan-out None: every kept entry), `excluded` its excluded positions."""
    p0, p1 = int(rowptr[r]), int(rowptr[r + 1])
    excl = set(int(p) for p in excluded)
    kept = np.array([p for p in range(p0, p1) if p not in excl], np.int64)
    if k is None:
        return kept
    return kept[keep_mask(variates(np.asarray(col)[kept], key), kept.size, k)]


def hop_keys(seed, L, layer_dependency=False):
    return [hop_seed(seed, 0 if layer_dependency else h) for h in range(L)]


def neighborhood(rowptr, col, w_csr, seeds, fanouts, seed=0, layer_dependency=False, excluded=None):
    """(node_index, edge_index_list, edge_weight_list, global_col_list, hop_sizes) of a LABOR sample_blocks batch (layer 0
    first, as SampledBlocks' blocks).  excluded: {list position t: CSR positions} removed at every hop."""
    rowptr = np.asarray(rowptr, np.int64)
    col = np.asarray(col)
    n_rows = len(rowptr) - 1
    nodes = [int(v) for v in seeds]
    where = {v: i for i, v in enumerate(nodes)}
    keys = hop_keys(seed, len(fanouts), layer_dependency)
    hop_sizes, edges, weights, gcols = [len(nodes)], [], [], []
    for h, k in enumerate(reversed(list(fanouts))):
        rows, cols, ws, gs = [], [], [], []
        for t in range(len(nodes)):
            v = nodes[t]
            if v >= n_rows:
                continue
            ex = excluded.get(t, ()) if excluded else ()
            for p in row_positions(rowptr, col, v, k, keys[h], ex):
                c = int(col[p])
                if c not in where:
                    where[c] = len(nodes)
                    nodes.append(c)
                rows.append(t)
                cols.append(where[c])
                ws.append(w_csr[p])
                gs.append(c)
        edges.append(np.array([rows, cols], np.int32).reshape(2, -1))
        weights.append(np.array(ws, np.float32))
        gcols.append(np.array(gs, np.int32))
        hop_sizes.append(len(nodes))
    return np.array(nodes, np.int32), edges[::-1], weights[::-1], gcols[::-1], hop_sizes
