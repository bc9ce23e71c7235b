# coding=utf-8
"""Numpy restatement of the weighted fan-out rule (include/tfgk.h, "weighted block sampler"): rng.cuh's log_rn and key in
float64 with every operation rounded on its own, the per-row draw with and without replacement, and the weighted
neighbourhood of sample_blocks / sample_neighborhood, hop by hop with a dict, optionally with excluded CSR positions."""
import math

import numpy as np

from oracle import tfg_oracle as o

RNG_STREAM_WEIGHTED = 3
_MASK64 = (1 << 64) - 1


def _d(h):
    return np.array([h], np.uint64).view(np.float64)[0]


_LG = [_d(0x3FE5555555555593), _d(0x3FD999999997FA04), _d(0x3FD2492494229359), _d(0x3FCC71C51D8E78AF),
       _d(0x3FC7466496CB03DE), _d(0x3FC39A09D078C69F), _d(0x3FC2F112DF3E5244)]
_LN2_HI, _LN2_LO = _d(0x3FE62E42FEE00000), _d(0x3DEA39EF35793C76)


def log_rn(u):
    """rng.cuh's log_rn over a float64 array of positive normal values."""
    u = np.asarray(u, np.float64)
    b = u.view(np.uint64)
    e = (b >> np.uint64(52)).astype(np.int64) - 1023
    mb = (b & np.uint64(0x000FFFFFFFFFFFFF)) | np.uint64(0x3FF0000000000000)
    big = mb > np.uint64(0x3FF6A09E667F3BCD)
    mb = np.where(big, mb - np.uint64(1 << 52), mb)
    e = e + big
    f = mb.view(np.float64) - 1.0
    s = f / (2.0 + f)
    z = s * s
    w = z * z
    Lg1, Lg2, Lg3, Lg4, Lg5, Lg6, Lg7 = _LG
    t1 = w * (Lg2 + w * (Lg4 + w * Lg6))
    t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)))
    R = t2 + t1
    hfsq = 0.5 * (f * f)
    dk = e.astype(np.float64)
    return dk * _LN2_HI - ((hfsq - (s * (hfsq + R) + dk * _LN2_LO)) - f)


def uniform(seed, stream, v, r, j):
    """u in (0, 1] of the key counter (v, r, stream, j) under `seed`: 53 bits of lanes 0 and 1."""
    v = np.asarray(v, np.uint32)
    shape = v.shape
    counter = np.stack([v, np.broadcast_to(np.asarray(r, np.uint32), shape),
                        np.full(shape, stream, np.uint32), np.broadcast_to(np.asarray(j, np.uint32), shape)], axis=-1)
    key = np.empty(shape + (2,), np.uint32)
    key[..., 0] = seed & 0xFFFFFFFF
    key[..., 1] = (seed >> 32) & 0xFFFFFFFF
    x = o.philox4x32(counter, key)
    u64 = x[..., 0].astype(np.uint64) | (x[..., 1].astype(np.uint64) << np.uint64(32))
    return ((u64 >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * 2.0 ** -53


def keys(seed, stream, v, r, j, w):
    """The keys' bits (uint64, sign cleared) of entries v of row r, draw j, weights w (float32, > 0)."""
    e = -log_rn(uniform(seed, stream, v, r, j)) / np.asarray(w, np.float32).astype(np.float64)
    return e.view(np.uint64) & np.uint64(0x7FFFFFFFFFFFFFFF)


def draw_row(w_kept, r, k, padding, seed, stream=RNG_STREAM_WEIGHTED):
    """Virtual positions drawn from one row whose kept entries have weights w_kept (in CSR order), fan-out k >= 0."""
    w_kept = np.asarray(w_kept, np.float32)
    cand = np.flatnonzero(w_kept > 0)
    d = cand.size
    if d == 0 or k == 0:
        return np.zeros(0, np.int64)
    if padding and k >= d:
        out = np.empty(k, np.int64)
        for j in range(k):
            kk = keys(seed, stream, cand, r, j + 1, w_kept[cand])
            out[j] = cand[np.lexsort((cand, kk))[0]]
        return out
    if k >= d:
        return cand.astype(np.int64)
    kk = keys(seed, stream, cand, r, 0, w_kept[cand])
    return np.sort(cand[np.lexsort((cand, kk))[:k]]).astype(np.int64)


def row_positions(rowptr, w_csr, r, k, padding, seed, excluded=(), stream=RNG_STREAM_WEIGHTED):
    """Real CSR positions drawn for global row r (fan-out None: every kept entry), `excluded` its excluded positions."""
    p0, p1 = int(rowptr[r]), int(rowptr[r + 1])
    excl = set(int(p) for p in excluded)
    kept = np.array([p for p in range(p0, p1) if p not in excl], np.int64)
    if k is None:
        return kept
    return kept[draw_row(w_csr[kept], r, k, padding, seed, stream)]


def hop_seed(seed, h):
    return (seed + h * 0x9E3779B97F4A7C15) & _MASK64


def neighborhood(rowptr, col, w_csr, seeds, fanouts, padding=False, seed=0, excluded=None):
    """(node_index, edge_index_list, edge_weight_list, hop_sizes) of a weighted sample_neighborhood / sample_blocks batch
    (layer 0 first, as SampledNeighborhood).  excluded: {list position t: CSR positions} removed at every hop."""
    rowptr = np.asarray(rowptr, np.int64)
    n_rows = len(rowptr) - 1
    nodes = [int(v) for v in seeds]
    where = {v: i for i, v in enumerate(nodes)}
    hop_sizes, edges, weights = [len(nodes)], [], []
    for h, k in enumerate(reversed(list(fanouts))):
        rows, cols, ws = [], [], []
        for t in range(len(nodes)):
            v = nodes[t]
            if v >= n_rows:
                continue
            ex = excluded.get(t, ()) if excluded else ()
            for p in row_positions(rowptr, w_csr, v, k, padding, hop_seed(seed, h), ex):
                c = int(col[p])
                if c not in where:
                    where[c] = len(nodes)
                    nodes.append(c)
                rows.append(t)
                cols.append(where[c])
                ws.append(w_csr[p])
        edges.append(np.array([rows, cols], np.int32).reshape(2, -1))
        weights.append(np.array(ws, np.float32))
        hop_sizes.append(len(nodes))
    return np.array(nodes, np.int32), edges[::-1], weights[::-1], hop_sizes


def ulp_error(got, x):
    """|got - ln(x)| in units of the last place of math.log(x)."""
    want = math.log(x)
    return abs(got - want) / max(math.ulp(want), 2.0 ** -1074)
