# coding=utf-8
"""Numpy restatements for the mini-batch sampler: K13 (the full-graph sampler's draws for a list of rows), the hop-by-hop
neighbourhood of RandomNeighborSampler.sample_neighborhood, and the reference's sampled-subgraph helpers
(utils/graph_utils.py:455-485, :538-551, :946-975 of tf_geometric) restated with Python sets and dicts."""
import numpy as np

from oracle import tfg_oracle as o

_MASK64 = (1 << 64) - 1


def hop_seed(seed, h):
    return (seed + h * 0x9E3779B97F4A7C15) & _MASK64


def sample_rows(rowptr, rows, k=None, ratio=None, padding=False, seed=0, stream=o.RNG_STREAM_SAMPLER):
    """(list position int32 [S], CSR position int32 [S], offsets int64 [R+1]): row t's slice is what the full-graph
    sampler draws for global row rows[t]."""
    _, pos, rp = o.neighbor_sample_csr(rowptr, k, ratio, padding, seed, stream)
    t_out, p_out, counts = [], [], []
    for t, r in enumerate(np.asarray(rows, np.int64)):
        p = pos[rp[r]:rp[r + 1]]
        t_out.append(np.full(len(p), t, np.int32))
        p_out.append(p.astype(np.int32))
        counts.append(len(p))
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    if not t_out:
        return np.zeros(0, np.int32), np.zeros(0, np.int32), offsets
    return np.concatenate(t_out), np.concatenate(p_out), offsets


def neighborhood(rowptr, col, w_csr, seeds, fanouts, padding=False, seed=0):
    """(node_index, edge_index_list, edge_weight_list, hop_sizes) of sample_neighborhood, built edge by edge with a dict:
    hop h draws fanouts[-1 - h] for every listed node with key hop_seed(seed, h); a column seen for the first time is
    appended to the list."""
    rowptr = np.asarray(rowptr, np.int64)
    n_rows = len(rowptr) - 1
    nodes = [int(v) for v in seeds]
    where = {v: i for i, v in enumerate(nodes)}
    assert len(where) == len(nodes), "duplicate seeds"
    hop_sizes, edges, weights = [len(nodes)], [], []
    for h, k in enumerate(reversed(list(fanouts))):
        _, pos, rp = o.neighbor_sample_csr(rowptr, k, None, padding, hop_seed(seed, h))
        rows, cols, ws = [], [], []
        for t in range(len(nodes)):
            v = nodes[t]
            if v >= n_rows:
                continue
            for p in pos[rp[v]:rp[v + 1]]:
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


def reindex_sampled_edge_index(sampled_edge_index, sampled_node_index):
    table = {}
    for i, v in enumerate(np.asarray(sampled_node_index).reshape(-1).tolist()):
        if v in table:
            raise ValueError("duplicate key")
        table[v] = i
    ei = np.asarray(sampled_edge_index)
    return np.vectorize(lambda v: table.get(int(v), -1), otypes=[np.int32])(ei).reshape(ei.shape)


def compute_edge_mask_by_node_index(edge_index, node_index):
    s = set(np.asarray(node_index).reshape(-1).tolist())
    ei = np.asarray(edge_index)
    return np.array([int(a) in s and int(b) in s for a, b in zip(ei[0], ei[1])], bool)


def extract_unique_edge(edge_index, edge_weight=None, mode="undirected"):
    ei = np.asarray(edge_index, np.int32)
    seen, keep = set(), []
    for i in range(ei.shape[1]):
        e = ei[:, i]
        e = tuple(sorted(e)) if mode == "undirected" else tuple(e)
        if e not in seen:
            seen.add(e)
            keep.append(i)
    w = None if edge_weight is None else np.asarray(edge_weight, np.float32)[keep]
    return ei[:, keep], w
