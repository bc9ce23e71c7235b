# coding=utf-8
"""TEST DOUBLE for link prediction on blocks (ops.link_block_sample, ops.link_tail_negatives and
K6's ops.edge_dot) on top of tests/block_fake_backend.py: numpy statements
of the pair begin (first-occurrence relabelling of the endpoints), the tail negatives, the exclusion lists (the kernel's
sort and per-row binary search) and the virtual-to-real position mapping, and a link block sampler that samples the CSR
with the excluded positions removed through the block sampler's restatement.  Injected with monkeypatch; the product has
no such path.  `calls` counts the fake entries and records the flags of every CSR build."""
import numpy as np

import block_fake_backend
import link_oracle as lo
from fake_backend import _np, _t


def pair_begin_np(pairs, N):
    """(seeds, local [2, P], n_bad): the distinct valid endpoints pair by pair (source, then destination) in
    first-occurrence order, the pairs relabelled (-1 for an id outside [0, N)) and the number of such endpoints."""
    pairs = np.asarray(pairs, np.int64).reshape(2, -1)
    where, seeds, n_bad = {}, [], 0
    for v in pairs.T.reshape(-1).tolist():
        if v < 0 or v >= N:
            n_bad += 1
        elif v not in where:
            where[v] = len(seeds)
            seeds.append(v)
    local = np.array([[where.get(int(v), -1) for v in side] for side in pairs], np.int32).reshape(2, -1)
    return np.array(seeds, np.int32), local, n_bad


def tail_negatives_np(src, q, N, seed, stream=2):
    n = len(src) * q
    return np.stack([np.repeat(np.asarray(src, np.int32), q),
                     lo.random_below64(seed, stream, np.arange(n, dtype=np.uint64), N).astype(np.int32)]).reshape(2, n)


def exclusion_lists_np(rowptr, col, nodes, cap, ts, td):
    """(excl_off int64 [cap + 1], excl_pos) as the kernels build them: the targets sorted by (source, destination) with
    two stable passes, then each targeted row's columns tested by binary search against its sorted destinations."""
    ts, td = np.asarray(ts, np.int64), np.asarray(td, np.int64)
    order = np.argsort(td.astype(np.uint32), kind="stable")
    ts, td = ts[order], td[order]
    order = np.argsort(ts.astype(np.uint32), kind="stable")
    ts, td = ts[order], td[order]
    counts, lists = np.zeros(cap, np.int64), []
    for t in range(cap):
        dests = td[ts == t]
        pos = []
        if dests.size and t < len(nodes) and 0 <= nodes[t] < len(rowptr) - 1:
            r = int(nodes[t])
            for p in range(rowptr[r], rowptr[r + 1]):
                i = np.searchsorted(dests, col[p])
                if i < dests.size and dests[i] == col[p]:
                    pos.append(p)
        counts[t] = len(pos)
        lists.append(pos)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return off, np.array([p for lst in lists for p in lst], np.int64)


def virtual_to_real_np(excluded, v):
    """The position in its row of the v-th kept entry, given the row's ascending excluded offsets: v plus the number of
    excluded offsets e_j with e_j - j <= v (the kernels' binary search)."""
    e = np.asarray(excluded, np.int64)
    return int(v) + int(np.searchsorted(e - np.arange(e.size), v, side="right"))


def install(monkeypatch):
    block_calls = block_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops
    calls = {"link_block_sample": 0, "link_tail_negatives": 0, "edge_dot": 0, "csr_build": block_calls["csr_build"],
             "csr_build_plan": []}
    block_sample = ops.block_sample
    plain_csr_build = ops.csr_build

    def csr_build(row, col, n_rows, n_cols=None, ids_in_range=False, plan=True):
        calls["csr_build_plan"].append((bool(ids_in_range), bool(plan)))
        return plain_csr_build(row, col, n_rows, n_cols, ids_in_range)

    def edge_dot(h, row, col, out=None):
        calls["edge_dot"] += 1
        hn = _np(h)
        return _t((hn[_np(row)] * hn[_np(col)]).sum(axis=1).astype(np.float32))

    def link_block_sample(rowptr, col, w_csr, pairs, n_pos, fanouts, keys, node_map, exclude=None, padding=False,
                          rng_stream=1):
        calls["link_block_sample"] += 1
        assert np.all(_np(node_map) == -1), "the map must be clean between calls"
        ops._check_block_fanouts(fanouts, padding)
        if exclude not in (None, "self", "reverse"):
            raise ValueError("link_block_sample: exclude must be None, 'self' or 'reverse'")
        rp, c, w, N = _np(rowptr).astype(np.int64), _np(col), _np(w_csr), node_map.numel()
        pairs = _np(pairs)
        seeds, local, n_bad = pair_begin_np(pairs, N)
        excluded = None
        if exclude is not None:
            ts, td = local[0, :n_pos], pairs[1, :n_pos]
            if exclude == "reverse":
                ts, td = np.concatenate([ts, local[1, :n_pos]]), np.concatenate([td, pairs[0, :n_pos]])
            cap = 2 * pairs.shape[1]
            off, pos = exclusion_lists_np(rp, c, seeds, cap, ts, td)
            keep = np.ones(c.size, bool)
            keep[pos] = False
            counts = np.diff(rp) - np.bincount(np.searchsorted(rp, pos, side="right") - 1, minlength=rp.size - 1)
            rp = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
            c, w = c[keep], w[keep]
            excluded = (_t(off), cap)
        if n_bad:
            return _t(seeds), [len(seeds)] * (len(fanouts) + 1), [], n_bad, _t(local), excluded
        nodes, sizes, hops, _, _ = block_sample(_t(rp), _t(c), _t(w), _t(seeds), fanouts, keys, node_map, padding,
                                                rng_stream)
        return nodes, sizes, hops, 0, _t(local), excluded

    def link_tail_negatives(src, q, num_nodes, seed, out_row, out_col, rng_stream=2):
        calls["link_tail_negatives"] += 1
        neg = tail_negatives_np(_np(src), q, num_nodes, seed, rng_stream)
        out_row.copy_(_t(neg[0]))
        out_col.copy_(_t(neg[1]))

    monkeypatch.setattr(ops, "csr_build", csr_build)
    monkeypatch.setattr(ops, "edge_dot", edge_dot)
    monkeypatch.setattr(ops, "link_block_sample", link_block_sample)
    monkeypatch.setattr(ops, "link_tail_negatives", link_tail_negatives)
    return calls
