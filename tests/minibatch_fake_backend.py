# coding=utf-8
"""TEST DOUBLE for K13 and the relabelling entries (ops.neighbor_sample_rows, ops.reindex, ops.frontier): the CPU fake
kernel layer of tests/fake_backend.py plus numpy restatements, so that the host logic of the mini-batch sampler and the
sampled-subgraph helpers runs without a GPU.  Injected with monkeypatch; the product has no such path."""
import numpy as np

import fake_backend
import minibatch_ref as ref
from fake_backend import _np, _t


def install(monkeypatch):
    fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def neighbor_sample_rows(rowptr, rows, k=None, ratio=None, padding=False, seed=0, rng_stream=1):
        if not isinstance(padding, bool) and padding == ops.SAMPLE_HEAD:
            padding = "head"
        rows = _np(rows)
        n_rows = rowptr.numel() - 1
        if rows.size and (rows.min() < 0 or rows.max() >= n_rows):
            raise IndexError("listed rows outside [0, {})".format(n_rows))
        t, p, rp = ref.sample_rows(_np(rowptr), rows, k, ratio, padding, seed, rng_stream)
        return _t(t), _t(p), _t(rp)

    def reindex(nodes, ids, node_map):
        nodes, N = _np(nodes), node_map.numel()
        assert np.all(_np(node_map) == -1), "the map must be clean between calls"
        if nodes.size and (nodes.min() < 0 or nodes.max() >= N):
            raise IndexError("node ids outside [0, {})".format(N))
        table = {}
        for i, v in enumerate(nodes.tolist()):
            table.setdefault(v, i)
        out = np.array([table.get(v, -1) for v in _np(ids).tolist()], np.int32)
        return _t(out), len(nodes) - len(table)

    def frontier(nodes, n_nodes, cols, node_map):
        assert np.all(_np(node_map) == -1), "the map must be clean between calls"
        buf = _np(nodes)
        table = {v: i for i, v in enumerate(buf[:n_nodes].tolist())}
        n = n_nodes
        local = []
        for c in _np(cols).tolist():
            if c not in table:
                table[c] = n
                buf[n] = c
                n += 1
            local.append(table[c])
        nodes.copy_(_t(buf))
        return _t(np.array(local, np.int32)), n - n_nodes, 0

    monkeypatch.setattr(ops, "neighbor_sample_rows", neighbor_sample_rows)
    monkeypatch.setattr(ops, "reindex", reindex)
    monkeypatch.setattr(ops, "frontier", frontier)
