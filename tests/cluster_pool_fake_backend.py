# coding=utf-8
"""TEST DOUBLE for K8 (ops.graph_tmm / ops.graph_rmm, the per-graph dense algebra of DiffPool and MinCutPool): the CPU
fake kernel layer of tests/edge_grad_fake_backend.py plus numpy restatements of tfgk_graph_tmm_f32 and
tfgk_graph_rmm_f32, so that the host logic of the pooling API runs without a GPU.  Injected with monkeypatch; the
product has no such path."""
import numpy as np

import edge_grad_fake_backend
from fake_backend import _np, _t


def tmm_reference(S, Y, gptr, gnodes=None):
    """out[g*C + c] = sum over graph g's node-list positions p (node gnodes[p] or p) of S[n, c] * Y[n] (float32 sums)."""
    S, Y = np.asarray(S, np.float32), np.asarray(Y, np.float32)
    G, C, D = len(gptr) - 1, S.shape[1], Y.shape[1]
    out = np.zeros((G * C, D), np.float32)
    for g in range(G):
        nodes = np.arange(gptr[g], gptr[g + 1])
        if gnodes is not None:
            nodes = np.asarray(gnodes)[nodes]
        out[g * C:(g + 1) * C] = S[nodes].T @ Y[nodes]
    return out


def rmm_reference(Y, B, node_graph, C, trans=False, beta=0.0, out=None):
    """out[n] = beta * out[n] + Y[n] @ B_g (or @ B_g^T), B_g = rows g*C .. g*C + C - 1 of B."""
    Y, B = np.asarray(Y, np.float32), np.asarray(B, np.float32)
    blocks = B.reshape(-1, C, B.shape[1])[np.asarray(node_graph)]          # [N, C, K]
    res = np.einsum("nk,nck->nc", Y, blocks) if trans else np.einsum("nc,nck->nk", Y, blocks)
    res = res.astype(np.float32)
    if beta != 0.0:
        res = (np.float32(beta) * np.asarray(out, np.float32) + res).astype(np.float32)
    return res


def install(monkeypatch):
    edge_grad_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def graph_tmm(S, Y, gptr, num_graphs, gnodes=None, out=None):
        res = _t(tmm_reference(_np(S), _np(Y), _np(gptr), _np(gnodes)))
        if out is not None:
            out.copy_(res)
            return out
        return res

    def graph_rmm(Y, B, node_graph, num_clusters, trans=False, beta=0.0, out=None):
        res = _t(rmm_reference(_np(Y), _np(B), _np(node_graph), int(num_clusters), trans, beta, _np(out)))
        if out is not None:
            out.copy_(res)
            return out
        return res

    monkeypatch.setattr(ops, "graph_tmm", graph_tmm)
    monkeypatch.setattr(ops, "graph_rmm", graph_rmm)
