# coding=utf-8
"""tf_geometric_b200 - an H100 (sm_90a) message-passing backend behind tf_geometric's own API surface.

    import tf_geometric_b200 as tfg
    graph = tfg.Graph(x, edge_index).to_device()
    layer = tfg.layers.GCN(128, activation=tfg.nn.relu)
    layer.build_cache_for_graph(graph)
    h = layer([graph.x, graph.edge_index, graph.edge_weight], cache=graph.cache)

Scope: the gather -> edge-apply -> segment-aggregate path under tfg.nn.gcn / gat / *_graph_sage / appnp
(SURVEY.md section 8).  All arithmetic runs in libtfgk.so (hand-written CUDA, include/tfgk.h); importing the package
works without a GPU, calling any operator does not (there is no CPU fallback).
"""
from . import _ffi, ops, nn, layers, utils, dist, peer
from .data.graph import Graph, BatchGraph
from .sparse import SparseMatrix
from ._rng import set_seed

__version__ = "0.1.0"
