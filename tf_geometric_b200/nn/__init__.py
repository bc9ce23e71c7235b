# coding=utf-8
"""Functional API: the names a tf_geometric user finds under `tfg.nn`, resolved from this package's own modules
(message-passing hot path and the rows of SURVEY.md section 8f)."""
from . import conv, kernel, link, pool, sampling
from ..ops import relu

_EXPORTS = {
    kernel.map_reduce: ("aggregate_neighbors", "identity_mapper", "neighbor_count_mapper", "gcn_mapper", "sum_reducer",
                        "mean_reducer", "max_reducer", "sum_updater", "identity_updater"),
    kernel.segment: ("segment_softmax", "segment_count"),
    conv.gcn: ("gcn", "gcn_norm_adj", "gcn_norm_edge", "gcn_build_cache_by_adj", "gcn_build_cache_for_graph", "compute_cache_key"),
    conv.gat: ("gat",),
    conv.graph_sage: ("mean_graph_sage", "sum_graph_sage", "gcn_graph_sage", "mean_pool_graph_sage", "max_pool_graph_sage",
                        "lstm_graph_sage"),
    conv.appnp: ("appnp",),
    conv.propagation: ("sgc", "ssgc", "tagcn", "gin", "gin_updater", "le_conv", "chebynet", "chebynet_norm_edge", "get_laplacian"),
    pool.common_pool: ("mean_pool", "sum_pool", "max_pool", "min_pool"),
    pool.set2set: ("set2set",),
    pool.topk_pool: ("topk_pool",),
    pool.score_pool: ("sag_pool", "sort_pool"),
    pool.diff_pool: ("diff_pool", "diff_pool_coarsen"),
    pool.min_cut_pool: ("min_cut_pool", "min_cut_pool_coarsen", "min_cut_pool_compute_losses"),
    pool.cluster_pool: ("cluster_pool",),
    pool.asap: ("asap",),
    sampling.drop_edge: ("drop_edge",),
    link.predict_edge: ("predict_edge",),
}
for _module, _names in _EXPORTS.items():
    for _name in _names:
        globals()[_name] = getattr(_module, _name)
__all__ = ["relu"] + [n for names in _EXPORTS.values() for n in names]
