# coding=utf-8
from . import graph_utils
from .graph_utils import (add_self_loop_edge, remove_self_loop_edge, convert_edge_to_directed, merge_duplicated_edge,
                          convert_edge_to_upper, convert_edge_index_to_edge_hash, convert_edge_hash_to_edge_index,
                          adj_norm_edge, compute_num_or_size_splits, negative_sampling,
                          negative_sampling_with_start_node, edge_train_test_split, convert_dense_adj_to_edge,
                          convert_dense_assign_to_edge, convert_x_to_3d, reindex_sampled_edge_index,
                          compute_edge_mask_by_node_index, extract_unique_edge)
from .sampling import (RandomNeighborSampler, UniformNeighborSampler, SampledNeighborhood, SampledBlocks, Block,
                       SelfLoopBlock, GcnBlock, SourceRows, HostFeatureTable, rank_source_rows, HostNeighborSampler,
                       LinkBlocks, layerwise_chunk_bytes)
from .layerwise import layerwise_inference
