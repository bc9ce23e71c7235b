# coding=utf-8
"""tfg.layers.GCN (reference layers/conv/gcn.py:12-156)."""
import warnings

import torch

from ... import ops
from ...sparse import SparseMatrix
from ...nn.conv.gcn import gcn, gcn_build_cache_for_graph, gcn_build_cache_by_adj
from ...utils.graph_utils import compute_num_or_size_splits
from ...utils.sampling import GcnBlock
from .._base import Layer


class GCN(Layer):
    """Graph Convolutional Layer: act(norm(A) (x W) + b)."""

    def __init__(self, units, activation=None, use_kernel=True, use_bias=True,
                 norm="both", add_self_loop=True, sym=True, renorm=True, improved=False,
                 edge_drop_rate=0.0, num_splits=None, num_or_size_splits=None,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 / torch.float8_e4m3fn for inference with bf16 / fp8
        message rows (nn.gcn)."""
        super().__init__(*args, **kwargs)
        ops.conv_message_dtype(message_dtype)     # ValueError for anything but fp32 / bf16 / fp8 e4m3
        self.message_dtype = message_dtype
        self.units = units
        self.activation = activation
        self.use_kernel = use_kernel
        self.use_bias = use_bias
        self.edge_drop_rate = edge_drop_rate
        self.kernel = None
        self.bias = None
        self.norm = norm
        self.add_self_loop = add_self_loop
        self.sym = sym
        self.renorm = renorm
        self.improved = improved
        self.kernel_regularizer = kernel_regularizer
        self.bias_regularizer = bias_regularizer
        if num_splits is not None and num_or_size_splits is not None:
            raise Exception("cannot provide both num_splits and num_or_size_splits for GCN")
        self.num_splits = num_splits
        self.num_or_size_splits = num_or_size_splits

    def build(self, input_shapes, device=None):
        num_features = input_shapes[0][-1]
        if self.num_splits is not None:
            num_h_features = self.units if self.use_kernel else num_features
            self.num_or_size_splits = compute_num_or_size_splits(num_h_features, self.num_splits)
        if self.use_kernel:
            self.kernel = self.add_weight("kernel", [num_features, self.units], "glorot_uniform", device=device)
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units if self.use_kernel else num_features], "zeros",
                                        device=device)

    def build_cache_by_adj(self, sparse_adj, override=False, cache=None):
        return gcn_build_cache_by_adj(sparse_adj, self.norm, self.add_self_loop, self.sym, self.renorm, self.improved,
                                      override=override, cache=cache)

    def build_cache_for_graph(self, graph, override=False):
        gcn_build_cache_for_graph(graph, self.norm, self.add_self_loop, self.sym, self.renorm, self.improved,
                                  override=override)

    def cache_normed_edge(self, graph, override=False):
        warnings.warn("'GCN.cache_normed_edge(graph, override)' is deprecated, use "
                      "'GCN.build_cache_for_graph(graph, override)' instead", DeprecationWarning)
        return self.build_cache_for_graph(graph, override=override)

    def partitioned_projections(self):
        """All-row projections this layer needs on a partitioned graph: [(key, [(weight, bias, act code)])].  None when
        the input is narrower than the output (ops.spmm_proj_shape) on the GPU: the rows of x are gathered and projected
        after aggregation instead (dist.gcn_partitioned)."""
        if not self.use_kernel or (self.kernel.is_cuda and ops.spmm_proj_shape(self.kernel.shape[0], self.kernel.shape[1])):
            return []
        return [((id(self.kernel),), [(self.kernel, None, ops.ACT_NONE)])]

    def _call_partitioned(self, x_local, pg):
        from ... import dist as tdist
        if not (self.norm == "both" and self.add_self_loop and self.sym):
            raise NotImplementedError("partitioned GCN implements the default normalisation (norm='both', self loops, sym)")
        return tdist.gcn_partitioned(pg, x_local, self.kernel, self.bias, self.activation, renorm=self.renorm,
                                     improved=self.improved)

    def call(self, inputs, cache=None, split=True, training=None, mask=None):
        """inputs: [x, sparse_adj], [x, edge_index] or [x, edge_index, edge_weight]; on a sampled block
        [x_src or batch.source_rows(x), block.with_gcn_norm()] (nn.gcn); on several GPUs [x_local, partitioned_graph]
        (tf_geometric_b200.dist.PartitionedGraph; x_local may be the result of its share())."""
        if hasattr(inputs[1], "part") and hasattr(inputs[1], "project_all_rows"):
            if ops.conv_message_dtype(self.message_dtype) is not None:
                raise NotImplementedError("message_dtype={} is not implemented for partitioned graphs".format(
                    str(ops.conv_message_dtype(self.message_dtype)).replace("torch.", "")))
            return self._call_partitioned(inputs[0], inputs[1])
        if isinstance(inputs[1], GcnBlock):
            if len(inputs) == 3:
                if torch.is_tensor(inputs[2]) and inputs[2].requires_grad:
                    raise NotImplementedError("GCN on a sampled block has no edge-weight gradient")
                raise ValueError("a sampled block carries its edge weights: pass [x, block.with_gcn_norm()]")
            x, sparse_adj = inputs
        elif isinstance(inputs[1], SparseMatrix):
            x, sparse_adj = inputs
        elif len(inputs) == 3:
            x, edge_index, edge_weight = inputs
            sparse_adj = SparseMatrix(edge_index, value=edge_weight, shape=[len(x), len(x)])
        else:
            x, edge_index = inputs
            sparse_adj = SparseMatrix(edge_index, shape=[len(x), len(x)])
        return gcn(x, sparse_adj, self.kernel, self.bias, activation=self.activation,
                   norm=self.norm, add_self_loop=self.add_self_loop, sym=self.sym, renorm=self.renorm,
                   improved=self.improved, edge_drop_rate=self.edge_drop_rate,
                   num_or_size_splits=self.num_or_size_splits if split else None,
                   training=bool(training), cache=cache, message_dtype=self.message_dtype)
