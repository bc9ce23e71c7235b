# coding=utf-8
"""tfg.layers.APPNP (reference layers/conv/appnp.py:9-130)."""
import warnings

from ... import ops
from ...nn.conv.gcn import gcn_build_cache_for_graph, gcn_build_cache_by_adj
from ...nn.conv.appnp import appnp
from .._base import Layer


class APPNP(Layer):

    def __init__(self, units_list, dense_activation=ops.relu, activation=None, k=10, alpha=0.1,
                 dense_drop_rate=0.0, last_dense_drop_rate=0.0, edge_drop_rate=0.0,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.appnp)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units_list = units_list
        self.dense_activation = dense_activation
        self.activation = activation
        self.k = k
        self.alpha = alpha
        self.dense_drop_rate = dense_drop_rate
        self.last_dense_drop_rate = last_dense_drop_rate
        self.edge_drop_rate = edge_drop_rate
        self.kernel_regularizer = kernel_regularizer
        self.bias_regularizer = bias_regularizer
        self.kernels = []
        self.biases = []

    def build(self, input_shapes, device=None):
        last_units = input_shapes[0][-1]
        for i, units in enumerate(self.units_list):
            self.kernels.append(self.add_weight("kernel_{}".format(i), [last_units, units], device=device))
            self.biases.append(self.add_weight("bias_{}".format(i), [units], "zeros", device=device))
            last_units = units

    def build_cache_by_adj(self, sparse_adj, override=False, cache=None):
        return gcn_build_cache_by_adj(sparse_adj, override=override, cache=cache)

    def build_cache_for_graph(self, graph, override=False):
        gcn_build_cache_for_graph(graph, override=override)

    def cache_normed_edge(self, graph, override=False):
        warnings.warn("'APPNP.cache_normed_edge(graph, override)' is deprecated, use "
                      "'APPNP.build_cache_for_graph(graph, override)' instead", DeprecationWarning)
        return self.build_cache_for_graph(graph, override=override)

    def call(self, inputs, cache=None, training=None, mask=None):
        if len(inputs) == 3:
            x, edge_index, edge_weight = inputs
        else:
            x, edge_index = inputs
            edge_weight = None
        return appnp(x, edge_index, edge_weight, self.kernels, self.biases,
                     dense_activation=self.dense_activation, activation=self.activation, k=self.k, alpha=self.alpha,
                     dense_drop_rate=self.dense_drop_rate, last_dense_drop_rate=self.last_dense_drop_rate,
                     edge_drop_rate=self.edge_drop_rate, cache=cache, training=bool(training),
                     message_dtype=self.message_dtype)
