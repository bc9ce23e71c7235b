# coding=utf-8
"""tfg.layers.{SGC, SSGC, TAGCN, GIN, LEConv} (reference layers/conv/{sgc,ssgc,tagcn,gin,le_conv}.py)."""
import torch

from ... import ops
from ...nn.conv.gcn import gcn_build_cache_for_graph, gcn_build_cache_by_adj
from ...nn.conv.propagation import sgc, ssgc, tagcn, gin, le_conv, chebynet, chebynet_norm_edge
from .._base import Layer


def _unpack(inputs):
    if len(inputs) == 3:
        return inputs
    x, edge_index = inputs
    return x, edge_index, None


class SGC(Layer):
    def __init__(self, units, k=1, activation=None, use_bias=True, renorm=True, improved=False,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.sgc)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units, self.k, self.activation, self.use_bias = units, k, activation, use_bias
        self.renorm, self.improved = renorm, improved
        self.kernel = None
        self.bias = None

    def build(self, input_shapes, device=None):
        self.kernel = self.add_weight("kernel", [input_shapes[0][-1], self.units], device=device)
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units], "zeros", device=device)

    def build_cache_for_graph(self, graph, override=False):
        gcn_build_cache_for_graph(graph, renorm=self.renorm, improved=self.improved, override=override)

    def build_cache_by_adj(self, sparse_adj, override=False, cache=None):
        return gcn_build_cache_by_adj(sparse_adj, renorm=self.renorm, improved=self.improved, override=override, cache=cache)

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight = _unpack(inputs)
        return sgc(x, edge_index, edge_weight, self.k, self.kernel, self.bias, activation=self.activation,
                   renorm=self.renorm, improved=self.improved, cache=cache, message_dtype=self.message_dtype)


class SSGC(Layer):
    def __init__(self, units_list=None, k=10, alpha=0.1, dense_activation=ops.relu, activation=None,
                 dense_drop_rate=0.0, last_dense_drop_rate=0.0, edge_drop_rate=0.0,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.ssgc)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units_list, self.k, self.alpha = units_list, k, alpha
        self.dense_activation, self.activation = dense_activation, activation
        self.dense_drop_rate, self.last_dense_drop_rate, self.edge_drop_rate = dense_drop_rate, last_dense_drop_rate, edge_drop_rate
        self.kernels, self.biases = [], []

    def build(self, input_shapes, device=None):
        last_units = input_shapes[0][-1]
        for i, units in enumerate(self.units_list or []):
            self.kernels.append(self.add_weight("kernel_{}".format(i), [last_units, units], device=device))
            self.biases.append(self.add_weight("bias_{}".format(i), [units], "zeros", device=device))
            last_units = units

    def build_cache_for_graph(self, graph, override=False):
        gcn_build_cache_for_graph(graph, override=override)

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight = _unpack(inputs)
        return ssgc(x=x, edge_index=edge_index, edge_weight=edge_weight,
                    kernels=self.kernels if self.units_list else None, biases=self.biases if self.units_list else None,
                    k=self.k, alpha=self.alpha, dense_activation=self.dense_activation, activation=self.activation,
                    dense_drop_rate=self.dense_drop_rate, last_dense_drop_rate=self.last_dense_drop_rate,
                    edge_drop_rate=self.edge_drop_rate, cache=cache, training=bool(training),
                    message_dtype=self.message_dtype)


class TAGCN(Layer):
    def __init__(self, units, k=3, activation=None, use_bias=True, renorm=False, improved=False,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.tagcn)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units, self.k, self.activation, self.use_bias = units, k, activation, use_bias
        self.renorm, self.improved = renorm, improved
        self.kernel = None
        self.bias = None

    def build(self, input_shapes, device=None):
        self.kernel = self.add_weight("kernel", [input_shapes[0][-1] * (self.k + 1), self.units], device=device)
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units], "zeros", device=device)

    def build_cache_for_graph(self, graph, override=False):
        gcn_build_cache_for_graph(graph, renorm=self.renorm, improved=self.improved, override=override)

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight = _unpack(inputs)
        return tagcn(x, edge_index, edge_weight, self.k, self.kernel, self.bias, activation=self.activation,
                     renorm=self.renorm, improved=self.improved, cache=cache, message_dtype=self.message_dtype)


class GIN(Layer):
    def __init__(self, mlp_model, eps=0, train_eps=False, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.gin)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.mlp_model = mlp_model
        self.eps = eps
        if train_eps:
            self.eps = self.add_weight("eps", [], "zeros")

    def build(self, input_shapes, device=None):
        pass

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index = inputs[0], inputs[1]
        return gin(x, edge_index, self.mlp_model, self.eps, training=training, message_dtype=self.message_dtype)


class LEConv(Layer):
    def __init__(self, units, activation=None, self_use_bias=True, aggr_self_use_bias=True, aggr_neighbor_use_bias=False,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.le_conv)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units, self.activation = units, activation
        self.self_use_bias, self.aggr_self_use_bias, self.aggr_neighbor_use_bias = \
            self_use_bias, aggr_self_use_bias, aggr_neighbor_use_bias
        self.self_kernel = self.self_bias = self.aggr_self_kernel = self.aggr_self_bias = None
        self.aggr_neighbor_kernel = self.aggr_neighbor_bias = None

    def build(self, input_shapes, device=None):
        f = input_shapes[0][-1]
        self.self_kernel = self.add_weight("self_kernel", [f, self.units], device=device)
        if self.self_use_bias:
            self.self_bias = self.add_weight("self_bias", [self.units], "zeros", device=device)
        self.aggr_self_kernel = self.add_weight("aggr_self_kernel", [f, self.units], device=device)
        if self.aggr_self_use_bias:
            self.aggr_self_bias = self.add_weight("aggr_self_bias", [self.units], "zeros", device=device)
        self.aggr_neighbor_kernel = self.add_weight("aggr_neighbor_kernel", [f, self.units], device=device)
        if self.aggr_neighbor_use_bias:
            self.aggr_neighbor_bias = self.add_weight("aggr_neighbor_bias", [self.units], "zeros", device=device)

    def call(self, inputs, training=None, mask=None, cache=None):
        x, edge_index, edge_weight = _unpack(inputs)
        return le_conv(x, edge_index, edge_weight, self.self_kernel, self.self_bias, self.aggr_self_kernel,
                       self.aggr_self_bias, self.aggr_neighbor_kernel, self.aggr_neighbor_bias, activation=self.activation,
                       message_dtype=self.message_dtype)


class ChebyNet(Layer):
    """tfg.layers.ChebyNet (reference layers/conv/chebynet.py): weights kernel0..kernel{k-1}, bias."""

    def __init__(self, units, k, activation=None, use_bias=True, normalization_type="sym", use_dynamic_lambda_max=False,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.chebynet)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units, self.k, self.activation, self.use_bias = units, k, activation, use_bias
        self.normalization_type, self.use_dynamic_lambda_max = normalization_type, use_dynamic_lambda_max
        self.kernels = []
        self.bias = None

    def build(self, input_shapes, device=None):
        f = input_shapes[0][-1]
        for i in range(self.k):
            self.kernels.append(self.add_weight("kernel{}".format(i), [f, self.units], device=device))
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units], "zeros", device=device)

    def build_cache_for_graph(self, graph, override=False):
        if override:
            graph.cache["chebynet_normed_edge_{}".format(self.normalization_type)] = None
        chebynet_norm_edge(graph.edge_index, graph.num_nodes, graph.edge_weight, self.normalization_type,
                           use_dynamic_lambda_max=self.use_dynamic_lambda_max, cache=graph.cache)

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight = _unpack(inputs)
        return chebynet(x, edge_index, edge_weight, self.k, self.kernels, self.bias, self.activation,
                        self.normalization_type, use_dynamic_lambda_max=self.use_dynamic_lambda_max, cache=cache,
                        message_dtype=self.message_dtype)
