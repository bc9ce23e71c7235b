# coding=utf-8
"""tfg.layers.{Mean,Sum,GCN,MeanPool,MaxPool,LSTM}GraphSage (reference layers/conv/graph_sage.py:8-421)."""
import math

import torch

from ... import ops, autograd
from ...nn.conv.graph_sage import (mean_graph_sage, sum_graph_sage, gcn_graph_sage, mean_pool_graph_sage,
                                   max_pool_graph_sage, _lstm_sage)
from .._base import Layer


def _unpack(inputs):
    if len(inputs) == 3:
        return inputs
    x, edge_index = inputs
    return x, edge_index, None


class _PairSage(Layer):
    _fn = None

    def __init__(self, units, activation=ops.relu, use_bias=True, concat=True, normalize=False,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.mean_graph_sage / sum_graph_sage)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units = units
        self.activation = activation
        self.use_bias = use_bias
        self.concat = concat
        self.normalize = normalize
        if concat and (units % 2 != 0):
            raise Exception("units must be a event number if concat is True")
        self.kernel_regularizer = kernel_regularizer
        self.bias_regularizer = bias_regularizer
        self.self_kernel = None
        self.neighbor_kernel = None
        self.bias = None

    def build(self, input_shapes, device=None):
        num_features = input_shapes[0][-1]
        kernel_units = self.units // 2 if self.concat else self.units
        self.self_kernel = self.add_weight("self_kernel", [num_features, kernel_units], device=device)
        self.neighbor_kernel = self.add_weight("neighbor_kernel", [num_features, kernel_units], device=device)
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units], "zeros", device=device)

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight = _unpack(inputs)
        return type(self)._fn(x, edge_index, edge_weight, self.self_kernel, self.neighbor_kernel, bias=self.bias,
                              activation=self.activation, concat=self.concat, normalize=self.normalize,
                              message_dtype=self.message_dtype)


class MeanGraphSage(_PairSage):
    _fn = staticmethod(mean_graph_sage)


class SumGraphSage(_PairSage):
    _fn = staticmethod(sum_graph_sage)


class GCNGraphSage(Layer):

    def __init__(self, units, activation=ops.relu, use_bias=True, normalize=False,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.gcn_graph_sage)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units = units
        self.activation = activation
        self.use_bias = use_bias
        self.normalize = normalize
        self.kernel_regularizer = kernel_regularizer
        self.bias_regularizer = bias_regularizer
        self.kernel = None
        self.bias = None

    def build(self, input_shapes, device=None):
        num_features = input_shapes[0][-1]
        self.kernel = self.add_weight("kernel", [num_features, self.units], device=device)
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units], "zeros", device=device)

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight = _unpack(inputs)
        return gcn_graph_sage(x, edge_index, edge_weight, self.kernel, self.bias, self.activation, self.normalize,
                              cache=cache, message_dtype=self.message_dtype)


class _PoolSage(Layer):
    _fn = None
    _names = ("neighbor_mlp_kernel", "neighbor_mlp_bias", "neighbor_kernel")

    def __init__(self, units, activation=ops.relu, use_bias=True, concat=True, normalize=False,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """message_dtype: None / torch.float32, or torch.bfloat16 for inference with bf16 message rows (nn.mean_pool_graph_sage / max_pool_graph_sage)."""
        super().__init__(*args, **kwargs)
        ops.message_dtype(message_dtype)          # ValueError for anything but fp32 / bf16
        self.message_dtype = message_dtype
        self.units = units
        self.activation = activation
        self.use_bias = use_bias
        self.concat = concat
        if concat and (units % 2 != 0):
            raise Exception("units must be a event number if concat is True")
        self.normalize = normalize
        self.kernel_regularizer = kernel_regularizer
        self.bias_regularizer = bias_regularizer
        self.self_kernel = None
        self.bias = None

    def build(self, input_shapes, device=None):
        num_features = input_shapes[0][-1]
        kernel_units = self.units // 2 if self.concat else self.units
        mlp_k, mlp_b, neigh_k = self._names
        self.self_kernel = self.add_weight("self_kernel", [num_features, kernel_units], device=device)
        self.add_weight(mlp_k, [num_features, kernel_units * 4], device=device)
        if self.use_bias:
            self.add_weight(mlp_b, [kernel_units * 4], "zeros", device=device)
        self.add_weight(neigh_k, [kernel_units * 4, kernel_units], device=device)
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units], "zeros", device=device)

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight = _unpack(inputs)
        mlp_k, mlp_b, neigh_k = self._names
        return type(self)._fn(x, edge_index, edge_weight, self.self_kernel, getattr(self, mlp_k), getattr(self, neigh_k),
                              neighbor_mlp_bias=getattr(self, mlp_b) if self.use_bias else None, bias=self.bias,
                              activation=self.activation, concat=self.concat, normalize=self.normalize,
                              message_dtype=self.message_dtype)


class MeanPoolGraphSage(_PoolSage):
    _fn = staticmethod(mean_pool_graph_sage)


class MaxPoolGraphSage(_PoolSage):
    # weight names of the reference's MaxPoolGraphSage.build (layers/conv/graph_sage.py:327-338)
    _names = ("mlp_kernel", "mlp_bias", "neighs_kernel")
    _fn = staticmethod(max_pool_graph_sage)


class LSTMGraphSage(Layer):
    """LSTM aggregator (reference layers/conv/graph_sage.py:357-421): inputs [x, edge_index] or [x, edge_index,
    edge_weight] (the weight is ignored, as in the reference).  The layer owns a torch.nn.LSTM (cuDNN), initialised like
    tf.keras.layers.LSTM (glorot-uniform kernel, orthogonal recurrent kernel, zero bias with the forget-gate slice at 1;
    gate order i, f, g, o in both frameworks), fed the sequence-major [K, N, F] neighbour tensor and run with cuDNN's TF32
    math off in the forward and the backward.  `load_keras_lstm_weights` takes Keras-layout LSTM weights."""

    def __init__(self, units, activation=ops.relu, use_bias=True, concat=True, normalize=False,
                 kernel_regularizer=None, bias_regularizer=None, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.units = units
        self.activation = activation
        self.use_bias = use_bias
        self.concat = concat
        self.normalize = normalize
        if concat and (units % 2 != 0):
            raise Exception("units must be a event number if concat is True")
        self.kernel_regularizer = kernel_regularizer
        self.bias_regularizer = bias_regularizer
        self.lstm = None
        self.self_kernel = None
        self.neighbor_kernel = None
        self.bias = None

    def build(self, input_shapes, device=None):
        num_features = input_shapes[0][-1]
        kernel_units = self.units // 2 if self.concat else self.units
        self.__dict__.pop("lstm", None)
        self.lstm = torch.nn.LSTM(num_features, kernel_units, device=device)
        gen = None
        if self._seed is not None:
            gen = torch.Generator(device="cpu")
            gen.manual_seed(self._seed + sum(ord(c) for c in "lstm"))
        limit = math.sqrt(6.0 / (num_features + 4 * kernel_units))
        kernel = (torch.rand((num_features, 4 * kernel_units), generator=gen) * 2.0 - 1.0) * limit
        recurrent = torch.nn.init.orthogonal_(torch.empty((kernel_units, 4 * kernel_units)), generator=gen)
        bias = torch.zeros((4 * kernel_units,))
        bias[kernel_units:2 * kernel_units] = 1.0                           # Keras unit_forget_bias
        self._copy_keras_lstm(kernel, recurrent, bias)
        for p in self.lstm.parameters():
            p.requires_grad_(self._trainable)
        self.self_kernel = self.add_weight("self_kernel", [num_features, kernel_units], device=device)
        self.neighbor_kernel = self.add_weight("neighbor_kernel", [kernel_units, kernel_units], device=device)
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units], "zeros", device=device)

    def load_keras_lstm_weights(self, kernel, recurrent_kernel, bias):
        """Copy tf.keras.layers.LSTM weights (kernel [F, 4U], recurrent_kernel [U, 4U], bias [4U]; numpy or tensors)
        into the torch LSTM: weight_ih = kernel^T, weight_hh = recurrent_kernel^T, bias_ih = bias, bias_hh = 0.  Builds
        the layer first (F = kernel rows) when it has not been called yet."""
        kernel = torch.as_tensor(kernel, dtype=torch.float32)
        if not self.built:
            self.build([(None, kernel.shape[0])], device=ops.default_device())
            self.built = True
        self._copy_keras_lstm(kernel, recurrent_kernel, bias)

    def _copy_keras_lstm(self, kernel, recurrent_kernel, bias):
        cell = self.lstm
        with torch.no_grad():
            cell.weight_ih_l0.copy_(torch.as_tensor(kernel, dtype=torch.float32).t())
            cell.weight_hh_l0.copy_(torch.as_tensor(recurrent_kernel, dtype=torch.float32).t())
            cell.bias_ih_l0.copy_(torch.as_tensor(bias, dtype=torch.float32))
            cell.bias_hh_l0.zero_()

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index = inputs[0], inputs[1]
        return _lstm_sage(x, edge_index, lambda padded: autograd.run_lstm_fp32(self.lstm, padded).mean(dim=0), True,
                          self.self_kernel, self.neighbor_kernel, self.bias, self.activation, self.concat,
                          self.normalize)
