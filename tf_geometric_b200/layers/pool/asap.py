# coding=utf-8
"""ASAP layer with the reference's constructor and weights (layers/pool/asap.py); inputs = [x, edge_index, edge_weight,
node_graph_index]."""
import torch

from ...nn.pool.asap import asap
from .._base import Layer


class ASAP(Layer):
    """OOP API for ASAP: Adaptive Structure Aware Pooling.  attention_units defaults to the number of input features and
    must equal it (nn.asap raises ValueError otherwise)."""

    def __init__(self, k=None, ratio=None, drop_rate=0.0, attention_units=None, le_conv_activation=torch.sigmoid,
                 le_conv_use_bias=True, kernel_regularizer=None, bias_regularizer=None, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.attention_units = attention_units
        self.k, self.ratio, self.drop_rate = k, ratio, drop_rate
        self.le_conv_activation = le_conv_activation
        self.le_conv_use_bias = le_conv_use_bias
        for name in ("attention_gcn_kernel", "attention_gcn_bias", "attention_query_kernel", "attention_query_bias",
                     "attention_score_kernel", "attention_score_bias", "le_conv_self_kernel", "le_conv_self_bias",
                     "le_conv_aggr_self_kernel", "le_conv_aggr_self_bias", "le_conv_aggr_neighbor_kernel"):
            setattr(self, name, None)

    def build(self, input_shapes, device=None):
        num_features = input_shapes[0][-1]
        if self.attention_units is None:
            self.attention_units = num_features
        units = self.attention_units
        if units != num_features:
            raise ValueError("ASAP: attention_units ({}) must equal the number of input features ({}): le_conv's "
                             "[attention_units, 1] kernels are applied to the cluster features".format(units, num_features))
        self.add_weight("attention_gcn_kernel", [num_features, units], device=device)
        self.add_weight("attention_gcn_bias", [units], initializer="zeros", device=device)
        self.add_weight("attention_query_kernel", [units, units], device=device)
        self.add_weight("attention_query_bias", [units], initializer="zeros", device=device)
        self.add_weight("attention_score_kernel", [units * 2, 1], device=device)
        self.add_weight("attention_score_bias", [1], initializer="zeros", device=device)
        self.add_weight("le_conv_self_kernel", [units, 1], device=device)
        if self.le_conv_use_bias:
            self.add_weight("le_conv_self_bias", [1], initializer="zeros", device=device)
        self.add_weight("le_conv_aggr_self_kernel", [units, 1], device=device)
        if self.le_conv_use_bias:
            self.add_weight("le_conv_aggr_self_bias", [1], initializer="zeros", device=device)
        self.add_weight("le_conv_aggr_neighbor_kernel", [units, 1], device=device)

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight, node_graph_index = inputs
        return asap(x, edge_index, edge_weight, node_graph_index,
                    self.attention_gcn_kernel, self.attention_gcn_bias,
                    self.attention_query_kernel, self.attention_query_bias,
                    self.attention_score_kernel, self.attention_score_bias,
                    self.le_conv_self_kernel, self.le_conv_self_bias,
                    self.le_conv_aggr_self_kernel, self.le_conv_aggr_self_bias,
                    self.le_conv_aggr_neighbor_kernel, None,
                    k=self.k, ratio=self.ratio, le_conv_activation=self.le_conv_activation,
                    drop_rate=self.drop_rate, training=training, cache=cache)
