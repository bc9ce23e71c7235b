# coding=utf-8
"""DiffPool and MinCutPool layers with the reference's constructors (layers/pool/diff_pool.py,
layers/pool/min_cut_pool.py); inputs = [x, edge_index, edge_weight, node_graph_index].

Deviation: the reference's MinCutPool registers its losses with Keras' `add_loss`, which has no torch counterpart.  Here
the caller asks for them with `return_losses=True` (or `return_loss_func=True`) and adds them to its loss, as the
reference's demo/demo_min_cut_pool.py does."""
from ...nn.pool.diff_pool import diff_pool
from ...nn.pool.min_cut_pool import min_cut_pool
from .._base import Layer


class _ClusterPoolLayer(Layer):

    def __init__(self, feature_gnn, assign_gnn, units, num_clusters, activation=None, use_bias=True,
                 bias_regularizer=None, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.feature_gnn = feature_gnn
        self.assign_gnn = assign_gnn
        self.num_clusters = num_clusters
        self.activation = activation
        if use_bias and units is None:
            raise Exception("The \"units\" parameter is required when you set use_bias=True.")
        self.units = units
        self.use_bias = use_bias
        self.bias = None

    def build(self, input_shapes, device=None):
        if self.use_bias:
            self.add_weight("bias", shape=[self.units], initializer="zeros", device=device)


class DiffPool(_ClusterPoolLayer):
    """OOP API for DiffPool: inputs [x, edge_index, edge_weight, node_graph_index] -> the pooled batch."""

    def call(self, inputs, cache=None, training=None, mask=None):
        x, edge_index, edge_weight, node_graph_index = inputs
        return diff_pool(x, edge_index, edge_weight, node_graph_index, self.feature_gnn, self.assign_gnn,
                         self.num_clusters, bias=self.bias, activation=self.activation, training=training, cache=cache)


class MinCutPool(_ClusterPoolLayer):
    """OOP API for MinCutPool: inputs [x, edge_index, edge_weight, node_graph_index] -> the pooled batch, and
    (cut_loss, orth_loss) or a callable returning them when asked (no add_loss; see the module docstring)."""

    def __init__(self, feature_gnn, assign_gnn, units, num_clusters, activation=None, use_bias=True,
                 gnn_use_normed_edge=True, bias_regularizer=None, *args, **kwargs):
        super().__init__(feature_gnn, assign_gnn, units, num_clusters, activation, use_bias, bias_regularizer, *args,
                         **kwargs)
        self.gnn_use_normed_edge = gnn_use_normed_edge

    def call(self, inputs, cache=None, training=None, mask=None, return_loss_func=False, return_losses=False):
        x, edge_index, edge_weight, node_graph_index = inputs
        return min_cut_pool(x, edge_index, edge_weight, node_graph_index, self.feature_gnn, self.assign_gnn,
                            self.num_clusters, bias=self.bias, activation=self.activation,
                            gnn_use_normed_edge=self.gnn_use_normed_edge, return_loss_func=return_loss_func,
                            return_losses=return_losses, cache=cache, training=training)
