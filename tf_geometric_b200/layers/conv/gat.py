# coding=utf-8
"""tfg.layers.GAT: the weight set and calling convention of the reference layer (layers/conv/gat.py:7-101) over the
fused attention kernel.

Weights (names as in the reference, so that checkpoints map 1:1): query_kernel / query_bias and key_kernel / key_bias
[F, attention_units] / [attention_units], kernel [F, units] (or [F, units * num_heads] when the heads are averaged
instead of concatenated), bias [units]."""
from ... import ops
from ...nn.conv.gat import gat
from .._base import Layer

_WEIGHT_SLOTS = ("query_kernel", "query_bias", "key_kernel", "key_bias", "kernel", "bias")


class GAT(Layer):

    def __init__(self, units, attention_units=None, activation=None, use_bias=True, num_heads=1,
                 split_value_heads=True, query_activation=ops.relu, key_activation=ops.relu, edge_drop_rate=0.0,
                 kernel_regularizer=None, bias_regularizer=None, *args, message_dtype=None, **kwargs):
        """
        :param units: output width
        :param attention_units: width of the query / key projections (default: units); must divide by num_heads
        :param num_heads: attention heads; split_value_heads=True concatenates per-head slices of the values,
            False lets every head see full-width values and averages the heads
        :param edge_drop_rate: dropout on the attention coefficients while training
        :param message_dtype: None / torch.float32, or torch.bfloat16 / torch.float8_e4m3fn for inference with bf16 / fp8
            keys and values (nn.gat)
        """
        super().__init__(*args, **kwargs)
        ops.conv_message_dtype(message_dtype)     # ValueError for anything but fp32 / bf16 / fp8 e4m3
        self.message_dtype = message_dtype
        for slot in _WEIGHT_SLOTS:                  # declared up front like the reference, created lazily in build()
            setattr(self, slot, None)
        self.units, self.num_heads, self.split_value_heads = units, num_heads, split_value_heads
        self.attention_units = attention_units if attention_units is not None else units
        self.activation, self.query_activation, self.key_activation = activation, query_activation, key_activation
        self.use_bias, self.edge_drop_rate = use_bias, edge_drop_rate
        self.kernel_regularizer, self.bias_regularizer = kernel_regularizer, bias_regularizer

    def build(self, input_shapes, device=None):
        num_features = input_shapes[0][-1]
        value_units = self.units * (1 if self.split_value_heads else self.num_heads)
        for prefix in ("query", "key"):
            setattr(self, prefix + "_kernel",
                    self.add_weight(prefix + "_kernel", [num_features, self.attention_units], device=device))
            setattr(self, prefix + "_bias", self.add_weight(prefix + "_bias", [self.attention_units], "zeros", device=device))
        self.kernel = self.add_weight("kernel", [num_features, value_units], device=device)
        if self.use_bias:
            self.bias = self.add_weight("bias", [self.units], "zeros", device=device)

    def partitioned_projections(self):
        """All-row projections this layer needs on a partitioned graph: K | V side by side (Q only for local rows)."""
        k_act, _ = ops.activation_code(self.key_activation)
        return [((id(self.key_kernel), id(self.kernel)),
                 [(self.key_kernel, self.key_bias, k_act), (self.kernel, None, ops.ACT_NONE)])]

    def call(self, inputs, training=None, mask=None, cache=None):
        """inputs = [x, edge_index] (a third entry, edge_weight, is accepted and ignored like in the reference); on a
        sampled block [x_src or batch.source_rows(x), block.with_self_loops()] (nn.gat); on several GPUs
        [x_local, partitioned_graph] (tf_geometric_b200.dist.PartitionedGraph)."""
        if hasattr(inputs[1], "part") and hasattr(inputs[1], "project_all_rows"):
            from ... import dist as tdist
            if ops.conv_message_dtype(self.message_dtype) is not None:
                raise NotImplementedError("message_dtype={} is not implemented for partitioned graphs".format(
                    str(ops.conv_message_dtype(self.message_dtype)).replace("torch.", "")))
            if not self.split_value_heads:
                raise NotImplementedError("partitioned GAT concatenates the heads (split_value_heads=True)")
            return tdist.gat_partitioned(inputs[1], inputs[0], self.query_kernel, self.query_bias, self.query_activation,
                                         self.key_kernel, self.key_bias, self.key_activation, self.kernel, self.bias,
                                         self.activation, num_heads=self.num_heads)
        return gat(inputs[0], inputs[1], self.query_kernel, self.query_bias, self.query_activation, self.key_kernel,
                   self.key_bias, self.key_activation, self.kernel, self.bias, self.activation, num_heads=self.num_heads,
                   split_value_heads=self.split_value_heads, edge_drop_rate=self.edge_drop_rate, training=bool(training),
                   cache=cache, message_dtype=self.message_dtype)
