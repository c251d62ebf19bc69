"""Graph-global information exchange — H100-backed mirror of tf2_gnn.layers.graph_global_exchange
(/root/reference/tf2_gnn/layers/graph_global_exchange.py:12-183).

Every variant first computes a per-graph representation (WeightedSumGraphRepresentation with
scoring_mlp_layers=[hidden_dim]), broadcasts it back to the graph's nodes (gather by node_to_graph_map) and
combines it with the node states: mean ((x + g) / 2), GRUCell(inputs=g, state=x) or MLP([g || x]).  The
graph-side halves of the GRU / MLP (g K + b0, g W1[:H]) are computed once per GRAPH and gathered inside the
combine kernel — row-wise identical arithmetic, V/G times fewer FLOPs.
"""
from __future__ import annotations

from typing import Any, List, NamedTuple, Optional

import torch

from ..runtime import to_device_f32
from ..utils.param_helpers import get_activation_function
from . import graph_autograd, node_ops
from .message_passing.message_passing import Variable, glorot_uniform
from .nodes_to_graph_representation import (NodesToGraphRepresentationInput, WeightedSumGraphRepresentation, _MLP)


class GraphGlobalExchangeInput(NamedTuple):
    """graph_global_exchange.py:12-17."""

    node_embeddings: Any
    node_to_graph_map: Any
    num_graphs: Any


class GraphGlobalExchange:
    """Update node representations based on graph-global information (graph_global_exchange.py:20-103)."""

    def __init__(self, hidden_dim: int, weighting_fun: str = "softmax", num_heads: int = 4, dropout_rate: float = 0.0):
        self._hidden_dim = int(hidden_dim)
        self._weighting_fun = weighting_fun
        self._num_heads = int(num_heads)
        self._dropout_rate = float(dropout_rate)
        self._node_to_graph_representation_layer: Optional[WeightedSumGraphRepresentation] = None
        self.dropout_state = None
        self.built = False

    def build(self, tensor_shapes: GraphGlobalExchangeInput, name: Optional[str] = None):
        name = name or type(self).__name__
        self._node_to_graph_representation_layer = WeightedSumGraphRepresentation(
            graph_representation_size=self._hidden_dim, weighting_fun=self._weighting_fun, num_heads=self._num_heads,
            scoring_mlp_layers=[self._hidden_dim])
        self._node_to_graph_representation_layer.build(
            NodesToGraphRepresentationInput((None, self._hidden_dim), None, None),
            name=f"{name}/WeightedSumGraphRepresentation")
        self.built = True

    @property
    def variables(self) -> List[Variable]:
        return list(self._node_to_graph_representation_layer.variables)

    trainable_variables = variables

    def __call__(self, inputs: GraphGlobalExchangeInput, training: bool = False):
        if not self.built:
            self.build(GraphGlobalExchangeInput((None, self._hidden_dim), (None,), ()))
        return self.call(inputs, training=training)

    def _prepare(self, inputs: GraphGlobalExchangeInput, training: bool):
        """graph_global_exchange.py:83-103: the node states, the per-graph representations [G, H], node_to_graph_map and
        graph_ptr.  With the exchange's own dropout active the representations come back per NODE ([V, H]) and the map is
        None: tf.nn.dropout acts on the per-node copies (:98-101), the mask differs per node."""
        x = to_device_f32(inputs.node_embeddings)
        n2g = inputs.node_to_graph_map
        if not isinstance(n2g, torch.Tensor):
            n2g = torch.as_tensor(n2g)
        n2g = n2g.to(device=x.device, dtype=torch.int32).contiguous()
        num_graphs = int(inputs.num_graphs)
        graph_ptr = node_ops.graph_offsets(n2g, num_graphs)
        self._node_to_graph_representation_layer.dropout_state = self.dropout_state
        graph_reprs = self._node_to_graph_representation_layer.call(
            NodesToGraphRepresentationInput(x, n2g, num_graphs), training=training, graph_ptr=graph_ptr)
        if training and self._dropout_rate > 0.0:
            per_node = graph_autograd.gather_graph_rows(graph_reprs, n2g, graph_ptr)
            return x, node_ops.dropout(per_node, self._dropout_rate, self.dropout_state), None, graph_ptr
        return x, graph_reprs, n2g, graph_ptr


class GraphGlobalMeanExchange(GraphGlobalExchange):
    """(x + g[node_to_graph_map]) / 2 (graph_global_exchange.py:106-124)."""

    def call(self, inputs: GraphGlobalExchangeInput, training: bool = False):
        x, g, index, graph_ptr = self._prepare(inputs, training)
        if node_ops._needs_grad(x, g):
            if index is None:
                from .differentiable import _AddFunction
                return _AddFunction.apply(x, g, 0.5, 0.5)
            return graph_autograd.gathered_add(x, g, index, graph_ptr, scale=0.5)
        return node_ops.gathered_add(x, g, index, scale=0.5)


class GraphGlobalGRUExchange(GraphGlobalExchange):
    """GRUCell(inputs=g[node_to_graph_map], states=[x]) (graph_global_exchange.py:127-153)."""

    def build(self, tensor_shapes: GraphGlobalExchangeInput, name: Optional[str] = None):
        name = name or type(self).__name__
        H = self._hidden_dim
        self._gru_kernel = Variable(f"{name}/gru_cell/kernel:0", glorot_uniform((H, 3 * H)))
        self._gru_recurrent_kernel = Variable(f"{name}/gru_cell/recurrent_kernel:0", glorot_uniform((H, 3 * H)))
        self._gru_bias = Variable(f"{name}/gru_cell/bias:0",
                                  torch.zeros((2, 3 * H), dtype=torch.float32, device=self._gru_kernel.value.device))
        super().build(tensor_shapes, name)

    @property
    def variables(self) -> List[Variable]:
        return [self._gru_kernel, self._gru_recurrent_kernel, self._gru_bias] + super().variables

    trainable_variables = variables

    def call(self, inputs: GraphGlobalExchangeInput, training: bool = False):
        x, g, index, graph_ptr = self._prepare(inputs, training)
        if node_ops._needs_grad(x, g, self._gru_kernel.value, self._gru_recurrent_kernel.value, self._gru_bias.value):
            if index is None:
                from .differentiable import gru_cell
                return gru_cell(g, x, self._gru_kernel.value, self._gru_recurrent_kernel.value, self._gru_bias.value)
            return graph_autograd.gru_cell(g, index, graph_ptr, x, self._gru_kernel.value, self._gru_recurrent_kernel.value,
                                           self._gru_bias.value)
        return node_ops.gru_cell(g, index, x, self._gru_kernel.value, self._gru_recurrent_kernel.value,
                                 self._gru_bias.value)


class GraphGlobalMLPExchange(GraphGlobalExchange):
    """MLP(out_size=H)(concat([g[node_to_graph_map], x])) (graph_global_exchange.py:156-183); dpu_utils' MLP default is one
    hidden layer of out_size units, ReLU, no biases."""

    def build(self, tensor_shapes: GraphGlobalExchangeInput, name: Optional[str] = None):
        name = name or type(self).__name__
        H = self._hidden_dim
        self._mlp = _MLP(f"{name}/MLP", 2 * H, H, 1, False, get_activation_function("relu"), 0.0)
        super().build(tensor_shapes, name)

    @property
    def variables(self) -> List[Variable]:
        return list(self._mlp.variables) + super().variables

    trainable_variables = variables

    def call(self, inputs: GraphGlobalExchangeInput, training: bool = False):
        x, g, index, graph_ptr = self._prepare(inputs, training)
        H = self._hidden_dim
        W1, W2 = self._mlp.kernels[0].value, self._mlp.kernels[1].value
        needs_grad = node_ops._needs_grad(x, g, W1, W2)
        if needs_grad and index is None:
            # tf.concat([per_node_graph_representations, node_embeddings], -1) -> MLP (graph_global_exchange.py:176-181)
            return self._mlp(torch.cat([g, x], dim=-1), training, self.dropout_state)
        # first layer split by rows: [g || x] W1 = g W1[:H] + x W1[H:]; the graph half once per graph (or per node when the
        # training-time dropout already materialised per-node copies: index is None then).  The slices of W1 are views: under
        # autograd the two halves' gradients land in the one variable.
        relu = get_activation_function("relu")
        gp = node_ops.dense(g, W1[:H])
        xp = node_ops.dense(x, W1[H:])
        if needs_grad:
            hidden = graph_autograd.gathered_add(xp, gp, index, graph_ptr, scale=1.0, activation=relu)
        else:
            hidden = node_ops.gathered_add(xp, gp, index, scale=1.0, activation=relu)
        return node_ops.dense(hidden, W2)
