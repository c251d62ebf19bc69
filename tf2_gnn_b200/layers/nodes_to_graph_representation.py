"""Graph representation aggregation layer — H100-backed mirror of
tf2_gnn.layers.nodes_to_graph_representation (/root/reference/tf2_gnn/layers/nodes_to_graph_representation.py:8-229).

WeightedSumGraphRepresentation: per-node scores (MLP) -> per-(graph, head) softmax or sigmoid weights -> weighted
sum of the transformed node representations per graph.  node_to_graph_map is non-decreasing, so each graph is a
contiguous row range and the segment reductions run without atomics (csrc/graph_ops.cu).
"""
from __future__ import annotations

from typing import Any, List, NamedTuple, Optional

import torch

from ..runtime import to_device_f32
from ..utils.param_helpers import get_activation_function
from . import differentiable, graph_autograd, node_ops
from .message_passing.message_passing import Variable, glorot_uniform


class NodesToGraphRepresentationInput(NamedTuple):
    """nodes_to_graph_representation.py:8-14."""

    node_embeddings: Any
    node_to_graph_map: Any
    num_graphs: Any


def _activation_by_name(name: Optional[str]):
    """dpu_utils.tf2utils.get_activation_function_by_name: case-insensitive, None / "linear" -> identity."""
    if name is None or name.lower() in ("linear", "none"):
        return None
    return get_activation_function(name.lower())


class _MLP:
    """dpu_utils.tf2utils.MLP(out_size, hidden_layers, use_biases, activation_fun, dropout_rate)."""

    def __init__(self, name: str, in_dim: int, out_size: int, hidden_layers, use_biases: bool, activation,
                 dropout_rate: float):
        if isinstance(hidden_layers, int):
            hidden_layers = [out_size] * hidden_layers
        sizes = [int(in_dim)] + [int(h) for h in hidden_layers] + [int(out_size)]
        self.kernels = [Variable(f"{name}/dense_{i}/kernel:0", glorot_uniform((sizes[i], sizes[i + 1])))
                        for i in range(len(sizes) - 1)]
        dev = self.kernels[0].value.device
        self.biases = ([Variable(f"{name}/dense_{i}/bias:0", torch.zeros(sizes[i + 1], dtype=torch.float32, device=dev))
                        for i in range(len(sizes) - 1)] if use_biases else None)
        self.activation = activation
        self.dropout_rate = float(dropout_rate)

    @property
    def variables(self) -> List[Variable]:
        return self.kernels + (self.biases or [])

    def __call__(self, x: torch.Tensor, training: bool = False, rng=None) -> torch.Tensor:
        return node_ops.mlp(x, [k.value for k in self.kernels],
                            [b.value for b in self.biases] if self.biases else None, self.activation, training,
                            self.dropout_rate, rng)


class NodesToGraphRepresentation:
    """Abstract base (nodes_to_graph_representation.py:17-51)."""

    def __init__(self, graph_representation_size: int, **kwargs):
        self._graph_representation_size = int(graph_representation_size)
        self.built = False

    def __call__(self, inputs: NodesToGraphRepresentationInput, training: bool = False):
        if not self.built:
            self.build(NodesToGraphRepresentationInput(tuple(inputs.node_embeddings.shape), None, None))
        return self.call(inputs, training=training)


class WeightedSumGraphRepresentation(NodesToGraphRepresentation):
    """nodes_to_graph_representation.py:54-229; same constructor arguments and defaults."""

    def __init__(self, graph_representation_size: int, num_heads: int, weighting_fun: str = "softmax",
                 scoring_mlp_layers: List[int] = [128], scoring_mlp_activation_fun: str = "ReLU",
                 scoring_mlp_use_biases: bool = False, scoring_mlp_dropout_rate: float = 0.2,
                 transformation_mlp_layers: List[int] = [128], transformation_mlp_activation_fun: str = "ReLU",
                 transformation_mlp_use_biases: bool = False, transformation_mlp_dropout_rate: float = 0.2,
                 transformation_mlp_result_lower_bound: Optional[float] = None,
                 transformation_mlp_result_upper_bound: Optional[float] = None, **kwargs):
        super().__init__(graph_representation_size, **kwargs)
        assert graph_representation_size % num_heads == 0, \
            f"Number of heads {num_heads} needs to divide final representation size {graph_representation_size}!"
        assert weighting_fun.lower() in {"none", "average", "softmax", "sigmoid"}, \
            f"Weighting function {weighting_fun} unknown, {{'softmax', 'sigmoid', 'none', 'average'}} supported."
        self._num_heads = int(num_heads)
        self._weighting_fun = weighting_fun.lower()
        self._scoring_cfg = (list(scoring_mlp_layers), _activation_by_name(scoring_mlp_activation_fun),
                             bool(scoring_mlp_use_biases), float(scoring_mlp_dropout_rate))
        self._transformation_mlp_activation_fun = _activation_by_name(transformation_mlp_activation_fun)
        self._transformation_cfg = (list(transformation_mlp_layers), self._transformation_mlp_activation_fun,
                                    bool(transformation_mlp_use_biases), float(transformation_mlp_dropout_rate))
        self._transformation_mlp_result_lower_bound = transformation_mlp_result_lower_bound
        self._transformation_mlp_result_upper_bound = transformation_mlp_result_upper_bound
        self._scoring_mlp: Optional[_MLP] = None
        self._transformation_mlp: Optional[_MLP] = None
        self.dropout_state = None

    def build(self, input_shapes: NodesToGraphRepresentationInput, name: str = "WeightedSumGraphRepresentation"):
        in_dim = int(tuple(input_shapes.node_embeddings)[-1])
        if self._weighting_fun not in ("none", "average"):
            layers, act, biases, rate = self._scoring_cfg
            self._scoring_mlp = _MLP(f"{name}/ScoringMLP", in_dim, self._num_heads, layers, biases, act, rate)
        layers, act, biases, rate = self._transformation_cfg
        self._transformation_mlp = _MLP(f"{name}/TransformationMLP", in_dim, self._graph_representation_size, layers,
                                        biases, act, rate)
        self.built = True

    @property
    def variables(self) -> List[Variable]:
        out = list(self._scoring_mlp.variables) if self._scoring_mlp is not None else []
        return out + (list(self._transformation_mlp.variables) if self._transformation_mlp is not None else [])

    trainable_variables = variables

    def call(self, inputs: NodesToGraphRepresentationInput, training: bool = False, graph_ptr=None):
        x = to_device_f32(inputs.node_embeddings)
        n2g = inputs.node_to_graph_map
        if not isinstance(n2g, torch.Tensor):
            n2g = torch.as_tensor(n2g)
        n2g = n2g.to(device=x.device, dtype=torch.int32).contiguous()
        num_graphs = int(inputs.num_graphs)
        if graph_ptr is None:
            graph_ptr = node_ops.graph_offsets(n2g, num_graphs)
        scores = None
        if self._weighting_fun not in ("none", "average"):                       # (1) scores per node / head
            scores = self._scoring_mlp(x, training, self.dropout_state)           # [V, H]
        reprs = self._transformation_mlp(x, training, self.dropout_state)         # (2) representations
        reprs = differentiable.activation(reprs, self._transformation_mlp_activation_fun)
        lower, upper = self._transformation_mlp_result_lower_bound, self._transformation_mlp_result_upper_bound
        if node_ops._needs_grad(scores, reprs):
            # same forward kernels as below; backward on the graphs' row ranges (graph_autograd.py)
            return graph_autograd.readout(scores, reprs, n2g, graph_ptr, self._num_heads, self._weighting_fun, lower, upper)
        weights = None
        if self._weighting_fun == "sigmoid":
            weights = _sigmoid(scores)
        elif self._weighting_fun == "softmax":
            weights = node_ops.segment_softmax(scores, graph_ptr)
        node_ops.clamp_(reprs, lower, upper)
        return node_ops.weighted_segment_sum(reprs, weights, graph_ptr, self._num_heads,      # (3) aggregate by graph
                                             mean=self._weighting_fun == "average")


class WASGraphRepresentation(NodesToGraphRepresentation):
    """_W_eighted _A_verage and _S_um graph representation (nodes_to_graph_representation.py:232-314): a softmax- and a
    sigmoid-weighted WeightedSumGraphRepresentation, concatenated and projected without bias; same constructor arguments
    and defaults."""

    def __init__(self, graph_representation_size: int = 128, num_heads: int = 8, pooling_mlp_layers: List[int] = [128, 128],
                 pooling_mlp_activation_fun: str = "elu", pooling_mlp_use_biases: bool = True,
                 pooling_mlp_dropout_rate: float = 0.0, **kwargs):
        super().__init__(graph_representation_size, **kwargs)

        def pooling(weighting_fun: str) -> WeightedSumGraphRepresentation:
            return WeightedSumGraphRepresentation(
                graph_representation_size=graph_representation_size, num_heads=num_heads, weighting_fun=weighting_fun,
                scoring_mlp_layers=pooling_mlp_layers, scoring_mlp_dropout_rate=pooling_mlp_dropout_rate,
                scoring_mlp_use_biases=pooling_mlp_use_biases, scoring_mlp_activation_fun=pooling_mlp_activation_fun,
                transformation_mlp_layers=pooling_mlp_layers, transformation_mlp_dropout_rate=pooling_mlp_dropout_rate,
                transformation_mlp_use_biases=pooling_mlp_use_biases,
                transformation_mlp_activation_fun=pooling_mlp_activation_fun)

        self._weighted_avg_graph_repr_layer = pooling("softmax")
        self._weighted_sum_graph_repr_layer = pooling("sigmoid")
        self._out_projection: Optional[Variable] = None
        self.dropout_state = None

    def build(self, input_shapes: NodesToGraphRepresentationInput, name: str = "WASGraphRepresentation"):
        self._weighted_avg_graph_repr_layer.build(
            input_shapes, name=f"{name}/WeightedAvgGraphRepresentation/WeightedSumGraphRepresentation")
        self._weighted_sum_graph_repr_layer.build(
            input_shapes, name=f"{name}/WeightedSumGraphRepresentation/WeightedSumGraphRepresentation")
        size = self._graph_representation_size
        self._out_projection = Variable(f"{name}/dense/kernel:0", glorot_uniform((2 * size, size)))
        self.built = True

    @property
    def variables(self) -> List[Variable]:
        return (self._weighted_avg_graph_repr_layer.variables + self._weighted_sum_graph_repr_layer.variables
                + [self._out_projection])

    trainable_variables = variables

    def call(self, inputs: NodesToGraphRepresentationInput, training: bool = False):
        self._weighted_avg_graph_repr_layer.dropout_state = self.dropout_state
        self._weighted_sum_graph_repr_layer.dropout_state = self.dropout_state
        avg_graph_repr = self._weighted_avg_graph_repr_layer.call(inputs, training=training)
        sum_graph_repr = self._weighted_sum_graph_repr_layer.call(inputs, training=training)
        return node_ops.dense(torch.cat([avg_graph_repr, sum_graph_repr], dim=-1), self._out_projection.value)


def _sigmoid(x: torch.Tensor) -> torch.Tensor:
    """tf.nn.sigmoid on the library's activation kernel."""
    from .. import _ffi
    from ..runtime import stream_ptr
    out = torch.empty_like(x)
    _ffi.check(_ffi.lib().tfgnn_b200_activation(x.data_ptr(), x.numel(), _ffi.ACT_SIGMOID, out.data_ptr(), stream_ptr()))
    return out
