"""GNN encoder — H100-backed mirror of tf2_gnn.layers.gnn (/root/reference/tf2_gnn/layers/gnn.py:21-329).

Same GNNInput namedtuple, hyper-parameter dict, layer loop and return convention.  The adjacency
lists are prepared ONCE per call (CSR sorted by type,target) and shared by all message-passing layers;
the reference rebuilds the in-degree table in every layer (message_passing.py:190).

Node-level glue on the library's kernels (layers/node_ops.py): initial projection / inter-layer Dense, residual
average, LayerNormalization, training-time dropout (Philox) — each differentiable through its own backward
kernel — and the graph global exchange layers (layers/graph_global_exchange.py, SURVEY.md §8f-3/4).
"""
from __future__ import annotations

from typing import Any, Dict, List, NamedTuple, Optional, Tuple

import torch

from ..runtime import PreparedBatch, prepared_batch_for, to_device_adj, to_device_f32
from ..utils.param_helpers import get_activation_function
from . import node_ops
from .graph_global_exchange import (GraphGlobalExchange, GraphGlobalExchangeInput, GraphGlobalGRUExchange,
                                    GraphGlobalMeanExchange, GraphGlobalMLPExchange)
from .message_passing import MessagePassing, MessagePassingInput, get_message_passing_class
from .message_passing.message_passing import Variable, glorot_uniform


class GNNInput(NamedTuple):
    """Input named tuple for the GNN (gnn.py:21-27)."""

    node_features: Any
    adjacency_lists: Tuple[Any, ...]
    node_to_graph_map: Any
    num_graphs: Any


class _Dense:
    """tf.keras.layers.Dense(units, use_bias=False, activation=...) on tfgnn_b200_dense_fwd."""

    def __init__(self, name: str, in_dim: int, units: int, activation):
        self.kernel = Variable(f"{name}/kernel:0", glorot_uniform((in_dim, units)))
        self.activation = activation

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        return node_ops.dense(x, self.kernel.value, None, self.activation)


class _LayerNorm:
    """tf.keras.layers.LayerNormalization() defaults: axis=-1, epsilon=1e-3, gamma=1, beta=0."""

    def __init__(self, name: str, dim: int, epsilon: float = 1e-3):
        dev = "cuda" if torch.cuda.is_available() else "cpu"
        self.gamma = Variable(f"{name}/gamma:0", torch.ones(dim, dtype=torch.float32, device=dev))
        self.beta = Variable(f"{name}/beta:0", torch.zeros(dim, dtype=torch.float32, device=dev))
        self.epsilon = epsilon

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        return node_ops.layer_norm(x, self.gamma.value, self.beta.value, self.epsilon)


class GNN:
    """Encode graph states using a combination of graph message passing layers and dense layers
    (gnn.py:30-329)."""

    @classmethod
    def get_default_hyperparameters(cls, mp_style: Optional[str] = None) -> Dict[str, Any]:
        """gnn.py:53-79: the GNN-level keys override the message-passing defaults."""
        these_hypers = {
            "message_calculation_class": "rgcn",
            "initial_node_representation_activation": "tanh",
            "dense_intermediate_layer_activation": "tanh",
            "num_layers": 4,
            "dense_every_num_layers": 2,
            "residual_every_num_layers": 2,
            "use_inter_layer_layernorm": False,
            "hidden_dim": 16,
            "layer_input_dropout_rate": 0.0,
            "global_exchange_mode": "gru",  # One of "mean", "mlp", "gru"
            "global_exchange_every_num_layers": 2,
            "global_exchange_weighting_fun": "softmax",  # One of "softmax", "sigmoid"
            "global_exchange_num_heads": 4,
            "global_exchange_dropout_rate": 0.2,
        }  # type: Dict[str, Any]
        if mp_style is not None:
            these_hypers["message_calculation_class"] = mp_style
        message_passing_class = get_message_passing_class(these_hypers["message_calculation_class"])
        message_passing_hypers = message_passing_class.get_default_hyperparameters()
        message_passing_hypers.update(these_hypers)
        return message_passing_hypers

    def __init__(self, params: Dict[str, Any]):
        self._params = params
        self._hidden_dim = params["hidden_dim"]
        self._num_layers = params["num_layers"]
        self._dense_every_num_layers = params["dense_every_num_layers"]
        self._residual_every_num_layers = params["residual_every_num_layers"]
        self._use_inter_layer_layernorm = params["use_inter_layer_layernorm"]
        self._initial_node_representation_activation_fn = get_activation_function(
            params["initial_node_representation_activation"])
        self._dense_intermediate_layer_activation_fn = get_activation_function(
            params["dense_intermediate_layer_activation"])
        self._message_passing_class = get_message_passing_class(params["message_calculation_class"])
        if not params["global_exchange_mode"].lower() in {"mean", "mlp", "gru"}:
            raise ValueError(
                f"Unknown global_exchange_mode mode {params['global_exchange_mode']} - has to be one of 'mean', 'mlp', 'gru'!")
        self._global_exchange_mode = params["global_exchange_mode"]
        self._global_exchange_every_num_layers = params["global_exchange_every_num_layers"]
        self._global_exchange_weighting_fun = params["global_exchange_weighting_fun"]
        self._global_exchange_num_heads = params["global_exchange_num_heads"]
        self._global_exchange_dropout_rate = params["global_exchange_dropout_rate"]
        self._initial_projection_layer: Optional[_Dense] = None
        self._mp_layers: List[MessagePassing] = []
        self._inter_layer_layernorms: List[_LayerNorm] = []
        self._dense_layers: Dict[str, _Dense] = {}
        self._global_exchange_layers: Dict[str, GraphGlobalExchange] = {}
        # Philox stream of the training-time dropout (b200_dropout_seed is not a reference hyper-parameter)
        self.dropout_state = node_ops.DropoutState(int(params.get("b200_dropout_seed", 0x5EED)))
        self.built = False

    def _exchange_layers(self) -> List[int]:
        return [i for i in range(self._num_layers) if i and i % self._global_exchange_every_num_layers == 0]

    def build(self, tensor_shapes: GNNInput):
        """gnn.py:117-232 (same name scopes, so reference checkpoints map by name)."""
        in_dim = int(tuple(tensor_shapes.node_features)[-1])
        adjacency_list_shapes = tuple(tensor_shapes.adjacency_lists)
        scope = f"{self._message_passing_class.__name__}_GNN"
        self._initial_projection_layer = _Dense(f"{scope}/gnn_initial_node_projection/dense", in_dim,
                                                self._hidden_dim, self._initial_node_representation_activation_fn)
        for layer_idx in range(self._num_layers):
            mp = self._message_passing_class(self._params)
            mp.build(MessagePassingInput((None, self._hidden_dim), adjacency_list_shapes))
            for v in mp.variables:
                v.name = f"{scope}/Layer_{layer_idx}/MessagePassing/{v.name}"
            self._mp_layers.append(mp)
            if self._use_inter_layer_layernorm:
                self._inter_layer_layernorms.append(
                    _LayerNorm(f"{scope}/Layer_{layer_idx}/LayerNorm/layer_normalization", self._hidden_dim))
            if layer_idx % self._dense_every_num_layers == 0:
                self._dense_layers[str(layer_idx)] = _Dense(
                    f"{scope}/Layer_{layer_idx}/Dense/dense", self._hidden_dim, self._hidden_dim,
                    self._dense_intermediate_layer_activation_fn)
            if layer_idx and layer_idx % self._global_exchange_every_num_layers == 0:       # gnn.py:172-200
                exchange_layer_class = {"mean": GraphGlobalMeanExchange, "gru": GraphGlobalGRUExchange,
                                        "mlp": GraphGlobalMLPExchange}[self._global_exchange_mode.lower()]
                exchange_layer = exchange_layer_class(
                    hidden_dim=self._hidden_dim, weighting_fun=self._global_exchange_weighting_fun,
                    num_heads=self._global_exchange_num_heads, dropout_rate=self._global_exchange_dropout_rate)
                exchange_layer.build(GraphGlobalExchangeInput((None, self._hidden_dim), (None,), ()),
                                     name=f"{scope}/Layer_{layer_idx}/Global_Exchange/{exchange_layer_class.__name__}")
                exchange_layer.dropout_state = self.dropout_state
                self._global_exchange_layers[str(layer_idx)] = exchange_layer
        self.built = True

    @property
    def variables(self) -> List[Variable]:
        out = [self._initial_projection_layer.kernel] if self._initial_projection_layer else []
        for i, mp in enumerate(self._mp_layers):
            out.extend(mp.variables)
            if self._use_inter_layer_layernorm:
                out.extend([self._inter_layer_layernorms[i].gamma, self._inter_layer_layernorms[i].beta])
            if str(i) in self._dense_layers:
                out.append(self._dense_layers[str(i)].kernel)
            if str(i) in self._global_exchange_layers:
                out.extend(self._global_exchange_layers[str(i)].variables)
        return out

    trainable_variables = variables
    weights = variables

    def __call__(self, inputs: GNNInput, training: bool = False, return_all_representations: bool = False, shard=None):
        if not self.built:
            self.build(GNNInput(tuple(inputs.node_features.shape),
                                tuple(tuple(a.shape) for a in inputs.adjacency_lists), None, None))
        return self.call(inputs, training=training, return_all_representations=return_all_representations, shard=shard)

    def call(self, inputs: GNNInput, training: bool = False, return_all_representations: bool = False, shard=None):
        """gnn.py:234-274.

        shard (sharding.TargetRangeShard): run on one rank of a graph cut by target range.  node_features and
        node_to_graph_map are the rank's rows [lo, hi), the adjacency lists hold global node ids (all edges, or those into
        [lo, hi)), num_graphs is the global count; the result is the rank's rows.  Every message-passing layer reads the
        all-gathered table (sharding.gather_node_states); the node-level glue runs on the rank's rows and dropout draws the
        unsharded masks of those rows; the readout of a global exchange is merged over the ranks in rank order.  Collective
        in forward and backward: every rank of the shard's group makes the same calls.  Weight gradients come out as the
        rank's part: sharding.sum_gradients_over_ranks(gnn.trainable_variables) sums them."""
        cur, all_reps = self._internal_call(inputs, training, want_all_representations=return_all_representations,
                                            shard=shard)
        if return_all_representations:
            return cur, all_reps
        return cur

    def _internal_call(self, inputs: GNNInput, training: bool = False, want_all_representations: bool = True, shard=None):
        """gnn.py:276-329.  When the caller does not ask for the per-layer representations (the reference's traced function
        always returns them and `call` drops them), a message-passing layer that is directly followed by its LayerNorm runs
        both in one fused call (`call_with_layernorm`) and the tuple holds None for that layer."""
        if shard is not None and self._message_passing_class.__name__ == "GNN_FiLM":
            raise NotImplementedError(
                "GNN: a GNN-FiLM stack on target-range shards is not built (its sharded gradients do not yet meet the "
                "float64 bar the unsharded stack meets); GNN_FiLM layers themselves train on shards through "
                "sharding.gather_node_states and PreparedBatch(..., target_range=(lo, hi))")
        feats = to_device_f32(inputs.node_features)
        adjs = tuple(to_device_adj(a, feats.device) for a in inputs.adjacency_lists)
        rows = None
        if shard is not None:
            if int(feats.shape[0]) != shard.hi - shard.lo:
                raise ValueError(f"a shard's node_features hold its {shard.hi - shard.lo} rows, got {int(feats.shape[0])}")
            from .. import sharding
            prepared = PreparedBatch(adjs, shard.num_nodes, target_range=(shard.lo, shard.hi))
            rows = shard.rows

            def layer_input(h):
                return sharding.gather_node_states(h, shard.bounds, shard.group)
        else:
            if all(a is b for a, b in zip(adjs, inputs.adjacency_lists)):
                prepared = prepared_batch_for(adjs, int(feats.shape[0]))
            else:
                prepared = PreparedBatch(adjs, int(feats.shape[0]))

            def layer_input(h):
                return h
        cur = self._initial_projection_layer(feats)
        last = cur
        all_reps = [cur]
        n2g = None
        if self._global_exchange_layers:
            n2g = node_ops.node_to_graph_index(inputs.node_to_graph_map, feats.device)
        dropout_rate = float(self._params.get("layer_input_dropout_rate", 0.0))
        for layer_idx, mp_layer in enumerate(self._mp_layers):
            if training:                                                             # gnn.py:285-289
                cur = node_ops.dropout(cur, dropout_rate, self.dropout_state, rows)
            if layer_idx % self._residual_every_num_layers == 0:                     # gnn.py:291-296
                tmp = cur
                if layer_idx > 0:
                    cur = node_ops.residual_average(cur, last)
                last = tmp
            has_exchange = bool(layer_idx and layer_idx % self._global_exchange_every_num_layers == 0)
            if (self._use_inter_layer_layernorm and not has_exchange and not want_all_representations
                    and hasattr(mp_layer, "call_with_layernorm")):
                ln = self._inter_layer_layernorms[layer_idx]
                if not mp_layer.built:
                    mp_layer.build(MessagePassingInput(tuple(cur.shape), tuple(tuple(a.shape) for a in adjs)))
                cur = mp_layer.call_with_layernorm(MessagePassingInput(layer_input(cur), adjs), ln.gamma.value,
                                                   ln.beta.value, ln.epsilon,
                                                   prepared=prepared)     # gnn.py:299-304 + 317-321 in one call
                all_reps.append(None)
            else:
                cur = mp_layer(MessagePassingInput(layer_input(cur), adjs), training=training, prepared=prepared)
                all_reps.append(cur)
                if has_exchange:                                                         # gnn.py:307-315
                    cur = self._global_exchange_layers[str(layer_idx)](
                        GraphGlobalExchangeInput(cur, n2g, int(inputs.num_graphs)), training=training, shard=shard)
                if self._use_inter_layer_layernorm:
                    cur = self._inter_layer_layernorms[layer_idx](cur)
            if layer_idx % self._dense_every_num_layers == 0:
                cur = self._dense_layers[str(layer_idx)](cur)
        return cur, tuple(all_reps)
