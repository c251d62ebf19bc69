"""Message passing layer — H100-backed mirror of tf2_gnn.layers.message_passing.message_passing
(/root/reference/tf2_gnn/layers/message_passing/message_passing.py:13-263).

Same class contract as the reference plugin seam: ``cls.get_default_hyperparameters()``,
``cls(params)``, ``.build(MessagePassingInput(shape, shapes))``,
``layer(MessagePassingInput(node_embeddings, adjacency_lists), training=False) -> [V, hidden_dim]``,
and the registry decorator / lookup.  The built-in subclasses (RGCN, RGAT, RGIN, GGNN,
GNN_Edge_MLP, GNN_FiLM) override ``call`` with ONE C-ABI call per layer; a user subclass that only
implements ``_message_function`` runs the generic path below, which keeps the reference's op
sequence (gather -> _message_function -> concat -> segment-reduce -> activation) on the library's
own gather / segment-reduce / activation kernels.
"""
from __future__ import annotations

from abc import abstractmethod
from typing import Any, Dict, List, NamedTuple, Optional, Sequence, Tuple

import torch

from ... import _ffi
from ...runtime import PreparedBatch, prepared_batch_for, require_cuda, to_device_adj, to_device_f32
from ...utils.param_helpers import get_activation_function, get_aggregation_function


class MessagePassingInput(NamedTuple):
    """A named tuple to hold input to the message passing layer (message_passing.py:13-17)."""

    node_embeddings: Any
    adjacency_lists: Tuple[Any, ...]


class _Shape(tuple):
    """tuple with the TensorShape-style as_list() the reference tests call."""

    def as_list(self):
        return list(self)


class Variable:
    """A named weight.  ``value`` is a float32 CUDA tensor laid out exactly like the reference's
    tf.Variable of the same name (so reference checkpoints map one to one)."""

    def __init__(self, name: str, value: torch.Tensor, trainable: bool = True):
        self.name = name
        self.value = value
        self.trainable = trainable

    @property
    def shape(self) -> _Shape:
        return _Shape(self.value.shape)

    def assign(self, new_value) -> None:
        new = to_device_f32(new_value, self.value.device)
        if tuple(new.shape) != tuple(self.value.shape):
            raise ValueError(f"shape mismatch assigning {self.name}: {tuple(new.shape)} vs {tuple(self.value.shape)}")
        with torch.no_grad():
            self.value.copy_(new)

    def numpy(self):
        return self.value.detach().cpu().numpy()

    def requires_grad_(self, flag: bool = True) -> "Variable":
        """Mark the weight as a leaf that accumulates .grad in the autograd-enabled (training) path."""
        self.value.requires_grad_(flag)
        return self

    @property
    def grad(self):
        return self.value.grad

    def __repr__(self):
        return f"<Variable {self.name} shape={tuple(self.value.shape)}>"


def glorot_uniform(shape: Sequence[int], generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """Keras' default kernel initialiser (Dense / add_weight): U(+-sqrt(6/(fan_in+fan_out)))."""
    fan_in, fan_out = int(shape[-2]), int(shape[-1])
    lim = (6.0 / (fan_in + fan_out)) ** 0.5
    w = (torch.rand(tuple(shape), generator=generator, dtype=torch.float32) * 2.0 - 1.0) * lim
    # Weights live on the GPU; without one (CPU-only shape/registry tests) they stay on the host and
    # any attempt to *run* the layer raises in runtime.require_cuda().
    return w.to(require_cuda()) if torch.cuda.is_available() else w


def _last_dim(shape) -> int:
    return int(tuple(shape)[-1])


class MessagePassing:
    """Abstract class to compute new graph states by neural message passing
    (message_passing.py:20-218).  Shapes: V nodes, L edge types, E edges of a type, D input
    dimension, H = hidden_dim output dimension."""

    @classmethod
    def get_default_hyperparameters(cls):
        return {
            "aggregation_function": "sum",  # One of sum, mean, max, sqrt_n
            "message_activation_function": "relu",  # One of relu, leaky_relu, elu, gelu, tanh
            "message_activation_before_aggregation": False,
            "hidden_dim": 7,
        }

    def __init__(self, params: Dict[str, Any], **kwargs):
        self.name = kwargs.get("name", type(self).__name__.lower())
        self._hidden_dim = int(params["hidden_dim"])
        aggregation_fn_name = params["aggregation_function"]
        self._aggregation_fn = get_aggregation_function(aggregation_fn_name)
        self._message_activation_before_aggregation = params.get(
            "message_activation_before_aggregation", False)
        activation_fn_name = params["message_activation_function"]
        self._activation_fn = get_activation_function(activation_fn_name)
        self._variables: List[Variable] = []
        self._path = params.get("b200_path", "auto")  # execution path knob (not in the reference)
        if self._path not in _ffi.PATH:
            raise ValueError(f"Unknown b200_path: {self._path}")
        self.built = False

    # -- variable bookkeeping (Keras-like surface used by the reference tests) -----------------
    def add_weight(self, name: str, shape: Sequence[int], trainable: bool = True,
                   initial_value: Optional[torch.Tensor] = None) -> Variable:
        if initial_value is None:
            value = glorot_uniform(shape)
        elif torch.cuda.is_available():
            value = to_device_f32(initial_value)
        else:
            value = torch.as_tensor(initial_value, dtype=torch.float32)
        var = Variable(name, value, trainable)
        self._variables.append(var)
        return var

    @property
    def variables(self) -> List[Variable]:
        return list(self._variables)

    weights = variables

    @property
    def trainable_variables(self) -> List[Variable]:
        return [v for v in self._variables if v.trainable]

    def set_weights_from_oracle_dict(self, w: Dict[str, Any]) -> None:
        """Load weights given in the oracle's dict layout (tests / smoke)."""
        raise NotImplementedError

    # -- plugin hooks ---------------------------------------------------------------------------
    @abstractmethod
    def _message_function(self, edge_source_states, edge_target_states,
                          num_incoming_to_node_per_message, edge_type_idx: int, training: bool):
        """Messages [E, H] for one edge type (message_passing.py:64-93)."""

    def build(self, input_shapes: MessagePassingInput):
        self.built = True

    def __call__(self, inputs: MessagePassingInput, training: bool = False, **kwargs):
        if not self.built:
            node_shape = tuple(getattr(inputs.node_embeddings, "shape"))
            adj_shapes = tuple(tuple(getattr(a, "shape", (None, 2))) for a in inputs.adjacency_lists)
            self.build(MessagePassingInput(node_shape, adj_shapes))
        return self.call(inputs, training=training, **kwargs)

    @staticmethod
    def _device_inputs(inputs: MessagePassingInput, prepared: Optional[PreparedBatch]):
        h = to_device_f32(inputs.node_embeddings)
        if h.dim() != 2:
            raise ValueError("node_embeddings must have shape [V, D]")
        if prepared is None:
            adjs = tuple(to_device_adj(a, h.device) for a in inputs.adjacency_lists)
            # host adjacency lists are converted per call, so only device tensors hit the cache
            if all(a is b for a, b in zip(adjs, inputs.adjacency_lists)):
                prepared = prepared_batch_for(adjs, h.shape[0])
            else:
                prepared = PreparedBatch(adjs, h.shape[0])
        elif prepared.num_source_nodes != h.shape[0]:
            raise ValueError("prepared batch was built for a different number of nodes")
        return h, prepared

    def call(self, inputs: MessagePassingInput, training: bool = False,
             prepared: Optional[PreparedBatch] = None):
        """Generic path for user plugins (message_passing.py:95-133)."""
        h, prepared = self._device_inputs(inputs, prepared)
        from ..node_ops import require_no_grad
        require_no_grad("the generic MessagePassing.call plugin path", h, *[v.value for v in self.variables])
        num_nodes = int(h.shape[0])
        messages_per_type = self._calculate_messages_per_type(prepared, h, training)
        edge_type_to_message_targets = [a[:, 1] for a in prepared.adjacency_lists]
        return self._compute_new_node_embeddings(h, messages_per_type, edge_type_to_message_targets,
                                                 num_nodes, training)

    def _compute_new_node_embeddings(self, cur_node_embeddings, messages_per_type,
                                     edge_type_to_message_targets, num_nodes, training):
        """message_passing.py:135-179."""
        dev = cur_node_embeddings.device
        if messages_per_type:
            message_targets = torch.cat([t.reshape(-1) for t in edge_type_to_message_targets], dim=0)
            messages = torch.cat(messages_per_type, dim=0)
        else:
            message_targets = torch.zeros((0,), dtype=torch.int32, device=dev)
            messages = torch.zeros((0, self._hidden_dim), dtype=torch.float32, device=dev)
        if self._message_activation_before_aggregation:
            messages = self._activation_fn(messages)
        aggregated = self._aggregation_fn(data=messages, segment_ids=message_targets, num_segments=num_nodes)
        if not self._message_activation_before_aggregation:
            aggregated = self._activation_fn(aggregated)
        return aggregated

    def _calculate_messages_per_type(self, prepared: PreparedBatch, node_embeddings, training=False):
        """message_passing.py:181-218."""
        from ..node_ops import gather_rows
        V = int(node_embeddings.shape[0])
        type_to_num_incoming_edges = prepared.in_degree()  # [L, V]
        messages_per_type = []
        for edge_type_idx, adj in enumerate(prepared.adjacency_lists):
            src_states = gather_rows(node_embeddings, adj, 0)
            tgt_states = gather_rows(node_embeddings, adj, 1)
            n_in = gather_rows(type_to_num_incoming_edges[edge_type_idx].reshape(V, 1), adj, 1).reshape(-1)
            messages_per_type.append(
                self._message_function(src_states, tgt_states, n_in, edge_type_idx, training))
        return messages_per_type


MESSAGE_PASSING_IMPLEMENTATIONS: Dict[str, type] = {}


def register_message_passing_implementation(cls):
    """Decorator used to register a message passing class implementation (message_passing.py:221-227)."""
    MESSAGE_PASSING_IMPLEMENTATIONS[cls.__name__.lower()] = cls
    return cls


def calculate_type_to_num_incoming_edges(node_embeddings, adjacency_lists):
    """float32 tensor [L, V]: number of type-l edges into node v (message_passing.py:230-263).

    >>> # node_embeddings: 5 nodes; adjacency_lists as in the reference doctest give
    >>> # [[0,1,0,0,2],[0,0,0,1,1],[0,1,0,0,0]]  (checked in tests/test_gpu_parity.py)
    """
    h = to_device_f32(node_embeddings)
    adjs = tuple(to_device_adj(a, h.device) for a in adjacency_lists)
    return PreparedBatch(adjs, int(h.shape[0])).in_degree()
