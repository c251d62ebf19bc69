"""GNN_Edge_MLP — mirror of tf2_gnn/layers/message_passing/gnn_edge_mlp.py:12-107 on the H100 path."""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import torch

from ... import _ffi
from ...runtime import PreparedBatch, stream_ptr
from ..node_ops import _needs_grad
from .message_passing import (MessagePassing, MessagePassingInput, Variable, _last_dim,
                              register_message_passing_implementation)


def _edge_mlp_forward(h, prepared: PreparedBatch, cfg, weights) -> torch.Tensor:
    """tfgnn_b200_edge_mlp_fwd: the layer's output rows [num_nodes, H]."""
    out = torch.empty((prepared.num_nodes, cfg["H"]), dtype=torch.float32, device=h.device)
    _ffi.check(_ffi.lib().tfgnn_b200_edge_mlp_fwd(
        prepared.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights), cfg["n_hidden"], cfg["H"],
        cfg["flags"], cfg["agg"], cfg["act"], cfg["path"], out.data_ptr(), stream_ptr()))
    return out


class _EdgeMLPLayerFunction(torch.autograd.Function):
    """Autograd hook of the fused layer (SURVEY.md §8f-1): forward = tfgnn_b200_edge_mlp_fwd, backward =
    tfgnn_b200_rgcn_bwd (no hidden layer) or tfgnn_b200_edge_mlp_bwd (one hidden layer).  The reference gets these
    gradients from tf.GradientTape (models/graph_task_model.py:338-365)."""

    @staticmethod
    def forward(ctx, h, prepared, cfg, *weights):
        out = _edge_mlp_forward(h, prepared, cfg, weights)
        ctx.prepared, ctx.cfg = prepared, cfg
        ctx.save_for_backward(h, out, *weights)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        h, out, *weights = ctx.saved_tensors
        cfg, prepared = ctx.cfg, ctx.prepared
        if cfg["n_hidden"] not in (0, 1):
            raise NotImplementedError("backward is built for edge MLPs with at most one hidden layer")
        grad_out = grad_out.contiguous()
        grad_h = torch.empty_like(h) if ctx.needs_input_grad[0] else None
        grad_w = [torch.empty_like(w) for w in weights]
        gh = grad_h.data_ptr() if grad_h is not None else None
        if cfg["n_hidden"] == 0:
            _ffi.check(_ffi.lib().tfgnn_b200_rgcn_bwd(
                prepared.handle, prepared.transposed().handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights),
                cfg["H"], cfg["flags"], cfg["agg"], cfg["act"], out.data_ptr(), grad_out.data_ptr(), gh,
                _ffi.ptr_array(grad_w), stream_ptr()))
        else:
            _ffi.check(_ffi.lib().tfgnn_b200_edge_mlp_bwd(
                prepared.handle, prepared.transposed().handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights),
                1, cfg["H"], cfg["flags"], cfg["agg"], cfg["act"], out.data_ptr(), grad_out.data_ptr(), gh,
                _ffi.ptr_array(grad_w), stream_ptr()))
        return (grad_h, None, None, *grad_w)


class EdgeMLP:
    """Weights of one dpu_utils.tf2utils.MLP(out_size=H, hidden_layers=n, use_biases=False):
    n hidden Dense(H, relu) + linear Dense(H) (gnn_edge_mlp.py:76-79)."""

    def __init__(self, layer: MessagePassing, scope: str, in_size: int, out_size: int, hidden_layers):
        sizes = [out_size] * hidden_layers if isinstance(hidden_layers, int) else list(hidden_layers)
        dims = [in_size] + sizes + [out_size]
        self.layers: List[Variable] = []
        for i in range(len(dims) - 1):
            lname = "dense_out" if i == len(dims) - 2 else f"dense_{i}"
            self.layers.append(layer.add_weight(f"{scope}/MLP/{lname}/kernel:0", (dims[i], dims[i + 1])))

    @property
    def num_hidden_layers(self) -> int:
        return len(self.layers) - 1


@register_message_passing_implementation
class GNN_Edge_MLP(MessagePassing):
    """h'_v = sum_l sum_{(u,v) in A_l} sigma(1/c_{v,l} * MLP_l(h_u || h_v))  (gnn_edge_mlp.py:13-44)."""

    @classmethod
    def get_default_hyperparameters(cls):
        these_hypers = {
            "use_target_state_as_input": True,
            "normalize_by_num_incoming": False,
            "num_edge_MLP_hidden_layers": 1,
        }
        mp_hypers = super().get_default_hyperparameters()
        mp_hypers.update(these_hypers)
        return mp_hypers

    def __init__(self, params: Dict[str, Any], **kwargs):
        super().__init__(params, **kwargs)
        self._use_target_state_as_input = params["use_target_state_as_input"]
        self._normalize_by_num_incoming = params["normalize_by_num_incoming"]
        self._num_edge_MLP_hidden_layers = params["num_edge_MLP_hidden_layers"]
        self._edge_type_mlps: List[EdgeMLP] = []

    def build(self, input_shapes: MessagePassingInput):
        D = _last_dim(input_shapes.node_embeddings)
        num_edge_types = len(input_shapes.adjacency_lists)
        edge_layer_input_size = 2 * D if self._use_target_state_as_input else D
        for i in range(num_edge_types):
            self._edge_type_mlps.append(
                EdgeMLP(self, f"edge_type_{i}", edge_layer_input_size, self._hidden_dim,
                        self._num_edge_MLP_hidden_layers))
        super().build(input_shapes)

    # -- C-ABI glue ---------------------------------------------------------------------------
    def _flags(self) -> int:
        f = 0
        if self._normalize_by_num_incoming:
            f |= _ffi.FLAG_NORMALIZE
        if self._message_activation_before_aggregation:
            f |= _ffi.FLAG_ACT_BEFORE_AGG
        if self._use_target_state_as_input:
            f |= _ffi.FLAG_USE_TARGET
        return f

    def _cfg(self) -> Dict[str, int]:
        """The layer's arguments of the fused entry points, the same for the training and the inference call."""
        act = self._activation_fn.code if self._activation_fn is not None else _ffi.ACT[None]
        return dict(H=self._hidden_dim, n_hidden=int(self._num_edge_MLP_hidden_layers), flags=self._flags(),
                    agg=self._aggregation_fn.code, act=act, path=_ffi.PATH[self._path])

    def _mlp_weights(self) -> List[torch.Tensor]:
        """Every edge type's MLP kernels, type by type."""
        return [v.value for mlp in self._edge_type_mlps for v in mlp.layers]

    def _check_types(self, prepared: PreparedBatch):
        if prepared.num_edge_types != len(self._edge_type_mlps):
            raise ValueError(f"layer was built for {len(self._edge_type_mlps)} edge types, "
                             f"got {prepared.num_edge_types} adjacency lists")

    def call(self, inputs: MessagePassingInput, training: bool = False,
             prepared: Optional[PreparedBatch] = None):
        h, prepared = self._device_inputs(inputs, prepared)
        self._check_types(prepared)
        cfg, weights = self._cfg(), self._mlp_weights()
        if _needs_grad(h, *weights):
            if not self._has_fused_backward(int(h.shape[1]), self._message_activation_before_aggregation):
                # two or more hidden layers / one hidden layer with max aggregation or activation before aggregation: the
                # reference's literal op order with per-op backward kernels (layers/differentiable.py)
                from ..differentiable import edge_mlp_family_forward
                return edge_mlp_family_forward(self, h, prepared)
            return _EdgeMLPLayerFunction.apply(h, prepared, cfg, *weights)
        return _edge_mlp_forward(h, prepared, cfg, weights)

    def _has_fused_backward(self, D: int, activation_before: bool = False) -> bool:
        """The edge MLPs tfgnn_b200_rgcn_bwd (no hidden layer: every aggregation, the activation before or after it; with
        max aggregation or the activation before it up to hidden_dim 512) and tfgnn_b200_edge_mlp_bwd (one hidden layer, the
        class defaults of GNN_Edge_MLP and RGIN: sum / mean / sqrt_n with the activation after it, up to hidden_dim 512)
        differentiate.  `activation_before`: the layer applies its activation before the aggregation (RGIN ignores it)."""
        n, H = int(self._num_edge_MLP_hidden_layers), self._hidden_dim
        if D % 4 or H % 4:
            return False
        transform_then_aggregate = activation_before or self._aggregation_fn.name == "max"
        if n == 0:
            return H <= 512 or not transform_then_aggregate
        return n == 1 and H <= 512 and not transform_then_aggregate

    def call_with_layernorm(self, inputs: MessagePassingInput, gamma: torch.Tensor, beta: torch.Tensor, epsilon: float,
                            prepared: Optional[PreparedBatch] = None) -> torch.Tensor:
        """LayerNormalization(layer(inputs)) — the pair gnn.py:299-321 runs with use_inter_layer_layernorm — as ONE call
        (tfgnn_b200_rgcn_ln_fwd): for RGCN-style layers the normalisation happens in the fused kernel's epilogue.  Other
        configurations, and any call that records gradients, compose the two ops."""
        h, prepared = self._device_inputs(inputs, prepared)
        weights = self._mlp_weights()
        fusable = (int(self._num_edge_MLP_hidden_layers) == 0 and not self._use_target_state_as_input
                   and type(self)._compute_is_plain_edge_mlp())
        if not fusable or _needs_grad(h, gamma, beta, *weights):
            from ..node_ops import layer_norm
            return layer_norm(self.call(MessagePassingInput(h, inputs.adjacency_lists), prepared=prepared), gamma, beta,
                              epsilon)
        self._check_types(prepared)
        cfg = self._cfg()
        out = torch.empty((prepared.num_nodes, cfg["H"]), dtype=torch.float32, device=h.device)
        _ffi.check(_ffi.lib().tfgnn_b200_rgcn_ln_fwd(
            prepared.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights), cfg["H"], cfg["flags"], cfg["agg"],
            cfg["act"], cfg["path"], gamma.data_ptr(), beta.data_ptr(), float(epsilon), out.data_ptr(), stream_ptr()))
        return out

    @classmethod
    def _compute_is_plain_edge_mlp(cls) -> bool:
        """True for the classes whose call() is the plain edge-MLP layer (GNN_Edge_MLP, RGCN); GGNN / RGIN / GNN-FiLM add
        their own node update or modulation and take the composed path."""
        return cls.__name__ in ("GNN_Edge_MLP", "RGCN")

    def call_allgather(self, node_embeddings: torch.Tensor, prepared: PreparedBatch, replica_ptrs, own_rank: int,
                       multicast_ptr: int = 0) -> None:
        """The layer on a target-range shard with the all-gather fused into the kernel's epilogue
        (tfgnn_b200_rgcn_fwd_allgather, SURVEY.md §8e case 2): `node_embeddings` is this rank's full [V, D] source table,
        `replica_ptrs[r]` the device address, mapped into this process, of rank r's [V, H] OUTPUT table (e.g.
        sharding.PeerNodeTables).  Output rows [target_begin, target_end) of every replica are written; nothing is
        returned.  Raises NotImplementedError when the shard does not take the fused kernel (use the plain call + an
        all-gather then).  `multicast_ptr`: a multicast (NVSwitch) mapping of the same tables, if the platform has one: the
        epilogue then issues one multimem.st instead of one store per peer."""
        from ctypes import c_void_p
        if int(self._num_edge_MLP_hidden_layers) != 0 or self._use_target_state_as_input:
            raise NotImplementedError("call_allgather needs an RGCN-style layer (no hidden layers, source state only)")
        self._check_types(prepared)
        reps = (c_void_p * len(replica_ptrs))(*[int(p) for p in replica_ptrs])
        _ffi.check(_ffi.lib().tfgnn_b200_rgcn_fwd_allgather(
            prepared.handle, node_embeddings.data_ptr(), int(node_embeddings.shape[1]), _ffi.ptr_array(self._mlp_weights()),
            self._hidden_dim, self._flags(), self._aggregation_fn.code, self._activation_fn.code, reps, len(replica_ptrs),
            int(own_rank), c_void_p(int(multicast_ptr) or None), stream_ptr()))

    def _message_function(self, edge_source_states, edge_target_states, num_incoming_to_node_per_message,
                          edge_type_idx: int, training: bool):
        raise NotImplementedError("built-in layers run fused; _message_function is only a plugin hook")

    def set_weights_from_oracle_dict(self, w: Dict[str, Any]) -> None:
        for mlp, mats in zip(self._edge_type_mlps, w["edge_mlps"]):
            for var, m in zip(mlp.layers, mats):
                var.assign(m)
