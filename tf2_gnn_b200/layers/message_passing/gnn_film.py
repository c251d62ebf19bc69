"""GNN_FiLM — mirror of tf2_gnn/layers/message_passing/gnn_film.py:13-108 on the H100 path."""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import torch

from ... import _ffi
from ...runtime import PreparedBatch, stream_ptr
from ...utils.param_helpers import get_activation_function
from .gnn_edge_mlp import EdgeMLP, GNN_Edge_MLP
from ..differentiable import edge_mlp_family_forward
from ..node_ops import _needs_grad, dense
from .message_passing import MessagePassingInput, _last_dim, register_message_passing_implementation


def _film_forward(h, prepared: PreparedBatch, cfg, kernels, film) -> torch.Tensor:
    """tfgnn_b200_film_fwd: the layer's output rows [num_nodes, H]; kernels = the edge MLPs', film = the FiLM kernels."""
    out = torch.empty((prepared.num_nodes, cfg["H"]), dtype=torch.float32, device=h.device)
    _ffi.check(_ffi.lib().tfgnn_b200_film_fwd(
        prepared.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(kernels), cfg["n_hidden"], _ffi.ptr_array(film),
        cfg["H"], cfg["flags"], cfg["agg"], cfg["act"], cfg["path"], out.data_ptr(), stream_ptr()))
    return out


def _film_in_forward(h, film_in, prepared: PreparedBatch, cfg, kernels, film) -> torch.Tensor:
    """tfgnn_b200_film_in_fwd: as _film_forward with the FiLM input table film_in [V_owned, L*S] and the last FiLM
    kernels."""
    out = torch.empty((prepared.num_nodes, cfg["H"]), dtype=torch.float32, device=h.device)
    _ffi.check(_ffi.lib().tfgnn_b200_film_in_fwd(
        prepared.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(kernels), cfg["n_hidden"], film_in.data_ptr(),
        cfg["S"], _ffi.ptr_array(film), cfg["H"], cfg["flags"], cfg["agg"], cfg["act"], cfg["path"], out.data_ptr(),
        stream_ptr()))
    return out


class _FilmLayerFunction(torch.autograd.Function):
    """Autograd hook of the FiLM layer without hidden layers: forward = tfgnn_b200_film_fwd, backward =
    tfgnn_b200_film_bwd (aggregate-then-transform, no per-edge tensors).  weights = the L edge-MLP kernels, then the L
    FiLM kernels.  The reference gets these gradients from tf.GradientTape (models/graph_task_model.py:338-365)."""

    @staticmethod
    def forward(ctx, h, prepared, cfg, *weights):
        L = len(weights) // 2
        out = _film_forward(h, prepared, cfg, weights[:L], weights[L:])
        ctx.prepared, ctx.cfg = prepared, cfg
        ctx.save_for_backward(h, out, *weights)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        h, out, *weights = ctx.saved_tensors
        cfg, prepared = ctx.cfg, ctx.prepared
        L = len(weights) // 2
        grad_out = grad_out.contiguous()
        grad_h = torch.empty_like(h) if ctx.needs_input_grad[0] else None
        grad_w = [torch.empty_like(w) for w in weights]
        _ffi.check(_ffi.lib().tfgnn_b200_film_bwd(
            prepared.handle, prepared.transposed().handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights[:L]),
            _ffi.ptr_array(weights[L:]), cfg["H"], cfg["flags"], cfg["agg"], cfg["act"], out.data_ptr(),
            grad_out.data_ptr(), grad_h.data_ptr() if grad_h is not None else None, _ffi.ptr_array(grad_w[:L]),
            _ffi.ptr_array(grad_w[L:]), stream_ptr()))
        return (grad_h, None, None, *grad_w)


class _FilmInLayerFunction(torch.autograd.Function):
    """Autograd hook of the FiLM layer with hidden FiLM-MLP layers: forward = tfgnn_b200_film_in_fwd, backward =
    tfgnn_b200_film_in_bwd.  film_in [V, L*S] holds every type's last hidden FiLM activation z_l (computed at node level by
    the caller, whose Dense ops differentiate the hidden chain); weights = the L edge-MLP kernels, then the L last FiLM
    kernels [S, 2H]."""

    @staticmethod
    def forward(ctx, h, film_in, prepared, cfg, *weights):
        L = len(weights) // 2
        out = _film_in_forward(h, film_in, prepared, cfg, weights[:L], weights[L:])
        ctx.prepared, ctx.cfg = prepared, cfg
        ctx.save_for_backward(h, film_in, out, *weights)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        h, film_in, out, *weights = ctx.saved_tensors
        cfg, prepared = ctx.cfg, ctx.prepared
        L = len(weights) // 2
        grad_out = grad_out.contiguous()
        grad_h = torch.empty_like(h) if ctx.needs_input_grad[0] else None
        grad_in = torch.empty_like(film_in) if ctx.needs_input_grad[1] else None
        grad_w = [torch.empty_like(w) for w in weights]
        _ffi.check(_ffi.lib().tfgnn_b200_film_in_bwd(
            prepared.handle, prepared.transposed().handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights[:L]),
            film_in.data_ptr(), cfg["S"], _ffi.ptr_array(weights[L:]), cfg["H"], cfg["flags"], cfg["agg"], cfg["act"],
            out.data_ptr(), grad_out.data_ptr(), grad_h.data_ptr() if grad_h is not None else None,
            grad_in.data_ptr() if grad_in is not None else None, _ffi.ptr_array(grad_w[:L]), _ffi.ptr_array(grad_w[L:]),
            stream_ptr()))
        return (grad_h, grad_in, None, None, *grad_w)


@register_message_passing_implementation
class GNN_FiLM(GNN_Edge_MLP):
    """h'_v = sum_l sum_{(u,v) in A_l} sigma(1/c_{v,l} * gamma_{l,v} * (W_l h_u) + beta_{l,v}),
    [gamma|beta] = F_l(h_v)  (gnn_film.py:14-47)."""

    @classmethod
    def get_default_hyperparameters(cls):
        these_hypers = {
            "use_target_state_as_input": False,
            "normalize_by_num_incoming": False,
            "num_edge_MLP_hidden_layers": 0,
            "film_parameter_MLP_hidden_layers": [],
        }
        mp_hypers = super().get_default_hyperparameters()
        mp_hypers.update(these_hypers)
        return mp_hypers

    def __init__(self, params: Dict[str, Any], **kwargs):
        super().__init__(params, **kwargs)
        self._film_parameter_MLP_hidden_layers = params["film_parameter_MLP_hidden_layers"]
        self._edge_type_film_layer_computations: List[EdgeMLP] = []

    def build(self, input_shapes: MessagePassingInput):
        D = _last_dim(input_shapes.node_embeddings)
        for i in range(len(input_shapes.adjacency_lists)):
            # an int is that many hidden layers of width 2H, as dpu_utils' MLP builds them
            hidden = self._film_parameter_MLP_hidden_layers
            self._edge_type_film_layer_computations.append(
                EdgeMLP(self, f"edge_type_{i}-FiLM", D, 2 * self._hidden_dim,
                        hidden if isinstance(hidden, int) else list(hidden)))
        super().build(input_shapes)

    def call(self, inputs: MessagePassingInput, training: bool = False,
             prepared: Optional[PreparedBatch] = None):
        h, prepared = self._device_inputs(inputs, prepared)
        self._check_types(prepared)
        cfg, kernels = self._cfg(), self._mlp_weights()
        film = [m.layers[-1].value for m in self._edge_type_film_layer_computations]
        film_hidden = any(m.num_hidden_layers for m in self._edge_type_film_layer_computations)
        if _needs_grad(h, *[v.value for v in self.variables]):
            # both fused backwards take edge MLPs without hidden layers: `kernels` holds one kernel per type
            if self._has_fused_backward(int(h.shape[1])):
                return _FilmLayerFunction.apply(h, prepared, cfg, *kernels, *film)
            if film_hidden and self._has_fused_film_mlp_backward(int(h.shape[1]), prepared):
                film_in = self._film_inputs(h, prepared)
                return _FilmInLayerFunction.apply(h, film_in, prepared, dict(cfg, S=self._film_input_width()), *kernels,
                                                  *film)
            # edge-MLP hidden layers / max aggregation / activation before aggregation / widths that are not multiples of
            # 4 / target-range shards: the reference's literal op order with per-op backward kernels
            # (layers/differentiable.py)
            return edge_mlp_family_forward(
                self, h, prepared,
                film_kernels=[[v.value for v in m.layers] for m in self._edge_type_film_layer_computations])
        if film_hidden:
            film_in = self._film_inputs(h, prepared)
            return _film_in_forward(h, film_in, prepared, dict(cfg, S=self._film_input_width()), kernels, film)
        return _film_forward(h, prepared, cfg, kernels, film)

    def _film_input_width(self) -> int:
        """S: the width of the last hidden FiLM-MLP layer (the same for every type)."""
        return int(self._edge_type_film_layer_computations[0].layers[-1].value.shape[0])

    def _film_inputs(self, h: torch.Tensor, prepared: PreparedBatch) -> torch.Tensor:
        """[V_owned, L*S]: type l's hidden FiLM-MLP chain z_l = relu(.. relu(h_v F^(0)_l) ..) on the owned target rows
        (gnn_film.py:99-101 evaluates it on every edge's gathered target row; it depends on the target only)."""
        relu = get_activation_function("relu")
        lo, hi = prepared.target_range
        rows = h[lo:hi]
        zs = []
        for m in self._edge_type_film_layer_computations:
            z = rows
            for var in m.layers[:-1]:
                z = dense(z, var.value, None, relu)
            zs.append(z)
        return torch.cat(zs, dim=1)

    def _has_fused_backward(self, D: int) -> bool:
        """The configurations tfgnn_b200_film_bwd differentiates (the reference's PPI_GNN_FiLM.json among them)."""
        return (int(self._num_edge_MLP_hidden_layers) == 0
                and not any(m.num_hidden_layers for m in self._edge_type_film_layer_computations)
                and self._aggregation_fn.name != "max" and not self._message_activation_before_aggregation
                and D % 4 == 0 and self._hidden_dim % 4 == 0)

    def _has_fused_film_mlp_backward(self, D: int, prepared: PreparedBatch) -> bool:
        """The configurations with hidden FiLM-MLP layers that tfgnn_b200_film_in_bwd differentiates, on whole batches."""
        return (int(self._num_edge_MLP_hidden_layers) == 0
                and self._aggregation_fn.name != "max" and not self._message_activation_before_aggregation
                and D % 4 == 0 and self._hidden_dim % 4 == 0 and self._film_input_width() % 4 == 0
                and prepared.target_range == (0, prepared.num_source_nodes))

    def set_weights_from_oracle_dict(self, w: Dict[str, Any]) -> None:
        super().set_weights_from_oracle_dict(w)
        for mlp, mats in zip(self._edge_type_film_layer_computations, w["film_mlps"]):
            for var, m in zip(mlp.layers, mats):
                var.assign(m)
