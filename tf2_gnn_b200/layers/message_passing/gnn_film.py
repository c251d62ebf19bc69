"""GNN_FiLM — mirror of tf2_gnn/layers/message_passing/gnn_film.py:13-108 on the H100 path."""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import torch

from ... import _ffi
from ...runtime import PreparedBatch, stream_ptr
from .gnn_edge_mlp import EdgeMLP, GNN_Edge_MLP
from ..differentiable import edge_mlp_family_forward
from ..node_ops import _needs_grad
from .message_passing import MessagePassingInput, _last_dim, register_message_passing_implementation


class _FilmLayerFunction(torch.autograd.Function):
    """Autograd hook of the FiLM layer without hidden layers: forward = tfgnn_b200_film_fwd, backward =
    tfgnn_b200_film_bwd (aggregate-then-transform, no per-edge tensors).  weights = the L edge-MLP kernels, then the L
    FiLM kernels.  The reference gets these gradients from tf.GradientTape (models/graph_task_model.py:338-365)."""

    @staticmethod
    def forward(ctx, h, prepared, cfg, *weights):
        L = len(weights) // 2
        out = torch.empty((prepared.num_nodes, cfg["H"]), dtype=torch.float32, device=h.device)
        _ffi.check(_ffi.lib().tfgnn_b200_film_fwd(
            prepared.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights[:L]), 0, _ffi.ptr_array(weights[L:]),
            cfg["H"], cfg["flags"], cfg["agg"], cfg["act"], cfg["path"], out.data_ptr(), stream_ptr()))
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
            self._edge_type_film_layer_computations.append(
                EdgeMLP(self, f"edge_type_{i}-FiLM", D, 2 * self._hidden_dim,
                        list(self._film_parameter_MLP_hidden_layers)))
        super().build(input_shapes)

    def call(self, inputs: MessagePassingInput, training: bool = False,
             prepared: Optional[PreparedBatch] = None):
        h, prepared = self._device_inputs(inputs, prepared)
        self._check_types(prepared)
        if _needs_grad(h, *[v.value for v in self.variables]):
            if self._has_fused_backward(int(h.shape[1])):
                act = self._activation_fn.code if self._activation_fn is not None else _ffi.ACT[None]
                cfg = dict(H=self._hidden_dim, flags=self._flags(), agg=self._aggregation_fn.code, act=act,
                           path=_ffi.PATH[self._path])
                weights = ([m.layers[0].value for m in self._edge_type_mlps]
                           + [m.layers[0].value for m in self._edge_type_film_layer_computations])
                return _FilmLayerFunction.apply(h, prepared, cfg, *weights)
            # hidden layers / max aggregation / activation before aggregation: the reference's literal op order with
            # per-op backward kernels (layers/differentiable.py)
            return edge_mlp_family_forward(
                self, h, prepared,
                film_kernels=[[v.value for v in m.layers] for m in self._edge_type_film_layer_computations])
        if any(m.num_hidden_layers for m in self._edge_type_film_layer_computations):
            raise NotImplementedError("film_parameter_MLP_hidden_layers != [] is not built yet")
        out = torch.empty((prepared.num_nodes, self._hidden_dim), dtype=torch.float32, device=h.device)
        ptrs, _keep = self._mlp_weight_ptrs()
        film = [m.layers[0].value for m in self._edge_type_film_layer_computations]
        _ffi.check(_ffi.lib().tfgnn_b200_film_fwd(
            prepared.handle, h.data_ptr(), int(h.shape[1]), ptrs, int(self._num_edge_MLP_hidden_layers),
            _ffi.ptr_array(film), self._hidden_dim, self._flags(), self._aggregation_fn.code,
            self._activation_fn.code, _ffi.PATH[self._path], out.data_ptr(), stream_ptr()))
        return out

    def _has_fused_backward(self, D: int) -> bool:
        """The configurations tfgnn_b200_film_bwd differentiates (the reference's PPI_GNN_FiLM.json among them)."""
        return (int(self._num_edge_MLP_hidden_layers) == 0 and not list(self._film_parameter_MLP_hidden_layers)
                and self._aggregation_fn.name != "max" and not self._message_activation_before_aggregation
                and D % 4 == 0 and self._hidden_dim % 4 == 0)

    def set_weights_from_oracle_dict(self, w: Dict[str, Any]) -> None:
        super().set_weights_from_oracle_dict(w)
        for mlp, mats in zip(self._edge_type_film_layer_computations, w["film_mlps"]):
            for var, m in zip(mlp.layers, mats):
                var.assign(m)
