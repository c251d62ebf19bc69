"""GGNN — mirror of tf2_gnn/layers/message_passing/ggnn.py:12-89 on the H100 path."""
from __future__ import annotations

from typing import Any, Dict, Optional

import torch

from ... import _ffi
from ...runtime import PreparedBatch, stream_ptr
from ..differentiable import edge_mlp_family_forward, gru_cell
from ..node_ops import _needs_grad
from .gnn_edge_mlp import GNN_Edge_MLP, _EdgeMLPLayerFunction
from .message_passing import MessagePassingInput, _last_dim, register_message_passing_implementation


def _ggnn_forward(h, prepared: PreparedBatch, cfg, gru_kernel, gru_recurrent_kernel, gru_bias, weights) -> torch.Tensor:
    """tfgnn_b200_ggnn_fwd: the layer's output rows [num_nodes, H]."""
    out = torch.empty((prepared.num_nodes, cfg["H"]), dtype=torch.float32, device=h.device)
    _ffi.check(_ffi.lib().tfgnn_b200_ggnn_fwd(
        prepared.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights), cfg["n_hidden"], cfg["H"],
        cfg["flags"], cfg["agg"], gru_kernel.data_ptr(), gru_recurrent_kernel.data_ptr(), gru_bias.data_ptr(),
        cfg["path"], out.data_ptr(), stream_ptr()))
    return out


class _GGNNFunction(torch.autograd.Function):
    """Autograd hook of the GGNN layer (SURVEY.md §8f-1): forward = tfgnn_b200_ggnn_fwd, backward =
    tfgnn_b200_ggnn_bwd (everything but h is recomputed)."""

    @staticmethod
    def forward(ctx, h, prepared, cfg, gru_kernel, gru_recurrent_kernel, gru_bias, *weights):
        out = _ggnn_forward(h, prepared, cfg, gru_kernel, gru_recurrent_kernel, gru_bias, weights)
        ctx.prepared, ctx.cfg = prepared, cfg
        ctx.save_for_backward(h, gru_kernel, gru_recurrent_kernel, gru_bias, *weights)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        h, gru_kernel, gru_recurrent_kernel, gru_bias, *weights = ctx.saved_tensors
        cfg, prepared = ctx.cfg, ctx.prepared
        if cfg["n_hidden"] != 0:
            raise NotImplementedError("GGNN backward is built for message MLPs without hidden layers only")
        grad_out = grad_out.contiguous()
        grad_h = torch.empty_like(h)
        grad_w = [torch.empty_like(w) for w in weights]
        g_k, g_u, g_b = (torch.empty_like(t) for t in (gru_kernel, gru_recurrent_kernel, gru_bias))
        _ffi.check(_ffi.lib().tfgnn_b200_ggnn_bwd(
            prepared.handle, prepared.transposed().handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights),
            cfg["H"], cfg["flags"], cfg["agg"], gru_kernel.data_ptr(), gru_recurrent_kernel.data_ptr(),
            gru_bias.data_ptr(), grad_out.data_ptr(), grad_h.data_ptr(), _ffi.ptr_array(grad_w), g_k.data_ptr(),
            g_u.data_ptr(), g_b.data_ptr(), stream_ptr()))
        return (grad_h, None, None, g_k, g_u, g_b, *grad_w)


class _GruUpdateFunction(torch.autograd.Function):
    """GGNN's node update out = GRUCell(agg, h) on its own (ggnn.py:84-87): forward = tfgnn_b200_gru_update_fwd (the update
    tfgnn_b200_ggnn_fwd runs), backward = tfgnn_b200_gru_update_bwd.  h = the layer's state rows."""

    @staticmethod
    def forward(ctx, agg, h, path, gru_kernel, gru_recurrent_kernel, gru_bias):
        agg, h = agg.contiguous(), h.contiguous()
        out = torch.empty_like(agg)
        _ffi.check(_ffi.lib().tfgnn_b200_gru_update_fwd(
            agg.data_ptr(), h.data_ptr(), int(agg.shape[0]), int(agg.shape[1]), gru_kernel.data_ptr(),
            gru_recurrent_kernel.data_ptr(), gru_bias.data_ptr(), path, out.data_ptr(), stream_ptr()))
        ctx.save_for_backward(agg, h, gru_kernel, gru_recurrent_kernel, gru_bias)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        agg, h, gru_kernel, gru_recurrent_kernel, gru_bias = ctx.saved_tensors
        grad_out = grad_out.contiguous()
        g_agg, g_h = torch.empty_like(agg), torch.empty_like(h)
        g_k, g_u, g_b = (torch.empty_like(t) for t in (gru_kernel, gru_recurrent_kernel, gru_bias))
        _ffi.check(_ffi.lib().tfgnn_b200_gru_update_bwd(
            agg.data_ptr(), h.data_ptr(), int(agg.shape[0]), int(agg.shape[1]), gru_kernel.data_ptr(),
            gru_recurrent_kernel.data_ptr(), gru_bias.data_ptr(), grad_out.data_ptr(), g_agg.data_ptr(), g_h.data_ptr(),
            g_k.data_ptr(), g_u.data_ptr(), g_b.data_ptr(), stream_ptr()))
        return g_agg, g_h, None, g_k, g_u, g_b


@register_message_passing_implementation
class GGNN(GNN_Edge_MLP):
    """h'_v = GRUCell(h_v, sum_l sum_{(u,v) in A_l} W_l h_u)  (ggnn.py:13-45).  The node embedding
    dimension must equal hidden_dim (ggnn.py:30).  GRU = Keras GRUCell(units=H) with TF2 defaults:
    kernel [D,3H], recurrent_kernel [H,3H], bias [2,3H], gates z|r|h, reset_after=True."""

    @classmethod
    def get_default_hyperparameters(cls):
        these_hypers = {
            "use_target_state_as_input": False,
            "normalize_by_num_incoming": True,
            "num_edge_MLP_hidden_layers": 0,
        }
        mp_hypers = super().get_default_hyperparameters()
        mp_hypers.update(these_hypers)
        return mp_hypers

    def __init__(self, params: Dict[str, Any], **kwargs):
        super().__init__(params, **kwargs)
        self._gru_kernel = None
        self._gru_recurrent_kernel = None
        self._gru_bias = None

    def build(self, input_shapes: MessagePassingInput):
        D = _last_dim(input_shapes.node_embeddings)
        H = self._hidden_dim
        self._gru_kernel = self.add_weight("gru_cell/kernel:0", (D, 3 * H))
        # Keras uses an orthogonal recurrent initialiser; Glorot keeps the same shape contract.
        self._gru_recurrent_kernel = self.add_weight("gru_cell/recurrent_kernel:0", (H, 3 * H))
        self._gru_bias = self.add_weight("gru_cell/bias:0", (2, 3 * H),
                                         initial_value=torch.zeros((2, 3 * H), dtype=torch.float32))
        super().build(input_shapes)

    def call(self, inputs: MessagePassingInput, training: bool = False,
             prepared: Optional[PreparedBatch] = None):
        h, prepared = self._device_inputs(inputs, prepared)
        self._check_types(prepared)
        if int(h.shape[1]) != self._hidden_dim:
            raise ValueError("GGNN: the node embedding dimension must equal hidden_dim")
        cfg, weights = self._cfg(), self._mlp_weights()
        gru = (self._gru_kernel.value, self._gru_recurrent_kernel.value, self._gru_bias.value)
        if _needs_grad(h, *gru, *weights):
            if self._ggnn_bwd_takes_it():
                return _GGNNFunction.apply(h, prepared, cfg, *gru, *weights)
            return self._composed_forward(h, prepared, cfg, gru, weights)
        return _ggnn_forward(h, prepared, cfg, *gru, weights)

    def _ggnn_bwd_takes_it(self) -> bool:
        """The configurations _GGNNFunction trains (tfgnn_b200_ggnn_bwd): linear messages from the source state only,
        hidden_dim % 4 == 0, max aggregation up to hidden_dim 512."""
        H = self._hidden_dim
        return (int(self._num_edge_MLP_hidden_layers) == 0 and not self._use_target_state_as_input and H % 4 == 0
                and (self._aggregation_fn.name != "max" or H <= 512))

    def _composed_forward(self, h: torch.Tensor, prepared: PreparedBatch, cfg, gru, weights) -> torch.Tensor:
        """Every other message MLP under autograd: the messages through GNN_Edge_MLP's own routing without activation
        (GGNN ignores activation-before, as its forward does), then the GRU update.  On the fused message paths this runs
        the kernels of tfgnn_b200_ggnn_fwd in the same order, so training and inference give the same bits."""
        if self._has_fused_backward(int(h.shape[1])):
            cfg = dict(cfg, flags=cfg["flags"] & ~_ffi.FLAG_ACT_BEFORE_AGG, act=_ffi.ACT[None])
            agg = _EdgeMLPLayerFunction.apply(h, prepared, cfg, *weights)
        else:
            agg = edge_mlp_family_forward(self, h, prepared, final_activation=False, activation_before=False)
        lo, hi = prepared.target_range
        if self._hidden_dim % 4 == 0:   # the shapes tfgnn_b200_gru_update_bwd differentiates
            return _GruUpdateFunction.apply(agg, h[lo:hi], _ffi.PATH[self._path], *gru)
        return gru_cell(agg, h[lo:hi], *gru)

    def set_weights_from_oracle_dict(self, w: Dict[str, Any]) -> None:
        super().set_weights_from_oracle_dict(w)
        self._gru_kernel.assign(w["gru_kernel"])
        self._gru_recurrent_kernel.assign(w["gru_recurrent_kernel"])
        self._gru_bias.assign(w["gru_bias"])
