"""RGAT — mirror of tf2_gnn/layers/message_passing/rgat.py:11-163 on the H100 path."""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import torch

from ... import _ffi
from ...runtime import PreparedBatch, stream_ptr
from ..node_ops import _needs_grad
from .message_passing import (MessagePassing, MessagePassingInput, Variable, _last_dim,
                              register_message_passing_implementation)


def _rgat_forward(h, prepared: PreparedBatch, cfg, kernels, attention) -> torch.Tensor:
    """tfgnn_b200_rgat_fwd: the layer's output rows [num_nodes, H]."""
    out = torch.empty((prepared.num_nodes, cfg["H"]), dtype=torch.float32, device=h.device)
    _ffi.check(_ffi.lib().tfgnn_b200_rgat_fwd(
        prepared.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(kernels), _ffi.ptr_array(attention),
        cfg["H"], cfg["K"], cfg["act"], cfg["path"], out.data_ptr(), stream_ptr()))
    return out


class _RgatLayerFunction(torch.autograd.Function):
    """Autograd hook of the RGAT layer: forward = tfgnn_b200_rgat_fwd (so training output equals inference output),
    backward = tfgnn_b200_rgat_bwd (no per-edge tensors, no float atomics).  weights = the L projection kernels, then the L
    attention parameters.  The reference gets these gradients from tf.GradientTape (models/graph_task_model.py:338-365)."""

    @staticmethod
    def forward(ctx, h, prepared, cfg, *weights):
        L = len(weights) // 2
        out = _rgat_forward(h, prepared, cfg, weights[:L], weights[L:])
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
        _ffi.check(_ffi.lib().tfgnn_b200_rgat_bwd(
            prepared.handle, prepared.transposed().handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights[:L]),
            _ffi.ptr_array(weights[L:]), cfg["H"], cfg["K"], cfg["act"], cfg["path"], out.data_ptr(), grad_out.data_ptr(),
            grad_h.data_ptr() if grad_h is not None else None, _ffi.ptr_array(grad_w[:L]), _ffi.ptr_array(grad_w[L:]),
            stream_ptr()))
        return (grad_h, None, None, *grad_w)


@register_message_passing_implementation
class RGAT(MessagePassing):
    """Relational graph attention (rgat.py:12-51): per type a bias-free Dense W_l [D,H] applied to
    source and target states, K-head scores leaky_relu(a_l . [W_l h_u || W_l h_v]), softmax over ALL
    incoming edges of a node (all types jointly, rgat.py:135-151), weighted sum, activation."""

    @classmethod
    def get_default_hyperparameters(cls):
        these_hypers = {"num_heads": 3}
        mp_hypers = super().get_default_hyperparameters()
        mp_hypers.update(these_hypers)
        return mp_hypers

    def __init__(self, params: Dict[str, Any], **kwargs):
        super().__init__(params, **kwargs)
        self._num_heads: int = params["num_heads"]
        self._edge_type_to_message_computation_layer: List[Variable] = []
        self._edge_type_to_attention_parameters: List[Variable] = []

    def build(self, input_shapes: MessagePassingInput):
        D = _last_dim(input_shapes.node_embeddings)
        per_head_dim = self._hidden_dim // self._num_heads
        for i in range(len(input_shapes.adjacency_lists)):
            self._edge_type_to_message_computation_layer.append(
                self.add_weight(f"edge_type_{i}/Edge_weight_{i}/kernel:0", (D, self._hidden_dim)))
            self._edge_type_to_attention_parameters.append(
                self.add_weight(f"edge_type_{i}/Edge_attention_parameters_{i}:0",
                                (self._num_heads, 2 * per_head_dim)))
        super().build(input_shapes)

    def call(self, inputs: MessagePassingInput, training: bool = False,
             prepared: Optional[PreparedBatch] = None):
        h, prepared = self._device_inputs(inputs, prepared)
        self._check_shape(prepared)
        kernels = [v.value for v in self._edge_type_to_message_computation_layer]
        attention = [v.value for v in self._edge_type_to_attention_parameters]
        if _needs_grad(h, *[v.value for v in self.variables]):
            if self._has_fused_backward(int(h.shape[1])):
                return _RgatLayerFunction.apply(h, prepared, self._cfg(), *kernels, *attention)
            # other shapes: the reference's literal op order with per-op backward kernels (layers/differentiable.py)
            from ..differentiable import rgat_forward
            return rgat_forward(self, h, prepared)
        return _rgat_forward(h, prepared, self._cfg(), kernels, attention)

    def _cfg(self) -> Dict[str, int]:
        """The layer's arguments of tfgnn_b200_rgat_fwd / _bwd, the same for the training and the inference call."""
        act = self._activation_fn.code if self._activation_fn is not None else _ffi.ACT[None]
        return dict(H=self._hidden_dim, K=int(self._num_heads), act=act, path=_ffi.PATH[self._path])

    def _check_shape(self, prepared: PreparedBatch) -> None:
        if prepared.num_edge_types != len(self._edge_type_to_message_computation_layer):
            raise ValueError("number of adjacency lists differs from the number the layer was built for")
        if self._hidden_dim % self._num_heads:
            raise ValueError("hidden_dim must be divisible by num_heads (rgat.py:72)")

    def _has_fused_backward(self, D: int) -> bool:
        """The shapes tfgnn_b200_rgat_bwd differentiates, on whole batches and target-range shards (the reference's
        PPI_RGAT.json and bench.py's cfg3 among them): D and the per-head width multiples of 4, hidden_dim <= 512."""
        H, K = self._hidden_dim, int(self._num_heads)
        return (K > 0 and H % K == 0 and D % 4 == 0 and (H // K) % 4 == 0 and H <= 512
                and self._path != "atomic")

    def _message_function(self, *args, **kwargs):
        raise NotImplementedError("built-in layers run fused; _message_function is only a plugin hook")

    def set_weights_from_oracle_dict(self, w: Dict[str, Any]) -> None:
        for var, m in zip(self._edge_type_to_message_computation_layer, w["edge_kernels"]):
            var.assign(m)
        for var, m in zip(self._edge_type_to_attention_parameters, w["edge_attention"]):
            var.assign(m)
