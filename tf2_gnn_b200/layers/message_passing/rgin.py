"""RGIN — mirror of tf2_gnn/layers/message_passing/rgin.py:13-106 on the H100 path."""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import torch

from ... import _ffi
from ...runtime import PreparedBatch, stream_ptr
from ...utils.param_helpers import get_activation_function
from .gnn_edge_mlp import GNN_Edge_MLP, _EdgeMLPLayerFunction
from ..differentiable import edge_mlp_family_forward
from ..node_ops import _needs_grad, dense
from .message_passing import MessagePassingInput, Variable, register_message_passing_implementation


@register_message_passing_implementation
class RGIN(GNN_Edge_MLP):
    """h'_v = sigma(MLP_aggr(sum_l sum_{(u,v) in A_l} MLP_l(h_u)))  (rgin.py:14-59)."""

    @classmethod
    def get_default_hyperparameters(cls):
        these_hypers = {
            "use_target_state_as_input": False,
            "num_edge_MLP_hidden_layers": 1,
            "num_aggr_MLP_hidden_layers": None,
        }
        gnn_edge_mlp_hypers = super().get_default_hyperparameters()
        gnn_edge_mlp_hypers.update(these_hypers)
        return gnn_edge_mlp_hypers

    def __init__(self, params: Dict[str, Any], **kwargs):
        super().__init__(params, **kwargs)
        self._num_aggr_MLP_hidden_layers: Optional[int] = params["num_aggr_MLP_hidden_layers"]
        self._aggregation_mlp: Optional[List[Variable]] = None

    def build(self, input_shapes: MessagePassingInput):
        if self._num_aggr_MLP_hidden_layers is not None:
            H = self._hidden_dim
            n = int(self._num_aggr_MLP_hidden_layers)
            self._aggregation_mlp = []
            for i in range(n + 1):
                lname = "dense_out" if i == n else f"dense_{i}"
                self._aggregation_mlp.append(self.add_weight(f"aggregation_MLP/MLP/{lname}/kernel:0", (H, H)))
        super().build(input_shapes)

    def call(self, inputs: MessagePassingInput, training: bool = False,
             prepared: Optional[PreparedBatch] = None):
        h, prepared = self._device_inputs(inputs, prepared)
        self._check_types(prepared)
        if _needs_grad(h, *[v.value for v in self.variables]):
            if self._has_fused_backward(int(h.shape[1])):
                # the inference forward's op sequence, each op with its fused backward: edge MLP (activation-before is
                # ignored, rgin.py:88-106), then the aggregation MLP and the activation
                aggr = [v.value for v in (self._aggregation_mlp or [])]
                act = self._activation_fn.code if (self._activation_fn is not None and not aggr) else _ffi.ACT[None]
                cfg = dict(H=self._hidden_dim, n_hidden=int(self._num_edge_MLP_hidden_layers),
                           flags=self._flags() & ~_ffi.FLAG_ACT_BEFORE_AGG, agg=self._aggregation_fn.code, act=act,
                           path=_ffi.PATH[self._path])
                out = _EdgeMLPLayerFunction.apply(h, prepared, cfg, *self._mlp_weight_ptrs()[1])
                relu = get_activation_function("relu")
                for i, W in enumerate(aggr):
                    out = dense(out, W, None, self._activation_fn if i == len(aggr) - 1 else relu)
                return out
            # two or more hidden layers / one hidden layer with max aggregation: the reference's literal op order with
            # per-op backward kernels (layers/differentiable.py)
            return edge_mlp_family_forward(
                self, h, prepared, activation_before=False,
                aggr_kernels=[v.value for v in self._aggregation_mlp] if self._aggregation_mlp is not None else None)
        out = torch.empty((prepared.num_nodes, self._hidden_dim), dtype=torch.float32, device=h.device)
        ptrs, _keep = self._mlp_weight_ptrs()
        aggr = [v.value for v in (self._aggregation_mlp or [])]
        _ffi.check(_ffi.lib().tfgnn_b200_rgin_fwd(
            prepared.handle, h.data_ptr(), int(h.shape[1]), ptrs, int(self._num_edge_MLP_hidden_layers),
            self._hidden_dim, self._flags(), self._aggregation_fn.code, self._activation_fn.code,
            _ffi.ptr_array(aggr), len(aggr), _ffi.PATH[self._path], out.data_ptr(), stream_ptr()))
        return out

    def set_weights_from_oracle_dict(self, w: Dict[str, Any]) -> None:
        super().set_weights_from_oracle_dict(w)
        if self._aggregation_mlp is not None:
            for var, m in zip(self._aggregation_mlp, w["aggr_mlp"]):
                var.assign(m)
