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


def _rgin_forward(h, prepared: PreparedBatch, cfg, weights, aggr) -> torch.Tensor:
    """tfgnn_b200_rgin_fwd: the layer's output rows [num_nodes, H]; `aggr` = the aggregation MLP's kernels."""
    out = torch.empty((prepared.num_nodes, cfg["H"]), dtype=torch.float32, device=h.device)
    _ffi.check(_ffi.lib().tfgnn_b200_rgin_fwd(
        prepared.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(weights), cfg["n_hidden"], cfg["H"],
        cfg["flags"], cfg["agg"], cfg["act"], _ffi.ptr_array(aggr), len(aggr), cfg["path"], out.data_ptr(), stream_ptr()))
    return out


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
        cfg, weights = self._cfg(), self._mlp_weights()
        aggr = [v.value for v in (self._aggregation_mlp or [])]
        if _needs_grad(h, *[v.value for v in self.variables]):
            if self._has_fused_backward(int(h.shape[1])):
                # the inference forward's op sequence, each op with its fused backward: edge MLP (activation-before is
                # ignored, rgin.py:88-106), then the aggregation MLP and the activation
                cfg = dict(cfg, flags=cfg["flags"] & ~_ffi.FLAG_ACT_BEFORE_AGG, act=_ffi.ACT[None] if aggr else cfg["act"])
                out = _EdgeMLPLayerFunction.apply(h, prepared, cfg, *weights)
                relu = get_activation_function("relu")
                for i, W in enumerate(aggr):
                    out = dense(out, W, None, self._activation_fn if i == len(aggr) - 1 else relu)
                return out
            # two or more hidden layers / one hidden layer with max aggregation: the reference's literal op order with
            # per-op backward kernels (layers/differentiable.py)
            return edge_mlp_family_forward(self, h, prepared, activation_before=False, aggr_kernels=aggr or None)
        return _rgin_forward(h, prepared, cfg, weights, aggr)

    def set_weights_from_oracle_dict(self, w: Dict[str, Any]) -> None:
        super().set_weights_from_oracle_dict(w)
        if self._aggregation_mlp is not None:
            for var, m in zip(self._aggregation_mlp, w["aggr_mlp"]):
                var.assign(m)
