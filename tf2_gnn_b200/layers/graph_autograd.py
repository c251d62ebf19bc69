"""Training path of the graph readout and the global exchange combines on graph ROW RANGES.

node_to_graph_map is non-decreasing, so a graph is the row range graph_ptr[g] .. graph_ptr[g+1].  The forward of every
function here is the inference forward (the segment kernels of csrc/graph_ops.cu: the training forward is bitwise the
torch.no_grad() forward); the backward is one row-parallel pass plus, where a per-graph value was broadcast to the
graph's nodes, tfgnn_b200_segment_sum_rows.  No float atomics (gradients are bitwise reproducible) and no per-node copy
of a per-graph value.  layers/differentiable.py keeps the reference's literal op order for the same layers; the tests use
it as the second opinion.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import _ffi
from ..runtime import stream_ptr
from . import node_ops
from .node_ops import _ptr


def segment_sum_rows(data: torch.Tensor, n2g: torch.Tensor, graph_ptr: torch.Tensor) -> torch.Tensor:
    """out[g] = sum of data[v] over the rows of graph g: the adjoint of table[node_to_graph_map]."""
    data = data.contiguous()
    G, C = int(graph_ptr.shape[0]) - 1, int(data.shape[1])
    out = torch.empty((G, C), dtype=torch.float32, device=data.device)
    _ffi.check(_ffi.lib().tfgnn_b200_segment_sum_rows(data.data_ptr(), n2g.data_ptr(), graph_ptr.data_ptr(),
                                                      int(data.shape[0]), G, C, out.data_ptr(), stream_ptr()))
    return out


# ---- readout ----------------------------------------------------------------------------------------------------
class _ReadoutFunction(torch.autograd.Function):
    """scores [V, K] (or None) and the transformation result [V, GD] before the clamp -> graph representations [G, GD]
    (nodes_to_graph_representation.py:176-227)."""

    @staticmethod
    def forward(ctx, scores, reprs, n2g, graph_ptr, num_heads, weighting_fun, lower, upper):
        weights = node_ops.readout_weights(scores, graph_ptr, weighting_fun)
        reprs = reprs.contiguous()
        clamped = reprs if lower is None and upper is None else node_ops.clamp_(reprs.clone(), lower, upper)
        out = node_ops.weighted_segment_sum(clamped, weights, graph_ptr, num_heads, mean=weighting_fun == "average")
        ctx.cfg = (n2g, graph_ptr, num_heads, weighting_fun, lower, upper)
        ctx.save_for_backward(reprs, weights, out)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        reprs, weights, out = ctx.saved_tensors
        n2g, graph_ptr, num_heads, weighting_fun, lower, upper = ctx.cfg
        grad_out = grad_out.contiguous()
        grad_reprs = torch.empty_like(reprs)
        grad_scores = torch.empty_like(weights) if weights is not None else None
        _ffi.check(_ffi.lib().tfgnn_b200_readout_bwd(
            reprs.data_ptr(), _ptr(weights), n2g.data_ptr(), graph_ptr.data_ptr(), out.data_ptr(), grad_out.data_ptr(),
            int(reprs.shape[0]), int(out.shape[0]), int(reprs.shape[1]), num_heads, _ffi.READOUT_MODE[weighting_fun],
            float(lower or 0.0), float(upper or 0.0), 0 if lower is None else 1, 0 if upper is None else 1,
            grad_reprs.data_ptr(), _ptr(grad_scores), stream_ptr()))
        return grad_scores, grad_reprs, None, None, None, None, None, None


def readout(scores: Optional[torch.Tensor], reprs: torch.Tensor, n2g: torch.Tensor, graph_ptr: torch.Tensor, num_heads: int,
            weighting_fun: str, lower: Optional[float], upper: Optional[float]) -> torch.Tensor:
    return _ReadoutFunction.apply(scores, reprs, n2g, graph_ptr, int(num_heads), weighting_fun, lower, upper)


# ---- readout on a target-range shard -------------------------------------------------------------------------------
class _ShardReadoutFunction(torch.autograd.Function):
    """The readout of graphs whose rows may lie on several ranks.  Forward: tfgnn_b200_readout_partial over the rank's rows,
    an all-gather of the [G, 2K + GD] partials, tfgnn_b200_readout_merge in rank order: every rank gets the same [G, GD]
    bits.  Backward: the gradient arriving at the graph rows on each rank is that rank's part (e.g. the segment sum over its
    own rows of what it broadcast to them); the parts are all-gathered and added in rank order, and tfgnn_b200_readout_bwd
    runs on the rank's rows with the full-graph gradient, the merged result and, for softmax, the weights from the global
    normaliser."""

    @staticmethod
    def forward(ctx, scores, reprs, n2g, graph_ptr, num_graphs, num_heads, weighting_fun, lower, upper, shard):
        from .. import sharding
        mode = _ffi.READOUT_MODE[weighting_fun]
        reprs = reprs.contiguous()
        clamped = reprs if lower is None and upper is None else node_ops.clamp_(reprs.clone(), lower, upper)
        weights = None
        if weighting_fun in ("softmax", "sigmoid"):
            scores = scores.contiguous()
        if weighting_fun == "sigmoid":
            weights = node_ops.sigmoid(scores)
        G, GD, V = int(num_graphs), int(reprs.shape[1]), int(reprs.shape[0])
        K = 1 if weighting_fun == "none" else int(num_heads)
        partial = torch.empty((G, 2 * K + GD), dtype=torch.float32, device=reprs.device)
        w_in = scores if weighting_fun == "softmax" else weights
        _ffi.check(_ffi.lib().tfgnn_b200_readout_partial(_ptr(w_in), clamped.data_ptr(), n2g.data_ptr(),
                                                         graph_ptr.data_ptr(), V, G, GD, int(num_heads), mode,
                                                         partial.data_ptr(), stream_ptr()))
        parts = sharding.all_gather_stacked(partial, shard.group)
        out = torch.empty((G, GD), dtype=torch.float32, device=reprs.device)
        gmax = gsum = None
        if weighting_fun == "softmax":
            gmax = torch.empty((G, K), dtype=torch.float32, device=reprs.device)
            gsum = torch.empty_like(gmax)
        _ffi.check(_ffi.lib().tfgnn_b200_readout_merge(parts.data_ptr(), int(parts.shape[0]), G, GD, int(num_heads), mode,
                                                       out.data_ptr(), _ptr(gmax), _ptr(gsum), stream_ptr()))
        ctx.cfg = (n2g, graph_ptr, int(num_heads), weighting_fun, lower, upper, shard)
        ctx.save_for_backward(reprs, scores if weighting_fun == "softmax" else weights, out, gmax, gsum)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        from .. import sharding
        reprs, w_saved, out, gmax, gsum = ctx.saved_tensors
        n2g, graph_ptr, num_heads, weighting_fun, lower, upper, shard = ctx.cfg
        grad_full = sharding.sum_over_ranks(grad_out.contiguous(), shard.group)
        V = int(reprs.shape[0])
        weights = w_saved
        if weighting_fun == "softmax":                    # exp(score - max_g) / sum_g with the merged normaliser
            weights = torch.empty_like(w_saved)
            m_rows, s_rows = node_ops.gather_rows(gmax, n2g), node_ops.gather_rows(gsum, n2g)
            _ffi.check(_ffi.lib().tfgnn_b200_softmax_apply(w_saved.data_ptr(), m_rows.data_ptr(), s_rows.data_ptr(),
                                                           weights.numel(), weights.data_ptr(), stream_ptr()))
        grad_reprs = torch.empty_like(reprs)
        grad_scores = torch.empty_like(weights) if weights is not None else None
        _ffi.check(_ffi.lib().tfgnn_b200_readout_bwd(
            reprs.data_ptr(), _ptr(weights), n2g.data_ptr(), graph_ptr.data_ptr(), out.data_ptr(), grad_full.data_ptr(),
            V, int(out.shape[0]), int(reprs.shape[1]), num_heads, _ffi.READOUT_MODE[weighting_fun],
            float(lower or 0.0), float(upper or 0.0), 0 if lower is None else 1, 0 if upper is None else 1,
            grad_reprs.data_ptr(), _ptr(grad_scores), stream_ptr()))
        return grad_scores, grad_reprs, None, None, None, None, None, None, None, None


def shard_readout(scores: Optional[torch.Tensor], reprs: torch.Tensor, n2g: torch.Tensor, graph_ptr: torch.Tensor,
                  num_graphs: int, num_heads: int, weighting_fun: str, lower: Optional[float], upper: Optional[float],
                  shard) -> torch.Tensor:
    """The readout of the rank's rows (n2g, graph_ptr: those rows, global graph ids) merged over the ranks of `shard`:
    [num_graphs, GD], the same bits on every rank.  Collective: every rank calls it, forward and backward."""
    if weighting_fun == "average":
        raise NotImplementedError("average weighting is not built for target-range shards")
    return _ShardReadoutFunction.apply(scores, reprs, n2g, graph_ptr, int(num_graphs), int(num_heads), weighting_fun, lower,
                                       upper, shard)


# ---- per-node copies (only where a per-node dropout mask needs them) ----------------------------------------------
class _GatherGraphRowsFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, n2g, graph_ptr):
        ctx.index = (n2g, graph_ptr)
        return node_ops.gather_rows(table.contiguous(), n2g)

    @staticmethod
    def backward(ctx, grad_out):
        return segment_sum_rows(grad_out, *ctx.index), None, None


def gather_graph_rows(table: torch.Tensor, n2g: torch.Tensor, graph_ptr: torch.Tensor) -> torch.Tensor:
    """table[node_to_graph_map] (graph_global_exchange.py:94-96)."""
    if node_ops._needs_grad(table):
        return _GatherGraphRowsFunction.apply(table, n2g, graph_ptr)
    return node_ops.gather_rows(table.contiguous(), n2g)


# ---- exchange combines on (x [V, H], per-graph rows [G, .], node_to_graph_map) -------------------------------------
class _GatheredAddFunction(torch.autograd.Function):
    """act((a[v] + b[n2g[v]]) * scale); b is never expanded to [V, H]."""

    @staticmethod
    def forward(ctx, a, b, n2g, graph_ptr, scale, activation):
        out = node_ops.gathered_add(a, b.contiguous(), n2g, scale, activation)
        ctx.cfg = (n2g, graph_ptr, scale, activation)
        ctx.save_for_backward(out)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (out,) = ctx.saved_tensors
        n2g, graph_ptr, scale, activation = ctx.cfg
        grad_pre = grad_out.contiguous()
        if activation is not None:
            grad_act = torch.empty_like(grad_pre)
            _ffi.check(_ffi.lib().tfgnn_b200_activation_bwd(out.data_ptr(), grad_pre.data_ptr(), grad_pre.numel(),
                                                            activation.code, grad_act.data_ptr(), stream_ptr()))
            grad_pre = grad_act
        if scale != 1.0:
            grad_pre = node_ops._axpby(grad_pre, scale, None, 0.0)
        return grad_pre, segment_sum_rows(grad_pre, n2g, graph_ptr), None, None, None, None


def gathered_add(a: torch.Tensor, b: torch.Tensor, n2g: torch.Tensor, graph_ptr: torch.Tensor, scale: float = 1.0,
                 activation=None) -> torch.Tensor:
    if activation is not None and activation.name == "gelu":
        raise NotImplementedError("gathered_add backward: gelu needs the pre-activation, which the forward does not keep")
    return _GatheredAddFunction.apply(a.contiguous(), b, n2g, graph_ptr, float(scale), activation)


class _GruGateIndexedFunction(torch.autograd.Function):
    """Keras GRUCell(reset_after=True) gate math with gx = graph_repr K + b0 per GRAPH, gh = h U + b1 per node."""

    @staticmethod
    def forward(ctx, gx, gh, h, n2g, graph_ptr):
        gx, gh, h = gx.contiguous(), gh.contiguous(), h.contiguous()
        out = node_ops.gru_gate_fwd(gx, n2g, gh, h)
        ctx.index = (n2g, graph_ptr)
        ctx.save_for_backward(gx, gh, h)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        gx, gh, h = ctx.saved_tensors
        n2g, graph_ptr = ctx.index
        grad_out = grad_out.contiguous()
        dgx, dgh, dh = torch.empty_like(gx), torch.empty_like(gh), torch.empty_like(h)
        _ffi.check(_ffi.lib().tfgnn_b200_gru_gate_bwd_indexed(
            gx.data_ptr(), n2g.data_ptr(), graph_ptr.data_ptr(), gh.data_ptr(), h.data_ptr(), grad_out.data_ptr(),
            int(h.shape[0]), int(gx.shape[0]), int(h.shape[1]), dgx.data_ptr(), dgh.data_ptr(), dh.data_ptr(), stream_ptr()))
        return dgx, dgh, dh, None, None


def gru_cell(graph_reprs: torch.Tensor, n2g: torch.Tensor, graph_ptr: torch.Tensor, state: torch.Tensor, kernel, recurrent_kernel,
             bias) -> torch.Tensor:
    """GRUCell(inputs=graph_reprs[node_to_graph_map], states=[state]): both input-side GEMMs (forward, and grad of the
    kernel / of graph_reprs in the backward) have G rows."""
    gx, gh = node_ops.gru_gate_inputs(graph_reprs, state, kernel, recurrent_kernel, bias)
    return _GruGateIndexedFunction.apply(gx, gh, state, n2g, graph_ptr)
