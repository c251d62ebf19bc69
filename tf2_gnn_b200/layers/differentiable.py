"""Differentiable generic message passing (SURVEY.md §8f-1).

The reference trains EVERY variant by letting tf.GradientTape differentiate its literal op sequence
(message_passing.py:95-218: gather -> _message_function -> concat -> optional activation -> unsorted_segment_* ->
activation).  The fused forward kernels reorder that sequence; RGCN-style layers, GGNN, GNN-FiLM without hidden layers, and
GNN_Edge_MLP / RGIN (with or without its aggregation MLP) with at most one hidden layer in the edge MLPs have fused backward
kernels (csrc/backward.cu).  Without a hidden layer in the edge MLPs, max aggregation and activation before aggregation have
them too (the transform-then-aggregate form, up to hidden_dim 512).  RGAT has one (tfgnn_b200_rgat_bwd) when D and the
per-head width are multiples of 4 and hidden_dim <= 512.  Every other configuration of the Edge-MLP family — two
or more hidden layers in the edge MLPs, one hidden layer combined with max aggregation or activation before aggregation,
hidden layers in GNN-FiLM's MLPs, GNN-FiLM with max aggregation or activation before aggregation, D or H not a multiple of
4 — and RGAT outside those shapes train through THIS module: the
reference's own op order, each op a C-ABI kernel with a C-ABI backward (gather_rows <-> unsorted_segment_sum are each
other's adjoint).  It materialises [E, D] tensors exactly like the reference does; it is the correctness path for
training, not the fast path for inference (inference never comes here).

torch is used as the autograd tape and for data movement (cat / slicing) only.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from .. import _ffi
from ..runtime import PreparedBatch, stream_ptr
from . import node_ops


def _f32(shape, like):
    return torch.empty(shape, dtype=torch.float32, device=like.device)


# ---- gather / segment reduce (adjoint pair) ---------------------------------------------------------------------
class _GatherFunction(torch.autograd.Function):
    """table[ids] — tf.nn.embedding_lookup (message_passing.py:197-206) and tf.gather (graph_global_exchange.py:94-96):
    backward = segment sum."""

    @staticmethod
    def forward(ctx, table, ids, column):
        ctx.ids, ctx.column, ctx.n = ids, column, int(table.shape[0])
        return node_ops.gather_rows(table.contiguous(), ids, column)

    @staticmethod
    def backward(ctx, g):
        return node_ops.segment_sum(g.contiguous(), ctx.ids, ctx.n, ctx.column), None, None


def gather(table: torch.Tensor, adj: torch.Tensor, column: int) -> torch.Tensor:
    """table[adj[:, column]]."""
    if node_ops._needs_grad(table):
        return _GatherFunction.apply(table, adj, column)
    return node_ops.gather_rows(table.contiguous(), adj, column)


class _SegmentReduceFunction(torch.autograd.Function):
    """tf.math.unsorted_segment_{sum,mean,sqrt_n,max} (message_passing.py:172-174) keyed by a 1-D int32 id tensor."""

    @staticmethod
    def forward(ctx, data, ids, num_segments, agg):
        data = data.contiguous()
        M, H = int(data.shape[0]), int(data.shape[1])
        out = _f32((num_segments, H), data)
        _ffi.check(_ffi.lib().tfgnn_b200_unsorted_segment_reduce(data.data_ptr(), ids.data_ptr(), 1, M, H, num_segments,
                                                                 _ffi.AGG[agg], out.data_ptr(), stream_ptr()))
        ctx.ids, ctx.agg, ctx.num_segments = ids, agg, num_segments
        ctx.save_for_backward(data, out)
        return out

    @staticmethod
    def backward(ctx, g):
        data, out = ctx.saved_tensors
        g = g.contiguous()
        M, H = int(data.shape[0]), int(data.shape[1])
        lib = _ffi.lib()
        if M == 0:
            return _f32((M, H), data), None, None, None
        if ctx.agg == "max":
            grad = _f32((M, H), data)
            _ffi.check(lib.tfgnn_b200_segment_max_bwd(data.data_ptr(), ctx.ids.data_ptr(), 1, out.data_ptr(), g.data_ptr(), M, H,
                                                      ctx.num_segments, grad.data_ptr(), stream_ptr()))
            return grad, None, None, None
        grad = node_ops.gather_rows(g, ctx.ids)
        if ctx.agg in ("mean", "sqrt_n"):
            ones = torch.ones((M, 1), dtype=torch.float32, device=data.device)
            per_msg = node_ops.gather_rows(node_ops.segment_sum(ones, ctx.ids, ctx.num_segments), ctx.ids)
            scaled = _f32((M, H), data)
            _ffi.check(lib.tfgnn_b200_row_scale(grad.data_ptr(), per_msg.data_ptr(), M, H, 2 if ctx.agg == "mean" else 3,
                                                scaled.data_ptr(), stream_ptr()))
            grad = scaled
        return grad, None, None, None


# ---- elementwise ------------------------------------------------------------------------------------------------
class _ActivationFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, code):
        x = x.contiguous()
        out = torch.empty_like(x)
        _ffi.check(_ffi.lib().tfgnn_b200_activation(x.data_ptr(), x.numel(), code, out.data_ptr(), stream_ptr()))
        ctx.code = code
        ctx.save_for_backward(x if code == _ffi.ACT["gelu"] else out)
        return out

    @staticmethod
    def backward(ctx, g):
        (ref,) = ctx.saved_tensors
        g = g.contiguous()
        out = torch.empty_like(g)
        _ffi.check(_ffi.lib().tfgnn_b200_activation_bwd(ref.data_ptr(), g.data_ptr(), g.numel(), ctx.code, out.data_ptr(),
                                                        stream_ptr()))
        return out, None


def activation(x: torch.Tensor, act) -> torch.Tensor:
    if act is None:
        return x
    if node_ops._needs_grad(x):
        return _ActivationFunction.apply(x, act.code)
    return act(x)


class _RowScaleFunction(torch.autograd.Function):
    """messages * 1/(n + 1e-7) (gnn_edge_mlp.py:102-106); the scale carries no gradient (it is a count)."""

    @staticmethod
    def forward(ctx, x, s, mode):
        x = x.contiguous()
        out = torch.empty_like(x)
        if x.shape[0]:
            _ffi.check(_ffi.lib().tfgnn_b200_row_scale(x.data_ptr(), s.data_ptr(), int(x.shape[0]), int(x.shape[1]), mode,
                                                       out.data_ptr(), stream_ptr()))
        ctx.s, ctx.mode = s, mode
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        out = torch.empty_like(g)
        if g.shape[0]:
            _ffi.check(_ffi.lib().tfgnn_b200_row_scale(g.data_ptr(), ctx.s.data_ptr(), int(g.shape[0]), int(g.shape[1]),
                                                       ctx.mode, out.data_ptr(), stream_ptr()))
        return out, None, None


def _mul_add(a, lda, b, ldb, c, ldc, M, H, out, ldo):
    if M:
        _ffi.check(_ffi.lib().tfgnn_b200_mul_add(a, lda, b, ldb, c, ldc, M, H, out, ldo, stream_ptr()))


class _FilmFunction(torch.autograd.Function):
    """film[:, :H] * messages + film[:, H:] (gnn_film.py:103-107)."""

    @staticmethod
    def forward(ctx, film, messages):
        film, messages = film.contiguous(), messages.contiguous()
        E, H = int(messages.shape[0]), int(messages.shape[1])
        out = torch.empty_like(messages)
        _mul_add(film.data_ptr(), 2 * H, messages.data_ptr(), H, film.data_ptr() + 4 * H, 2 * H, E, H, out.data_ptr(), H)
        ctx.save_for_backward(film, messages)
        return out

    @staticmethod
    def backward(ctx, g):
        film, messages = ctx.saved_tensors
        g = g.contiguous()
        E, H = int(messages.shape[0]), int(messages.shape[1])
        g_film = torch.empty_like(film)
        g_msg = torch.empty_like(messages)
        _mul_add(g.data_ptr(), H, messages.data_ptr(), H, 0, 0, E, H, g_film.data_ptr(), 2 * H)       # d/dgamma = g * m
        if E:
            g_film[:, H:] = g                                                                      # d/dbeta  = g (copy)
        _mul_add(g.data_ptr(), H, film.data_ptr(), 2 * H, 0, 0, E, H, g_msg.data_ptr(), H)           # d/dm     = g * gamma
        return g_film, g_msg


# ---- the literal layer ------------------------------------------------------------------------------------------
def _mlp(x: torch.Tensor, kernels: Sequence[torch.Tensor]) -> torch.Tensor:
    """dpu_utils MLP of the message functions: bias-free, ReLU hidden layers, linear output."""
    from ..utils.param_helpers import get_activation_function
    relu = get_activation_function("relu")
    cur = x
    for i, W in enumerate(kernels):
        cur = node_ops.dense(cur, W, None, relu if i < len(kernels) - 1 else None)
    return cur


def edge_mlp_family_forward(layer, h: torch.Tensor, prepared: PreparedBatch, *, film_kernels: Optional[List] = None,
                            aggr_kernels: Optional[List[torch.Tensor]] = None, final_activation: bool = True,
                            activation_before: Optional[bool] = None) -> torch.Tensor:
    """message_passing.py:95-218 with GNN_Edge_MLP._message_function (gnn_edge_mlp.py:84-107), optionally GNN_FiLM's
    modulation (gnn_film.py:83-108) and RGIN's aggregation MLP (rgin.py:88-106), in the reference's op order."""
    if prepared.target_range != (0, prepared.num_source_nodes):
        raise NotImplementedError("training through a target-range shard is not built")
    V = int(h.shape[0])
    in_degree = prepared.in_degree()                                   # [L, V] (message_passing.py:190)
    messages_per_type, targets = [], []
    for l, adj in enumerate(prepared.adjacency_lists):
        E = int(adj.shape[0])
        src = gather(h, adj, 0)                                         # :197-200
        tgt = gather(h, adj, 1) if (layer._use_target_state_as_input or film_kernels is not None) else None   # :201-204
        x = torch.cat([src, tgt], dim=1) if layer._use_target_state_as_input else src
        m = _mlp(x, [v.value for v in layer._edge_type_mlps[l].layers])  # gnn_edge_mlp.py:100
        if layer._normalize_by_num_incoming:                            # :102-106
            n_in = node_ops.gather_rows(in_degree[l].reshape(V, 1).contiguous(), adj, 1)
            m = _RowScaleFunction.apply(m, n_in, 1)
        if film_kernels is not None:                                    # gnn_film.py:99-107
            film = _mlp(tgt, film_kernels[l])
            m = _FilmFunction.apply(film, m)
        messages_per_type.append(m)
        targets.append(adj[:, 1])
    H = layer._hidden_dim
    if messages_per_type:
        messages = torch.cat(messages_per_type, dim=0)                  # message_passing.py:166-167
        ids = torch.cat([t.reshape(-1) for t in targets], dim=0).contiguous()
    else:
        messages = torch.zeros((0, H), dtype=torch.float32, device=h.device)
        ids = torch.zeros((0,), dtype=torch.int32, device=h.device)
    before = layer._message_activation_before_aggregation if activation_before is None else activation_before
    if before:
        messages = activation(messages, layer._activation_fn)           # :169-170
    agg = _SegmentReduceFunction.apply(messages, ids, V, layer._aggregation_fn.name)   # :172-174
    if aggr_kernels is not None:
        agg = _mlp(agg, aggr_kernels)                                   # rgin.py:103-104
    if final_activation and not before:
        agg = activation(agg, layer._activation_fn)                     # :176-177
    return agg



# ==================================================================================================================
# Attention / graph-level pieces: RGAT (rgat.py:91-163), readout (nodes_to_graph_representation.py:170-229) and
# global exchange (graph_global_exchange.py:83-183) in the reference's op order, every op with its adjoint kernel.
# ==================================================================================================================
class _AddFunction(torch.autograd.Function):
    """alpha * a + beta * b."""

    @staticmethod
    def forward(ctx, a, b, alpha, beta):
        ctx.ab = (alpha, beta)
        return node_ops._axpby(a.contiguous(), alpha, b.contiguous(), beta)

    @staticmethod
    def backward(ctx, g):
        alpha, beta = ctx.ab
        g = g.contiguous()
        return node_ops._axpby(g, alpha, None, 0.0), node_ops._axpby(g, beta, None, 0.0), None, None


def _head_scale(x, w, K):
    out = torch.empty_like(x)
    if x.shape[0]:
        _ffi.check(_ffi.lib().tfgnn_b200_head_scale(x.data_ptr(), w.data_ptr(), int(x.shape[0]), K, int(x.shape[1]) // K,
                                                    out.data_ptr(), stream_ptr()))
    return out


class _HeadScaleFunction(torch.autograd.Function):
    """weights[:, k, None] * x[:, k, :] per head (rgat.py:152-155; nodes_to_graph_representation.py:219-220)."""

    @staticmethod
    def forward(ctx, x, w):
        x, w = x.contiguous(), w.contiguous()
        ctx.K = int(w.shape[1])
        ctx.save_for_backward(x, w)
        return _head_scale(x, w, ctx.K)

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        g = g.contiguous()
        gx = _head_scale(g, w, ctx.K)
        gw = torch.empty_like(w)
        if x.shape[0]:
            _ffi.check(_ffi.lib().tfgnn_b200_head_dot(g.data_ptr(), x.data_ptr(), int(x.shape[0]), ctx.K,
                                                      int(x.shape[1]) // ctx.K, gw.data_ptr(), stream_ptr()))
        return gx, gw


class _SegmentSoftmaxFunction(torch.autograd.Function):
    """exp(unsorted_segment_log_softmax(scores[:, k], ids, n)) for every head k at once (rgat.py:147-151;
    dpu_utils unsorted_segment_softmax, nodes_to_graph_representation.py:179-185).
    backward: d_score = alpha * (d_alpha - segment_sum(alpha * d_alpha)[ids])."""

    @staticmethod
    def forward(ctx, scores, ids, num_segments):
        scores = scores.contiguous()
        M, K = int(scores.shape[0]), int(scores.shape[1])
        lib = _ffi.lib()
        alpha = torch.empty_like(scores)
        if M:
            seg_max = _f32((num_segments, K), scores)
            _ffi.check(lib.tfgnn_b200_unsorted_segment_reduce(scores.data_ptr(), ids.data_ptr(), 1, M, K, num_segments,
                                                              _ffi.AGG["max"], seg_max.data_ptr(), stream_ptr()))
            m_e = node_ops.gather_rows(seg_max, ids)
            e = torch.empty_like(scores)
            _ffi.check(lib.tfgnn_b200_softmax_apply(scores.data_ptr(), m_e.data_ptr(), None, M * K, e.data_ptr(), stream_ptr()))
            z_e = node_ops.gather_rows(node_ops.segment_sum(e, ids, num_segments), ids)
            _ffi.check(lib.tfgnn_b200_softmax_apply(scores.data_ptr(), m_e.data_ptr(), z_e.data_ptr(), M * K, alpha.data_ptr(),
                                                    stream_ptr()))
        ctx.ids, ctx.n = ids, num_segments
        ctx.save_for_backward(alpha)
        return alpha

    @staticmethod
    def backward(ctx, g):
        (alpha,) = ctx.saved_tensors
        g = g.contiguous()
        M, K = int(alpha.shape[0]), int(alpha.shape[1])
        out = torch.empty_like(alpha)
        if M:
            t = torch.empty_like(alpha)
            _mul_add(alpha.data_ptr(), K, g.data_ptr(), K, 0, 0, M, K, t.data_ptr(), K)                 # alpha * d_alpha
            s_e = node_ops.gather_rows(node_ops.segment_sum(t, ctx.ids, ctx.n), ctx.ids)
            u = torch.empty_like(alpha)
            _mul_add(alpha.data_ptr(), K, s_e.data_ptr(), K, 0, 0, M, K, u.data_ptr(), K)               # alpha * sum
            out = node_ops._axpby(t, 1.0, u, -1.0)
        return out, None, None


def _attention_matrices(a: torch.Tensor, K: int, d: int):
    """The einsum "vki,ki->vk" of rgat.py:115-121 as two dense products: scores = P_src A_src + P_tgt A_tgt with the block
    matrices A_src[k*d+i, k] = a[k, i], A_tgt[k*d+i, k] = a[k, d+i] (slice copies only: autograd routes the gradient back to a)."""
    H = K * d
    a_src = torch.zeros((H, K), dtype=torch.float32, device=a.device)
    a_tgt = torch.zeros((H, K), dtype=torch.float32, device=a.device)
    for k in range(K):
        a_src[k * d:(k + 1) * d, k] = a[k, :d]
        a_tgt[k * d:(k + 1) * d, k] = a[k, d:]
    return a_src, a_tgt


def rgat_forward(layer, h: torch.Tensor, prepared: PreparedBatch) -> torch.Tensor:
    """RGAT._message_function + _compute_new_node_embeddings (rgat.py:91-163) in the reference's op order."""
    from ..utils.param_helpers import get_activation_function
    if prepared.target_range != (0, prepared.num_source_nodes):
        raise NotImplementedError("training through a target-range shard is not built")
    V, H, K = int(h.shape[0]), layer._hidden_dim, int(layer._num_heads)
    d = H // K
    leaky = get_activation_function("leaky_relu")
    msgs, scores, targets = [], [], []
    for l, adj in enumerate(prepared.adjacency_lists):
        W = layer._edge_type_to_message_computation_layer[l].value
        a = layer._edge_type_to_attention_parameters[l].value
        P = node_ops.dense(h, W)                                        # Dense applied to every node once: rows are identical
        ps = gather(P, adj, 0)                                          # :102-105
        pt = gather(P, adj, 1)                                          # :106-109
        a_src, a_tgt = _attention_matrices(a, K, d)
        sc = _AddFunction.apply(node_ops.dense(ps, a_src), node_ops.dense(pt, a_tgt), 1.0, 1.0)   # :111-121
        scores.append(activation(sc, leaky))
        msgs.append(ps)
        targets.append(adj[:, 1])
    if msgs:
        M = torch.cat(msgs, dim=0)
        S = torch.cat(scores, dim=0)
        ids = torch.cat([t.reshape(-1) for t in targets], dim=0).contiguous()
    else:
        M = torch.zeros((0, H), dtype=torch.float32, device=h.device)
        S = torch.zeros((0, K), dtype=torch.float32, device=h.device)
        ids = torch.zeros((0,), dtype=torch.int32, device=h.device)
    alpha = _SegmentSoftmaxFunction.apply(S, ids, V)                    # :141-151 (all heads)
    weighted = _HeadScaleFunction.apply(M, alpha)                       # :152-155
    out = _SegmentReduceFunction.apply(weighted, ids, V, "sum")         # :156-160
    return activation(out, layer._activation_fn)                        # :162-163


class _GruGateFunction(torch.autograd.Function):
    """Keras GRUCell(reset_after=True) gate math on gx = inputs K + b0, gh = h U + b1."""

    @staticmethod
    def forward(ctx, gx, gh, h):
        gx, gh, h = gx.contiguous(), gh.contiguous(), h.contiguous()
        out = node_ops.gru_gate_fwd(gx, None, gh, h)
        ctx.save_for_backward(gx, gh, h)
        return out

    @staticmethod
    def backward(ctx, g):
        gx, gh, h = ctx.saved_tensors
        g = g.contiguous()
        dgx, dgh, dh = torch.empty_like(gx), torch.empty_like(gh), torch.empty_like(h)
        _ffi.check(_ffi.lib().tfgnn_b200_gru_gate_bwd(gx.data_ptr(), gh.data_ptr(), h.data_ptr(), g.data_ptr(), int(h.shape[0]),
                                                      int(h.shape[1]), dgx.data_ptr(), dgh.data_ptr(), dh.data_ptr(),
                                                      stream_ptr()))
        return dgx, dgh, dh


def gru_cell(inputs: torch.Tensor, state: torch.Tensor, kernel, recurrent_kernel, bias) -> torch.Tensor:
    """tf.keras.layers.GRUCell (TF2 defaults), differentiable: the direct path of the state through z * h is added to the
    recurrent path by the autograd tape."""
    gx, gh = node_ops.gru_gate_inputs(inputs, state, kernel, recurrent_kernel, bias)
    return _GruGateFunction.apply(gx, gh, state)


def weighted_sum_graph_representation(rep, x: torch.Tensor, n2g: torch.Tensor, num_graphs: int, training: bool) -> torch.Tensor:
    """WeightedSumGraphRepresentation.call (nodes_to_graph_representation.py:170-229), differentiable."""
    from .. import _ffi as ffi
    weights = None
    if rep._weighting_fun not in ("none", "average"):
        scores = rep._scoring_mlp(x, training, rep.dropout_state)
        if rep._weighting_fun == "sigmoid":
            weights = _ActivationFunction.apply(scores, ffi.ACT_SIGMOID)
        else:
            weights = _SegmentSoftmaxFunction.apply(scores, n2g, num_graphs)
    reprs = rep._transformation_mlp(x, training, rep.dropout_state)
    if rep._transformation_mlp_activation_fun is not None:
        reprs = activation(reprs, rep._transformation_mlp_activation_fun)
    if rep._transformation_mlp_result_lower_bound is not None or rep._transformation_mlp_result_upper_bound is not None:
        raise NotImplementedError("training with clipped transformation results is not built")
    if weights is not None:
        reprs = _HeadScaleFunction.apply(reprs, weights)
        return _SegmentReduceFunction.apply(reprs, n2g, num_graphs, "sum")
    return _SegmentReduceFunction.apply(reprs, n2g, num_graphs, "mean" if rep._weighting_fun == "average" else "sum")


def per_node_graph_representations(exchange, x: torch.Tensor, n2g: torch.Tensor, num_graphs: int, training: bool):
    """GraphGlobalExchange._compute_per_node_graph_representations (graph_global_exchange.py:83-103), differentiable."""
    rep = exchange._node_to_graph_representation_layer
    rep.dropout_state = exchange.dropout_state
    g = weighted_sum_graph_representation(rep, x, n2g, num_graphs, training)
    per_node = _GatherFunction.apply(g, n2g, 0)
    if training and exchange._dropout_rate > 0.0:
        per_node = node_ops.dropout(per_node, exchange._dropout_rate, exchange.dropout_state)
    return per_node
