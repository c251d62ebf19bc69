"""Node-level and graph-level ops of GNN._internal_call (gnn.py:279-327) on the library's kernels, each with
the gradient the reference obtains from tf.GradientTape (models/graph_task_model.py:338-365).

Every function takes and returns CUDA float32 tensors; when autograd is recording and an input requires grad the
op runs through a torch.autograd.Function whose backward is again a C-ABI call — no torch arithmetic on the path.
Ops whose backward is not built (the graph readout / exchange family) raise under autograd instead of silently
cutting the gradient (ADVICE r1: "training through the GNN stack silently truncates gradients").
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from .. import _ffi
from ..runtime import stream_ptr


def _needs_grad(*tensors) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def require_no_grad(what: str, *tensors) -> None:
    if _needs_grad(*tensors):
        raise NotImplementedError(
            f"{what}: the backward pass of this op is not built; run it under torch.no_grad() or detach its inputs "
            "(it never silently drops a gradient)")


# ---- Dense ------------------------------------------------------------------------------------------------------
def _dense_fwd(x, W, bias, act_code):
    V, K = int(x.shape[0]), int(x.shape[1])
    N = int(W.shape[1])
    out = torch.empty((V, N), dtype=torch.float32, device=x.device)
    if bias is None:
        _ffi.check(_ffi.lib().tfgnn_b200_dense_fwd(x.data_ptr(), W.data_ptr(), out.data_ptr(), V, K, N, act_code, 0,
                                                   stream_ptr()))
    else:
        _ffi.check(_ffi.lib().tfgnn_b200_dense_bias_fwd(x.data_ptr(), W.data_ptr(), bias.data_ptr(), out.data_ptr(), V, K,
                                                        N, act_code, 0, stream_ptr()))
    return out


class _DenseFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, W, bias, act_code):
        out = _dense_fwd(x, W, bias, act_code)
        ctx.act_code = act_code
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x, W, bias if bias is not None else W.new_empty(0), out)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x, W, bias, out = ctx.saved_tensors
        bias = bias if ctx.has_bias else None
        grad_out = grad_out.contiguous()
        V, K, N = int(x.shape[0]), int(x.shape[1]), int(W.shape[1])
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gW = torch.empty_like(W) if ctx.needs_input_grad[1] else None
        gb = torch.empty_like(bias) if (bias is not None and ctx.needs_input_grad[2]) else None
        _ffi.check(_ffi.lib().tfgnn_b200_dense_bwd(
            x.data_ptr(), W.data_ptr(), _ptr(bias), out.data_ptr(), grad_out.data_ptr(), V, K, N, ctx.act_code,
            _ptr(gx), _ptr(gW), _ptr(gb), stream_ptr()))
        return gx, gW, gb, None


def dense(x: torch.Tensor, W: torch.Tensor, bias: Optional[torch.Tensor] = None, activation=None) -> torch.Tensor:
    """tf.keras.layers.Dense(units, use_bias=bias is not None, activation=activation)."""
    code = activation.code if activation is not None else 0
    x = x.contiguous()
    if _needs_grad(x, W, bias):
        return _DenseFunction.apply(x, W, bias, code)
    return _dense_fwd(x, W, bias, code)


def mlp(x: torch.Tensor, kernels, biases=None, hidden_activation=None, training: bool = False, dropout_rate: float = 0.0,
        rng: Optional["DropoutState"] = None, rows=None) -> torch.Tensor:
    """dpu_utils.tf2utils.MLP: hidden Dense layers with `hidden_activation` (ReLU by default), linear output layer;
    under training, dropout on the input of every layer (`rows`: see dropout)."""
    from ..utils.param_helpers import get_activation_function
    act = hidden_activation or get_activation_function("relu")
    cur = x
    n = len(kernels)
    for i, W in enumerate(kernels):
        if training and dropout_rate > 0.0:
            cur = dropout(cur, dropout_rate, rng, rows)
        b = biases[i] if biases is not None else None
        cur = dense(cur, W, b, act if i < n - 1 else None)
    return cur


# ---- LayerNormalization -----------------------------------------------------------------------------------------
def _ln_fwd(x, gamma, beta, eps):
    out = torch.empty_like(x)
    _ffi.check(_ffi.lib().tfgnn_b200_layer_norm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), int(x.shape[0]),
                                                int(x.shape[1]), eps, out.data_ptr(), stream_ptr()))
    return out


class _LayerNormFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        ctx.eps = eps
        ctx.save_for_backward(x, gamma)
        return _ln_fwd(x, gamma, beta, eps)

    @staticmethod
    def backward(ctx, grad_out):
        x, gamma = ctx.saved_tensors
        grad_out = grad_out.contiguous()
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gg, gb = torch.empty_like(gamma), torch.empty_like(gamma)
        _ffi.check(_ffi.lib().tfgnn_b200_layer_norm_bwd(x.data_ptr(), gamma.data_ptr(), grad_out.data_ptr(), int(x.shape[0]),
                                                        int(x.shape[1]), ctx.eps, _ptr(gx), gg.data_ptr(), gb.data_ptr(),
                                                        stream_ptr()))
        return gx, gg, gb, None


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, epsilon: float = 1e-3) -> torch.Tensor:
    x = x.contiguous()
    if _needs_grad(x, gamma, beta):
        return _LayerNormFunction.apply(x, gamma, beta, float(epsilon))
    return _ln_fwd(x, gamma, beta, float(epsilon))


# ---- residual average, scaling ----------------------------------------------------------------------------------
def _axpby(a, alpha, b, beta):
    out = torch.empty_like(a)
    _ffi.check(_ffi.lib().tfgnn_b200_axpby(a.data_ptr(), float(alpha), _ptr(b), float(beta), a.numel(), out.data_ptr(),
                                           stream_ptr()))
    return out


class _AverageFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, last):
        out = torch.empty_like(x)
        _ffi.check(_ffi.lib().tfgnn_b200_residual_average(x.data_ptr(), last.data_ptr(), out.data_ptr(), x.numel(),
                                                          stream_ptr()))
        return out

    @staticmethod
    def backward(ctx, grad_out):
        half = _axpby(grad_out.contiguous(), 0.5, None, 0.0)
        return half, half


def residual_average(x: torch.Tensor, last: torch.Tensor) -> torch.Tensor:
    """cur += last; cur /= 2 (gnn.py:294-295)."""
    x, last = x.contiguous(), last.contiguous()
    if _needs_grad(x, last):
        return _AverageFunction.apply(x, last)
    out = torch.empty_like(x)
    _ffi.check(_ffi.lib().tfgnn_b200_residual_average(x.data_ptr(), last.data_ptr(), out.data_ptr(), x.numel(),
                                                      stream_ptr()))
    return out


# ---- dropout ----------------------------------------------------------------------------------------------------
class DropoutState:
    """Seed + running offset of the Philox stream (one per model, like a tf.random.Generator): every dropout call
    consumes ceil(n / 4) counter values, so masks of successive calls are independent and a run is reproducible
    from its seed."""

    def __init__(self, seed: int = 0):
        self.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self.offset = 0

    def take(self, n: int) -> int:
        off = self.offset
        self.offset += (int(n) + 3) // 4
        return off


_default_dropout_state = DropoutState(0x5EED)


def _dropout_apply(x, rate, seed, offset, first=0):
    out = torch.empty_like(x)
    if first:
        _ffi.check(_ffi.lib().tfgnn_b200_dropout_at(x.data_ptr(), x.numel(), float(rate), seed, offset, first,
                                                    out.data_ptr(), stream_ptr()))
    else:
        _ffi.check(_ffi.lib().tfgnn_b200_dropout(x.data_ptr(), x.numel(), float(rate), seed, offset, out.data_ptr(),
                                                 stream_ptr()))
    return out


class _DropoutFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, rate, seed, offset, first):
        ctx.cfg = (rate, seed, offset, first)
        return _dropout_apply(x, rate, seed, offset, first)

    @staticmethod
    def backward(ctx, grad_out):
        rate, seed, offset, first = ctx.cfg
        return _dropout_apply(grad_out.contiguous(), rate, seed, offset, first), None, None, None, None


def dropout(x: torch.Tensor, rate: float, state: Optional[DropoutState] = None, rows=None) -> torch.Tensor:
    """tf.nn.dropout(x, rate) (gnn.py:285-289).  rate == 0 is the identity, as in TensorFlow.

    rows=(first_row, total_rows): x is rows [first_row, first_row + len(x)) of a [total_rows, C] table (a target-range
    shard, sharding.TargetRangeShard.rows).  The call then consumes the stream of the whole table and draws exactly the
    masks the unsharded call draws for those rows, so every rank of a sharded model stays in step with the unsharded run."""
    if rate <= 0.0:
        return x
    state = state or _default_dropout_state
    x = x.contiguous()
    first = 0
    if rows is None:
        offset = state.take(x.numel())
    else:
        cols = math.prod(int(n) for n in x.shape[1:])
        if not 0 <= int(rows[0]) <= int(rows[0]) + int(x.shape[0]) <= int(rows[1]):
            raise ValueError(f"dropout rows={tuple(rows)}: rows [{int(rows[0])}, {int(rows[0]) + int(x.shape[0])}) of x "
                             f"must lie inside a table of {int(rows[1])} rows")
        first = int(rows[0]) * cols
        offset = state.take(int(rows[1]) * cols)
    if _needs_grad(x):
        return _DropoutFunction.apply(x, float(rate), state.seed, offset, first)
    return _dropout_apply(x, float(rate), state.seed, offset, first)


# ---- gather / segment sum by int32 ids (forward only) -------------------------------------------------------------
def _id_column(ids: torch.Tensor, column: int):
    """(pointer, stride) of the ids: a contiguous int32 vector, or column `column` of a contiguous [E, 2] adjacency list."""
    return ids.data_ptr() + 4 * column, (2 if ids.dim() == 2 else 1)


def gather_rows(table: torch.Tensor, ids: torch.Tensor, column: int = 0) -> torch.Tensor:
    """table[ids] (ids as in _id_column)."""
    n, C = int(ids.shape[0]), int(table.shape[1])
    out = torch.empty((n, C), dtype=torch.float32, device=table.device)
    if n:
        _ffi.check(_ffi.lib().tfgnn_b200_gather_rows(table.data_ptr(), int(table.shape[0]), C, *_id_column(ids, column), n,
                                                     out.data_ptr(), stream_ptr()))
    return out


def segment_sum(data: torch.Tensor, ids: torch.Tensor, num_segments: int, column: int = 0) -> torch.Tensor:
    """tf.math.unsorted_segment_sum(data, ids, num_segments), the adjoint of gather_rows (ids as in _id_column)."""
    out = torch.empty((num_segments, int(data.shape[1])), dtype=torch.float32, device=data.device)
    _ffi.check(_ffi.lib().tfgnn_b200_unsorted_segment_reduce(data.data_ptr(), *_id_column(ids, column), int(data.shape[0]),
                                                             int(data.shape[1]), num_segments, _ffi.AGG["sum"],
                                                             out.data_ptr(), stream_ptr()))
    return out


# ---- graph-level primitives (forward only) ----------------------------------------------------------------------
def node_to_graph_index(node_to_graph_map, device: torch.device) -> torch.Tensor:
    """node_to_graph_map as a contiguous int32 tensor on `device`."""
    if not isinstance(node_to_graph_map, torch.Tensor):
        node_to_graph_map = torch.as_tensor(node_to_graph_map)
    return node_to_graph_map.to(device=device, dtype=torch.int32).contiguous()


def graph_offsets(node_to_graph_map: torch.Tensor, num_graphs: int, validate: bool = False) -> torch.Tensor:
    V = int(node_to_graph_map.shape[0])
    out = torch.empty(int(num_graphs) + 1, dtype=torch.int32, device=node_to_graph_map.device)
    _ffi.check(_ffi.lib().tfgnn_b200_graph_offsets(node_to_graph_map.data_ptr(), V, int(num_graphs), out.data_ptr(),
                                                   1 if validate else 0, stream_ptr()))
    return out


def segment_softmax(scores: torch.Tensor, graph_ptr: torch.Tensor) -> torch.Tensor:
    require_no_grad("segment_softmax", scores)
    scores = scores.contiguous()
    out = torch.empty_like(scores)
    _ffi.check(_ffi.lib().tfgnn_b200_segment_softmax(scores.data_ptr(), graph_ptr.data_ptr(), int(graph_ptr.shape[0]) - 1,
                                                     int(scores.shape[1]), out.data_ptr(), stream_ptr()))
    return out


def sigmoid(x: torch.Tensor) -> torch.Tensor:
    """tf.nn.sigmoid on the library's activation kernel."""
    out = torch.empty_like(x)
    _ffi.check(_ffi.lib().tfgnn_b200_activation(x.data_ptr(), x.numel(), _ffi.ACT_SIGMOID, out.data_ptr(), stream_ptr()))
    return out


def readout_weights(scores: Optional[torch.Tensor], graph_ptr: torch.Tensor, weighting_fun: str) -> Optional[torch.Tensor]:
    """The per-(node, head) weights of the graph readout (nodes_to_graph_representation.py:174-186): None for "none" and
    "average"."""
    if weighting_fun == "softmax":
        return segment_softmax(scores, graph_ptr)
    if weighting_fun == "sigmoid":
        return sigmoid(scores)
    return None


def weighted_segment_sum(node_reprs: torch.Tensor, weights: Optional[torch.Tensor], graph_ptr: torch.Tensor,
                         num_heads: int, mean: bool = False) -> torch.Tensor:
    require_no_grad("weighted_segment_sum", node_reprs, weights)
    node_reprs = node_reprs.contiguous()
    G, GD = int(graph_ptr.shape[0]) - 1, int(node_reprs.shape[1])
    out = torch.empty((G, GD), dtype=torch.float32, device=node_reprs.device)
    _ffi.check(_ffi.lib().tfgnn_b200_weighted_segment_sum(node_reprs.data_ptr(), _ptr(weights), graph_ptr.data_ptr(), G, GD,
                                                          int(num_heads), 1 if mean else 0, out.data_ptr(), stream_ptr()))
    return out


def gathered_add(a: torch.Tensor, b: torch.Tensor, index: Optional[torch.Tensor], scale: float = 1.0,
                 activation=None) -> torch.Tensor:
    """act((a[v] + b[index[v]]) * scale)."""
    require_no_grad("gathered_add", a, b)
    a = a.contiguous()
    out = torch.empty_like(a)
    _ffi.check(_ffi.lib().tfgnn_b200_gathered_add(a.data_ptr(), b.data_ptr(), _ptr(index), int(a.shape[0]), int(a.shape[1]),
                                                  float(scale), activation.code if activation is not None else 0,
                                                  out.data_ptr(), stream_ptr()))
    return out


def gru_gate_inputs(inputs: torch.Tensor, state: torch.Tensor, kernel: torch.Tensor, recurrent_kernel: torch.Tensor,
                    bias: torch.Tensor):
    """The two Dense halves of a Keras GRUCell(reset_after=True): gx = inputs K + b0, gh = state U + b1."""
    return dense(inputs, kernel, bias[0]), dense(state, recurrent_kernel, bias[1])


def gru_gate_fwd(gx: torch.Tensor, gx_row_index: Optional[torch.Tensor], gh: torch.Tensor,
                 state: torch.Tensor) -> torch.Tensor:
    """The GRUCell gate math on gx[gx_row_index[v]] (gx[v] without an index), gh[v] and state[v]."""
    out = torch.empty_like(state)
    _ffi.check(_ffi.lib().tfgnn_b200_gru_gate_fwd(gx.data_ptr(), _ptr(gx_row_index), gh.data_ptr(), state.data_ptr(),
                                                  int(state.shape[0]), int(state.shape[1]), out.data_ptr(), stream_ptr()))
    return out


def gru_cell(inputs: torch.Tensor, inputs_row_index: Optional[torch.Tensor], state: torch.Tensor, kernel: torch.Tensor,
             recurrent_kernel: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """tf.keras.layers.GRUCell(units=H) (TF2 defaults: reset_after=True, bias [2,3H], gates z|r|h) applied to
    inputs[inputs_row_index[v]] with state[v].  The input half (inputs K + b0) is computed once per row of `inputs`
    (e.g. once per GRAPH for the global exchange) and picked up per node inside the gate kernel."""
    require_no_grad("gru_cell", inputs, state, kernel, recurrent_kernel, bias)
    gx, gh = gru_gate_inputs(inputs, state, kernel, recurrent_kernel, bias)
    return gru_gate_fwd(gx, inputs_row_index, gh, state.contiguous())


def clamp_(x: torch.Tensor, lower: Optional[float], upper: Optional[float]) -> torch.Tensor:
    if lower is None and upper is None:
        return x
    _ffi.check(_ffi.lib().tfgnn_b200_clamp(x.data_ptr(), x.numel(), float(lower or 0.0), float(upper or 0.0),
                                           0 if lower is None else 1, 0 if upper is None else 1, stream_ptr()))
    return x
