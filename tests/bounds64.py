"""Element-wise float64 error bounds for float32 kernel results, and the one assertion that checks a result against them.

A kernel that evaluates sums of products in float32 (in any order, with fp32 FMAs or 3xTF32 tensor-core products) makes
an error in every output element that is at most a small multiple of u = 2^-24 times the SAME computation carried out on
absolute values: |h|, |W|, the positive normalisations, no cancellation.  So the bound of an element is that absolute
evaluation, and a kernel passes when |got - ref64| <= rel * bound for every element.  Unlike a criterion scaled by the
largest element of the tensor, this holds every row to its own scale: a hub row 100x larger than the rest, or one graph of
100 000 nodes next to graphs of one node, no longer hides a defect in the ordinary rows.

Activations.  The bound is taken on the pre-activation; an activation with Lipschitz constant Lip moves it by at most that
factor (relu, leaky_relu, tanh, elu: 1; gelu: 1.13; selu: scale * alpha = 1.76).  Relative error is meaningless next to a
relu zero crossing, an absolute bound on the pre-activation is not.  Max aggregation needs no special case (max is
1-Lipschitz in the sup norm); hidden MLP layers use relu, which is the identity on the non-negative absolute evaluation.

Attention and softmax weights (RGAT, the softmax readout) are convex weights; the float32 error of a weight alpha is about
u * |s| * alpha for scores s, which adds max |m| * 2 * max |s| to the convex combination of |m|.

Backward.  dZ = grad_out * act'(Z) is evaluated at a pre-activation that is itself inexact; with act2max = max |act''|
the error of act'(Z) is at most act2max * (error of Z).  The bound of every gradient is the float64 backward on absolute
values, without the activation, fed |grad_out| * (Lip + act2max * forward_bound_pre).  relu, leaky_relu and selu have
no act'' (their derivative jumps at 0): their gradients stay on the norm-wise tests.

GGNN is not covered: its outputs are convex combinations (sigmoid gates) of the state and a tanh candidate, all bounded by
1, so the max-scaled check of the parity tests is already an element-wise one there.
"""
from __future__ import annotations

from functools import lru_cache
from typing import Optional

import numpy as np
import torch

import reference64 as r64
import reference64_edge_mlp as rm
from oracle import message_passing_oracle as mo

LOWEST = float(np.finfo(np.float32).min)   # the unsorted_segment_max identity of an empty segment


# ---- activation constants ------------------------------------------------------------------------------------------
def _grid():
    return torch.linspace(-12.0, 12.0, 480001, dtype=torch.float64)


@lru_cache(maxsize=None)
def lipschitz(act: Optional[str]) -> float:
    """max |act'| over a fine grid (1 for relu, leaky_relu, tanh, elu; 1.129 for gelu; 1.758 for selu)."""
    if act is None:
        return 1.0
    _, d = r64.act_and_grad(_grid(), act)
    return float(d.abs().max())


@lru_cache(maxsize=None)
def act2max(act: Optional[str]) -> float:
    """max |act''| over a fine grid (0.770 for tanh, 0.798 for gelu, 1 for elu).  relu, leaky_relu and selu have none."""
    if act in ("relu", "leaky_relu", "selu"):
        raise ValueError(f"{act}' jumps at 0: its gradients have no element-wise bound")
    if act is None:
        return 0.0
    z = _grid()
    _, d = r64.act_and_grad(z, act)
    return float(((d[1:] - d[:-1]) / (z[1:] - z[:-1])).abs().max())


# ---- forward bounds ------------------------------------------------------------------------------------------------
def _abs_weights(w):
    if w is None:
        return None
    if isinstance(w, dict):
        return {k: _abs_weights(v) for k, v in w.items()}
    if isinstance(w, (list, tuple)):
        return [_abs_weights(v) for v in w]
    return np.abs(np.asarray(w, dtype=np.float64))


def forward_bound(kind: str, params, weights, h, adjs, pre_activation: bool = False) -> np.ndarray:
    """Element bound of a message-passing layer's output (kinds of mo.message_passing_forward, except GGNN): the float64
    oracle on |h| and |weights| with relu in place of the activation, times the activation's Lipschitz constant.
    pre_activation=True leaves out that factor."""
    kind = kind.lower()
    if kind == "ggnn":
        raise ValueError("GGNN has no element bound here (see the module docstring)")
    act = params["message_activation_function"]
    if kind == "rgat":
        b = rgat_bound(params, weights, h, adjs)
    else:
        p = dict(params, message_activation_function="relu")
        b = mo.message_passing_forward(kind, p, _abs_weights(weights), np.abs(np.asarray(h, np.float64)), adjs,
                                       dtype=np.float64)
        b = np.where(b <= LOWEST, 0.0, b)          # empty segments of max aggregation: exact
    return b if pre_activation else lipschitz(act) * b


def rgat_bound(params, weights, h, adjs) -> np.ndarray:
    """Pre-activation bound of RGAT, per target row v and head k: max_{e->v} max_c |m_e|[k, c] * (1 + 2 max_{e->v} |s_e|[k]),
    |m_e| and |s_e| the message and the attention score evaluated on absolute values; 0 for a row without edges."""
    H, K = int(params["hidden_dim"]), int(params["num_heads"])
    d = H // K
    ha = np.abs(np.asarray(h, np.float64))
    V = ha.shape[0]
    mmax = np.zeros((V, K))
    smax = np.zeros((V, K))
    for l, adj in enumerate(adjs):
        adj = np.asarray(adj).reshape(-1, 2)
        if not len(adj):
            continue
        W = np.abs(np.asarray(weights["edge_kernels"][l], np.float64))
        a = np.abs(np.asarray(weights["edge_attention"][l], np.float64))
        P = ha @ W                                              # node-level table: row u is |h_u| |W_l|
        ps, pt = P[adj[:, 0]].reshape(-1, K, d), P[adj[:, 1]].reshape(-1, K, d)
        s = np.einsum("eki,ki->ek", ps, a[:, :d]) + np.einsum("eki,ki->ek", pt, a[:, d:])
        np.maximum.at(mmax, adj[:, 1], ps.max(axis=2))
        np.maximum.at(smax, adj[:, 1], s)
    return np.repeat(mmax * (1.0 + 2.0 * smax), d, axis=1)


# ---- graph reductions ----------------------------------------------------------------------------------------------
def graph_ids(graph_ptr) -> np.ndarray:
    ptr = np.asarray(graph_ptr, np.int64)
    return np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))


def segment_bound(x, graph_ptr, agg: str = "sum", weights=None, num_heads: int = 1) -> np.ndarray:
    """Bound of a segment reduction over graph row ranges: the same reduction of |x| (times |weights[v, k]| on head k's
    columns); mean / sqrt_n divide by max(n, 1) / its square root; max is the segment max of |x| (0 for an empty graph)."""
    xa = np.abs(np.asarray(x, np.float64))
    ids = graph_ids(graph_ptr)
    G = len(graph_ptr) - 1
    if weights is not None:
        w = np.abs(np.asarray(weights, np.float64))
        xa = (xa.reshape(len(xa), num_heads, -1) * w[:, :, None]).reshape(xa.shape)
    if agg == "max":
        out = np.zeros((G, xa.shape[1]))
        np.maximum.at(out, ids, xa)
        return out
    out = np.zeros((G, xa.shape[1]))
    np.add.at(out, ids, xa)
    n = np.maximum(np.diff(np.asarray(graph_ptr, np.int64)), 1).astype(np.float64)[:, None]
    return out / n if agg == "mean" else out / np.sqrt(n) if agg == "sqrt_n" else out


def softmax_segment_bound(reprs, scores, graph_ptr, num_heads: int) -> np.ndarray:
    """Bound of the softmax-weighted graph sum, per graph and column of head k:
    sum_v alpha_vk |r_v| + max_v |r_v| * 2 * max_v |s_vk|, alpha the float64 softmax of the scores."""
    r = np.abs(np.asarray(reprs, np.float64))
    s = np.asarray(scores, np.float64)
    ids = graph_ids(graph_ptr)
    G, V, K = len(graph_ptr) - 1, r.shape[0], num_heads
    alpha = np.stack([mo.unsorted_segment_softmax(s[:, k], ids, G) for k in range(K)], axis=1)
    conv = segment_bound(r, graph_ptr, weights=alpha, num_heads=K)
    rmax = segment_bound(r, graph_ptr, agg="max")
    smax = segment_bound(s, graph_ptr, agg="max")
    return conv + rmax * 2.0 * np.repeat(smax, r.shape[1] // K, axis=1)


# ---- backward bounds -----------------------------------------------------------------------------------------------
def _effective_grad(grad_out, pre_bound, act):
    return np.abs(np.asarray(grad_out, np.float64)) * (lipschitz(act) + act2max(act) * np.asarray(pre_bound))


def rgcn_backward_bound(h, adjs, Ws, grad_out, *, agg, act, normalize, use_target=False):
    """Bounds of {out, grad_h, grad_W[l]} of the RGCN-style layer (reference64.rgcn_layer)."""
    kw = dict(agg=agg, normalize=normalize, use_target=use_target, absval=True)
    g = r64.Graph(adjs, np.asarray(h).shape[0])
    pre = r64.rgcn_layer(h, adjs, Ws, graph=g, **kw)["out"].numpy()
    res = r64.rgcn_layer(h, adjs, Ws, _effective_grad(grad_out, pre, act), graph=g, **kw)
    return {"out": lipschitz(act) * pre, "grad_h": res["grad_h"].numpy(), "grad_W": [w.numpy() for w in res["grad_W"]]}


def edge_mlp_backward_bound(h, adjs, Us, W2s, grad_out, *, agg, act, normalize, use_target=False):
    """Bounds of {out, grad_h, grad_U[l], grad_W2[l]} of the edge MLP with one hidden layer (reference64_edge_mlp)."""
    kw = dict(agg=agg, normalize=normalize, use_target=use_target, absval=True)
    g = r64.Graph(adjs, np.asarray(h).shape[0])
    pre = rm.edge_mlp_layer(h, adjs, Us, W2s, graph=g, **kw)["out"].numpy()
    res = rm.edge_mlp_layer(h, adjs, Us, W2s, _effective_grad(grad_out, pre, act), graph=g, **kw)
    return {"out": lipschitz(act) * pre, "grad_h": res["grad_h"].numpy(),
            "grad_U": [x.numpy() for x in res["grad_U"]], "grad_W2": [x.numpy() for x in res["grad_W2"]]}


def dense_backward_bound(x, W, bias, grad_out, act):
    """Bounds of {out, grad_x, grad_W, grad_bias} of out = act(x W + bias)."""
    xa, Wa = np.abs(np.asarray(x, np.float64)), np.abs(np.asarray(W, np.float64))
    pre = xa @ Wa + (0.0 if bias is None else np.abs(np.asarray(bias, np.float64)))
    ge = _effective_grad(grad_out, pre, act)
    return {"out": lipschitz(act) * pre, "grad_x": ge @ Wa.T, "grad_W": xa.T @ ge, "grad_bias": ge.sum(axis=0)}


# ---- the assertion -------------------------------------------------------------------------------------------------
def assert_within_bound(got, ref64, bound, rel: float = 1e-5, what: str = "", row_sizes=None,
                        row_label: str = "in-degree", tiles: bool = False) -> float:
    """Every element finite and |got - ref64| <= rel * bound.  Where bound == 0 (no incoming edge, an empty graph) got must
    equal float32(ref64) exactly; where ref64 is the unsorted_segment_max identity, got must be finfo(float32).min exactly.
    A failure names the worst element: row, column, error / bound, the row's size (row_sizes[row], `row_label`) and with
    tiles=True its 64-row and 128-row tile.  Returns the largest error / bound ratio (0 when every element is exact)."""
    got = np.asarray(got)
    ref = np.asarray(ref64, np.float64)
    bound = np.broadcast_to(np.asarray(bound, np.float64), ref.shape)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    assert np.all(bound >= 0) and np.all(np.isfinite(bound)), f"{what}: the bound itself is not finite"
    g = got.astype(np.float64)
    sentinel = ref <= LOWEST * 0.99
    exact = (bound == 0) | sentinel
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        want_exact = np.where(sentinel, LOWEST, ref.astype(np.float32).astype(np.float64))
        err = np.abs(g - ref)
        ratio = np.where(exact, np.where(g == want_exact, 0.0, np.inf), err / (rel * bound))
    ratio = np.where(np.isfinite(g), ratio, np.inf)
    if ratio.size == 0:
        return 0.0
    worst = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    r = float(ratio[worst]) * rel
    if ratio[worst] <= 1.0:
        return r
    row = int(worst[0])
    where = f"row {row}" + (f", column {int(worst[1])}" if len(worst) > 1 else "")
    if row_sizes is not None:
        where += f", {row_label} {int(np.asarray(row_sizes)[row])}"
    if tiles:
        where += f", 64-row tile {row // 64}, 128-row tile {row // 128}"
    n_bad = int(np.count_nonzero(ratio > 1.0))
    detail = (f"got {g[worst]!r}, want exactly {want_exact[worst]!r}" if exact[worst] or not np.isfinite(g[worst])
              else f"error {err[worst]:.3e} = {r:.3e} x bound {bound[worst]:.3e}")
    raise AssertionError(f"{what}: {n_bad} element(s) outside rel={rel:g} x bound; worst at {where}: {detail}")
