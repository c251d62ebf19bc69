"""float64 references of the transform-then-aggregate form of an edge MLP without hidden layer (max aggregation and / or
activation before aggregation) and of its backward (csrc/backward.cu, transform_aggregate_bwd; DESIGN.md §6).

Per edge e = (u -> v) of type l, with s = 1/(c_{v,l} + 1e-7) when normalised, else 1, and W_l = [W^s_l; W^t_l]:

    P_l = h W^s_l,   T_l = h W^t_l (target-state input, else 0),   x_e = (P_l[u] + T_l[v]) s
    y_e = act(x_e) (activation before aggregation) or x_e,   z[v] = agg_e y_e over all types jointly,  out = act(rn(v) z)

`literal_autograd` is the reference's op order (gather -> message -> scale -> activation -> unsorted_segment_* ->
activation) in torch autograd, with tf.math.unsorted_segment_max and its gradient (each message equal to the maximum gets
grad / count; empty segments hold the lowest float and pass no gradient).  `backward` restates the fused backward's steps in
numpy, optionally for the targets [lo, hi) of one shard only:

    1. P, T;  max: z and n[v, c] = #{e : y_e[c] == z[v, c]};   dZ = dOut act'(z) / max(n, 1)  or  dOut rn(v)
    2. w_e = dZ[v] [y_e == z[v]] (max) act'(x_e) (activation before) s;  dP_l[u] = sum_{e leaving u} w_e,
       dT_l[v] = sum_{e into v} w_e
    3. dW^s_l = h^T dP_l,  dW^t_l = h^T dT_l,  grad_h = sum_l dP_l W^s_l^T + dT_l W^t_l^T
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

from reference64 import F64, act_and_grad

LOWEST = float(np.finfo(np.float32).min)   # tf.math.unsorted_segment_max of an empty segment (float32)


def _act(x, act):
    return act_and_grad(x, act)[0]


class _SegmentMax(torch.autograd.Function):
    """tf.math.unsorted_segment_max and its registered gradient (math_grad.py _UnsortedSegmentMinOrMaxGrad)."""

    @staticmethod
    def forward(ctx, data, ids, num_segments):
        out = torch.full((num_segments, data.shape[1]), LOWEST, dtype=data.dtype)
        if data.shape[0]:
            out = out.scatter_reduce(0, ids[:, None].expand_as(data), data, reduce="amax", include_self=False)
        ctx.save_for_backward(data, ids, out)
        return out

    @staticmethod
    def backward(ctx, g):
        data, ids, out = ctx.saved_tensors
        eq = (data == out[ids]).to(data.dtype)
        n = torch.zeros_like(out).index_add_(0, ids, eq)
        return eq * (g / n.clamp(min=1))[ids], None, None


def literal_autograd(h, adjs, Ws, *, agg="max", act="relu", act_before=False, normalize=False, use_target=False):
    """The layer output in the reference's op order; h and Ws are float64 torch leaves."""
    V = h.shape[0]
    msgs, tgts = [], []
    for adj, W in zip(adjs, Ws):
        adj = torch.as_tensor(np.asarray(adj)).long()
        src, tgt = adj[:, 0], adj[:, 1]
        x = h.index_select(0, src)
        if use_target:
            x = torch.cat([x, h.index_select(0, tgt)], dim=1)
        m = x @ W
        if normalize:
            c = torch.bincount(tgt, minlength=V).to(h.dtype)
            m = m / (c[tgt] + 1e-7)[:, None]
        msgs.append(m)
        tgts.append(tgt)
    M, T = torch.cat(msgs), torch.cat(tgts)
    if act_before:
        M = _act(M, act)
    if agg == "max":
        out = _SegmentMax.apply(M, T, V)
    else:
        out = torch.zeros((V, M.shape[1]), dtype=h.dtype).index_add(0, T, M)
        if agg in ("mean", "sqrt_n"):
            n = torch.bincount(T, minlength=V).to(h.dtype).clamp(min=1)
            out = out / (n if agg == "mean" else n.sqrt())[:, None]
    return out if act_before else _act(out, act)


def backward(h, adjs, Ws, grad_out, *, agg="max", act="relu", act_before=False, normalize=False, use_target=False,
             lo: int = 0, hi: Optional[int] = None):
    """The fused backward's steps in float64 numpy: (out[lo:hi], grad_h, [grad_W_l]) of the targets [lo, hi) (default:
    all).  grad_out has hi - lo rows.  A shard's contribution: the contributions of a partition of [0, V) sum to the whole."""
    h = np.asarray(h, np.float64)
    V, D = h.shape
    hi = V if hi is None else hi
    L = len(adjs)
    H = Ws[0].shape[1]
    g = np.asarray(grad_out, np.float64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    f = lambda a: act_and_grad(t(a), act)
    edges = []
    for adj in adjs:
        a = np.asarray(adj, np.int64).reshape(-1, 2)
        c = np.bincount(a[:, 1], minlength=V).astype(np.float64)
        s = 1.0 / (c[a[:, 1]] + 1e-7) if normalize else np.ones(len(a))
        own = (a[:, 1] >= lo) & (a[:, 1] < hi)
        edges.append((a[own, 0], a[own, 1] - lo, s[own]))
    # 1. P, T, per-edge x and y, z and n
    P = [h @ np.asarray(W, np.float64)[:D] for W in Ws]
    T = [h[lo:hi] @ np.asarray(W, np.float64)[D:] if use_target else None for W in Ws]
    xs = [(P[l][u] + (T[l][v] if use_target else 0.0)) * s[:, None] for l, (u, v, s) in enumerate(edges)]
    ys = [f(x)[0].numpy() if act_before else x for x in xs]
    Vo = hi - lo
    cnt = np.zeros(Vo)
    for (_, v, _) in edges:
        cnt += np.bincount(v, minlength=Vo)
    if agg == "max":
        z = np.full((Vo, H), LOWEST)
        for (_, v, _), y in zip(edges, ys):
            np.maximum.at(z, v, y)
        n = np.zeros((Vo, H))
        for (_, v, _), y in zip(edges, ys):
            np.add.at(n, v, (y == z[v]).astype(np.float64))
        out_act, d_out = (z, np.ones_like(z)) if act_before else (x.numpy() for x in f(z))
        dZ = np.where(n > 0, g * d_out / np.maximum(n, 1), 0.0)
        out = out_act
    else:
        z = np.zeros((Vo, H))
        for (_, v, _), y in zip(edges, ys):
            np.add.at(z, v, y)
        rn = {"sum": np.ones(Vo), "mean": 1 / np.maximum(cnt, 1), "sqrt_n": 1 / np.sqrt(np.maximum(cnt, 1))}[agg]
        out = z * rn[:, None]
        dZ = g * rn[:, None]
    # 2. per-edge weights; dP over the edges leaving each source, dT over the edges into each target
    dP = [np.zeros((V, H)) for _ in range(L)]
    dT = [np.zeros((Vo, H)) for _ in range(L)]
    for l, ((u, v, s), x, y) in enumerate(zip(edges, xs, ys)):
        w = dZ[v].copy()
        if agg == "max":
            w *= (y == z[v])
        if act_before:
            w *= f(x)[1].numpy()
        w *= s[:, None]
        np.add.at(dP[l], u, w)
        np.add.at(dT[l], v, w)
    # 3. weight and node-state gradients
    grad_h = np.zeros((V, D))
    grad_W = []
    for l, W in enumerate(Ws):
        W = np.asarray(W, np.float64)
        gW = [h.T @ dP[l]]
        grad_h += dP[l] @ W[:D].T
        if use_target:
            gW.append(h[lo:hi].T @ dT[l])
            grad_h[lo:hi] += dT[l] @ W[D:].T
        grad_W.append(np.concatenate(gW))
    return out, grad_h, grad_W


def ggnn_autograd(h, adjs, Ws, K, U, b, *, agg="max", normalize=True):
    """GGNN (ggnn.py:68-89, Keras GRUCell with reset_after=True) on the literal message op order; all float64 leaves."""
    H = h.shape[1]
    a = literal_autograd(h, adjs, Ws, agg=agg, act=None, normalize=normalize)
    gx = a @ K + b[0]
    gh = h @ U + b[1]
    z = torch.sigmoid(gx[:, :H] + gh[:, :H])
    r = torch.sigmoid(gx[:, H:2 * H] + gh[:, H:2 * H])
    hh = torch.tanh(gx[:, 2 * H:] + r * gh[:, 2 * H:])
    return z * h + (1.0 - z) * hh


def max_margin(h, adjs, Ws, *, act="relu", act_before=False, normalize=False, use_target=False):
    """float64 precondition of the max tests: (the smallest relative gap between a segment's maximum and any message below
    it, the number of (v, c) with a tie).  A gap above fp32 rounding means fp32 and float64 pick the same messages."""
    h = np.asarray(h, np.float64)
    V, D = h.shape
    ys, vs = [], []
    for adj, W in zip(adjs, Ws):
        a = np.asarray(adj, np.int64).reshape(-1, 2)
        W = np.asarray(W, np.float64)
        c = np.bincount(a[:, 1], minlength=V).astype(np.float64)
        x = h[a[:, 0]] @ W[:D] + (h[a[:, 1]] @ W[D:] if use_target else 0.0)
        if normalize:
            x = x / (c[a[:, 1]] + 1e-7)[:, None]
        ys.append(act_and_grad(torch.from_numpy(x), act)[0].numpy() if act_before else x)
        vs.append(a[:, 1])
    y, v = np.concatenate(ys), np.concatenate(vs)
    z = np.full((V, y.shape[1]), -np.inf)
    np.maximum.at(z, v, y)
    ties = np.zeros_like(z)
    np.add.at(ties, v, (y == z[v]).astype(np.float64))
    below = y < z[v]
    gap = (z[v] - y)[below] / np.maximum(np.abs(z[v])[below], 1e-30)
    return (float(gap.min()) if gap.size else np.inf), int((ties > 1).sum())
