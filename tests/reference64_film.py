"""float64 reference of the GNN-FiLM layer (0 hidden layers in both MLPs, activation after the aggregation), forward and
backward, that scales to BASELINE sizes.

Per edge type l, with c_{v,l} the in-degree of v in type l and S_l the sparse matrix of reference64.Graph:

    A_l = S_l h,   T_l = c s h  (s = 1/(c + 1e-7) when normalised, else 1),   [gamma_l | beta_l] = h F_l
    Q_l = A_l W^s_l (+ T_l W^t_l),   Z = rn * sum_l (gamma_l * Q_l + c beta_l),   out = act(Z)
    dZ = rn * grad_out * act'(Z),   dQ_l = dZ * gamma_l,   dgamma_l = dZ * Q_l,   dbeta_l = c dZ
    dW_l = [A_l | T_l]^T dQ_l,   dF_l = h^T [dgamma_l | dbeta_l]
    grad_h = sum_l S_l^T (dQ_l W^s_l^T) + [dgamma_l | dbeta_l] F_l^T (+ c s dQ_l W^t_l^T)

One type is processed at a time and no [E, D] array is built: the largest temporaries are [V, 2H] / [V, 2D] tables.

absval=True evaluates the same products on |h|, |W|, |F|, |grad_out| with the identity activation.  Every partial sum the
kernels form is then bounded element-wise by one of the tables of that evaluation; "partial_max" is the largest entry of
all of them, which the exact-arithmetic tests check against 2^24 before they compare bits.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from reference64 import F64, Graph, _spmm, _t, act_and_grad


def _type_operands(g: Graph, h, l, D, normalize, use_target, with_transpose):
    """(S_l^T or None, [A_l | T_l], c s) of one type."""
    S, ST = g.matrices(l, normalize, transpose=with_transpose)
    A = _spmm(S, h)
    del S
    coeff = g.counts[l] * g.scale(l, normalize)
    X = torch.cat([A, coeff[:, None] * h], dim=1) if use_target else A
    return ST, X, coeff


def film_layer(h, adjs, Ws: Sequence, Fs: Sequence, grad_out=None, *, agg="sum", act="relu", normalize=False,
               use_target=False, absval=False, graph: Optional[Graph] = None) -> Dict[str, object]:
    """GNN-FiLM layer: out, grad_h, grad_W (list), grad_F (list), partial_max.  W_l is [D, H] ([2D, H] with use_target: rows
    [D, 2D) multiply the target state), F_l is [D, 2H] (gamma columns first)."""
    h = _t(h)
    Ws = [_t(w) for w in Ws]
    Fs = [_t(f) for f in Fs]
    g = graph if graph is not None else Graph(adjs, h.shape[0])
    if absval:
        h, Ws, Fs, act = h.abs(), [w.abs() for w in Ws], [f.abs() for f in Fs], None
        grad_out = None if grad_out is None else _t(grad_out).abs()
    V, D = h.shape
    H = Fs[0].shape[1] // 2 if Fs else (Ws[0].shape[1] if Ws else 0)
    rn = g.row_norm(agg)
    peak = [0.0]

    def seen(*xs):
        for x in xs:
            if x.numel():
                peak[0] = max(peak[0], float(x.abs().max()))

    Z = torch.zeros((V, H), dtype=F64)
    for l in range(g.L):
        _, X, _ = _type_operands(g, h, l, D, normalize, use_target, False)
        Q = X @ Ws[l]
        GB = h @ Fs[l]
        seen(X, Q, GB)
        Z += GB[:, :H] * Q + g.counts[l][:, None] * GB[:, H:]
        del X, Q, GB
    if rn is not None:
        Z *= rn[:, None]
    seen(Z)
    out, dact = act_and_grad(Z, act)
    del Z
    res = {"out": out}
    if grad_out is None:
        res["partial_max"] = peak[0]
        return res
    dZ = _t(grad_out) * dact
    del dact
    if rn is not None:
        dZ *= rn[:, None]
    grad_h = torch.zeros_like(h)
    dHt = torch.zeros_like(h)
    grad_W, grad_F = [], []
    for l in range(g.L):
        ST, X, coeff = _type_operands(g, h, l, D, normalize, use_target, True)
        GB = h @ Fs[l]
        dQ = dZ * GB[:, :H]
        dGB = torch.cat([dZ * (X @ Ws[l]), g.counts[l][:, None] * dZ], dim=1)
        del GB
        grad_W.append(X.T @ dQ)
        grad_F.append(h.T @ dGB)
        del X
        dA = dQ @ Ws[l][:D].T
        grad_h += _spmm(ST, dA)
        dHt += dGB @ Fs[l].T
        seen(dQ, dGB, dA, dHt, grad_W[-1], grad_F[-1])
        if use_target:
            dT = dQ @ Ws[l][D:].T
            seen(dT)
            dHt += coeff[:, None] * dT
            del dT
        del ST, dQ, dGB, dA
    seen(grad_h)
    grad_h += dHt
    seen(dHt, grad_h)
    res.update(grad_h=grad_h, grad_W=grad_W, grad_F=grad_F, partial_max=peak[0])
    return res


def film_autograd(h, adjs, Ws, Fs, *, agg="sum", act="relu", normalize=False, use_target=False):
    """The reference's literal per-edge op order (message_passing.py:95-218 with gnn_film.py:83-108) in float64 torch
    autograd, for small graphs: h, Ws and Fs must be leaves with requires_grad."""
    V = h.shape[0]
    H = Fs[0].shape[1] // 2
    msgs, tgts = [], []
    for adj, W, F in zip(adjs, Ws, Fs):
        adj = adj if isinstance(adj, torch.Tensor) else torch.from_numpy(adj)
        src, tgt = adj[:, 0].long(), adj[:, 1].long()
        hs, ht = h.index_select(0, src), h.index_select(0, tgt)
        m = (torch.cat([hs, ht], dim=1) if use_target else hs) @ W
        if normalize:
            c = torch.bincount(tgt, minlength=V).to(h.dtype)
            m = m / (c[tgt] + 1e-7)[:, None]
        f = ht @ F
        msgs.append(f[:, :H] * m + f[:, H:])
        tgts.append(tgt)
    M, T = torch.cat(msgs), torch.cat(tgts)
    out = torch.zeros((V, H), dtype=h.dtype).index_add(0, T, M)
    if agg in ("mean", "sqrt_n"):
        n = torch.bincount(T, minlength=V).to(h.dtype).clamp(min=1)
        out = out / (n if agg == "mean" else n.sqrt())[:, None]
    return act_and_grad(out, act)[0]
