"""float64 reference of the edge MLP with one hidden layer (GNN_Edge_MLP and RGIN defaults), forward and backward, that
scales to BASELINE sizes.  RGIN's aggregation MLP (0 or more hidden layers) is included.

Per edge e = (u -> v) of type l, with U_l = [U^s_l; U^t_l] ([D, H] or [2D, H]) and W2_l [H, H]:

    Xs_l = h U^s_l,   Xt_l = h U^t_l (target-state input, else 0),   P_e = Xs_l[u] + Xt_l[v],   m_e = [P_e > 0]
    A_l[v] = s_{v,l} sum_{e into v} relu(P_e)   (s = 1/(c_{v,l} + 1e-7) when normalised, else 1)
    Z = rn * sum_l A_l W2_l,   out = act(Z)   or, with an aggregation MLP, out = act(relu(..relu(Z M_0)..) M_n)
    dZ = rn * dZ_out,   dW2_l = A_l^T dZ,   dA_l = s_l (dZ W2_l^T)
    dXs_l[u] = sum_{e leaving u} dA_l[v] m_e,   dXt_l[v] = sum_{e into v} dA_l[v] m_e
    dU^s_l = h^T dXs_l,   dU^t_l = h^T dXt_l,   grad_h = sum_l dXs_l U^s_l^T + dXt_l U^t_l^T

The mask uses '>' (the derivative of relu at 0 is 0), as the kernels and TF's ReluGrad do.  One type is processed at a
time, and per-edge quantities are evaluated in chunks of at most `chunk` edges: no [E, H] array is ever held.  The
largest temporaries are [V, H] tables.

absval=True evaluates the same products on |h|, |U|, |W2|, |M|, |grad_out| with every mask set and the identity
activation.  Every partial sum the kernels form is then bounded element-wise by one of the tables of that evaluation:
"partial_max" is the largest entry of all of them, and "operand_max" the largest entry of any tensor-core GEMM operand
(h, U, W2, M, A, dZ, dXs, dXt and the aggregation MLP's activations).  "min_abs_P" is min |P_e| over every edge and column
(float64), for the margin precondition of tolerance tests whose inputs are not on a grid; "min_abs_aggr_pre" is the same
for the hidden pre-activations of the aggregation MLP.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from reference64 import F64, Graph, _t, act_and_grad

CHUNK = 1 << 19


def _edge_pass(g: Graph, l: int, Xs, Xt, absval: bool, chunk: int, dA=None, want_A=True):
    """One chunked pass over the edges of type l: (sum_e relu(P_e) per target or None, dXs, dXt, min |P_e|).
    dXs / dXt are computed when dA (the scaled per-target gradient of A_l) is given."""
    src, tgt = g.edges[l]
    V, H = Xs.shape
    S = torch.zeros((V, H), dtype=F64) if want_A else None
    dXs = torch.zeros((V, H), dtype=F64) if dA is not None else None
    dXt = torch.zeros((V, H), dtype=F64) if (dA is not None and Xt is not None) else None
    min_p = float("inf")
    for c0 in range(0, int(src.shape[0]), chunk):
        s, t = src[c0:c0 + chunk], tgt[c0:c0 + chunk]
        P = Xs.index_select(0, s)
        if Xt is not None:
            P += Xt.index_select(0, t)
        if P.numel():
            min_p = min(min_p, float(P.abs().min()))
        m = torch.ones_like(P) if absval else (P > 0).to(F64)
        if want_A:
            S.index_add_(0, t, P * m)
        del P
        if dA is not None:
            contrib = dA.index_select(0, t) * m
            dXs.index_add_(0, s, contrib)
            if dXt is not None:
                dXt.index_add_(0, t, contrib)
            del contrib
        del m
    return S, dXs, dXt, min_p


def edge_mlp_layer(h, adjs, Us: Sequence, W2s: Sequence, grad_out=None, *, agg="sum", act="relu", normalize=False,
                   use_target=False, aggr_ws: Optional[Sequence] = None, absval=False, graph: Optional[Graph] = None,
                   chunk: int = CHUNK) -> Dict[str, object]:
    """Edge MLP with one hidden layer, optionally followed by RGIN's aggregation MLP (aggr_ws = its kernels, ReLU on the
    hidden ones, `act` after the last): out, grad_h, grad_U (list), grad_W2 (list), grad_aggr (list), partial_max,
    operand_max, min_abs_P."""
    h = _t(h)
    Us = [_t(u) for u in Us]
    W2s = [_t(w) for w in W2s]
    aggr_ws = [_t(w) for w in (aggr_ws or [])]
    g = graph if graph is not None else Graph(adjs, h.shape[0])
    if absval:
        h, Us, W2s, aggr_ws, act = h.abs(), [u.abs() for u in Us], [w.abs() for w in W2s], [w.abs() for w in aggr_ws], None
        grad_out = None if grad_out is None else _t(grad_out).abs()
    V, D = h.shape
    H = W2s[0].shape[1] if W2s else (Us[0].shape[1] if Us else 0)
    rn = g.row_norm(agg)
    peak, opnd, min_p = [0.0], [0.0], [float("inf")]

    def seen(*xs, operand=False):
        for x in xs:
            if x is not None and x.numel():
                m = float(x.abs().max())
                peak[0] = max(peak[0], m)
                if operand:
                    opnd[0] = max(opnd[0], m)

    seen(h, *Us, *W2s, *aggr_ws, operand=True)

    def tables(l):
        Xs = h @ Us[l][:D]
        Xt = h @ Us[l][D:] if use_target else None
        seen(Xs, Xt)
        return Xs, Xt

    Z = torch.zeros((V, H), dtype=F64)
    for l in range(g.L):
        Xs, Xt = tables(l)
        S, _, _, mp = _edge_pass(g, l, Xs, Xt, absval, chunk)
        min_p[0] = min(min_p[0], mp)
        del Xs, Xt
        A = S * g.scale(l, normalize)[:, None]
        seen(S, A, operand=False)
        seen(A, operand=True)
        Z += A @ W2s[l]
        del S, A
    if rn is not None:
        Z *= rn[:, None]
    seen(Z)
    # aggregation MLP: ys[i] = input of layer i, pres[i] = its pre-activation
    ys, pres = [Z], []
    for i, M in enumerate(aggr_ws):
        seen(ys[-1], operand=True)
        pre = ys[-1] @ M
        seen(pre)
        pres.append(pre)
        if i < len(aggr_ws) - 1:
            ys.append(pre if absval else torch.relu(pre))
    last = pres[-1] if aggr_ws else Z
    out, dact = act_and_grad(last, act)
    hidden_pre = [float(p.abs().min()) for p in pres[:-1] if p.numel()]
    res = {"out": out, "min_abs_P": min_p[0], "min_abs_aggr_pre": min(hidden_pre, default=float("inf"))}
    if grad_out is None:
        res.update(partial_max=peak[0], operand_max=opnd[0])
        return res
    d = _t(grad_out) * dact
    del dact
    grad_aggr = [None] * len(aggr_ws)
    for i in range(len(aggr_ws) - 1, -1, -1):
        seen(d, operand=True)
        grad_aggr[i] = ys[i].T @ d
        d = d @ aggr_ws[i].T
        if i > 0 and not absval:
            d = d * (pres[i - 1] > 0).to(F64)
        seen(grad_aggr[i], d)
    del ys, pres
    dZ = d
    if rn is not None:
        dZ = dZ * rn[:, None]
    seen(dZ, operand=True)
    grad_h = torch.zeros_like(h)
    grad_U, grad_W2 = [], []
    for l in range(g.L):
        Xs, Xt = tables(l)
        dA = (dZ @ W2s[l].T) * g.scale(l, normalize)[:, None]
        S, dXs, dXt, _ = _edge_pass(g, l, Xs, Xt, absval, chunk, dA=dA)
        del Xs, Xt
        A = S * g.scale(l, normalize)[:, None]
        grad_W2.append(A.T @ dZ)
        del S, A
        seen(dA, grad_W2[-1])
        seen(dXs, dXt, operand=True)
        gu = h.T @ dXs
        grad_h += dXs @ Us[l][:D].T
        if use_target:
            gu = torch.cat([gu, h.T @ dXt], dim=0)
            seen(grad_h)   # the tensor-core GEMM's first term, before the target term is accumulated onto it
            grad_h += dXt @ Us[l][D:].T
        grad_U.append(gu)
        seen(gu, grad_h)
        del dA, dXs, dXt
    res.update(grad_h=grad_h, grad_U=grad_U, grad_W2=grad_W2, grad_aggr=grad_aggr, partial_max=peak[0],
               operand_max=opnd[0])
    return res


def edge_mlp_autograd(h, adjs, Us, W2s, *, agg="sum", act="relu", normalize=False, use_target=False, aggr_ws=None):
    """The reference's literal per-edge op order (message_passing.py:95-218 with gnn_edge_mlp.py:84-107 and rgin.py:88-106)
    in float64 torch autograd, for small graphs: h and the weights must be leaves with requires_grad.  W2s=None: edge MLPs
    without a hidden layer (m = x U)."""
    V = h.shape[0]
    H = (W2s or Us)[0].shape[1]
    msgs, tgts = [], []
    for l, (adj, U) in enumerate(zip(adjs, Us)):
        adj = adj if isinstance(adj, torch.Tensor) else torch.from_numpy(adj)
        src, tgt = adj[:, 0].long(), adj[:, 1].long()
        x = h.index_select(0, src)
        if use_target:
            x = torch.cat([x, h.index_select(0, tgt)], dim=1)
        m = x @ U if W2s is None else torch.relu(x @ U) @ W2s[l]
        if normalize:
            c = torch.bincount(tgt, minlength=V).to(h.dtype)
            m = m / (c[tgt] + 1e-7)[:, None]
        msgs.append(m)
        tgts.append(tgt)
    if msgs:
        M, T = torch.cat(msgs), torch.cat(tgts)
    else:
        M, T = torch.zeros((0, H), dtype=h.dtype), torch.zeros((0,), dtype=torch.int64)
    out = torch.zeros((V, H), dtype=h.dtype).index_add(0, T, M)
    if agg in ("mean", "sqrt_n"):
        n = torch.bincount(T, minlength=V).to(h.dtype).clamp(min=1)
        out = out / (n if agg == "mean" else n.sqrt())[:, None]
    for i, Mw in enumerate(aggr_ws or []):
        out = out @ Mw
        if i < len(aggr_ws) - 1:
            out = torch.relu(out)
    return act_and_grad(out, act)[0]
