"""float64 reference of the RGCN-style and GGNN layers, forward and backward, that scales to BASELINE sizes.

Per edge type l the layer is written with sparse matrices over the nodes:

    S_l[v, u] = s_{v,l} * (number of edges u -> v of type l),   s = 1/(c_{v,l} + 1e-7) when normalised, else 1
    A_l = S_l h,   P = sum_l A_l W_l (+ coeff_l h W_l^tgt),   Z = rn * P,   out = act(Z)
    dZ = grad_out * act'(Z),   dP = rn * dZ,   dW_l = A_l^T dP,   grad_h = sum_l S_l^T (dP W_l^T) (+ coeff_l dP W_l^tgt^T)

so no [E, D] array is ever built: one type is processed at a time, and the largest temporaries are [V, D] / [V, H]
tables (the cfg2 case of test_gpu_backward_scale.py, 1M nodes x 256 features, peaks at 22.6 GiB resident, its inputs
included).  The GRU adjoints of GGNN are written out by hand.

absval=True evaluates the same products on |S|, |h|, |W|, |grad_out| with the identity activation.  Every partial sum
the kernels form (gathered rows, the message contraction, the dW reduction over nodes, the dh reduction over the
source-keyed CSR) is bounded element-wise by the matching table of that evaluation, which is what the exact-arithmetic
tests check against 2^24 before they compare bits.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

SMALL_NUMBER = 1e-7   # tf2_gnn/utils/constants.py:2
LEAKY_RELU_ALPHA = 0.2
SELU_ALPHA = 1.6732632423543772
SELU_SCALE = 1.0507009873554805
GELU_C = 0.7978845608028654

F64 = torch.float64


def _t(x) -> torch.Tensor:
    return x.to(F64) if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x)).to(F64)


def act_and_grad(z: torch.Tensor, act: Optional[str]):
    """(act(z), act'(z)) of the reference's activation table; relu'(0) = 0 as in the kernels and in torch autograd."""
    if act is None:
        return z, torch.ones_like(z)
    if act == "relu":
        return torch.relu(z), (z > 0).to(F64)
    if act == "tanh":
        y = torch.tanh(z)
        return y, 1.0 - y * y
    if act == "leaky_relu":
        one = torch.ones_like(z)
        return torch.where(z > 0, z, LEAKY_RELU_ALPHA * z), torch.where(z > 0, one, LEAKY_RELU_ALPHA * one)
    if act == "elu":
        e = torch.exp(torch.clamp(z, max=0.0))
        return torch.where(z > 0, z, e - 1.0), torch.where(z > 0, torch.ones_like(z), e)
    if act == "selu":
        e = torch.exp(torch.clamp(z, max=0.0))
        return (SELU_SCALE * torch.where(z > 0, z, SELU_ALPHA * (e - 1.0)),
                SELU_SCALE * torch.where(z > 0, torch.ones_like(z), SELU_ALPHA * e))
    if act == "gelu":   # tanh approximation, utils/activation.py:7-14
        t = torch.tanh(GELU_C * (z + 0.044715 * z ** 3))
        return (0.5 * z * (1.0 + t),
                0.5 * (1.0 + t) + 0.5 * z * (1.0 - t * t) * GELU_C * (1.0 + 3.0 * 0.044715 * z * z))
    raise ValueError(f"unknown activation {act!r}")


class Graph:
    """Edge lists of one batch and the per-type in-degrees; builds the sparse S_l / S_l^T of one type on demand."""

    def __init__(self, adjs: Sequence, V: int):
        self.V = int(V)
        self.edges = []
        for a in adjs:
            a = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a).reshape(-1, 2))
            a = a.to(torch.int64)
            self.edges.append((a[:, 0].contiguous(), a[:, 1].contiguous()))
        self.counts = [torch.bincount(t, minlength=self.V).to(F64) for _, t in self.edges]
        self.in_degree = sum(self.counts) if self.counts else torch.zeros(self.V, dtype=F64)
        self.out_degree = (sum(torch.bincount(s, minlength=self.V) for s, _ in self.edges) if self.edges
                           else torch.zeros(self.V, dtype=torch.int64))

    @property
    def L(self) -> int:
        return len(self.edges)

    def scale(self, l: int, normalize: bool) -> torch.Tensor:
        return 1.0 / (self.counts[l] + SMALL_NUMBER) if normalize else torch.ones(self.V, dtype=F64)

    def matrices(self, l: int, normalize: bool, transpose: bool = True):
        """(S_l, S_l^T) as CSR; duplicate edges add up."""
        src, tgt = self.edges[l]
        vals = self.scale(l, normalize)[tgt]
        S = torch.sparse_coo_tensor(torch.stack([tgt, src]), vals, (self.V, self.V)).coalesce().to_sparse_csr()
        if not transpose:
            return S, None
        ST = torch.sparse_coo_tensor(torch.stack([src, tgt]), vals, (self.V, self.V)).coalesce().to_sparse_csr()
        return S, ST

    def row_norm(self, agg: str) -> Optional[torch.Tensor]:
        if agg == "sum":
            return None
        n = self.in_degree.clamp(min=1.0)
        if agg == "mean":
            return 1.0 / n
        if agg == "sqrt_n":
            return 1.0 / n.sqrt()
        raise ValueError(f"aggregation {agg!r} has no reference here")


def _spmm(S, x):
    return S @ x if S._nnz() else torch.zeros((S.shape[0], x.shape[1]), dtype=F64)


def _messages_fwd(g: Graph, h, Ws, normalize, use_target, want_max_a=False):
    """P = sum_l S_l h W_l^src (+ coeff_l h W_l^tgt) and max |A_l| over all types."""
    D = h.shape[1]
    P = torch.zeros((g.V, Ws[0].shape[1]), dtype=F64)
    max_a = 0.0
    for l in range(g.L):
        S, _ = g.matrices(l, normalize, transpose=False)
        A = _spmm(S, h)
        del S
        if want_max_a and A.numel():
            max_a = max(max_a, float(A.abs().max()))
        P.addmm_(A, Ws[l][:D])
        del A
        if use_target:
            coeff = g.counts[l] * g.scale(l, normalize)
            P.addmm_(coeff[:, None] * h, Ws[l][D:])
    return P, max_a


def _messages_bwd(g: Graph, h, Ws, dP, normalize, use_target):
    """(grad_h, [grad_W_l]) of P = sum_l S_l h W_l (+ target term) for the upstream gradient dP."""
    D = h.shape[1]
    grad_h = torch.zeros_like(h)
    grad_W = []
    for l in range(g.L):
        S, ST = g.matrices(l, normalize)
        A = _spmm(S, h)
        del S
        gw = A.T @ dP
        del A
        grad_h += _spmm(ST, dP @ Ws[l][:D].T)
        del ST
        if use_target:
            coeff = g.counts[l] * g.scale(l, normalize)
            gw = torch.cat([gw, (coeff[:, None] * h).T @ dP], dim=0)
            grad_h += coeff[:, None] * (dP @ Ws[l][D:].T)
        grad_W.append(gw)
    return grad_h, grad_W


def rgcn_layer(h, adjs, Ws, grad_out=None, *, agg="sum", act="relu", normalize=False, use_target=False,
               absval=False, graph: Optional[Graph] = None) -> Dict[str, object]:
    """RGCN-style layer (0 hidden layers, activation after the aggregation): out, grad_h, grad_W (list), max_abs_A.
    W_l is [D, H], or [2D, H] with use_target (rows [D, 2D) multiply the target state)."""
    h = _t(h)
    Ws = [_t(w) for w in Ws]
    g = graph if graph is not None else Graph(adjs, h.shape[0])
    if absval:
        h, Ws, act = h.abs(), [w.abs() for w in Ws], None
        grad_out = None if grad_out is None else _t(grad_out).abs()
    rn = g.row_norm(agg)
    P, max_a = _messages_fwd(g, h, Ws, normalize, use_target, want_max_a=True)
    if rn is not None:
        P *= rn[:, None]
    out, dact = act_and_grad(P, act)
    del P
    res = {"out": out, "max_abs_A": max_a}
    if grad_out is None:
        return res
    dP = _t(grad_out) * dact
    del dact
    if rn is not None:
        dP *= rn[:, None]
    res["grad_h"], res["grad_W"] = _messages_bwd(g, h, Ws, dP, normalize, use_target)
    return res


def ggnn_layer(h, adjs, Ws, K, U, b, grad_out=None, *, agg="sum", normalize=True,
               graph: Optional[Graph] = None) -> Dict[str, object]:
    """GGNN (ggnn.py:68-89; Keras GRUCell, reset_after=True): out, grad_h, grad_W (list), grad_K, grad_U, grad_b."""
    h, K, U, b = _t(h), _t(K), _t(U), _t(b)
    Ws = [_t(w) for w in Ws]
    g = graph if graph is not None else Graph(adjs, h.shape[0])
    H = h.shape[1]
    rn = g.row_norm(agg)
    aggd, _ = _messages_fwd(g, h, Ws, normalize, False)
    if rn is not None:
        aggd *= rn[:, None]
    gx = aggd @ K + b[0]
    gh = h @ U + b[1]
    z = torch.sigmoid(gx[:, :H] + gh[:, :H])
    r = torch.sigmoid(gx[:, H:2 * H] + gh[:, H:2 * H])
    ghh = gh[:, 2 * H:]
    hh = torch.tanh(gx[:, 2 * H:] + r * ghh)
    res = {"out": z * h + (1.0 - z) * hh}
    if grad_out is None:
        return res
    go = _t(grad_out)
    da = go * (1.0 - z) * (1.0 - hh * hh)          # d/d(candidate pre-activation)
    dz = go * (h - hh) * z * (1.0 - z)             # d/d(update-gate pre-activation)
    dr = da * ghh * r * (1.0 - r)                  # d/d(reset-gate pre-activation)
    dgx = torch.cat([dz, dr, da], dim=1)
    dgh = torch.cat([dz, dr, da * r], dim=1)
    grad_h = go * z + dgh @ U.T                    # through the convex combination + through gh = h U + b1
    del gx, gh, z, r, ghh, hh, da, dz, dr
    res["grad_b"] = torch.stack([dgx.sum(0), dgh.sum(0)])
    res["grad_K"] = aggd.T @ dgx
    res["grad_U"] = h.T @ dgh
    del aggd, dgh
    dP = dgx @ K.T                                 # d/d(agg), then through the row norm onto the message sum
    del dgx
    if rn is not None:
        dP *= rn[:, None]
    gm, res["grad_W"] = _messages_bwd(g, h, Ws, dP, normalize, False)
    res["grad_h"] = grad_h + gm
    return res
