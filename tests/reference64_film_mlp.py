"""float64 torch restatement of a GNN-FiLM layer with hidden layers in its FiLM MLPs (and optionally in its edge MLPs), in
the reference's literal per-edge op order (message_passing.py:95-218 with gnn_edge_mlp.py:84-107 and gnn_film.py:83-108):
every edge evaluates its type's FiLM MLP on its gathered target row, as gnn_film.py:99-107 does.  Differentiable, for small
graphs: gradients come from torch autograd."""
from __future__ import annotations

from typing import Dict, Sequence

import torch

from reference64 import act_and_grad


def mlp(x, kernels: Sequence[torch.Tensor]):
    """dpu_utils.tf2utils.MLP without biases: hidden Dense layers with ReLU, linear output layer."""
    for W in kernels[:-1]:
        x = torch.relu(x @ W)
    return x @ kernels[-1]


def film_mlp_autograd(h, adjs, edge_mlps, film_mlps, *, agg="sum", act="relu", normalize=False, use_target=False,
                      act_before=False):
    """h [V, D]; edge_mlps[l] / film_mlps[l]: the kernels of type l's edge MLP / FiLM MLP (last FiLM kernel [S, 2H], gamma
    columns first).  Aggregations sum / mean / sqrt_n."""
    V = h.shape[0]
    H = film_mlps[0][-1].shape[1] // 2
    msgs, tgts = [], []
    for adj, E, F in zip(adjs, edge_mlps, film_mlps):
        adj = adj if isinstance(adj, torch.Tensor) else torch.from_numpy(adj)
        src, tgt = adj[:, 0].long(), adj[:, 1].long()
        hs, ht = h.index_select(0, src), h.index_select(0, tgt)
        m = mlp(torch.cat([hs, ht], dim=1) if use_target else hs, E)
        if normalize:
            c = torch.bincount(tgt, minlength=V).to(h.dtype)
            m = m / (c[tgt] + 1e-7)[:, None]
        f = mlp(ht, F)                      # per edge, on the gathered target row
        msgs.append(f[:, :H] * m + f[:, H:])
        tgts.append(tgt)
    M, T = torch.cat(msgs), torch.cat(tgts)
    if act_before:
        M = act_and_grad(M, act)[0]
    out = torch.zeros((V, H), dtype=h.dtype).index_add(0, T, M)
    if agg in ("mean", "sqrt_n"):
        n = torch.bincount(T, minlength=V).to(h.dtype).clamp(min=1)
        out = out / (n if agg == "mean" else n.sqrt())[:, None]
    return out if act_before else act_and_grad(out, act)[0]


def hidden_preactivations(h, film_mlps) -> Dict[int, torch.Tensor]:
    """{type: [V, total hidden width]}: every hidden FiLM-MLP unit's pre-activation at every node (the per-edge values are
    these rows, gathered), to check that no ReLU input sits at 0 on the chosen data."""
    res = {}
    with torch.no_grad():
        for l, F in enumerate(film_mlps):
            x, pre = h, []
            for W in F[:-1]:
                p = x @ W
                pre.append(p)
                x = torch.relu(p)
            res[l] = torch.cat(pre, dim=1)
    return res
