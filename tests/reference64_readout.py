"""float64 reference of the graph readout, the three global exchanges and WASGraphRepresentation
(nodes_to_graph_representation.py:170-314, graph_global_exchange.py:83-183) in torch on the CPU: the literal formulas, made
differentiable, plus the closed-form readout backward and a host restatement of the chunked segment sum that
csrc/graph_ops.cu implements.  Weight dicts have the layout of oracle/message_passing_oracle.py."""
from typing import Any, Dict, List, Optional

import numpy as np
import torch

ACTS = {"relu": torch.relu, "tanh": torch.tanh, "elu": torch.nn.functional.elu,
        "leaky_relu": lambda x: torch.nn.functional.leaky_relu(x, 0.2), None: lambda x: x}

SEGMENT_CHUNK_ROWS = 64      # kSegRows of csrc/graph_ops.cu


def leaf(a) -> torch.Tensor:
    return torch.from_numpy(np.asarray(a)).double().requires_grad_()


def leaves_of(weights: Dict[str, Any]) -> Dict[str, Any]:
    """Every array of a weight dict as a float64 leaf (lists stay lists)."""
    return {k: [leaf(m) for m in v] if isinstance(v, (list, tuple)) else leaf(v) for k, v in weights.items()}


def graph_ptr_of(n2g: np.ndarray, G: int) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(np.bincount(np.asarray(n2g, np.int64), minlength=G))]).astype(np.int64)


def segment_sum(data: torch.Tensor, ids: torch.Tensor, G: int) -> torch.Tensor:
    return torch.zeros((G,) + tuple(data.shape[1:]), dtype=data.dtype).index_add(0, ids, data)


def mlp(x, kernels, biases=None, act="relu", masks=None):
    """dpu_utils MLP; masks (one per layer, 0 or 1/(1-rate) per element) is the dropout on every layer's input."""
    for i, W in enumerate(kernels):
        if masks is not None:
            x = x * torch.from_numpy(np.asarray(masks[i])).double()
        x = x @ W
        if biases is not None:
            x = x + biases[i]
        if i < len(kernels) - 1:
            x = ACTS[act](x)
    return x


def readout_from_scores(scores: Optional[torch.Tensor], reprs: torch.Tensor, n2g: np.ndarray, G: int, K: int, mode: str,
                        lower: Optional[float] = None, upper: Optional[float] = None) -> torch.Tensor:
    """:176-227 from the scoring MLP's output and the transformation result (after its activation, before the clamp).
    torch.clamp passes the gradient on lower <= x <= upper, ties included, which is what tf.maximum / tf.minimum do for
    their first argument."""
    ids = torch.from_numpy(np.asarray(n2g)).long()
    V, GD = reprs.shape
    if lower is not None:
        reprs = reprs.clamp(min=lower)
    if upper is not None:
        reprs = reprs.clamp(max=upper)
    if mode == "none":
        return segment_sum(reprs, ids, G)
    if mode == "average":
        cnt = torch.bincount(ids, minlength=G).clamp(min=1).to(reprs.dtype)
        return segment_sum(reprs, ids, G) / cnt[:, None]
    if mode == "sigmoid":
        w = torch.sigmoid(scores)
    else:
        mx = torch.full((G, K), -1e300, dtype=scores.dtype).scatter_reduce(0, ids[:, None].expand(-1, K), scores.detach(),
                                                                           reduce="amax")
        e = torch.exp(scores - mx[ids])
        w = e / segment_sum(e, ids, G)[ids]
    return segment_sum(w[:, :, None] * reprs.reshape(V, K, GD // K), ids, G).reshape(G, GD)


def readout_backward_closed_form(scores, reprs, n2g, G, K, mode, grad_out, lower=None, upper=None, weights=None):
    """The formulas tfgnn_b200_readout_bwd implements, in numpy float64: (grad_scores or None, grad_reprs).  `weights`
    replaces the weights computed from `scores` (the entry takes them as an input)."""
    reprs, grad_out = np.asarray(reprs, np.float64), np.asarray(grad_out, np.float64)
    ids = np.asarray(n2g, np.int64)
    V, GD = reprs.shape
    d = GD // K
    passes = np.ones_like(reprs, dtype=bool)
    R = reprs
    if lower is not None:
        passes &= R >= lower
        R = np.maximum(R, lower)
    if upper is not None:
        passes &= R <= upper
        R = np.minimum(R, upper)
    dO = grad_out[ids]
    if mode in ("none", "average"):
        scale = 1.0 if mode == "none" else 1.0 / np.maximum(np.bincount(ids, minlength=G), 1)[ids][:, None]
        return None, np.where(passes, dO * scale, 0.0)
    s = np.asarray(scores, np.float64) if weights is None else None
    if weights is not None:
        w = np.asarray(weights, np.float64)
    elif mode == "sigmoid":
        w = 1.0 / (1.0 + np.exp(-s))
    else:
        mx = np.full((G, K), -np.inf)
        np.maximum.at(mx, ids, s)
        e = np.exp(s - mx[ids])
        z = np.zeros((G, K))
        np.add.at(z, ids, e)
        w = e / z[ids]
    out = np.zeros((G, K, d))
    np.add.at(out, ids, w[:, :, None] * R.reshape(V, K, d))
    dw = (dO.reshape(V, K, d) * R.reshape(V, K, d)).sum(-1)
    grad_reprs = np.where(passes, np.repeat(w, d, axis=1) * dO, 0.0)
    if mode == "sigmoid":
        return dw * w * (1.0 - w), grad_reprs
    t = (grad_out.reshape(G, K, d) * out).sum(-1)
    return w * (dw - t[ids]), grad_reprs


def segment_sum_rows_chunked(data: np.ndarray, graph_ptr: np.ndarray, chunk_rows: int = SEGMENT_CHUNK_ROWS,
                             lanes: int = 8) -> np.ndarray:
    """The reduction order of tfgnn_b200_segment_sum_rows: rows in order inside chunks of `chunk_rows`; a graph that crosses
    chunk borders adds its chunk sums with `lanes` strided accumulators combined in lane order.  dtype of `data` is kept."""
    data = np.asarray(data)
    G, C = len(graph_ptr) - 1, data.shape[1]
    out = np.zeros((G, C), data.dtype)
    for g in range(G):
        beg, end = int(graph_ptr[g]), int(graph_ptr[g + 1])
        if beg == end:
            continue
        pieces = []
        for c in range(beg // chunk_rows, (end - 1) // chunk_rows + 1):
            acc = np.zeros(C, data.dtype)
            for v in range(max(beg, c * chunk_rows), min(end, (c + 1) * chunk_rows)):
                acc = acc + data[v]
            pieces.append(acc)
        if len(pieces) == 1:
            out[g] = pieces[0]
            continue
        lane_sums = [np.zeros(C, data.dtype) for _ in range(lanes)]
        for t, piece in enumerate(pieces):
            lane_sums[t % lanes] = lane_sums[t % lanes] + piece
        tot = lane_sums[0]
        for s in lane_sums[1:]:
            tot = tot + s
        out[g] = tot
    return out


def readout_layer(x: torch.Tensor, L: Dict[str, Any], n2g, G: int, K: int, mode: str, scoring_act="relu",
                  transformation_act="relu", lower=None, upper=None, scoring_masks=None,
                  transformation_masks=None) -> torch.Tensor:
    """WeightedSumGraphRepresentation.call on leaves L (see leaves_of); the MLPs' dropout as explicit masks."""
    scores = None
    if mode in ("softmax", "sigmoid"):
        scores = mlp(x, L["scoring_mlp"], L.get("scoring_biases"), scoring_act, scoring_masks)
    reprs = ACTS[transformation_act](mlp(x, L["transformation_mlp"], L.get("transformation_biases"), transformation_act,
                                         transformation_masks))
    return readout_from_scores(scores, reprs, n2g, G, K, mode, lower, upper)


def gru(inputs, state, kernel, recurrent_kernel, bias):
    H = state.shape[1]
    gx, gh = inputs @ kernel + bias[0], state @ recurrent_kernel + bias[1]
    z = torch.sigmoid(gx[:, :H] + gh[:, :H])
    r = torch.sigmoid(gx[:, H:2 * H] + gh[:, H:2 * H])
    hh = torch.tanh(gx[:, 2 * H:] + r * gh[:, 2 * H:])
    return z * state + (1 - z) * hh


def exchange(mode: str, x: torch.Tensor, L: Dict[str, Any], n2g, G: int, K: int, weighting: str,
             per_node_mask: Optional[np.ndarray] = None, scoring_masks=None, transformation_masks=None) -> torch.Tensor:
    """GraphGlobal{Mean,GRU,MLP}Exchange.call; per_node_mask (0 or 1/(1-rate) per element) is the exchange's dropout."""
    ids = torch.from_numpy(np.asarray(n2g)).long()
    per_node = readout_layer(x, L, n2g, G, K, weighting, scoring_masks=scoring_masks,
                             transformation_masks=transformation_masks)[ids]
    if per_node_mask is not None:
        per_node = per_node * torch.from_numpy(np.asarray(per_node_mask)).double()
    if mode == "mean":
        return (x + per_node) / 2
    if mode == "gru":
        return gru(per_node, x, L["gru_kernel"], L["gru_recurrent_kernel"], L["gru_bias"])
    return mlp(torch.cat([per_node, x], -1), L["mlp"])


def was(x: torch.Tensor, L_avg: Dict[str, Any], L_sum: Dict[str, Any], projection: torch.Tensor, n2g, G: int, K: int,
        act="elu") -> torch.Tensor:
    avg = readout_layer(x, L_avg, n2g, G, K, "softmax", act, act)
    tot = readout_layer(x, L_sum, n2g, G, K, "sigmoid", act, act)
    return torch.cat([avg, tot], -1) @ projection


def flat_grads(L: Dict[str, Any]) -> List[np.ndarray]:
    out = []
    for k in sorted(L):
        for t in (L[k] if isinstance(L[k], list) else [L[k]]):
            out.append(np.zeros(tuple(t.shape)) if t.grad is None else t.grad.numpy())
    return out
