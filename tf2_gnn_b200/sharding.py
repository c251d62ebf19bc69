"""Multi-GPU partitioning of the message-passing path (SURVEY.md §8e).  One process per GPU.

Two cases, both with host-side index bookkeeping only (numpy; bit-exact, tested on CPU with gloo):

1. A batch of DISJOINT graphs (every dataset of the reference: graph_dataset.py:218-222 offsets each
   graph's node ids, so edges never cross graphs and node_to_graph_map is non-decreasing).  Cut the
   batch at graph boundaries into `world_size` contiguous node ranges balanced by edge count and
   re-base the indices per shard.  The forward pass needs NO collective.

2. ONE graph larger than a shard: 1-D partition by target-node range.  Rank g owns output rows
   [lo_g, hi_g) and every edge whose target falls there (ids stay global); it needs h[src] for
   arbitrary sources, i.e. one all-gather of the node-state shards per layer
   (tfgnn_b200_prepare_sharded + torch.distributed.all_gather_into_tensor over NCCL/NVLink).
   Training (DESIGN.md §6): gather_node_states is the differentiable all-gather, its backward the
   reduce-scatter reduce_scatter_node_grads; regather_saved_tables() keeps only a rank's own rows of
   every gathered table until backward.  Weight gradients come out partial per rank: sum them with
   sum_gradients_over_ranks (or torch.distributed.all_reduce) before the optimiser step.  A whole GNN, readout and
   global exchange included, runs on a TargetRangeShard (section 2c).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch


# ------------------------------------------------------------------------------------------------
# 1. disjoint-graph batches: cut at graph boundaries
# ------------------------------------------------------------------------------------------------
def partition_by_graph(node_to_graph_map: np.ndarray, adjacency_lists: Sequence[np.ndarray],
                       world_size: int) -> List[Tuple[int, int]]:
    """Contiguous node ranges [(lo, hi)] per rank, cut only at graph boundaries, balanced by the
    number of edges (the HBM traffic of the layer is proportional to it)."""
    n2g = np.asarray(node_to_graph_map)
    V = int(n2g.shape[0])
    if V == 0:
        return [(0, 0)] * world_size
    if np.any(np.diff(n2g) < 0):
        raise ValueError("node_to_graph_map must be non-decreasing (graph_dataset.py:211-217)")
    num_graphs = int(n2g[-1]) + 1
    graph_start = np.searchsorted(n2g, np.arange(num_graphs), side="left")          # first node of each graph
    edges_per_graph = np.zeros(num_graphs, dtype=np.int64)
    for adj in adjacency_lists:
        adj = np.asarray(adj).reshape(-1, 2)
        if len(adj):
            edges_per_graph += np.bincount(n2g[adj[:, 1]], minlength=num_graphs)
    load = edges_per_graph + np.diff(np.append(graph_start, V))                    # edges + nodes per graph
    cum = np.cumsum(load)
    total = int(cum[-1])
    bounds, g_lo = [], 0
    for r in range(world_size):
        if r == world_size - 1:
            g_hi = num_graphs
        else:
            target = total * (r + 1) / world_size
            g_hi = int(np.searchsorted(cum, target, side="left")) + 1
            g_hi = min(max(g_hi, g_lo), num_graphs)
        lo = int(graph_start[g_lo]) if g_lo < num_graphs else V
        hi = int(graph_start[g_hi]) if g_hi < num_graphs else V
        bounds.append((lo, hi))
        g_lo = g_hi
    return bounds


def shard_disjoint_batch(node_features: np.ndarray, adjacency_lists: Sequence[np.ndarray],
                         node_to_graph_map: np.ndarray, bounds: Sequence[Tuple[int, int]], rank: int
                         ) -> Dict[str, object]:
    """The rank's sub-batch with indices re-based to its node range.  Raises if an edge crosses the cut
    (it cannot for batches built by graph_dataset.py)."""
    lo, hi = bounds[rank]
    out_adj = []
    for adj in adjacency_lists:
        adj = np.asarray(adj, dtype=np.int32).reshape(-1, 2)
        tgt_in = (adj[:, 1] >= lo) & (adj[:, 1] < hi)
        src_in = (adj[:, 0] >= lo) & (adj[:, 0] < hi)
        if np.any(tgt_in != src_in):
            raise ValueError("an edge crosses a graph boundary: not a batch of disjoint graphs")
        out_adj.append(np.ascontiguousarray(adj[tgt_in] - np.int32(lo)))
    n2g = np.asarray(node_to_graph_map)[lo:hi]
    first_graph = int(n2g[0]) if hi > lo else 0
    return {
        "node_features": np.asarray(node_features)[lo:hi],
        "adjacency_lists": out_adj,
        "node_to_graph_map": (n2g - first_graph).astype(np.int32),
        "num_graphs": int(n2g[-1]) - first_graph + 1 if hi > lo else 0,
        "node_range": (lo, hi),
    }


# ------------------------------------------------------------------------------------------------
# 2. one large graph: 1-D partition by target range
# ------------------------------------------------------------------------------------------------
def partition_target_range(num_nodes: int, world_size: int, in_degree: Optional[np.ndarray] = None
                           ) -> List[Tuple[int, int]]:
    """Contiguous target ranges per rank; balanced by in-degree (edges) when given, else by rows."""
    if in_degree is None:
        cuts = [(num_nodes * r) // world_size for r in range(world_size + 1)]
    else:
        cum = np.cumsum(np.asarray(in_degree, dtype=np.int64) + 1)
        total = int(cum[-1]) if num_nodes else 0
        cuts = [0] + [int(np.searchsorted(cum, total * r / world_size, side="left")) for r in range(1, world_size)]
        cuts.append(num_nodes)
        cuts = [min(max(c, 0), num_nodes) for c in cuts]
        cuts = list(np.maximum.accumulate(cuts))
    return [(int(cuts[r]), int(cuts[r + 1])) for r in range(world_size)]


def filter_edges_by_target(adjacency_lists: Sequence[np.ndarray], lo: int, hi: int) -> List[np.ndarray]:
    """Edges whose target lies in [lo, hi); ids stay GLOBAL (tfgnn_b200_prepare_sharded re-bases the
    targets itself).  Optional: the library also accepts the unfiltered lists."""
    out = []
    for adj in adjacency_lists:
        adj = np.asarray(adj, dtype=np.int32).reshape(-1, 2)
        keep = (adj[:, 1] >= lo) & (adj[:, 1] < hi)
        out.append(np.ascontiguousarray(adj[keep]))
    return out


def padded_shard_rows(bounds: Sequence[Tuple[int, int]]) -> int:
    """Rows per rank for an equal-size all_gather_into_tensor (ranges are padded to the largest)."""
    return max((hi - lo) for lo, hi in bounds) if bounds else 0


def assemble_gathered(gathered: np.ndarray, bounds: Sequence[Tuple[int, int]]) -> np.ndarray:
    """[world * padded_rows, D] (concatenated padded shards) -> [V, D]."""
    rows = padded_shard_rows(bounds)
    parts = [gathered[r * rows: r * rows + (hi - lo)] for r, (lo, hi) in enumerate(bounds)]
    return np.concatenate(parts, axis=0) if parts else gathered[:0]


# ------------------------------------------------------------------------------------------------
# the two collectives every function of this module goes through.  A caller may replace them (module attributes), e.g. with
# host-staged versions over gloo for several ranks on one device, where NCCL refuses to run.
# ------------------------------------------------------------------------------------------------
def all_gather_into_tensor(out, inp, group=None) -> None:
    """out [world * n, ...] = every rank's inp [n, ...], in rank order."""
    import torch.distributed as dist
    dist.all_gather_into_tensor(out, inp, group=group)


def reduce_scatter_tensor(out, inp, group=None) -> None:
    """out [n, ...] = the sum over ranks of block `rank` of inp [world * n, ...]."""
    import torch.distributed as dist
    dist.reduce_scatter_tensor(out, inp, op=dist.ReduceOp.SUM, group=group)


def all_gather_node_states(h_local, bounds: Sequence[Tuple[int, int]], group=None):
    """torch tensors on any device/backend: all-gather the per-rank row ranges into the full [V, D] table."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rows = padded_shard_rows(bounds)
    D = int(h_local.shape[1])
    send = h_local
    if int(h_local.shape[0]) != rows:
        send = torch.zeros((rows, D), dtype=h_local.dtype, device=h_local.device)
        send[: h_local.shape[0]] = h_local
    recv = torch.empty((world * rows, D), dtype=h_local.dtype, device=h_local.device)
    all_gather_into_tensor(recv, send.contiguous(), group)
    if all((hi - lo) == rows for lo, hi in bounds):
        return recv
    return torch.cat([recv[r * rows: r * rows + (hi - lo)] for r, (lo, hi) in enumerate(bounds)], dim=0)


# ------------------------------------------------------------------------------------------------
# 2a. training on target-range shards: reduce-scatter backward, re-gather instead of saving the table
# ------------------------------------------------------------------------------------------------
def reduce_scatter_node_grads(partial_full, bounds: Sequence[Tuple[int, int]], group=None):
    """The adjoint of all_gather_node_states.  Every rank passes its partial gradient w.r.t. the full [V, D] table
    (e.g. the grad_h a layer's backward writes on a shard); rank r gets the sum over ranks of rows [lo_r, hi_r),
    [hi_r - lo_r, D].  Uneven and empty ranges are padded to padded_shard_rows like the all-gather."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    rows = padded_shard_rows(bounds)
    D = int(partial_full.shape[1])
    if all((hi - lo) == rows for lo, hi in bounds):
        send = partial_full.contiguous()
    else:
        send = torch.zeros((world * rows, D), dtype=partial_full.dtype, device=partial_full.device)
        for r, (lo, hi) in enumerate(bounds):
            send[r * rows: r * rows + (hi - lo)] = partial_full[lo:hi]
    recv = torch.empty((rows, D), dtype=partial_full.dtype, device=partial_full.device)
    reduce_scatter_tensor(recv, send, group)
    lo, hi = bounds[rank]
    return recv[: hi - lo]


class _GatherNodeStates(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h_local, bounds, group):
        ctx.bounds, ctx.group = bounds, group
        return all_gather_node_states(h_local.detach(), bounds, group)

    @staticmethod
    def backward(ctx, grad_full):
        return reduce_scatter_node_grads(grad_full, ctx.bounds, ctx.group), None, None


def gather_node_states(h_local, bounds: Sequence[Tuple[int, int]], group=None):
    """Differentiable all_gather_node_states: the full [V, D] table from every rank's rows; its backward is
    reduce_scatter_node_grads, so the gradient of h_local is the sum of every rank's gradient w.r.t. its rows.
    Backward is collective: every rank must run it through the same chain of gathers.  The result remembers h_local,
    so that regather_saved_tables() can save h_local in its place."""
    bounds = tuple((int(lo), int(hi)) for lo, hi in bounds)
    full = _GatherNodeStates.apply(h_local, bounds, group)
    full._tfgnn_gathered_from = (h_local.detach(), bounds, group)
    return full


class _Regather:
    """What regather_saved_tables() saves for a gathered table: the rank's own rows."""

    def __init__(self, h_local, bounds, group):
        self.h_local, self.bounds, self.group = h_local, bounds, group
        self.version = h_local._version

    def gather(self):
        if self.h_local._version != self.version:
            raise RuntimeError("a node-state shard saved for backward was modified in place before the re-gather")
        return all_gather_node_states(self.h_local, self.bounds, self.group)


class regather_saved_tables(torch.autograd.graph.saved_tensors_hooks):
    """Context manager: while it is active, autograd saves a table made by gather_node_states as the rank's own rows
    (h_local) and all-gathers it again when backward unpacks it.

        with sharding.regather_saved_tables():
            for layer in layers:
                h_local = layer(MessagePassingInput(sharding.gather_node_states(h_local, bounds), adj), prepared=shard)
        loss.backward()

    A layer hook (e.g. the fused RGCN / GGNN backward) saves its input table; without this context every rank keeps
    the full [V, D] table of every layer until backward, with it O(hi - lo) rows per layer, and a full table exists only
    while its layer runs forward or backward.  Only the forward has to run inside the context.  The re-gather in
    backward is a collective: it works because every rank runs the same chain of layers, so every rank unpacks the
    saved tables in the same order.  Other saved tensors are kept as they are."""

    def __init__(self):
        super().__init__(self._pack, self._unpack)

    def _pack(self, t):
        src = getattr(t, "_tfgnn_gathered_from", None)
        return t if src is None else _Regather(*src)

    def _unpack(self, saved):
        return saved.gather() if isinstance(saved, _Regather) else saved


# ------------------------------------------------------------------------------------------------
# 2c. a model on target-range shards: per-graph values and weight gradients the same on every rank
# ------------------------------------------------------------------------------------------------
class TargetRangeShard:
    """One rank's part of a graph cut by target range: `bounds[r] = (lo_r, hi_r)` for every rank r of `group` (contiguous,
    covering [0, num_nodes)), this process is `rank`.  Pass it as `shard=` to GNN, WeightedSumGraphRepresentation and the
    GraphGlobal*Exchange layers; they then take the rank's rows [lo, hi) of every node table."""

    def __init__(self, bounds: Sequence[Tuple[int, int]], rank: int, group=None):
        self.bounds = tuple((int(lo), int(hi)) for lo, hi in bounds)
        if not self.bounds or self.bounds[0][0] != 0 or any(a[1] != b[0] for a, b in zip(self.bounds, self.bounds[1:])):
            raise ValueError(f"shard bounds must be contiguous ranges starting at 0, got {self.bounds}")
        if any(hi < lo for lo, hi in self.bounds):
            raise ValueError(f"shard bounds must have lo <= hi, got {self.bounds}")
        self.rank = int(rank)
        if not 0 <= self.rank < len(self.bounds):
            raise ValueError(f"rank {rank} outside a world of {len(self.bounds)}")
        self.group = group
        self.lo, self.hi = self.bounds[self.rank]
        self.num_nodes = self.bounds[-1][1]
        self.world_size = len(self.bounds)

    @property
    def rows(self) -> Tuple[int, int]:
        """(first global row, rows of the whole table): what node_ops.dropout takes to draw the unsharded masks."""
        return self.lo, self.num_nodes

    def __repr__(self) -> str:
        return f"TargetRangeShard(bounds={self.bounds}, rank={self.rank})"


def all_gather_stacked(t, group=None):
    """[world, *t.shape]: every rank's t (the same shape on every rank), in rank order."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    flat = t.contiguous().reshape(-1)
    out = torch.empty((world * flat.numel(),), dtype=t.dtype, device=t.device)
    if flat.numel():
        all_gather_into_tensor(out, flat, group)
    return out.view((world,) + tuple(t.shape))


def sum_in_rank_order(stacked):
    """stacked[0] + stacked[1] + ... added left to right on the device (tfgnn_b200_axpby): every rank that holds the same
    gathered parts gets the same bits, whatever the collective backend's own reduction order."""
    from .layers.node_ops import _axpby
    acc = stacked[0].contiguous()
    if int(stacked.shape[0]) == 1:
        return acc.clone()
    for r in range(1, int(stacked.shape[0])):
        acc = _axpby(acc, 1.0, stacked[r].contiguous(), 1.0)
    return acc


def sum_over_ranks(t, group=None):
    """The sum over ranks of every rank's t, added in rank order: bitwise the same on every rank."""
    return sum_in_rank_order(all_gather_stacked(t, group))


def sum_gradients_over_ranks(variables, group=None) -> None:
    """After a backward on target-range shards every weight gradient is the rank's part.  Replace each variable's `.grad`
    by the sum over ranks, added in rank order (one all-gather of all gradients, then a fixed-order sum on the device), so
    that every rank holds the same bits before the optimiser step.  A variable without a gradient on a rank counts as zeros
    there; every rank must pass the same variables in the same order.  `variables`: tensors or objects with `.value`."""
    tensors = [getattr(v, "value", v) for v in variables]
    if not tensors:
        return
    dev = tensors[0].device
    flat = torch.cat([(t.grad if t.grad is not None else torch.zeros_like(t)).reshape(-1).to(torch.float32)
                      for t in tensors]).to(dev)
    total = sum_over_ranks(flat, group)
    off = 0
    for t in tensors:
        n = t.numel()
        t.grad = total[off: off + n].view_as(t).to(t.dtype).clone()
        off += n


def sum_gradient_list_over_ranks(gradients, like, group=None):
    """sum_gradients_over_ranks for a list of gradients (torch.autograd.grad's result; None = no gradient on this rank) of
    the float32 tensors `like`.  Returns the sums over ranks, added in rank order: the same bits on every rank.  A gradient
    that is None on every rank stays None (an optimizer then skips the variable, as it does unsharded); one that is None on
    some ranks counts as zeros there.  One all-gather; every rank must pass the same variables in the same order."""
    like = list(like)
    if not like:
        return []
    dev = like[0].device
    present = torch.tensor([0.0 if g is None else 1.0 for g in gradients], dtype=torch.float32, device=dev)
    flat = torch.cat([(g if g is not None else torch.zeros_like(t)).reshape(-1).to(torch.float32)
                      for g, t in zip(gradients, like)] + [present])
    total = sum_over_ranks(flat, group)
    flags = total[-len(like):].cpu()
    out, off = [], 0
    for i, t in enumerate(like):
        n = t.numel()
        out.append(total[off: off + n].view_as(t).clone() if flags[i] > 0 else None)
        off += n
    return out


def broadcast_variables(variables, group=None) -> None:
    """Copy rank 0's values of `variables` (tensors or objects with `.value`, the same list on every rank) into every rank's,
    in place: e.g. the starting weights of a model trained on target-range shards.  Goes through all_gather_stacked, so it
    uses the module's two collectives only."""
    tensors = [getattr(v, "value", v) for v in variables]
    if not tensors:
        return
    dev = tensors[0].device
    flat = torch.cat([t.detach().reshape(-1).to(torch.float32) for t in tensors]).to(dev)
    first = all_gather_stacked(flat, group)[0]
    off = 0
    with torch.no_grad():
        for t in tensors:
            n = t.numel()
            t.copy_(first[off: off + n].view_as(t))
            off += n


# ------------------------------------------------------------------------------------------------
# 2b. the all-gather fused into the layer kernel: node-state tables in peer-mapped (symmetric) memory
# ------------------------------------------------------------------------------------------------
class PeerNodeTables:
    """Two [num_nodes, H] float32 node-state tables per rank, allocated in symmetric memory
    (torch.distributed._symmetric_memory: CUDA VMM allocations every rank of the group maps over NVLink), so that the
    epilogue of the fused layer kernel can store its output tiles straight into every rank's copy
    (GNN_Edge_MLP.call_allgather / tfgnn_b200_rgcn_fwd_allgather).  Layer k reads `table(k)` and writes `table(k + 1)` on
    all ranks; `barrier(k + 1)` is the rank synchronisation between layers.  Collective constructor."""

    def __init__(self, num_nodes: int, hidden_dim: int, group=None):
        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        group = group or dist.group.WORLD
        dev = torch.device("cuda", torch.cuda.current_device())
        self._tables, self._handles = [], []
        for _ in range(2):
            t = symm_mem.empty((int(num_nodes), int(hidden_dim)), dtype=torch.float32, device=dev)
            self._handles.append(symm_mem.rendezvous(t, group))
            self._tables.append(t)
        self.rank = int(self._handles[0].rank)
        self.world_size = int(self._handles[0].world_size)

    def table(self, k: int):
        return self._tables[k % 2]

    def replica_ptrs(self, k: int):
        """Device addresses of table k on every rank, as mapped into this process (index = rank)."""
        return [int(p) for p in self._handles[k % 2].buffer_ptrs]

    def multicast_ptr(self, k: int) -> int:
        """Multicast (NVSwitch / NVLS) address of table k: one store to it lands in every rank's table; 0 if unsupported."""
        h = self._handles[k % 2]
        try:
            return int(h.multicast_ptr) if h.has_multicast_support(h.device.type, h.device.index) else 0
        except TypeError:
            try:
                return int(h.multicast_ptr or 0)
            except Exception:
                return 0
        except Exception:
            return 0

    def barrier(self, k: int) -> None:
        """All ranks have finished writing table k (enqueued on the current stream: a signal exchange in device memory)."""
        self._handles[k % 2].barrier(channel=0)
