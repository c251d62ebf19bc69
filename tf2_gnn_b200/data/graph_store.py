"""A dataset fold packed on the device, and minibatches assembled from it by CUDA kernels.

Mirrors ``GraphDataset.graph_batch_iterator_from_graph_iterator`` / ``_add_graph_to_batch`` / ``_finalise_batch``
(tf2_gnn/data/graph_dataset.py:161-246): a minibatch is the disjoint union of some graphs, node ids offset by the
running node count, ``node_to_graph_map`` a constant block per graph, empty edge types ``int32[0, 2]``.  The
reference rebuilds these arrays with Python loops for every batch; here the graphs are uploaded ONCE (all graphs of
an edge type back to back, graph-local ids) and ``batch(graph_ids)`` launches ``tfgnn_b200_assemble_batch``
(batch_builder.cu).  Only the greedy "which graphs fit" rule (:181-188) stays on the host: it needs node counts only.

On target-range shards each rank assembles only its rows of a batch: ``shard_bounds`` cuts the batch (by the in-degree
table the store keeps on the host) and ``shard_batch`` launches ``tfgnn_b200_assemble_batch_rows``.
"""
from __future__ import annotations

import ctypes
from ctypes import c_int64, c_void_p
from typing import Any, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _ffi, sharding
from ..runtime import require_cuda, stream_ptr


class DeviceGraphStore:
    """graphs: sequence of samples with ``node_features`` ([n, F] array-like) and ``adjacency_lists`` (list of
    num_edge_types arrays reshapeable to [e, 2], graph-local node ids), as ``GraphSample`` in graph_dataset.py:17-41.
    Optional labels, given by every sample or by none: ``node_labels`` ([n, C], e.g. PPI's PPIGraphSample) and
    ``target_value`` (one float per graph, e.g. the JSONL property datasets); ``batch_labels`` assembles them."""

    def __init__(self, graphs: Sequence[Any], num_edge_types: int):
        self.device = require_cuda()
        self.num_edge_types = int(num_edge_types)
        node_labels = [_get(s, "node_labels", None) for s in graphs]
        targets = [_get(s, "target_value", None) for s in graphs]
        for what, vals in (("node_labels", node_labels), ("target_value", targets)):
            if any(v is None for v in vals) and any(v is not None for v in vals):
                raise ValueError(f"{what} must be given for every graph or for none")
        self.node_labels: Optional[torch.Tensor] = None
        self.target_value: Optional[torch.Tensor] = None
        self.num_node_target_labels: Optional[int] = None
        if graphs and node_labels[0] is not None:
            labels = [np.asarray(v, dtype=np.float32) for v in node_labels]
            C = labels[0].reshape(len(labels[0]), -1).shape[1]
            self.num_node_target_labels = int(C)
            self.node_labels = torch.from_numpy(np.concatenate([l.reshape(-1, C) for l in labels], axis=0)).to(self.device)
        if graphs and targets[0] is not None:
            self.target_value = torch.from_numpy(np.asarray(targets, dtype=np.float32).reshape(-1)).to(self.device)
        self._last_rows = None   # (graph ids, node source rows) of the last batch(): batch_labels gathers through them
        self._last_shard_rows = None   # (graph ids, lo, hi, node source rows) of the last shard_batch()
        feats, node_counts = [], []
        edges: List[List[np.ndarray]] = [[] for _ in range(self.num_edge_types)]
        edge_counts = np.zeros((self.num_edge_types, len(graphs)), dtype=np.int64)
        for g, sample in enumerate(graphs):
            nf = np.asarray(_get(sample, "node_features"), dtype=np.float32)
            nf = nf.reshape(len(nf), -1)
            feats.append(nf)
            node_counts.append(len(nf))
            adj = _get(sample, "adjacency_lists")
            for t in range(self.num_edge_types):
                a = np.asarray(adj[t], dtype=np.int32).reshape(-1, 2)
                edges[t].append(a)
                edge_counts[t, g] = len(a)
        self.num_graphs = len(graphs)
        # host copies of the offset tables: sizes of a batch are known without a device round trip
        self.node_offsets_host = np.concatenate([[0], np.cumsum(node_counts, dtype=np.int64)]).astype(np.int64)
        self.edge_offsets_host = [np.concatenate([[0], np.cumsum(edge_counts[t])]).astype(np.int64)
                                  for t in range(self.num_edge_types)]
        # in-degree of every stored node, summed over edge types: shard cuts need no device round trip either
        self.in_degree_host = stored_in_degree(self.node_offsets_host, edges)
        dev = self.device
        self.node_features = torch.from_numpy(
            np.concatenate(feats, axis=0) if feats else np.zeros((0, 0), np.float32)).to(dev)
        self.node_offsets = torch.from_numpy(self.node_offsets_host).to(dev)
        self.edge_offsets = [torch.from_numpy(o).to(dev) for o in self.edge_offsets_host]
        self.edges = [torch.from_numpy(np.concatenate(e, axis=0) if e else np.zeros((0, 2), np.int32)).to(dev)
                      for e in edges]

    # ---- host logic: which graphs go into a batch (graph_dataset.py:164-188) ----------------------------------
    def iter_batch_graph_ids(self, max_nodes_per_batch: int, graph_order: Optional[Sequence[int]] = None
                             ) -> Iterator[np.ndarray]:
        return greedy_batches(np.diff(self.node_offsets_host), max_nodes_per_batch, graph_order)

    # ---- device: assemble the batch ---------------------------------------------------------------------------------
    def batch(self, graph_ids, with_node_features: bool = True) -> Dict[str, Any]:
        """batch_features of graph_dataset.py:226-246 as CUDA tensors: node_features, node_to_graph_map,
        num_graphs_in_batch, adjacency_list_{t}."""
        ids_host = self._check_ids(graph_ids)
        Gb = int(ids_host.size)
        T = self.num_edge_types
        no, eo = self.node_offsets_host, self.edge_offsets_host
        Vb = int((no[ids_host + 1] - no[ids_host]).sum()) if Gb else 0
        Eb = [int((eo[t][ids_host + 1] - eo[t][ids_host]).sum()) if Gb else 0 for t in range(T)]
        features, rows = self._assemble(ids_host, Vb, Eb, None, with_node_features)
        if with_node_features:
            self._last_rows = (ids_host, rows)
        return features

    def shard_bounds(self, graph_ids, world_size: int) -> List[Tuple[int, int]]:
        """Batch rows [(lo, hi)] per rank of the batch of graph_ids: sharding.partition_target_range over the batch's node
        count, balanced by the in-degree of its nodes (all edge types).  Host tables only."""
        ids_host = self._check_ids(graph_ids)
        return shard_bounds_from_tables(self.node_offsets_host, self.in_degree_host, ids_host, world_size)

    def shard_batch(self, graph_ids, shard, with_node_features: bool = True) -> Dict[str, Any]:
        """A rank's part of batch(graph_ids) on target-range shards (sharding.TargetRangeShard over the batch's rows, e.g.
        from shard_bounds), with the keys of batch(): node_features and node_to_graph_map (batch graph ids) of rows
        [shard.lo, shard.hi), num_graphs_in_batch of the whole batch, and adjacency_list_{t} in batch node ids holding every
        edge of the graphs that overlap those rows (tfgnn_b200_assemble_batch_rows).  Edges into other ranks' rows are
        among them; GNN(shard=...) prepares only those into [lo, hi)."""
        ids_host = self._check_ids(graph_ids)
        T = self.num_edge_types
        no, eo = self.node_offsets_host, self.edge_offsets_host
        batch_off = np.concatenate([[0], np.cumsum(no[ids_host + 1] - no[ids_host])]).astype(np.int64)
        Vb = int(batch_off[-1])
        if shard.num_nodes != Vb:
            raise ValueError(f"shard bounds cover {shard.num_nodes} rows, the batch has {Vb}")
        lo, hi = shard.lo, shard.hi
        Eb = [0] * T
        if hi > lo:
            g_first = int(np.searchsorted(batch_off, lo, side="right")) - 1   # the graphs holding rows lo and hi - 1
            g_last = int(np.searchsorted(batch_off, hi - 1, side="right")) - 1
            win = ids_host[g_first: g_last + 1]
            Eb = [int((eo[t][win + 1] - eo[t][win]).sum()) for t in range(T)]
        features, rows = self._assemble(ids_host, Vb, Eb, (lo, hi), with_node_features)
        if with_node_features:
            self._last_shard_rows = (ids_host, lo, hi, rows)
        return features

    def _assemble(self, ids_host: np.ndarray, Vb: int, Eb: List[int], window: Optional[Tuple[int, int]],
                  with_node_features: bool):
        """(features, node source rows): tfgnn_b200_assemble_batch, or _assemble_batch_rows over window = (lo, hi)."""
        dev = self.device
        Gb = int(ids_host.size)
        T = self.num_edge_types
        n = Vb if window is None else window[1] - window[0]
        ids = torch.from_numpy(ids_host).to(dev, non_blocking=True)
        n2g = torch.empty((n,), dtype=torch.int32, device=dev)
        rows = torch.empty((n,), dtype=torch.int32, device=dev) if with_node_features else None
        adj = [torch.empty((Eb[t], 2), dtype=torch.int32, device=dev) for t in range(T)]
        lib = _ffi.lib()
        ws = torch.empty((max(int(lib.tfgnn_b200_assemble_batch_workspace_bytes(T, Gb)), 8),), dtype=torch.uint8, device=dev)
        eoff_ptrs = (c_void_p * max(T, 1))(*[o.data_ptr() for o in self.edge_offsets])
        edge_ptrs = (c_void_p * max(T, 1))(*[e.data_ptr() if e.numel() else None for e in self.edges])
        out_ptrs = (c_void_p * max(T, 1))(*[a.data_ptr() if a.numel() else None for a in adj])
        Eb_c = (c_int64 * max(T, 1))(*Eb)
        head = (self.node_offsets.data_ptr(), ctypes.cast(eoff_ptrs, _ffi._PP), ctypes.cast(edge_ptrs, _ffi._PP), T,
                self.num_graphs, ids.data_ptr() if Gb else None, Gb, Vb, Eb_c)
        tail = (n2g.data_ptr() if n else None, rows.data_ptr() if (rows is not None and n) else None,
                ctypes.cast(out_ptrs, _ffi._PP), ws.data_ptr(), stream_ptr())
        if window is None:
            _ffi.check(lib.tfgnn_b200_assemble_batch(*head, *tail))
        else:
            _ffi.check(lib.tfgnn_b200_assemble_batch_rows(*head, window[0], n, *tail))
        features: Dict[str, Any] = {"node_to_graph_map": n2g, "num_graphs_in_batch": Gb}
        if with_node_features:
            features["node_features"] = self._gather(self.node_features, rows)
        for t in range(T):
            features[f"adjacency_list_{t}"] = adj[t]
        return features, rows

    def _gather(self, table: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
        """table[rows] (tfgnn_b200_gather_rows)."""
        n = int(rows.shape[0])
        F = int(table.shape[1]) if table.dim() == 2 else 0
        out = torch.empty((n, F), dtype=torch.float32, device=self.device)
        if n and F:
            _ffi.check(_ffi.lib().tfgnn_b200_gather_rows(table.data_ptr(), int(table.shape[0]), F, rows.data_ptr(), 1, n,
                                                         out.data_ptr(), stream_ptr()))
        return out

    def batch_labels(self, graph_ids) -> Dict[str, Any]:
        """batch_labels of graph_dataset.py:226-246 as CUDA tensors: ``node_labels`` [num_nodes_in_batch, C] gathered through
        the node rows that assemble node_features, and ``target_value`` [num_graphs_in_batch] by graph id, for the labels
        the store holds.  Call it after batch(graph_ids), whose node rows it reuses (otherwise it assembles them)."""
        ids_host = self._check_ids(graph_ids)
        labels: Dict[str, Any] = {}
        if self.node_labels is not None:
            if self._last_rows is None or not np.array_equal(self._last_rows[0], ids_host):
                self.batch(ids_host)
            labels["node_labels"] = self._gather(self.node_labels, self._last_rows[1])
        if self.target_value is not None:
            labels["target_value"] = self._targets(ids_host)
        return labels

    def shard_batch_labels(self, graph_ids, shard) -> Dict[str, Any]:
        """The labels of shard_batch(graph_ids, shard): ``node_labels`` of rows [shard.lo, shard.hi) and ``target_value`` of all
        the batch's graphs (the per-graph loss runs on every rank).  Reuses the node rows of the last shard_batch call."""
        ids_host = self._check_ids(graph_ids)
        labels: Dict[str, Any] = {}
        if self.node_labels is not None:
            last = self._last_shard_rows
            if last is None or not np.array_equal(last[0], ids_host) or (last[1], last[2]) != (shard.lo, shard.hi):
                self.shard_batch(ids_host, shard)
            labels["node_labels"] = self._gather(self.node_labels, self._last_shard_rows[3])
        if self.target_value is not None:
            labels["target_value"] = self._targets(ids_host)
        return labels

    def _targets(self, ids_host: np.ndarray) -> torch.Tensor:
        Gb = int(ids_host.size)
        out = torch.empty((Gb,), dtype=torch.float32, device=self.device)
        if Gb:
            ids = torch.from_numpy(ids_host).to(self.device, non_blocking=True)
            _ffi.check(_ffi.lib().tfgnn_b200_gather_rows(self.target_value.data_ptr(), self.num_graphs, 1, ids.data_ptr(), 1,
                                                         Gb, out.data_ptr(), stream_ptr()))
        return out

    def _check_ids(self, graph_ids) -> np.ndarray:
        ids_host = np.asarray(graph_ids, dtype=np.int32).reshape(-1)
        if ids_host.size and (ids_host.min() < 0 or ids_host.max() >= self.num_graphs):
            raise IndexError("graph id out of range")
        return ids_host


def stored_in_degree(node_offsets: np.ndarray, edges: Sequence[Sequence[np.ndarray]]) -> np.ndarray:
    """int64[V]: the in-degree of every node of the packed node table, summed over edge types.  edges[t][g]: graph g's
    [e, 2] list of type t in graph-local ids; graph g owns rows [node_offsets[g], node_offsets[g + 1])."""
    V = int(node_offsets[-1])
    deg = np.zeros(V, dtype=np.int64)
    for per_graph in edges:
        counts = [len(a) for a in per_graph]
        if sum(counts):
            tgt = np.concatenate([np.asarray(a).reshape(-1, 2)[:, 1] for a in per_graph]).astype(np.int64)
            tgt += np.repeat(np.asarray(node_offsets[:-1], dtype=np.int64), counts)
            deg += np.bincount(tgt, minlength=V)[:V]
    return deg


def shard_bounds_from_tables(node_offsets: np.ndarray, in_degree: np.ndarray, graph_ids: np.ndarray,
                             world_size: int) -> List[Tuple[int, int]]:
    """DeviceGraphStore.shard_bounds on the store's host tables: node_offsets int64[G + 1] and in_degree int64[V] of the
    packed node table.  The batch's in-degree is its graphs' slices of the table in batch order."""
    ids = np.asarray(graph_ids, dtype=np.int64).reshape(-1)
    starts, ends = node_offsets[ids], node_offsets[ids + 1]
    Vb = int((ends - starts).sum())
    deg = (np.concatenate([in_degree[a:b] for a, b in zip(starts, ends)]) if ids.size else np.zeros(0, np.int64))
    return sharding.partition_target_range(Vb, int(world_size), deg)


def greedy_batches(node_counts: Sequence[int], max_nodes_per_batch: int,
                   graph_order: Optional[Sequence[int]] = None) -> Iterator[np.ndarray]:
    """The reference's batching rule (graph_dataset.py:164-188): graphs are taken in order and the batch under
    construction is emitted as soon as adding the next graph would exceed max_nodes_per_batch; a single over-sized
    graph still forms its own batch.  (When the very FIRST graph is over-sized the reference emits an empty batch and
    fails in np.concatenate; here empty batches are skipped.)  Yields int32 arrays of graph ids."""
    counts = np.asarray(node_counts, dtype=np.int64)
    order = np.arange(len(counts)) if graph_order is None else np.asarray(graph_order)
    cur: List[int] = []
    nodes = 0
    for g in order:
        n = int(counts[g])
        if nodes + n > max_nodes_per_batch:
            if cur:
                yield np.asarray(cur, dtype=np.int32)
            cur, nodes = [], 0
        cur.append(int(g))
        nodes += n
    if cur:
        yield np.asarray(cur, dtype=np.int32)


_REQUIRED = object()


def _get(sample, name, default=_REQUIRED):
    if isinstance(sample, dict):
        return sample[name] if default is _REQUIRED else sample.get(name, default)
    return getattr(sample, name) if default is _REQUIRED else getattr(sample, name, default)
