"""QM9Dataset — mirror of tf2_gnn.data.qm9_dataset (qm9_dataset.py:44-191) whose folds are DeviceGraphStores.

``load_data`` reads the fold files (``{train,valid,test}.jsonl.gz``, one molecule per line) into host arrays and checks
them; ``store(fold)`` builds the fold's ``DeviceGraphStore`` with ``target_value`` set.  The adjacency lists of a fold are
processed in ONE ``process_adjacency_lists`` call over the fold's disjoint union, not one call per molecule: every
processed list of the union is a per-edge map of its input followed by concatenations of whole lists, so a graph's
processed list of a type is the union's list of that type restricted to the graph's edges, in the same order.  Grouping
the union's lists by graph with a stable sort therefore gives, graph by graph, the lists the reference's
``process_adjacency_lists`` returns for each molecule.

The reference shuffles the train fold on every epoch (qm9_dataset.py:164-169); here the caller passes the order, e.g.
``store.iter_batch_graph_ids(max_nodes, np.random.permutation(store.num_graphs))``.
"""
from __future__ import annotations

import gzip
import json
import os
from enum import Enum
from typing import Any, Dict, List, NamedTuple, Optional, Set, Tuple

import numpy as np

from .utils import compute_number_of_edge_types, get_tied_edge_types, process_adjacency_lists


class DataFold(Enum):
    """graph_dataset.py:10-13."""

    TRAIN = 0
    VALIDATION = 1
    TEST = 2


_FOLD_FILES = {DataFold.TRAIN: "train.jsonl.gz", DataFold.VALIDATION: "valid.jsonl.gz", DataFold.TEST: "test.jsonl.gz"}


class QM9Fold(NamedTuple):
    """A fold's molecules on the host, packed: graph g owns node rows [node_offsets[g], node_offsets[g + 1]).
    fwd_edges[t]: the [e, 2] edges of forward type t (0-based) of all graphs, node ids offset by the graph's first row,
    graph by graph and, within a graph, in the order of its record."""

    node_features: np.ndarray   # float32 [N, F]
    node_offsets: np.ndarray    # int64 [G + 1]
    fwd_edges: List[np.ndarray]  # int32 [e_t, 2] per forward type
    target_value: np.ndarray    # float32 [G]


class QM9Dataset:
    @classmethod
    def get_default_hyperparameters(cls) -> Dict[str, Any]:
        """graph_dataset.py:70-73 and qm9_dataset.py:49-60."""
        return {
            "max_nodes_per_batch": 10000,
            "add_self_loop_edges": True,
            "tie_fwd_bkwd_edges": True,
            "task_id": 0,
        }

    def __init__(self, params: Dict[str, Any], metadata: Optional[Dict[str, Any]] = None, **kwargs):
        self._params = params
        self._metadata = metadata if metadata is not None else {}
        self._num_fwd_edge_types = 4
        self._tied_fwd_bkwd_edge_types = get_tied_edge_types(tie_fwd_bkwd_edges=params["tie_fwd_bkwd_edges"],
                                                             num_fwd_edge_types=self._num_fwd_edge_types)
        self._num_edge_types = compute_number_of_edge_types(tied_fwd_bkwd_edge_types=self._tied_fwd_bkwd_edge_types,
                                                            num_fwd_edge_types=self._num_fwd_edge_types,
                                                            add_self_loop_edges=params["add_self_loop_edges"])
        self._node_feature_shape: Optional[Tuple] = None
        self._loaded_data: Dict[DataFold, QM9Fold] = {}
        self._stores: Dict[DataFold, Any] = {}

    @property
    def name(self) -> str:
        return self.__class__.__name__

    @property
    def params(self) -> Dict[str, Any]:
        return self._params

    @property
    def metadata(self) -> Dict[str, Any]:
        return self._metadata

    @property
    def num_edge_types(self) -> int:
        return self._num_edge_types

    @property
    def node_feature_shape(self) -> Tuple:
        """The shape of one node's features (qm9_dataset.py:156-162)."""
        if self._node_feature_shape is None:
            some_data_fold = next(iter(self._loaded_data.values()))
            self._node_feature_shape = (int(some_data_fold.node_features.shape[1]),)
        return self._node_feature_shape

    # ---- host: read and check the fold files ------------------------------------------------------------------------
    def load_data(self, path, folds_to_load: Optional[Set[DataFold]] = None) -> None:
        """qm9_dataset.py:93-111: the folds' files from the directory `path` (all three folds by default)."""
        if path is None:
            raise ValueError("QM9Dataset.load_data: give the directory that holds the fold files")
        if folds_to_load is None:
            folds_to_load = {DataFold.TRAIN, DataFold.VALIDATION, DataFold.TEST}
        for fold in (DataFold.TRAIN, DataFold.VALIDATION, DataFold.TEST):
            if fold in folds_to_load:
                self._loaded_data[fold] = self._read_fold(os.path.join(os.fspath(path), _FOLD_FILES[fold]))
                self._stores.pop(fold, None)

    def fold(self, fold: DataFold) -> QM9Fold:
        """The fold's molecules as load_data read them (host arrays)."""
        if fold not in self._loaded_data:
            raise KeyError(f"QM9Dataset: fold {fold.name} is not loaded")
        return self._loaded_data[fold]

    def _read_fold(self, file_name: str) -> QM9Fold:
        """qm9_dataset.py:118-138 without the per-graph processing: each record is {"graph": [[src, type, dst], ...],
        "node_features": [[...], ...], "targets": [[t0], ..., [t12]]}; edge types count from 1 (:145-147)."""
        task_id = int(self._params["task_id"])
        T = self._num_fwd_edge_types
        feats, counts, graphs, targets = [], [], [], []
        with gzip.open(file_name, "rt") as f:
            for line_no, line in enumerate(f, 1):
                if not line.strip():
                    continue
                d = json.loads(line)
                nf = np.asarray(d["node_features"], dtype=np.float32)
                n = len(nf)
                g = np.asarray(d["graph"], dtype=np.int64).reshape(-1, 3)
                where = f"{file_name}:{line_no}"
                if len(g) and (g[:, 1].min() < 1 or g[:, 1].max() > T):
                    raise ValueError(f"{where}: edge type {int(g[(g[:, 1] < 1) | (g[:, 1] > T), 1][0])} outside 1..{T}")
                ends = g[:, [0, 2]]
                if len(g) and (ends.min() < 0 or ends.max() >= n):
                    raise IndexError(f"{where}: node id {int(ends[(ends < 0) | (ends >= n)][0])} outside [0, {n})")
                if not 0 <= task_id < len(d["targets"]):
                    raise IndexError(f"{where}: task_id {task_id} outside the {len(d['targets'])} targets")
                feats.append(nf.reshape(n, -1))
                counts.append(n)
                graphs.append(g)
                targets.append(float(d["targets"][task_id][0]))
        node_offsets = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)
        if graphs:
            edges = np.concatenate(graphs, axis=0)
            edges[:, 0] += np.repeat(node_offsets[:-1], [len(g) for g in graphs])
            edges[:, 2] += np.repeat(node_offsets[:-1], [len(g) for g in graphs])
        else:
            edges = np.zeros((0, 3), np.int64)
        fwd = [np.ascontiguousarray(edges[edges[:, 1] == t + 1][:, [0, 2]], dtype=np.int32) for t in range(T)]
        F = feats[0].shape[1] if feats else 0
        return QM9Fold(node_features=np.concatenate(feats, axis=0) if feats else np.zeros((0, F), np.float32),
                       node_offsets=node_offsets, fwd_edges=fwd, target_value=np.asarray(targets, dtype=np.float32))

    # ---- device: the fold's store -----------------------------------------------------------------------------------
    def store(self, fold: DataFold):
        """The fold as a DeviceGraphStore with target_value set (built on the first call, then kept)."""
        if fold not in self._stores:
            from .graph_store import DeviceGraphStore
            self._stores[fold] = DeviceGraphStore(self._samples(self.fold(fold)), self._num_edge_types)
        return self._stores[fold]

    def _samples(self, data: QM9Fold) -> List[Dict[str, Any]]:
        """Per-graph samples (node_features, processed adjacency_lists in graph-local ids, target_value) from one
        process_adjacency_lists call over the fold's disjoint union."""
        G = len(data.target_value)
        if G == 0:
            return []
        offsets = data.node_offsets
        lists, _ = process_adjacency_lists(adjacency_lists=data.fwd_edges, num_nodes=int(offsets[-1]),
                                           add_self_loop_edges=self._params["add_self_loop_edges"],
                                           tied_fwd_bkwd_edge_types=self._tied_fwd_bkwd_edge_types)
        per_type = []
        for a in lists:
            e = a.cpu().numpy()
            graph = np.searchsorted(offsets, e[:, 0], side="right") - 1   # both ends of an edge lie in one graph
            order = np.argsort(graph, kind="stable")
            local = (e[order] - offsets[graph[order], None]).astype(np.int32)
            per_type.append(np.split(local, np.cumsum(np.bincount(graph, minlength=G))[:-1]))
        feats = np.split(data.node_features, offsets[1:-1])
        return [{"node_features": feats[g], "adjacency_lists": [p[g] for p in per_type],
                 "target_value": float(data.target_value[g])} for g in range(G)]
