"""Device-side mirror of tf2_gnn.data's index bookkeeping (SURVEY.md §8f-2)."""
from .utils import (compute_number_of_edge_types, get_tied_edge_types, process_adjacency_lists)
from .graph_store import DeviceGraphStore, greedy_batches
from .qm9_dataset import DataFold, QM9Dataset

__all__ = ["compute_number_of_edge_types", "get_tied_edge_types", "process_adjacency_lists", "DeviceGraphStore", "greedy_batches",
           "DataFold", "QM9Dataset"]
