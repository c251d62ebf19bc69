"""GraphTaskModel — H100-backed mirror of tf2_gnn.models.graph_task_model (graph_task_model.py:14-419).

Same hyper-parameters and defaults; `gnn_`-prefixed parameters go to the GNN.  A training step runs the forward, the task
loss (a C-ABI entry with its own backward), torch.autograd.grad over trainable_variables and one optimizer entry
(tfgnn_b200_optimizer_step): gradients and the update are deterministic.  Batches come from a data.DeviceGraphStore:
features from `store.batch(graph_ids)`, labels from `store.batch_labels(graph_ids)`.

On target-range shards (sharding.TargetRangeShard, DESIGN.md §6 "Task models on shards") every rank trains on its rows of
the same batch (`store.shard_batch`): the node loss is merged over the ranks, the replicated per-graph head is counted once,
and the weight gradients are summed in rank order, so every rank applies the same update.
"""
from __future__ import annotations

import contextlib
import time
from abc import abstractmethod
from typing import Any, Dict, Iterable, List, Optional, Tuple

import torch

from .. import sharding
from ..layers import GNN, GNNInput
from ..layers.message_passing.message_passing import Variable
from .task_ops import Optimizer, PolynomialWarmupAndDecaySchedule


class GraphTaskModel:
    @classmethod
    def get_default_hyperparameters(cls, mp_style: Optional[str] = None) -> Dict[str, Any]:
        """graph_task_model.py:15-32."""
        params = {f"gnn_{name}": value for name, value in GNN.get_default_hyperparameters(mp_style).items()}
        these_hypers: Dict[str, Any] = {
            "optimizer": "Adam",  # One of "SGD", "RMSProp", "Adam"
            "learning_rate": 0.001,
            "learning_rate_warmup_steps": None,
            "learning_rate_decay_steps": None,
            "momentum": 0.85,
            "rmsprop_rho": 0.98,  # decay of gradients in RMSProp (unused otherwise)
            "gradient_clip_value": None,  # Set to float value to clip each gradient separately
            "gradient_clip_norm": None,  # Set to value to clip gradients by their norm
            "gradient_clip_global_norm": None,  # Set to value to clip gradients by their global norm
            "use_intermediate_gnn_results": False,
        }
        params.update(these_hypers)
        return params

    def __init__(self, params: Dict[str, Any], dataset, name: Optional[str] = None, **kwargs):
        self._params = params
        self.name = name or type(self).__name__
        self._num_edge_types = dataset.num_edge_types
        self._use_intermediate_gnn_results = params.get("use_intermediate_gnn_results", False)
        self._train_step_counter = 0
        self._optimizer: Optional[Optimizer] = None
        self._gnn: Optional[GNN] = None
        self.built = False

    # ---- build ------------------------------------------------------------------------------------------------------
    def build(self, input_shapes: Dict[str, Any]):
        """graph_task_model.py:93-123.  input_shapes: "node_features" (its last entry is the feature size) and
        "adjacency_list_{t}".  Subclasses build their head, then call this."""
        graph_params = {name[4:]: value for name, value in self._params.items() if name.startswith("gnn_")}
        self._gnn = GNN(graph_params)
        self._gnn.build(GNNInput(
            node_features=self.get_initial_node_feature_shape(input_shapes),
            adjacency_lists=tuple(input_shapes.get(f"adjacency_list_{t}", (None, 2)) for t in range(self._num_edge_types)),
            node_to_graph_map=(None,), num_graphs=()))
        for v in self.trainable_variables:
            v.requires_grad_(True)
        self.built = True

    def get_initial_node_feature_shape(self, input_shapes) -> Tuple:
        return tuple(input_shapes["node_features"])

    def compute_initial_node_features(self, inputs, training: bool) -> torch.Tensor:
        return inputs["node_features"]

    @property
    def dropout_state(self):
        """The model's one Philox stream (the GNN's, seeded by gnn_b200_dropout_seed): head dropout draws from it too."""
        return self._gnn.dropout_state

    def _task_variables(self) -> List[Variable]:
        return []

    @property
    def trainable_variables(self) -> List[Variable]:
        return list(self._gnn.trainable_variables) + self._task_variables()

    variables = trainable_variables

    # ---- forward ----------------------------------------------------------------------------------------------------
    @abstractmethod
    def compute_task_output(self, batch_features: Dict[str, Any], final_node_representations, training: bool,
                            shard=None) -> Any:
        """graph_task_model.py:131-156.  shard: the features are the rank's part of the batch (store.shard_batch)."""

    def compute_final_node_representations(self, inputs, training: bool, shard=None):
        """graph_task_model.py:158-179: (final, all representations incl. the initial one) when
        use_intermediate_gnn_results, else the final representations.  shard (sharding.TargetRangeShard): the GNN runs
        on the rank's rows (GNN.call), and so do the representations."""
        adjacency_lists = tuple(inputs[f"adjacency_list_{t}"] for t in range(self._num_edge_types))
        gnn_input = GNNInput(node_features=self.compute_initial_node_features(inputs, training),
                             adjacency_lists=adjacency_lists, node_to_graph_map=inputs["node_to_graph_map"],
                             num_graphs=inputs["num_graphs_in_batch"])
        return self._gnn(gnn_input, training=training, return_all_representations=self._use_intermediate_gnn_results,
                         shard=shard)

    def call(self, inputs, training: bool, shard=None):
        final_node_representations = self.compute_final_node_representations(inputs, training, shard)
        return self.compute_task_output(inputs, final_node_representations, training, shard=shard)

    def __call__(self, inputs, training: bool = False, shard=None):
        if not self.built:
            shapes = {"node_features": tuple(inputs["node_features"].shape)}
            shapes.update({f"adjacency_list_{t}": tuple(inputs[f"adjacency_list_{t}"].shape) for t in range(self._num_edge_types)})
            self.build(shapes)
        return self.call(inputs, training, shard)

    @abstractmethod
    def compute_task_metrics(self, batch_features: Dict[str, Any], task_output: Any,
                             batch_labels: Dict[str, Any], shard=None) -> Dict[str, Any]:
        """graph_task_model.py:185-205: must hold "loss"; values may be device tensors.  shard: the metrics of the whole
        batch, the same on every rank."""

    @abstractmethod
    def compute_epoch_metrics(self, task_results: List[Any]) -> Tuple[float, str]:
        """graph_task_model.py:207-222: (value, lower is better; description)."""

    # ---- optimizer --------------------------------------------------------------------------------------------------
    def _make_optimizer(self, learning_rate=None) -> Optimizer:
        """graph_task_model.py:224-276; the clip settings of _apply_gradients are part of the optimizer step here."""
        if learning_rate is None:
            learning_rate = self._params["learning_rate"]
            num_warmup_steps = self._params.get("learning_rate_warmup_steps")
            num_decay_steps = self._params.get("learning_rate_decay_steps")
            if num_warmup_steps is not None or num_decay_steps is not None:
                initial_learning_rate = 0.00001
                final_learning_rate = 0.00001
                if num_warmup_steps is None:
                    num_warmup_steps = -1  # Make sure that we have no warmup phase
                    initial_learning_rate = learning_rate
                if num_decay_steps is None:
                    num_decay_steps = 1  # Value doesn't matter, but needs to be non-zero
                    final_learning_rate = learning_rate
                learning_rate = PolynomialWarmupAndDecaySchedule(
                    learning_rate=learning_rate, warmup_steps=num_warmup_steps, decay_steps=num_decay_steps,
                    initial_learning_rate=initial_learning_rate, final_learning_rate=final_learning_rate, power=1.0)
        clip_val = self._params.get("gradient_clip_value")
        clip_norm_val = self._params.get("gradient_clip_norm")
        clip_global_norm_val = self._params.get("gradient_clip_global_norm")
        if clip_val is not None:
            if clip_norm_val is not None:
                raise ValueError("Both 'gradient_clip_value' and 'gradient_clip_norm' are set, but can only use one at a time.")
            if clip_global_norm_val is not None:
                raise ValueError("Both 'gradient_clip_value' and 'gradient_clip_global_norm' are set, but can only use one at a time.")
        elif clip_norm_val is not None and clip_global_norm_val is not None:
            raise ValueError("Both 'gradient_clip_norm' and 'gradient_clip_global_norm' are set, but can only use one at a time.")
        return Optimizer(self._params["optimizer"], learning_rate, momentum=self._params["momentum"],
                         rho=self._params["rmsprop_rho"], clip_value=clip_val, clip_norm=clip_norm_val,
                         clip_global_norm=clip_global_norm_val)

    def _apply_gradients(self, gradient_variable_pairs: Iterable[Tuple[Optional[torch.Tensor], Variable]]) -> None:
        """graph_task_model.py:278-324: variables without a gradient are skipped; clipping and the update are one
        tfgnn_b200_optimizer_step."""
        pairs = list(gradient_variable_pairs)
        if getattr(self, "_optimizer", None) is None:
            self._optimizer = self._make_optimizer()
        self._optimizer.apply_gradients([(g, v.value) for g, v in pairs])

    # ---- training loop ----------------------------------------------------------------------------------------------
    def train_step(self, batch_features: Dict[str, Any], batch_labels: Dict[str, Any], shard=None) -> Dict[str, Any]:
        """graph_task_model.py:338-365 with training=True: forward, loss, gradients of every trainable variable, one
        optimizer step.

        shard (sharding.TargetRangeShard): the features and labels are the rank's part of the batch (store.shard_batch,
        store.shard_batch_labels).  The forward runs under sharding.regather_saved_tables(), the metrics are the whole
        batch's, and the gradients are summed over the ranks in rank order before the optimizer step, so every rank that
        started from the same variables (sharding.broadcast_variables) holds the same variables, slots and step count
        after it.  Collective: every rank of the shard's group makes the same call."""
        context = sharding.regather_saved_tables() if shard is not None else contextlib.nullcontext()
        with context:
            task_output = self(batch_features, training=True, shard=shard)
        task_metrics = self.compute_task_metrics(batch_features, task_output, batch_labels, shard=shard)
        variables = self.trainable_variables
        values = [v.value for v in variables]
        gradients = torch.autograd.grad(task_metrics["loss"], values, allow_unused=True)
        if shard is not None:
            gradients = sharding.sum_gradient_list_over_ranks(gradients, values, shard.group)
        self._apply_gradients(zip(gradients, variables))
        self._train_step_counter += 1
        return task_metrics

    def _run_step(self, batch_features: Dict[str, Any], batch_labels: Dict[str, Any], training: bool,
                  shard=None) -> Dict[str, Any]:
        if training:
            return self.train_step(batch_features, batch_labels, shard=shard)
        with torch.no_grad():
            task_output = self(batch_features, training=False, shard=shard)
            return self.compute_task_metrics(batch_features, task_output, batch_labels, shard=shard)

    def run_one_epoch(self, store, batches: Iterable, quiet: bool = True, training: bool = True,
                      shard_group=None) -> Tuple[float, float, List[Any]]:
        """graph_task_model.py:367-398 over a data.DeviceGraphStore and an iterable of graph-id arrays (e.g.
        store.iter_batch_graph_ids(max_nodes)).  Returns (graph-average loss, graphs per second, task_results).  The
        per-batch losses stay on the device until the epoch ends.

        shard_group (a torch.distributed process group, e.g. torch.distributed.group.WORLD): train or evaluate every batch
        on target-range shards over the group's ranks.  Each batch is cut by store.shard_bounds, and each rank takes its
        part with store.shard_batch / shard_batch_labels.  Every rank must pass the same batches; every rank returns the same
        losses and metrics, and the slowest rank's graphs per second."""
        shard_rank = shard_world = None
        if shard_group is not None:
            import torch.distributed as dist
            shard_rank, shard_world = dist.get_rank(shard_group), dist.get_world_size(shard_group)
        epoch_time_start = time.time()
        task_results, losses, counts = [], [], []
        for step, graph_ids in enumerate(batches):
            if shard_group is None:
                shard = None
                batch_features = store.batch(graph_ids)
                batch_labels = store.batch_labels(graph_ids)
            else:
                shard = sharding.TargetRangeShard(store.shard_bounds(graph_ids, shard_world), shard_rank, shard_group)
                batch_features = store.shard_batch(graph_ids, shard)
                batch_labels = store.shard_batch_labels(graph_ids, shard)
            task_metrics = self._run_step(batch_features, batch_labels, training, shard)
            losses.append(task_metrics["loss"].detach())
            counts.append(int(batch_features["num_graphs_in_batch"]))
            task_results.append(task_metrics)
            if not quiet:
                print(f"   Step: {step:4d}", end="\r")
        host_losses = torch.stack(losses).cpu().double().tolist() if losses else []
        total_time = time.time() - epoch_time_start
        if shard_group is not None:
            elapsed = torch.tensor([total_time], dtype=torch.float64, device=store.device)
            total_time = float(sharding.all_gather_stacked(elapsed, shard_group).max())
        total_num_graphs = sum(counts)
        total_loss = sum(l * n for l, n in zip(host_losses, counts))
        return total_loss / float(total_num_graphs), float(total_num_graphs) / total_time, task_results

    # ---- prediction -------------------------------------------------------------------------------------------------
    def predict(self, store, batches: Iterable) -> torch.Tensor:
        """graph_task_model.py:401-408: the task outputs of all batches, concatenated."""
        task_outputs = []
        with torch.no_grad():
            for graph_ids in batches:
                out = self(store.batch(graph_ids), training=False)
                task_outputs.append(out[0] if isinstance(out, tuple) else out)
        return torch.cat(task_outputs, dim=0)
