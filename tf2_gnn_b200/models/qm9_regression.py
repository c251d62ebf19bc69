"""QM9RegressionTask — mirror of tf2_gnn.models.qm9_regression (qm9_regression.py:11-154).

The head is a gated sum over each molecule's atoms: out[g] = Σ_v σ(gate_v) · transform_v, where transform is a Dense
layer on the final node representations and gate a Dense layer on [initial features ‖ final representations].  Both are
the library's Dense-with-bias (node_ops.mlp); the sum is the sigmoid-weighted graph readout with one head and one column
(graph_autograd.readout, or shard_readout on target-range shards), which trains on the graphs' row ranges.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

import torch

from ..data.qm9_dataset import QM9Dataset
from ..layers import graph_autograd, node_ops
from ..layers.message_passing.message_passing import Variable
from ..layers.nodes_to_graph_representation import _MLP
from .graph_task_model import GraphTaskModel
from .task_ops import count_once, graph_regression_loss

# These magic constants were obtained during dataset generation, as result of normalising
# the values of target properties:
CHEMICAL_ACC_NORMALISING_FACTORS = [
    0.066513725,
    0.012235489,
    0.071939046,
    0.033730778,
    0.033486113,
    0.004278493,
    0.001330901,
    0.004165489,
    0.004128926,
    0.00409976,
    0.004527465,
    0.012292586,
    0.037467458,
]


class QM9RegressionTask(GraphTaskModel):
    @classmethod
    def get_default_hyperparameters(cls, mp_style: Optional[str] = None) -> Dict[str, Any]:
        super_params = super().get_default_hyperparameters(mp_style)
        these_hypers: Dict[str, Any] = {
            "use_intermediate_gnn_results": False,
            "out_layer_dropout_keep_prob": 1.0,
        }
        super_params.update(these_hypers)
        return super_params

    def __init__(self, params: Dict[str, Any], dataset, name: Optional[str] = None, **kwargs):
        super().__init__(params, dataset=dataset, name=name, **kwargs)
        assert isinstance(dataset, QM9Dataset)

        self._task_id = int(dataset.params["task_id"])
        # dpu_utils MLP(out_size=1, hidden_layers=[], use_biases=True, dropout_rate=out_layer_dropout_keep_prob): the
        # reference passes the "keep prob" as the dropout rate, and so does this port.
        self._dropout_rate = float(self._params["out_layer_dropout_keep_prob"])
        self._regression_gate: Optional[_MLP] = None
        self._regression_transform: Optional[_MLP] = None

    def build(self, input_shapes):
        """qm9_regression.py:64-81."""
        scope = self.__class__.__name__
        hidden_dim = self._params["gnn_hidden_dim"]
        feature_size = int(tuple(input_shapes["node_features"])[-1])
        self._regression_gate = _MLP(f"{scope}/node_gate/gate", feature_size + hidden_dim, 1, [], True, None,
                                     self._dropout_rate)
        self._regression_transform = _MLP(f"{scope}/node_transform/transform", hidden_dim, 1, [], True, None,
                                          self._dropout_rate)
        super().build(input_shapes)

    def _task_variables(self) -> List[Variable]:
        return self._regression_gate.variables + self._regression_transform.variables

    def _check_dropout_rate(self, training: bool) -> None:
        """tf.nn.dropout rejects a rate outside [0, 1) when the MLPs run in training mode; so does this port, before the
        step launches anything.  At inference the MLPs apply no dropout and any rate works."""
        rate = self._dropout_rate
        if training and not 0.0 <= rate < 1.0:
            raise ValueError(f"`rate` must be a scalar tensor or a float in the range [0, 1). Received: rate={rate}")

    def call(self, inputs, training: bool, shard=None):
        self._check_dropout_rate(training)
        return super().call(inputs, training, shard)

    def compute_task_output(self, batch_features, final_node_representations, training: bool, shard=None) -> Any:
        """qm9_regression.py:83-114: per-graph regression results [G].  shard: both MLPs run on the rank's rows and draw the
        unsharded dropout masks of those rows; the gated sum is merged over the ranks in rank order, so the result is the
        same on every rank."""
        self._check_dropout_rate(training)
        if self._params["use_intermediate_gnn_results"]:
            final_node_representations, _ = final_node_representations
        rows = shard.rows if shard is not None else None
        # The per-node regression uses only final node representations (transform first: the reference's call order
        # is the order in which the two MLPs draw from the Philox stream):
        per_node_output = self._regression_transform(final_node_representations, training, self.dropout_state,
                                                     rows)  # [V, 1]
        # The gating uses both initial and final node representations:
        per_node_weight = self._regression_gate(
            torch.cat([batch_features["node_features"], final_node_representations], dim=-1), training,
            self.dropout_state, rows)  # [V, 1]
        num_graphs = int(batch_features["num_graphs_in_batch"])
        n2g = node_ops.node_to_graph_index(batch_features["node_to_graph_map"], per_node_output.device)
        graph_ptr = node_ops.graph_offsets(n2g, num_graphs)
        if shard is None:
            per_graph_output = graph_autograd.readout(per_node_weight, per_node_output, n2g, graph_ptr, 1, "sigmoid", None,
                                                      None)
        else:
            per_graph_output = graph_autograd.shard_readout(per_node_weight, per_node_output, n2g, graph_ptr, num_graphs, 1,
                                                            "sigmoid", None, None, shard)
        return per_graph_output.reshape(-1)  # [G]

    def compute_task_metrics(self, batch_features, task_output, batch_labels, shard=None) -> Dict[str, Any]:
        """qm9_regression.py:116-130: "loss" (MSE), "batch_squared_error" and "batch_absolute_error" as 0-d CUDA tensors,
        "num_graphs".  shard: the per-graph output is the same on every rank, and its loss is counted once
        (task_ops.count_once)."""
        mse, mae = graph_regression_loss(count_once(task_output, shard), batch_labels["target_value"])
        num_graphs = int(batch_features["num_graphs_in_batch"])
        return {
            "loss": mse,
            "batch_squared_error": mse.detach() * num_graphs,
            "batch_absolute_error": mae * num_graphs,
            "num_graphs": num_graphs,
        }

    def compute_epoch_metrics(self, task_results: List[Any]) -> Tuple[float, str]:
        """qm9_regression.py:132-154: graph-weighted MSE and MAE of the epoch (MAE is the value) and the MAE over the
        task's chemical accuracy.  One host synchronisation."""
        total_num_graphs = sum(r["num_graphs"] for r in task_results)
        errors = [0.0, 0.0]
        if task_results:
            per_batch = torch.stack([torch.stack([r["batch_squared_error"], r["batch_absolute_error"]])
                                     for r in task_results]).cpu().double()
            errors = per_batch.sum(dim=0).tolist()
        epoch_mse = errors[0] / total_num_graphs
        epoch_mae = errors[1] / total_num_graphs
        return (
            epoch_mae,
            (
                f"Task {self._task_id} |"
                f" MSE = {epoch_mse:.3f} |"
                f" MAE = {epoch_mae:.3f} |"
                f" Error Ratio: {epoch_mae / CHEMICAL_ACC_NORMALISING_FACTORS[self._task_id]:.3f}"
            ),
        )
