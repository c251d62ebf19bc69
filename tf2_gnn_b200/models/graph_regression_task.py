"""GraphRegressionTask — mirror of tf2_gnn.models.graph_regression_task (graph_regression_task.py:15-203)."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

import torch

from ..layers import NodesToGraphRepresentationInput, WeightedSumGraphRepresentation
from ..layers.message_passing.message_passing import Variable
from ..layers.nodes_to_graph_representation import _MLP
from ..utils.param_helpers import get_activation_function
from .graph_task_model import GraphTaskModel
from .task_ops import count_once, graph_regression_loss


class GraphRegressionTask(GraphTaskModel):
    @classmethod
    def get_default_hyperparameters(cls, mp_style: Optional[str] = None) -> Dict[str, Any]:
        super_params = super().get_default_hyperparameters(mp_style)
        these_hypers: Dict[str, Any] = {
            "use_intermediate_gnn_results": True,
            "graph_aggregation_output_size": 32,
            "graph_aggregation_num_heads": 4,
            "graph_aggregation_layers": [32, 32],
            "graph_aggregation_dropout_rate": 0.1,
            "regression_mlp_layers": [64, 32],
            "regression_mlp_dropout": 0.1,
        }
        super_params.update(these_hypers)
        return super_params

    def __init__(self, params: Dict[str, Any], dataset, name: Optional[str] = None, **kwargs):
        super().__init__(params, dataset=dataset, name=name, **kwargs)

        def readout(weighting_fun: str) -> WeightedSumGraphRepresentation:
            return WeightedSumGraphRepresentation(
                graph_representation_size=self._params["graph_aggregation_output_size"],
                num_heads=self._params["graph_aggregation_num_heads"], weighting_fun=weighting_fun,
                scoring_mlp_layers=self._params["graph_aggregation_layers"],
                scoring_mlp_dropout_rate=self._params["graph_aggregation_dropout_rate"], scoring_mlp_activation_fun="elu",
                transformation_mlp_layers=self._params["graph_aggregation_layers"],
                transformation_mlp_dropout_rate=self._params["graph_aggregation_dropout_rate"],
                transformation_mlp_activation_fun="elu")

        self._weighted_avg_of_nodes_to_graph_repr = readout("softmax")
        self._weighted_sum_of_nodes_to_graph_repr = readout("sigmoid")
        self._regression_mlp: Optional[_MLP] = None

    def build(self, input_shapes):
        """graph_regression_task.py:73-108."""
        feature_size = int(tuple(input_shapes["node_features"])[-1])
        if self._params["use_intermediate_gnn_results"]:
            # the initial GNN input + the results of all layers
            node_repr_size = feature_size + self._params["gnn_hidden_dim"] * self._params["gnn_num_layers"]
        else:
            node_repr_size = feature_size + self._params["gnn_hidden_dim"]
        shapes = NodesToGraphRepresentationInput(node_embeddings=(None, node_repr_size), node_to_graph_map=(None,),
                                                 num_graphs=())
        scope = f"{self.__class__.__name__}/graph_representation_computation"
        self._weighted_avg_of_nodes_to_graph_repr.build(shapes, name=f"{scope}/weighted_avg/WeightedSumGraphRepresentation")
        self._weighted_sum_of_nodes_to_graph_repr.build(shapes, name=f"{scope}/weighted_sum/WeightedSumGraphRepresentation")
        # dpu_utils MLP(out_size=1, hidden_layers=regression_mlp_layers, use_biases=True, activation_fun=relu)
        self._regression_mlp = _MLP(f"{self.__class__.__name__}/MLP", 2 * self._params["graph_aggregation_output_size"], 1,
                                    self._params["regression_mlp_layers"], True, get_activation_function("relu"),
                                    self._params["regression_mlp_dropout"])
        super().build(input_shapes)

    def _task_variables(self) -> List[Variable]:
        return (self._weighted_avg_of_nodes_to_graph_repr.variables + self._weighted_sum_of_nodes_to_graph_repr.variables
                + self._regression_mlp.variables)

    def compute_task_output(self, batch_features, final_node_representations, training: bool, shard=None) -> Any:
        """graph_regression_task.py:110-150: per-graph regression results [G].  shard: the readouts merge the ranks' rows
        in rank order, so the graph representations and the head MLP (with the same dropout masks: every rank's stream is
        at the same offset) are the same on every rank."""
        if self._params["use_intermediate_gnn_results"]:
            _, intermediate_node_representations = final_node_representations
            # skip the first "intermediate" representation, the output of the initial feature -> GNN input layer
            node_representations = torch.cat((batch_features["node_features"],) + tuple(intermediate_node_representations[1:]),
                                             dim=-1)
        else:
            node_representations = torch.cat([batch_features["node_features"], final_node_representations], dim=-1)
        inputs = NodesToGraphRepresentationInput(node_embeddings=node_representations,
                                                 node_to_graph_map=batch_features["node_to_graph_map"],
                                                 num_graphs=batch_features["num_graphs_in_batch"])
        for layer in (self._weighted_avg_of_nodes_to_graph_repr, self._weighted_sum_of_nodes_to_graph_repr):
            layer.dropout_state = self.dropout_state
        weighted_avg_graph_repr = self._weighted_avg_of_nodes_to_graph_repr(inputs, training=training, shard=shard)
        weighted_sum_graph_repr = self._weighted_sum_of_nodes_to_graph_repr(inputs, training=training, shard=shard)
        graph_representations = torch.cat([weighted_avg_graph_repr, weighted_sum_graph_repr], dim=-1)   # [G, GD]
        per_graph_results = self._regression_mlp(graph_representations, training, self.dropout_state)  # [G, 1]
        return per_graph_results.reshape(-1)

    def compute_task_metrics(self, batch_features, task_output, batch_labels, shard=None) -> Dict[str, Any]:
        """{"loss": mse, "mae", "num_graphs"}; loss and mae are 0-d CUDA tensors.  shard: the per-graph output is the same on
        every rank, and its loss is counted once (task_ops.count_once)."""
        mse, mae = graph_regression_loss(count_once(task_output, shard), batch_labels["target_value"])
        return {"loss": mse, "mae": mae, "num_graphs": int(batch_features["num_graphs_in_batch"])}

    def compute_epoch_metrics(self, task_results: List[Any]) -> Tuple[float, str]:
        """graph_regression_task.py:168-182: graph-weighted MSE and MAE of the epoch (MAE is the value)."""
        total_num_graphs = sum(r["num_graphs"] for r in task_results)
        total_squared_error = sum(float(r["loss"]) * r["num_graphs"] for r in task_results)
        total_absolute_error = sum(float(r["mae"]) * r["num_graphs"] for r in task_results)
        epoch_mse = total_squared_error / total_num_graphs
        epoch_mae = total_absolute_error / total_num_graphs
        return epoch_mae, f" MSE = {epoch_mse:.3f} | MAE = {epoch_mae:.3f}"
