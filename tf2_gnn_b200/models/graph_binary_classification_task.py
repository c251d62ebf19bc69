"""GraphBinaryClassificationTask — mirror of tf2_gnn.models.graph_binary_classification_task
(graph_binary_classification_task.py:11-101)."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

from .graph_regression_task import GraphRegressionTask
from .task_ops import count_once, graph_binary_loss, sigmoid


class GraphBinaryClassificationTask(GraphRegressionTask):
    @classmethod
    def get_default_hyperparameters(cls, mp_style: Optional[str] = None) -> Dict[str, Any]:
        super_params = super().get_default_hyperparameters(mp_style)
        these_hypers: Dict[str, Any] = {}
        super_params.update(these_hypers)
        return super_params

    def compute_task_output(self, batch_features, final_node_representations, training: bool, shard=None) -> Any:
        per_graph_regression_results = super().compute_task_output(batch_features, final_node_representations, training,
                                                                   shard=shard)
        return sigmoid(per_graph_regression_results)

    def compute_task_metrics(self, batch_features, task_output, batch_labels, shard=None) -> Dict[str, Any]:
        """{"loss", "num_correct", "num_graphs"}; loss and num_correct are 0-d CUDA tensors.  shard: as
        GraphRegressionTask.compute_task_metrics."""
        ce, num_correct = graph_binary_loss(count_once(task_output, shard), batch_labels["target_value"])
        return {"loss": ce, "num_correct": num_correct, "num_graphs": int(batch_features["num_graphs_in_batch"])}

    def compute_epoch_metrics(self, task_results: List[Any]) -> Tuple[float, str]:
        total_num_graphs = sum(r["num_graphs"] for r in task_results)
        total_num_correct = sum(int(r["num_correct"]) for r in task_results)
        epoch_acc = total_num_correct / total_num_graphs
        return -epoch_acc, f"Accuracy = {epoch_acc:.3f}"
