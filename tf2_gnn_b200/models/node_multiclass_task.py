"""NodeMulticlassTask — mirror of tf2_gnn.models.node_multiclass_task (node_multiclass_task.py:26-72)."""
from __future__ import annotations

import math
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from ..layers import node_ops
from ..layers.message_passing.message_passing import Variable, glorot_uniform
from .graph_task_model import GraphTaskModel
from .task_ops import node_multiclass_loss


def micro_f1(counts) -> float:
    """micro_f1 (node_multiclass_task.py:10-23) from the int64 counts (tp, fp, fn): NaN whenever tp == 0."""
    tp, fp, fn = (int(c) for c in counts)
    with np.errstate(divide="ignore", invalid="ignore"):
        precision = np.float64(tp) / np.float64(tp + fp)
        recall = np.float64(tp) / np.float64(tp + fn)
        return float(np.float32((2 * precision * recall) / (precision + recall)))


class NodeMulticlassTask(GraphTaskModel):
    @classmethod
    def get_default_hyperparameters(cls, mp_style: Optional[str] = None) -> Dict[str, Any]:
        super_params = super().get_default_hyperparameters(mp_style)
        these_hypers: Dict[str, Any] = {}
        super_params.update(these_hypers)
        return super_params

    def __init__(self, params: Dict[str, Any], dataset, name: Optional[str] = None, **kwargs):
        super().__init__(params, dataset=dataset, name=name, **kwargs)
        if not hasattr(dataset, "num_node_target_labels"):
            raise ValueError(f"Provided dataset of type {type(dataset)} does not provide num_node_target_labels information.")
        self._num_labels = dataset.num_node_target_labels
        self.node_to_labels_layer: Optional[Tuple[Variable, Variable]] = None

    def build(self, input_shapes):
        """tf.keras.layers.Dense(units=num_labels, use_bias=True) under the class's name scope."""
        scope = f"{self.__class__.__name__}/dense"
        kernel = Variable(f"{scope}/kernel:0", glorot_uniform((self._params["gnn_hidden_dim"], self._num_labels)))
        bias = Variable(f"{scope}/bias:0", torch.zeros(self._num_labels, dtype=torch.float32, device=kernel.value.device))
        self.node_to_labels_layer = (kernel, bias)
        super().build(input_shapes)

    def _task_variables(self) -> List[Variable]:
        return list(self.node_to_labels_layer)

    def compute_task_output(self, batch_features, final_node_representations, training: bool, shard=None):
        """[V, num_labels] logits; on a shard, the rank's rows."""
        if self._use_intermediate_gnn_results:
            final_node_representations = final_node_representations[0]
        kernel, bias = self.node_to_labels_layer
        return (node_ops.dense(final_node_representations, kernel.value, bias.value),)

    def compute_task_metrics(self, batch_features, task_output, batch_labels, shard=None) -> Dict[str, Any]:
        """{"loss", "f1_score"} as 0-d CUDA tensors (one fused pass over the logits), and the counts behind the F1.  On a
        shard: those of the whole batch, from the ranks' partial sums and counts merged in rank order."""
        (per_node_logits,) = task_output
        loss, f1_score, counts = node_multiclass_loss(per_node_logits, batch_labels["node_labels"], shard)
        return {"loss": loss, "f1_score": f1_score, "f1_counts": counts}

    def compute_epoch_metrics(self, task_results: List[Any]) -> Tuple[float, str]:
        avg_microf1 = np.average([float(r["f1_score"]) for r in task_results])
        return -avg_microf1, f"Avg MicroF1: {avg_microf1:.3f}"
