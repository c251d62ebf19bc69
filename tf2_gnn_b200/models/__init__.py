"""Task models of tf2_gnn.models (SURVEY.md row 13): task heads, fused losses and a one-launch optimizer step."""
from .graph_task_model import GraphTaskModel
from .node_multiclass_task import NodeMulticlassTask, micro_f1
from .graph_regression_task import GraphRegressionTask
from .graph_binary_classification_task import GraphBinaryClassificationTask
from .qm9_regression import CHEMICAL_ACC_NORMALISING_FACTORS, QM9RegressionTask
from .task_ops import Optimizer, PolynomialWarmupAndDecaySchedule

__all__ = ["GraphTaskModel", "NodeMulticlassTask", "GraphRegressionTask", "GraphBinaryClassificationTask", "QM9RegressionTask",
           "CHEMICAL_ACC_NORMALISING_FACTORS", "Optimizer", "PolynomialWarmupAndDecaySchedule", "micro_f1"]
