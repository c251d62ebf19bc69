from .message_passing import (GGNN, MESSAGE_PASSING_IMPLEMENTATIONS, RGAT, RGIN, GNN_Edge_MLP, GNN_FiLM,
                              MessagePassing, MessagePassingInput, RGCN, get_known_message_passing_classes,
                              get_message_passing_class)
from .gnn import GNN, GNNInput
from .graph_global_exchange import (GraphGlobalExchange, GraphGlobalExchangeInput, GraphGlobalGRUExchange,
                                    GraphGlobalMeanExchange, GraphGlobalMLPExchange)
from .nodes_to_graph_representation import (NodesToGraphRepresentation, NodesToGraphRepresentationInput,
                                            WASGraphRepresentation, WeightedSumGraphRepresentation)
