"""The task-loss and optimizer entries are exported and bound, reject invalid arguments before any CUDA call with a message
naming the entry, and the model raises the reference's ValueError for conflicting clip settings.  No GPU needed."""
import ctypes

import pytest

from tf2_gnn_b200 import _ffi

ENTRIES = ("tfgnn_b200_node_multiclass_loss_fwd", "tfgnn_b200_node_multiclass_loss_bwd",
           "tfgnn_b200_graph_regression_loss_fwd", "tfgnn_b200_graph_regression_loss_bwd",
           "tfgnn_b200_graph_binary_loss_fwd", "tfgnn_b200_graph_binary_loss_bwd", "tfgnn_b200_optimizer_step")
FAKE = 0x1000   # never dereferenced: every call below fails validation first


def test_entries_are_exported_and_bound():
    lib = _ffi.lib()
    for name in ENTRIES:
        assert name in _ffi.EXPORTED_SYMBOLS
        assert getattr(lib, name).argtypes, f"{name} has no argtypes"


def _rejects(name, *args, says=None):
    lib = _ffi.lib()
    rc = getattr(lib, name)(*args)
    assert rc == _ffi.ERR_INVALID_ARGUMENT, f"{name}: rc {rc}"
    msg = lib.tfgnn_b200_last_error().decode()
    assert name in msg
    if says:
        assert says in msg
    with pytest.raises(ValueError):
        _ffi.check(rc)


def test_loss_entries_validate_sizes_and_pointers():
    _rejects("tfgnn_b200_node_multiclass_loss_fwd", FAKE, FAKE, 10, 0, FAKE, FAKE, FAKE, None, says="num_labels")
    _rejects("tfgnn_b200_node_multiclass_loss_fwd", FAKE, FAKE, -1, 3, FAKE, FAKE, FAKE, None)
    _rejects("tfgnn_b200_node_multiclass_loss_fwd", None, FAKE, 10, 3, FAKE, FAKE, FAKE, None, says="NULL")
    _rejects("tfgnn_b200_node_multiclass_loss_fwd", FAKE, FAKE, 10, 3, FAKE, None, FAKE, None, says="NULL")
    _rejects("tfgnn_b200_node_multiclass_loss_bwd", FAKE, FAKE, 10, 0, FAKE, FAKE, None, says="num_labels")
    _rejects("tfgnn_b200_node_multiclass_loss_bwd", FAKE, FAKE, 10, 3, None, FAKE, None, says="NULL")
    _rejects("tfgnn_b200_graph_regression_loss_fwd", FAKE, FAKE, -2, FAKE, FAKE, None)
    _rejects("tfgnn_b200_graph_regression_loss_fwd", FAKE, None, 4, FAKE, FAKE, None, says="NULL")
    _rejects("tfgnn_b200_graph_regression_loss_bwd", FAKE, FAKE, -2, FAKE, FAKE, None)
    _rejects("tfgnn_b200_graph_regression_loss_bwd", FAKE, FAKE, 4, FAKE, None, None, says="NULL")
    _rejects("tfgnn_b200_graph_binary_loss_fwd", FAKE, FAKE, -1, FAKE, FAKE, None)
    _rejects("tfgnn_b200_graph_binary_loss_fwd", FAKE, FAKE, 4, FAKE, None, None, says="NULL")
    _rejects("tfgnn_b200_graph_binary_loss_bwd", FAKE, FAKE, -1, FAKE, FAKE, None)
    _rejects("tfgnn_b200_graph_binary_loss_bwd", None, FAKE, 4, FAKE, FAKE, None, says="NULL")


def test_empty_backward_is_a_no_op_without_a_gpu():
    lib = _ffi.lib()
    assert lib.tfgnn_b200_node_multiclass_loss_bwd(None, None, 0, 5, None, None, None) == _ffi.OK
    assert lib.tfgnn_b200_graph_regression_loss_bwd(None, None, 0, None, None, None) == _ffi.OK
    assert lib.tfgnn_b200_graph_binary_loss_bwd(None, None, 0, None, None, None) == _ffi.OK


def _tables(n, ptr=FAKE, size=8):
    arr = lambda: (ctypes.c_void_p * max(n, 1))(*([ptr] * n))
    return arr(), arr(), arr(), arr(), (ctypes.c_int64 * max(n, 1))(*([size] * n))


def _step(kind=0, n=2, tables=None, momentum=0.9, step=0, clip_mode=0):
    p, g, a, b, s = tables or _tables(n)
    return ("tfgnn_b200_optimizer_step", kind, n, p, g, a, b, s, 0.01, momentum, 0.9, step, clip_mode, 1.0, None)


def test_optimizer_step_validates_every_argument():
    _rejects(*_step(kind=7), says="kind")
    _rejects(*_step(clip_mode=9), says="clip mode")
    _rejects(*_step(n=-1), says="negative")
    _rejects(*_step(step=-3), says="negative")
    p, g, a, b, s = _tables(2)
    _rejects("tfgnn_b200_optimizer_step", 2, 2, None, g, a, b, s, 0.01, 0.0, 0.9, 0, 0, 0.0, None, says="NULL")
    _rejects("tfgnn_b200_optimizer_step", 2, 2, p, g, a, None, s, 0.01, 0.0, 0.9, 0, 0, 0.0, None, says="slot")
    neg = (ctypes.c_int64 * 2)(4, -1)
    _rejects("tfgnn_b200_optimizer_step", 0, 2, p, g, a, b, neg, 0.01, 0.9, 0.9, 0, 0, 0.0, None, says="negative tensor size")
    g0 = (ctypes.c_void_p * 2)(FAKE, None)
    _rejects("tfgnn_b200_optimizer_step", 2, 2, p, g0, a, b, s, 0.01, 0.0, 0.9, 0, 0, 0.0, None, says="NULL")


def test_optimizer_step_with_nothing_to_update_is_a_no_op():
    lib = _ffi.lib()
    assert lib.tfgnn_b200_optimizer_step(*_step(n=0)[1:]) == _ffi.OK
    p, g, a, b, s = _tables(3, ptr=None, size=0)   # size-0 tensors: NULL pointers are fine, nothing is launched
    before = _ffi.launch_count()
    assert lib.tfgnn_b200_optimizer_step(2, 3, p, g, a, b, s, 0.01, 0.0, 0.9, 0, 3, 1.0, None) == _ffi.OK
    assert _ffi.launch_count() == before


class _Dataset:
    num_edge_types = 3
    num_node_target_labels = 4


@pytest.mark.parametrize("clips", [("gradient_clip_value", "gradient_clip_norm"),
                                   ("gradient_clip_value", "gradient_clip_global_norm"),
                                   ("gradient_clip_norm", "gradient_clip_global_norm")])
def test_conflicting_clip_settings_raise_value_error(clips):
    from tf2_gnn_b200.models import NodeMulticlassTask
    params = NodeMulticlassTask.get_default_hyperparameters()
    params.update({c: 1.0 for c in clips})
    model = NodeMulticlassTask(params, dataset=_Dataset())
    with pytest.raises(ValueError, match="can only use one at a time"):
        model._apply_gradients([])


def test_unknown_optimizer_and_defaults():
    from tf2_gnn_b200.models import GraphRegressionTask, NodeMulticlassTask
    params = GraphRegressionTask.get_default_hyperparameters()
    assert params["optimizer"] == "Adam" and params["learning_rate"] == 0.001 and params["use_intermediate_gnn_results"]
    assert params["gnn_message_calculation_class"] == "rgcn" and params["regression_mlp_layers"] == [64, 32]
    params["optimizer"] = "Adagrad"
    with pytest.raises(Exception, match="Unknown optimizer"):
        GraphRegressionTask(params, dataset=_Dataset())._make_optimizer()
    with pytest.raises(ValueError, match="num_node_target_labels"):
        NodeMulticlassTask(NodeMulticlassTask.get_default_hyperparameters(), dataset=type("D", (), {"num_edge_types": 1})())
