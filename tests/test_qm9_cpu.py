"""QM9Dataset and QM9RegressionTask without a GPU: the float64 restatement of the head (tests/reference64_qm9.py) against
torch float64 autograd; reading the fold files (1-based bond types, the target picked by task_id, the number of edge types
for both tie settings, malformed records); the task's constructor checks and the epoch metrics' string."""
import gzip
import json

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_qm9 as rq
from tf2_gnn_b200.data import DataFold, QM9Dataset
from tf2_gnn_b200.models import CHEMICAL_ACC_NORMALISING_FACTORS, QM9RegressionTask


# ---- the head's float64 restatement ---------------------------------------------------------------------------------
@pytest.mark.parametrize("sizes", [[1], [5], [1, 7, 1, 30], [300, 2, 17]])
def test_head_restatement_matches_float64_autograd(sizes):
    rng = np.random.default_rng(len(sizes))
    V, F, H, G = sum(sizes), 15, 8, len(sizes)
    n2g = np.repeat(np.arange(G), sizes)
    x0, x = rng.normal(size=(V, F)), rng.normal(size=(V, H))
    w = {"gate_kernel": rng.normal(size=(F + H, 1)), "gate_bias": rng.normal(size=(1,)),
         "transform_kernel": rng.normal(size=(H, 1)), "transform_bias": rng.normal(size=(1,))}
    grad_out = rng.normal(size=(G,))
    leaves = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in w.items()}
    z = torch.tensor(np.concatenate([x0, x], axis=1), requires_grad=True)
    xt = torch.tensor(x, requires_grad=True)
    t = xt @ leaves["transform_kernel"] + leaves["transform_bias"]
    s = z @ leaves["gate_kernel"] + leaves["gate_bias"]
    out = torch.zeros(G, dtype=torch.float64).index_add(0, torch.from_numpy(n2g), (torch.sigmoid(s) * t)[:, 0])
    np.testing.assert_allclose(rq.head_forward(x0, x, n2g, G, w), out.detach().numpy(), rtol=1e-12, atol=1e-12)
    names = ["gate_input", "transform_input"] + list(w)
    want = torch.autograd.grad(out, [z, xt] + [leaves[k] for k in w], torch.from_numpy(grad_out))
    got = rq.head_backward(x0, x, n2g, w, grad_out)
    for name, a in zip(names, want):
        np.testing.assert_allclose(got[name], a.numpy(), rtol=1e-12, atol=1e-12, err_msg=name)


# ---- reading the fold files -------------------------------------------------------------------------------------------
def _params(**kw):
    p = QM9Dataset.get_default_hyperparameters()
    p.update(kw)
    return p


def test_default_hyperparameters_are_the_reference_ones():
    assert QM9Dataset.get_default_hyperparameters() == {"max_nodes_per_batch": 10000, "add_self_loop_edges": True,
                                                         "tie_fwd_bkwd_edges": True, "task_id": 0}
    p = QM9RegressionTask.get_default_hyperparameters()
    assert p["use_intermediate_gnn_results"] is False and p["out_layer_dropout_keep_prob"] == 1.0
    assert len(CHEMICAL_ACC_NORMALISING_FACTORS) == rq.NUM_TARGETS


@pytest.mark.parametrize("tie,self_loops,want", [(True, True, 5), (False, True, 9), (True, False, 4), (False, False, 8),
                                                 ([0, 2], True, 7)])
def test_number_of_edge_types(tie, self_loops, want):
    assert QM9Dataset(_params(tie_fwd_bkwd_edges=tie, add_self_loop_edges=self_loops)).num_edge_types == want


@pytest.mark.parametrize("task_id", [0, 4, 12])
def test_records_are_read_with_one_based_types_and_the_task_target(tmp_path, task_id):
    rng = np.random.default_rng(task_id)
    recs = rq.write_dataset(str(tmp_path), rng, sizes=(7, 3, 2))
    ds = QM9Dataset(_params(task_id=task_id))
    ds.load_data(str(tmp_path), {DataFold.TRAIN, DataFold.TEST})
    with pytest.raises(KeyError):
        ds.fold(DataFold.VALIDATION)
    for fold, name in ((DataFold.TRAIN, "train.jsonl.gz"), (DataFold.TEST, "test.jsonl.gz")):
        data, rs = ds.fold(fold), recs[name]
        sizes = [len(r["node_features"]) for r in rs]
        np.testing.assert_array_equal(data.node_offsets, np.concatenate([[0], np.cumsum(sizes)]))
        np.testing.assert_array_equal(data.node_features, np.concatenate([np.asarray(r["node_features"]) for r in rs]))
        np.testing.assert_array_equal(data.target_value, np.float32([r["targets"][task_id][0] for r in rs]))
        for t in range(4):   # qm9_dataset.py:143-147, node ids offset by the graph's first row
            want = [(a + data.node_offsets[g], b + data.node_offsets[g])
                    for g, r in enumerate(rs) for a, typ, b in r["graph"] if typ == t + 1]
            np.testing.assert_array_equal(data.fwd_edges[t], np.asarray(want, np.int32).reshape(-1, 2))
    assert ds.node_feature_shape == (rq.NUM_FEATURES,)


def _write_one(tmp_path, rec):
    with gzip.open(tmp_path / "train.jsonl.gz", "wt") as f:
        f.write(json.dumps(rq.molecule(np.random.default_rng(0))) + "\n")
        f.write(json.dumps(rec) + "\n")


@pytest.mark.parametrize("edge,error", [([0, 0, 1], ValueError), ([0, 5, 1], ValueError), ([0, 1, 9], IndexError),
                                        ([-1, 2, 1], IndexError)])
def test_malformed_edges_raise(tmp_path, edge, error):
    rec = rq.molecule(np.random.default_rng(1), num_atoms=9)
    rec["graph"].append(edge)
    _write_one(tmp_path, rec)
    with pytest.raises(error):
        QM9Dataset(_params()).load_data(str(tmp_path), {DataFold.TRAIN})


@pytest.mark.parametrize("task_id", [13, -1])
def test_task_id_outside_the_targets_raises(tmp_path, task_id):
    _write_one(tmp_path, rq.molecule(np.random.default_rng(2)))
    with pytest.raises(IndexError):
        QM9Dataset(_params(task_id=task_id)).load_data(str(tmp_path), {DataFold.TRAIN})


# ---- the task model ------------------------------------------------------------------------------------------------------
def test_task_rejects_other_datasets_and_reads_the_task_id():
    class Other:
        num_edge_types = 5
    with pytest.raises(AssertionError):
        QM9RegressionTask(QM9RegressionTask.get_default_hyperparameters(), dataset=Other())
    model = QM9RegressionTask(QM9RegressionTask.get_default_hyperparameters(), dataset=QM9Dataset(_params(task_id=3)))
    assert model._task_id == 3


def test_training_with_the_default_rate_raises_before_the_forward():
    model = QM9RegressionTask(QM9RegressionTask.get_default_hyperparameters(), dataset=QM9Dataset(_params()))
    with pytest.raises(ValueError, match=r"range \[0, 1\)\. Received: rate=1\.0"):
        model.call({}, training=True)        # raises before it reads the batch


def test_epoch_metrics_string():
    model = QM9RegressionTask(QM9RegressionTask.get_default_hyperparameters(), dataset=QM9Dataset(_params(task_id=2)))
    # two batches: 3 graphs with MSE 0.5 and MAE 0.25, 1 graph with MSE 2.0 and MAE 1.5
    results = [{"loss": torch.tensor(0.5), "batch_squared_error": torch.tensor(1.5),
                "batch_absolute_error": torch.tensor(0.75), "num_graphs": 3},
               {"loss": torch.tensor(2.0), "batch_squared_error": torch.tensor(2.0),
                "batch_absolute_error": torch.tensor(1.5), "num_graphs": 1}]
    value, text = model.compute_epoch_metrics(results)
    # MSE = 3.5 / 4 = 0.875, MAE = 2.25 / 4 = 0.5625, error ratio 0.5625 / 0.071939046 = 7.8191...
    assert value == pytest.approx(0.5625)
    assert text == "Task 2 | MSE = 0.875 | MAE = 0.562 | Error Ratio: 7.819"
