"""QM9Dataset and QM9RegressionTask on the GPU, on seeded synthetic molecules in the QM9 file format: the fold's store
against the reference's per-molecule process_adjacency_lists, the head's forward and gradients against float64 at ~500k
nodes and at its edge cases, one train_step with QM9_RGCN.json's hyper-parameters against the float64 optimizer applied to
the model's autograd gradients, bitwise reproducibility with out-layer dropout, the default rate (inference runs, training
raises before any launch) and the reference's test_train_improvement restated for QM9."""
import random

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_qm9 as rq
import reference64_task as rt
from oracle import adjacency_oracle as ao
from reference64_qm9 import QM9_RGCN

pytestmark = pytest.mark.gpu
LOSS_TOL = 3e-5       # the bars of test_gpu_task_models.py
OPT_TOL = 1e-6


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def normwise(got, ref, tol, what=""):
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    err = np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30)
    assert err <= tol, f"{what}: norm-wise error {err:.3e} > {tol:g}"


def _dataset(tmp_path, seed=0, sizes=(200, 50, 50), **params):
    from tf2_gnn_b200.data import QM9Dataset
    records = rq.write_dataset(str(tmp_path), np.random.default_rng(seed), sizes)
    p = QM9Dataset.get_default_hyperparameters()
    p.update(params)
    ds = QM9Dataset(p)
    ds.load_data(str(tmp_path))
    return ds, records


def _model(ds, **hyper):
    from tf2_gnn_b200.models import QM9RegressionTask
    params = QM9RegressionTask.get_default_hyperparameters()
    params.update(hyper)
    return QM9RegressionTask(params, ds)


# ---- 1. the fold's store --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie,self_loops", [(True, True), (False, True), ([1, 3], False)])
def test_store_lists_match_the_reference_graph_by_graph(tmp_path, tie, self_loops):
    _need_gpu()
    from tf2_gnn_b200.data import DataFold
    ds, records = _dataset(tmp_path, 1, (120, 10, 10), tie_fwd_bkwd_edges=tie, add_self_loop_edges=self_loops)
    store = ds.store(DataFold.TRAIN)
    assert store is ds.store(DataFold.TRAIN) and store.num_edge_types == ds.num_edge_types
    tied = ao.get_tied_edge_types(tie, 4)
    edges = [e.cpu().numpy() for e in store.edges]
    feats = store.node_features.cpu().numpy()
    no = store.node_offsets_host
    for g, rec in enumerate(records["train.jsonl.gz"]):
        n = len(rec["node_features"])
        raw = [[(a, b) for a, t, b in rec["graph"] if t == k + 1] for k in range(4)]
        want, _ = ao.process_adjacency_lists(raw, n, self_loops, tied)
        assert len(want) == ds.num_edge_types
        for t in range(ds.num_edge_types):
            eo = store.edge_offsets_host[t]
            np.testing.assert_array_equal(edges[t][eo[g]:eo[g + 1]], want[t], err_msg=f"graph {g} type {t}")
        np.testing.assert_array_equal(feats[no[g]:no[g + 1]], np.asarray(rec["node_features"], np.float32))
    np.testing.assert_array_equal(store.target_value.cpu().numpy(),
                                  np.float32([r["targets"][0][0] for r in records["train.jsonl.gz"]]))


# ---- 2. the head against float64 ------------------------------------------------------------------------------------
def _head_case(sizes, seed):
    from tf2_gnn_b200.data import QM9Dataset
    rng = np.random.default_rng(seed)
    F, H = rq.NUM_FEATURES, 128
    ds = QM9Dataset(QM9Dataset.get_default_hyperparameters())
    model = _model(ds, gnn_hidden_dim=H, out_layer_dropout_keep_prob=0.0)
    shapes = {"node_features": (None, F)}
    shapes.update({f"adjacency_list_{t}": (None, 2) for t in range(ds.num_edge_types)})
    model.build(shapes)
    for v in model._task_variables():          # non-zero biases and gates away from 1/2
        v.value.data.copy_(torch.from_numpy(rng.normal(0, 0.5, tuple(v.value.shape)).astype(np.float32)))
    V, G = int(sum(sizes)), len(sizes)
    n2g = np.repeat(np.arange(G), sizes).astype(np.int32)
    x0 = rng.uniform(-1, 1, (V, F)).astype(np.float32)
    x = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    batch = {"node_features": torch.from_numpy(x0).cuda().requires_grad_(True),
             "node_to_graph_map": torch.from_numpy(n2g).cuda(), "num_graphs_in_batch": G}
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    out = model.compute_task_output(batch, xt, training=True)
    grad_out = rng.normal(size=G).astype(np.float32)
    gate, transform = model._regression_gate, model._regression_transform
    variables = [gate.kernels[0], gate.biases[0], transform.kernels[0], transform.biases[0]]
    grads = torch.autograd.grad(out, [batch["node_features"], xt] + [v.value for v in variables],
                                torch.from_numpy(grad_out).cuda())
    w = {k: v.value.detach().double().cpu().numpy()
         for k, v in zip(("gate_kernel", "gate_bias", "transform_kernel", "transform_bias"), variables)}
    normwise(out.detach().cpu().numpy(), rq.head_forward(x0, x, n2g, G, w), LOSS_TOL, "forward")
    ref = rq.head_backward(x0, x, n2g, w, grad_out)
    normwise(grads[0].cpu().numpy(), ref["gate_input"][:, :F], LOSS_TOL, "node_features")
    normwise(grads[1].cpu().numpy(), ref["transform_input"] + ref["gate_input"][:, F:], LOSS_TOL, "final representations")
    for g, name in zip(grads[2:], w):
        normwise(g.cpu().numpy(), ref[name], LOSS_TOL, name)
    with torch.no_grad():                      # the inference forward gives the training forward's bits
        assert torch.equal(model.compute_task_output(batch, xt, training=False), out)


@pytest.mark.parametrize("case", ["qm9_500k", "one_node_graph", "one_graph", "longer_than_a_chunk"])
def test_head_matches_float64(case):
    _need_gpu()
    rng = np.random.default_rng(11)
    sizes = {"qm9_500k": rng.integers(9, 30, 26_000),           # ~500k nodes
             "one_node_graph": [1, 12, 1, 1, 20, 1],
             "one_graph": [23],
             "longer_than_a_chunk": [3, 1000, 5, 257, 256]}[case]   # the readout's row chunk is 256 rows
    _head_case(list(sizes), 3)


# ---- 3. train_step against the float64 optimizer ----------------------------------------------------------------------
def test_train_step_applies_the_float64_optimizer_to_the_autograd_gradients(tmp_path):
    _need_gpu()
    from tf2_gnn_b200.data import DataFold
    torch.manual_seed(5)
    ds, _ = _dataset(tmp_path, 5, (60, 5, 5))
    store = ds.store(DataFold.TRAIN)
    model = _model(ds, **QM9_RGCN, out_layer_dropout_keep_prob=0.1)
    ids = np.arange(store.num_graphs)
    feats, labels = store.batch(ids), store.batch_labels(ids)
    model(feats, training=False)                                    # build
    variables = model.trainable_variables
    w0 = [v.value.detach().double().cpu().numpy() for v in variables]
    off = model.dropout_state.offset
    out = model(feats, training=True)
    loss = model.compute_task_metrics(feats, out, labels)["loss"]
    grads = torch.autograd.grad(loss, [v.value for v in variables], allow_unused=True)
    grads = [None if g is None else g.double().cpu().numpy() for g in grads]
    assert sum(g is not None for g in grads) >= len(variables) - 2
    model.dropout_state.offset = off                                # the step draws the same dropout masks
    model.train_step(feats, labels)
    p = model._params
    ref = rt.Optimizer64("rmsprop", p["learning_rate"], momentum=p["momentum"], rho=p["rmsprop_rho"], clip_mode="value",
                         clip=p["gradient_clip_value"])
    ref.apply(w0, grads)
    for v, r in zip(variables, w0):
        normwise(v.value.detach().cpu().numpy(), r, OPT_TOL, v.name)


# ---- 4. bitwise reproducibility --------------------------------------------------------------------------------------
def test_two_models_from_one_seed_stay_bitwise_equal_with_dropout(tmp_path):
    _need_gpu()
    from tf2_gnn_b200.data import DataFold
    ds, _ = _dataset(tmp_path, 6, (80, 5, 5))
    store = ds.store(DataFold.TRAIN)
    ids = np.arange(store.num_graphs)

    def run():
        torch.manual_seed(6)
        model = _model(ds, **QM9_RGCN, out_layer_dropout_keep_prob=0.2)
        losses = [model.train_step(store.batch(ids), store.batch_labels(ids))["loss"].item() for _ in range(3)]
        return losses, [v.value.detach().cpu().numpy() for v in model.trainable_variables]

    l1, w1 = run()
    l2, w2 = run()
    assert l1 == l2
    for a, b in zip(w1, w2):
        assert np.array_equal(a, b)


# ---- 5. the default rate ----------------------------------------------------------------------------------------------
def test_default_rate_runs_at_inference_and_raises_before_any_launch_in_training(tmp_path):
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.data import DataFold
    torch.manual_seed(7)
    ds, _ = _dataset(tmp_path, 7, (30, 5, 5))
    store = ds.store(DataFold.TRAIN)
    model = _model(ds)                                 # out_layer_dropout_keep_prob = 1.0, the reference's default
    ids = np.arange(store.num_graphs)
    feats, labels = store.batch(ids), store.batch_labels(ids)
    preds = model.predict(store, store.iter_batch_graph_ids(100))
    assert preds.shape == (store.num_graphs,) and bool(torch.isfinite(preds).all())
    _, _, results = model.run_one_epoch(store, store.iter_batch_graph_ids(100), training=False)
    mae, text = model.compute_epoch_metrics(results)
    assert np.isfinite(mae) and text.startswith("Task 0 | MSE = ")
    w = [v.value.detach().clone() for v in model.trainable_variables]
    torch.cuda.synchronize()
    before, offset = _ffi.launch_count(), model.dropout_state.offset
    with pytest.raises(ValueError, match=r"range \[0, 1\)\. Received: rate=1\.0"):
        model.train_step(feats, labels)
    assert _ffi.launch_count() == before and model.dropout_state.offset == offset
    assert all(torch.equal(a, v.value) for a, v in zip(w, model.trainable_variables))


# ---- 6. the reference's test_train_improvement (tf2_gnn/test/models/test_graph_regression_task.py:93-138) ---------------
def test_train_improvement(tmp_path):
    _need_gpu()
    from tf2_gnn_b200.data import DataFold
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    ds, _ = _dataset(tmp_path, 8, (600, 100, 10))
    train, valid = ds.store(DataFold.TRAIN), ds.store(DataFold.VALIDATION)
    model = _model(ds, **dict(QM9_RGCN, gnn_num_layers=4, learning_rate=0.001), out_layer_dropout_keep_prob=0.0)

    def epoch(store, training):
        order = np.random.permutation(store.num_graphs) if training else None
        loss, _, results = model.run_one_epoch(store, store.iter_batch_graph_ids(2000, order), training=training)
        return loss, model.compute_epoch_metrics(results)[0]

    valid0 = epoch(valid, False)
    for _ in range(3):
        epoch(train, True)
    valid1 = epoch(valid, False)
    assert valid1[1] < valid0[1], (valid0, valid1)
    assert valid1[0] < valid0[0], (valid0, valid1)
