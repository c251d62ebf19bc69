"""Task losses, the optimizer step and the task models (tf2_gnn.models) on the GPU: every loss entry against float64 at PPI
shape and at its edge cases, five steps of every optimizer x clip mode against the float64 Keras rules, one train_step of
NodeMulticlassTask and GraphRegressionTask against the float64 optimizer applied to the model's autograd gradients, bitwise
reproducibility, and the reference's test_train_improvement restated on its JSONL data (tests/golden/*.jsonl.gz)."""
import gzip
import json
import math
import os
import random

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_task as rt

pytestmark = pytest.mark.gpu
LOSS_TOL = 3e-5
OPT_TOL = 1e-6
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def normwise(got, ref, tol, what=""):
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    den = max(np.linalg.norm(ref), 1e-30)
    err = np.linalg.norm(got - ref) / den
    assert err <= tol, f"{what}: norm-wise error {err:.3e} > {tol:g}"


def _cuda(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a), dtype=dtype).cuda()


# ---- losses -------------------------------------------------------------------------------------------------------
def _node_loss_case(x, y):
    from tf2_gnn_b200.models import task_ops
    xt = _cuda(x).requires_grad_(True)
    loss, f1, counts = task_ops.node_multiclass_loss(xt, _cuda(y))
    (grad,) = torch.autograd.grad(loss, xt)
    ref_loss, ref_grad, ref_counts, ref_f1 = rt.node_multiclass_loss(x, y)
    assert tuple(counts.cpu().tolist()) == ref_counts
    if math.isnan(ref_f1):
        assert math.isnan(float(f1))
    else:
        assert float(f1) == pytest.approx(ref_f1, rel=1e-6)
    if x.shape[0] == 0:
        assert math.isnan(float(loss)) and grad.shape == (0, x.shape[1])
        return
    normwise([float(loss)], [ref_loss], LOSS_TOL, "node loss")
    normwise(grad.cpu().numpy(), ref_grad, LOSS_TOL, "node grad")


def test_node_multiclass_loss_at_ppi_shape():
    _need_gpu()
    rng = np.random.default_rng(0)
    x = rng.normal(0, 4, (8000, 121)).astype(np.float32)
    y = (rng.uniform(size=(8000, 121)) < 0.3).astype(np.float32)
    _node_loss_case(x, y)


@pytest.mark.parametrize("case", ["saturated", "zero_logits", "zero_labels", "one_node", "no_nodes"])
def test_node_multiclass_loss_edge_cases(case):
    _need_gpu()
    rng = np.random.default_rng(1)
    x = rng.normal(0, 2, (300, 7)).astype(np.float32)
    y = (rng.uniform(size=(300, 7)) < 0.5).astype(np.float32)
    if case == "saturated":
        x = np.where(rng.uniform(size=x.shape) < 0.5, 80.0, -80.0).astype(np.float32)
    elif case == "zero_logits":
        x[:, :3] = 0.0                           # sigmoid(0) = 0.5 rounds to 0 (half to even)
    elif case == "zero_labels":
        y[:] = 0.0                               # tp == 0: F1 is NaN, as in the reference
    elif case == "one_node":
        x, y = x[:1], y[:1]
    else:
        x, y = x[:0], y[:0]
    _node_loss_case(x, y)


@pytest.mark.parametrize("G", [1, 7, 5000])
def test_graph_regression_loss(G):
    _need_gpu()
    from tf2_gnn_b200.models import task_ops
    rng = np.random.default_rng(G)
    p, t = rng.normal(size=G).astype(np.float32), rng.normal(size=G).astype(np.float32)
    pt = _cuda(p).requires_grad_(True)
    mse, mae = task_ops.graph_regression_loss(pt, _cuda(t))
    (grad,) = torch.autograd.grad(mse, pt)
    ref_mse, ref_mae, ref_grad = rt.graph_regression_loss(p, t)
    normwise([float(mse), float(mae)], [ref_mse, ref_mae], LOSS_TOL, "mse, mae")
    normwise(grad.cpu().numpy(), ref_grad, LOSS_TOL, "grad pred")


@pytest.mark.parametrize("G", [1, 9, 5000])
def test_graph_binary_loss(G):
    _need_gpu()
    from tf2_gnn_b200.models import task_ops
    rng = np.random.default_rng(G + 1)
    p = rng.uniform(0, 1, G).astype(np.float32)
    if G > 4:
        p[:4] = [0.0, 1.0, 1e-9, 0.5]           # clipped at both ends, and a tie that rounds to 0
    t = (rng.uniform(size=G) < 0.5).astype(np.float32)
    pt = _cuda(p).requires_grad_(True)
    loss, correct = task_ops.graph_binary_loss(pt, _cuda(t))
    (grad,) = torch.autograd.grad(loss, pt)
    ref_loss, ref_grad, ref_correct = rt.graph_binary_loss(p, t)
    assert int(correct) == ref_correct
    normwise([float(loss)], [ref_loss], LOSS_TOL, "bce")
    normwise(grad.cpu().numpy(), ref_grad, LOSS_TOL, "grad prob")
    if G > 4:
        assert (grad[:3] == 0).all()


def test_empty_graph_batches_give_nan_losses():
    _need_gpu()
    from tf2_gnn_b200.models import task_ops
    e = torch.zeros(0, device="cuda")
    assert all(math.isnan(float(v)) for v in task_ops.graph_regression_loss(e, e))
    loss, correct = task_ops.graph_binary_loss(e, e)
    assert math.isnan(float(loss)) and int(correct) == 0


# ---- optimizer ----------------------------------------------------------------------------------------------------
# GNN-shaped variables: RGCN kernels, a non-multiple-of-4 Dense, a size-1 bias, a GRU bias, one without a gradient
SHAPES = [(64, 64), (64, 64), (50, 64), (64, 121), (121,), (1,), (2, 3 * 17), (33, 7), (5,)]
NO_GRAD = 8


def _run_optimizer(kind, clip_mode, clip, steps=5, seed=0, momentum=0.85):
    from tf2_gnn_b200.models import Optimizer
    rng = np.random.default_rng(seed)
    w0 = [rng.normal(0, 0.3, s).astype(np.float32) for s in SHAPES]
    grads = [[None if i == NO_GRAD else rng.normal(0, 1.0 + i, s).astype(np.float32) for i, s in enumerate(SHAPES)]
             for _ in range(steps)]
    kw = {{"value": "clip_value", "norm": "clip_norm", "global_norm": "clip_global_norm"}[clip_mode]: clip} if clip_mode else {}
    opt = Optimizer(kind, lambda step: 1e-2 / (1 + step), momentum=momentum, rho=0.98, **kw)
    ws = [_cuda(w) for w in w0]
    for gs in grads:
        opt.apply_gradients([(None if g is None else _cuda(g), w) for g, w in zip(gs, ws)])
    ref = rt.Optimizer64(kind, lambda step: 1e-2 / (1 + step), momentum=momentum if kind != "adam" else 0.0, rho=0.98,
                         clip_mode=clip_mode, clip=clip)
    wr = [w.astype(np.float64) for w in w0]
    for gs in grads:
        ref.apply(wr, gs)
    return [w.cpu().numpy() for w in ws], wr, w0


@pytest.mark.parametrize("clip_mode,clip", [(None, 0.0), ("value", 0.7), ("norm", 5.0), ("global_norm", 20.0)])
@pytest.mark.parametrize("kind", ["sgd", "rmsprop", "adam"])
def test_optimizer_five_steps_match_float64(kind, clip_mode, clip):
    _need_gpu()
    got, ref, w0 = _run_optimizer(kind, clip_mode, clip)
    for i, (g, r) in enumerate(zip(got, ref)):
        normwise(g, r, OPT_TOL, f"{kind}/{clip_mode} variable {i} {SHAPES[i]}")
    np.testing.assert_array_equal(got[NO_GRAD], w0[NO_GRAD])
    again, _, _ = _run_optimizer(kind, clip_mode, clip)
    for a, b in zip(got, again):
        assert np.array_equal(a, b), "optimizer step is not bitwise reproducible"


@pytest.mark.parametrize("kind", ["sgd", "rmsprop"])
def test_momentum_free_optimizers_match_float64(kind):
    _need_gpu()
    got, ref, _ = _run_optimizer(kind, "global_norm", 20.0, momentum=0.0)
    for i, (g, r) in enumerate(zip(got, ref)):
        normwise(g, r, OPT_TOL, f"{kind} momentum 0 variable {i}")


def test_optimizer_launches_once_and_once_more_for_norms():
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.models import Optimizer
    ws = [torch.randn(s, device="cuda") for s in SHAPES]
    for clip, launches in ((None, 1), ("clip_norm", 2), ("clip_global_norm", 2)):
        opt = Optimizer("adam", 1e-3, **({clip: 1.0} if clip else {}))
        before = _ffi.launch_count()
        opt.apply_gradients([(torch.randn_like(w), w) for w in ws])
        assert _ffi.launch_count() - before == launches


# ---- models -------------------------------------------------------------------------------------------------------
def _synthetic_store(rng, num_graphs, node_range, F, L, C=None, edges_per_node=4):
    from tf2_gnn_b200.data import DeviceGraphStore
    graphs = []
    for _ in range(num_graphs):
        n = int(rng.integers(*node_range))
        s = {"node_features": rng.uniform(-1, 1, (n, F)).astype(np.float32),
             "adjacency_lists": [rng.integers(0, n, (edges_per_node * n, 2)).astype(np.int32) for _ in range(L)]}
        if C:
            s["node_labels"] = (rng.uniform(size=(n, C)) < 0.3).astype(np.float32)
        else:
            s["target_value"] = float(rng.normal(3.0, 1.0))
        graphs.append(s)
    return DeviceGraphStore(graphs, L)


def _node_model(store, dropout):
    from tf2_gnn_b200.models import NodeMulticlassTask
    params = NodeMulticlassTask.get_default_hyperparameters("rgcn")
    params.update(gnn_hidden_dim=64, gnn_num_layers=3, gnn_global_exchange_every_num_layers=10000,
                  gnn_layer_input_dropout_rate=dropout, optimizer="Adam", learning_rate=0.005)
    return NodeMulticlassTask(params, dataset=store)


def _regression_model(store, dropout):
    from tf2_gnn_b200.models import GraphRegressionTask
    params = GraphRegressionTask.get_default_hyperparameters()   # rgcn, 4 layers, GRU exchange every 2 layers
    params.update(optimizer="RMSProp", gradient_clip_global_norm=1.0, learning_rate=0.002)
    if not dropout:
        params.update(gnn_global_exchange_dropout_rate=0.0, graph_aggregation_dropout_rate=0.0, regression_mlp_dropout=0.0)
    return GraphRegressionTask(params, dataset=store)


@pytest.mark.parametrize("task", ["node_multiclass", "graph_regression"])
def test_train_step_applies_the_float64_optimizer_to_the_autograd_gradients(task):
    _need_gpu()
    rng = np.random.default_rng(5)
    torch.manual_seed(5)
    if task == "node_multiclass":
        store = _synthetic_store(rng, 3, (250, 400), 50, 3, C=121)
        model = _node_model(store, 0.1)
    else:
        store = _synthetic_store(rng, 40, (9, 30), 15, 3)
        model = _regression_model(store, True)
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
    ref = rt.Optimizer64(p["optimizer"].lower(), p["learning_rate"], momentum=p["momentum"], rho=p["rmsprop_rho"],
                         clip_mode="global_norm" if p["gradient_clip_global_norm"] else None,
                         clip=p["gradient_clip_global_norm"] or 0.0)
    ref.apply(w0, grads)
    for v, r in zip(variables, w0):
        normwise(v.value.detach().cpu().numpy(), r, OPT_TOL, v.name)


@pytest.mark.parametrize("task", ["node_multiclass", "graph_regression"])
def test_two_models_from_one_seed_stay_bitwise_equal_with_dropout(task):
    _need_gpu()

    def run():
        rng = np.random.default_rng(6)
        torch.manual_seed(6)
        if task == "node_multiclass":
            store = _synthetic_store(rng, 3, (250, 400), 50, 3, C=121)
            model = _node_model(store, 0.2)
        else:
            store = _synthetic_store(rng, 40, (9, 30), 15, 3)
            model = _regression_model(store, True)
        ids = np.arange(store.num_graphs)
        losses = [float(model.train_step(store.batch(ids), store.batch_labels(ids))["loss"]) for _ in range(3)]
        return losses, [v.value.detach().cpu().numpy() for v in model.trainable_variables]

    l1, w1 = run()
    l2, w2 = run()
    assert l1 == l2
    for a, b in zip(w1, w2):
        assert np.array_equal(a, b)


def test_store_labels_follow_the_batch_rows():
    _need_gpu()
    rng = np.random.default_rng(7)
    store = _synthetic_store(rng, 6, (3, 9), 4, 2, C=5)
    ids = np.array([4, 1, 3])
    feats, labels = store.batch(ids), store.batch_labels(ids)
    no = store.node_offsets_host
    rows = np.concatenate([np.arange(no[g], no[g + 1]) for g in ids])
    np.testing.assert_array_equal(labels["node_labels"].cpu().numpy(), store.node_labels.cpu().numpy()[rows])
    assert set(feats) == {"node_features", "node_to_graph_map", "num_graphs_in_batch", "adjacency_list_0", "adjacency_list_1"}
    assert store.num_node_target_labels == 5 and store.num_edge_types == 2
    reg = _synthetic_store(rng, 6, (3, 9), 4, 2)
    np.testing.assert_array_equal(reg.batch_labels(ids)["target_value"].cpu().numpy(), reg.target_value.cpu().numpy()[ids])


# ---- the reference's test_train_improvement (tf2_gnn/test/models/test_graph_regression_task.py:93-138) ---------------
def _load_jsonl(name, binary_threshold=None):
    """JsonLGraphPropertyDataset defaults: 3 forward edge types tied to their backward edges, self loops."""
    from tf2_gnn_b200.data import get_tied_edge_types, process_adjacency_lists
    tied = get_tied_edge_types(True, 3)
    num_edge_types = 2 * 3 - len(tied) + 1
    samples = []
    with gzip.open(os.path.join(GOLDEN, name), "rt") as f:
        for line in f:
            d = json.loads(line)
            nf = d["graph"]["node_features"]
            adjs, _ = process_adjacency_lists(d["graph"]["adjacency_lists"], len(nf), True, tied)
            target = float(d["Property"])
            if binary_threshold is not None:
                target = float(target > binary_threshold)
            samples.append({"node_features": nf, "adjacency_lists": [a.cpu().numpy() for a in adjs[:num_edge_types]],
                            "target_value": target})
    return samples, num_edge_types


def _jsonl_stores(binary=False):
    from tf2_gnn_b200.data import DeviceGraphStore
    threshold = None
    if binary:
        with gzip.open(os.path.join(GOLDEN, "train.jsonl.gz"), "rt") as f:
            threshold = float(np.median([float(json.loads(l)["Property"]) for l in f]))
    train, T = _load_jsonl("train.jsonl.gz", threshold)
    valid, _ = _load_jsonl("valid.jsonl.gz", threshold)
    return DeviceGraphStore(train, T), DeviceGraphStore(valid, T)


def _epoch(model, store, training):
    order = np.random.permutation(store.num_graphs) if training else None
    return model.run_one_epoch(store, store.iter_batch_graph_ids(10000, order), training=training)


def test_train_improvement():
    _need_gpu()
    from tf2_gnn_b200.models import GraphRegressionTask
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    train, valid = _jsonl_stores()
    model = GraphRegressionTask(GraphRegressionTask.get_default_hyperparameters(), dataset=train)
    valid0_loss, _, valid0_results = _epoch(model, valid, False)
    valid0_metric, _ = model.compute_epoch_metrics(valid0_results)
    train1_loss, _, train1_results = _epoch(model, train, True)
    train1_metric, _ = model.compute_epoch_metrics(train1_results)
    valid1_loss, _, valid1_results = _epoch(model, valid, False)
    valid1_metric, _ = model.compute_epoch_metrics(valid1_results)
    assert valid0_loss > valid1_loss
    assert valid0_metric > valid1_metric
    train2_loss, _, train2_results = _epoch(model, train, True)
    train2_metric, _ = model.compute_epoch_metrics(train2_results)
    assert train1_loss > train2_loss
    assert train1_metric > train2_metric


def test_binary_classification_train_improvement():
    _need_gpu()
    from tf2_gnn_b200.models import GraphBinaryClassificationTask
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    train, _ = _jsonl_stores(binary=True)
    model = GraphBinaryClassificationTask(GraphBinaryClassificationTask.get_default_hyperparameters(), dataset=train)
    losses = [_epoch(model, train, True)[0] for _ in range(5)]
    assert losses[-1] < losses[0], losses
    _, _, results = _epoch(model, train, False)
    acc = -model.compute_epoch_metrics(results)[0]
    assert 0.0 <= acc <= 1.0
    preds = model.predict(train, train.iter_batch_graph_ids(10000))
    assert preds.shape == (train.num_graphs,) and ((preds >= 0) & (preds <= 1)).all()
