"""One training step of the task models (tf2_gnn_b200.models) on an H100, split into its parts.

    python tools/bench_train_step.py [--steps 20] [--warmup 3] [--shapes ppi,qm9,qm9_task] [--out result.json]

Shapes:
  ppi  NodeMulticlassTask with PPI_RGCN.json's hyper-parameters: 8000 nodes in 3 graphs, 3 edge types, ~230k edges,
       H = 320, 50 features, 121 labels, Adam.
  qm9  GraphRegressionTask (default GNN: RGCN, GRU exchange, use_intermediate_gnn_results) on a QM9-like batch: ~500k nodes
       in graphs of 9-29 nodes, 4 edge types, 15 features, H = 128, RMSProp with global-norm clipping.
  qm9_task  QM9RegressionTask with QM9_RGCN.json's model parameters (8 RGCN layers, H = 128, RMSProp, value clipping) and
       out-layer dropout 0, on ~500k nodes of synthetic QM9-like molecules (9-29 atoms, a tree plus ring bonds of 4 types,
       15-wide one-hot features) written as a train fold to a temporary directory and read through QM9Dataset.
Timed with CUDA events, each over `steps` calls after `warmup`:
  step          model.train_step (forward, loss, torch.autograd.grad, optimizer step)
  fwd_bwd       forward with the task head and loss, and torch.autograd.grad over the trainable variables
  loss          the loss entries alone (forward + backward) on the step's task output
  optimizer     Optimizer.apply_gradients alone on the step's gradients
  head          qm9_task only: the gated-sum head (both Dense layers and the readout) forward and backward on the step's
                final node representations
The optimizer's line also gives its kernel launches per call and the bytes it moves (parameters, gradients and slots read,
parameters and slots written; the gradients once more for a norm reduction) over its time.  Fails without a GPU; the card's
name and power limit are read in the same run.
"""
import argparse
import gzip
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    rec = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        rec["power_limit_W"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:   # the numbers are then reported without the power limit
        rec["power_limit_W"] = f"unavailable: {type(e).__name__}"
    return rec


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def make_store(rng, sizes, F, L, edges_per_node, C=None):
    from tf2_gnn_b200.data import DeviceGraphStore
    graphs = []
    for n in sizes:
        n = int(n)
        g = {"node_features": rng.uniform(-1, 1, (n, F)).astype(np.float32),
             "adjacency_lists": [rng.integers(0, n, (int(edges_per_node * n), 2)).astype(np.int32) for _ in range(L)]}
        if C:
            g["node_labels"] = (rng.uniform(size=(n, C)) < 0.3).astype(np.float32)
        else:
            g["target_value"] = float(rng.normal(3.0, 1.0))
        graphs.append(g)
    return DeviceGraphStore(graphs, L)


# QM9_RGCN.json's model parameters (the reference's default_hypers)
QM9_RGCN = dict(gnn_residual_every_num_layers=2, gnn_num_layers=8, gnn_initial_node_representation_activation="tanh",
                gnn_dense_intermediate_layer_activation="tanh", gnn_layer_input_dropout_rate=0.0,
                gnn_message_activation_function="leaky_relu", rmsprop_rho=0.98, momentum=0.85,
                gnn_aggregation_function="sum", gnn_dense_every_num_layers=32, learning_rate=0.0005720408870458782,
                gnn_use_inter_layer_layernorm=True, gnn_hidden_dim=128, gradient_clip_value=1.0, optimizer="RMSProp")


def qm9_records(rng, num_molecules):
    """Synthetic molecules in the QM9 file format: 9-29 atoms, a random spanning tree plus up to 3 ring bonds, bond types
    1..4, one-hot features of width 15, 13 targets."""
    for _ in range(num_molecules):
        n = int(rng.integers(9, 30))
        bonds = [(int(rng.integers(0, v)), v) for v in range(1, n)]
        bonds += [tuple(int(a) for a in rng.choice(n, 2, replace=False)) for _ in range(int(rng.integers(0, 4)))]
        feats = np.zeros((n, 15), dtype=np.int64)
        feats[np.arange(n), rng.integers(0, 15, n)] = 1
        yield {"graph": [[a, int(rng.integers(1, 5)), b] for a, b in bonds], "node_features": feats.tolist(),
               "targets": [[float(rng.normal())] for _ in range(13)]}


def build(shape, rng):
    from tf2_gnn_b200.models import GraphRegressionTask, NodeMulticlassTask
    if shape == "qm9_task":
        from tf2_gnn_b200.data import DataFold, QM9Dataset
        from tf2_gnn_b200.models import QM9RegressionTask
        dataset = QM9Dataset(QM9Dataset.get_default_hyperparameters())
        with tempfile.TemporaryDirectory() as tmp:
            with gzip.open(os.path.join(tmp, "train.jsonl.gz"), "wt", compresslevel=1) as f:
                for rec in qm9_records(rng, 26_000):
                    f.write(json.dumps(rec) + "\n")
            dataset.load_data(tmp, {DataFold.TRAIN})
        store = dataset.store(DataFold.TRAIN)
        params = QM9RegressionTask.get_default_hyperparameters()
        params.update(QM9_RGCN, out_layer_dropout_keep_prob=0.0)
        desc = (f"QM9RegressionTask QM9_RGCN: {int(store.node_offsets_host[-1])} nodes in {store.num_graphs} molecules, "
                f"{store.num_edge_types} edge types, {sum(int(e.shape[0]) for e in store.edges)} edges, H=128, RMSProp + "
                f"value clip")
        return store, QM9RegressionTask(params, dataset), desc
    if shape == "ppi":
        store = make_store(rng, [2400, 3500, 2100], 50, 3, 230_000 / 8000 / 3, C=121)
        params = NodeMulticlassTask.get_default_hyperparameters("rgcn")
        params.update(gnn_num_layers=4, gnn_hidden_dim=320, gnn_use_target_state_as_input=False,
                      gnn_normalize_by_num_incoming=True, gnn_num_edge_MLP_hidden_layers=0, gnn_layer_input_dropout_rate=0.1,
                      gnn_dense_every_num_layers=10000, gnn_residual_every_num_layers=10000,
                      gnn_global_exchange_every_num_layers=10000, gnn_use_inter_layer_layernorm=False,
                      gnn_message_activation_function="ReLU", gnn_aggregation_function="sum", optimizer="Adam")
        return store, NodeMulticlassTask(params, dataset=store), "NodeMulticlassTask PPI_RGCN: 8000 nodes, ~230k edges, H=320, Adam"
    sizes = rng.integers(9, 30, size=26_000)
    store = make_store(rng, sizes, 15, 4, 1.0)
    params = GraphRegressionTask.get_default_hyperparameters()
    params.update(gnn_hidden_dim=128, optimizer="RMSProp", gradient_clip_global_norm=1.0)
    desc = f"GraphRegressionTask QM9-like: {int(sizes.sum())} nodes in {len(sizes)} graphs, H=128, RMSProp + global-norm clip"
    return store, GraphRegressionTask(params, dataset=store), desc


def bench(shape, steps, warmup):
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.models import task_ops
    rng = np.random.default_rng(0)
    torch.manual_seed(0)
    store, model, desc = build(shape, rng)
    ids = np.arange(store.num_graphs)
    feats, labels = store.batch(ids), store.batch_labels(ids)
    model.train_step(feats, labels)   # builds the model and creates the optimizer's slots
    variables = model.trainable_variables
    state = {}

    def fwd_bwd():
        out = model(feats, training=True)
        loss = model.compute_task_metrics(feats, out, labels)["loss"]
        state["out"] = out
        state["grads"] = torch.autograd.grad(loss, [v.value for v in variables], allow_unused=True)

    def loss_only():
        out = state["out"]
        x = (out[0] if isinstance(out, tuple) else out).detach().requires_grad_(True)
        if shape == "ppi":
            loss = task_ops.node_multiclass_loss(x, labels["node_labels"])[0]
        else:
            loss = task_ops.graph_regression_loss(x, labels["target_value"])[0]
        torch.autograd.grad(loss, x)

    opt = model._optimizer

    def opt_only():
        opt.apply_gradients([(g, v.value) for g, v in zip(state["grads"], variables)])

    rec = {"shape": shape, "desc": desc}
    rec["step_ms"] = timed(lambda: model.train_step(feats, labels), steps, warmup)
    rec["fwd_bwd_ms"] = timed(fwd_bwd, steps, warmup)
    rec["loss_ms"] = timed(loss_only, steps, warmup)
    before = _ffi.launch_count()
    opt_only()
    rec["optimizer_launches"] = _ffi.launch_count() - before
    rec["optimizer_ms"] = timed(opt_only, steps, warmup)
    if shape == "qm9_task":
        final = model.compute_final_node_representations(feats, True).detach().requires_grad_(True)
        head_vars = [v.value for v in model._task_variables()]

        def head_only():
            out = model.compute_task_output(feats, final, True)
            torch.autograd.grad(out.sum(), [final] + head_vars)

        rec["head_ms"] = timed(head_only, steps, warmup)
    n = sum(v.value.numel() for g, v in zip(state["grads"], variables) if g is not None)
    slots = sum(s is not None for s in opt.slots(variables[0].value))
    # read w, g and the slots, write w and the slots; a norm reduction reads g once more
    per_elem = 4 * (2 + 2 * slots + 1 + (1 if opt.clip_mode in (_ffi.CLIP_NORM, _ffi.CLIP_GLOBAL_NORM) else 0))
    rec["optimizer_elements"] = n
    rec["optimizer_bytes"] = n * per_elem
    rec["optimizer_GBps"] = n * per_elem / (rec["optimizer_ms"] * 1e-3) / 1e9
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default="ppi,qm9,qm9_task")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_step needs a CUDA device")
    result = {"card": card(), "results": []}
    for shape in args.shapes.split(","):
        rec = bench(shape, args.steps, args.warmup)
        print(json.dumps(rec), flush=True)
        result["results"].append(rec)
    print(json.dumps({"card": result["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
