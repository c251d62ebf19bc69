"""One training step of the task models (tf2_gnn_b200.models) on an H100, split into its parts.

    python tools/bench_train_step.py [--steps 20] [--warmup 3] [--shapes ppi,qm9] [--out result.json]

Shapes:
  ppi  NodeMulticlassTask with PPI_RGCN.json's hyper-parameters: 8000 nodes in 3 graphs, 3 edge types, ~230k edges,
       H = 320, 50 features, 121 labels, Adam.
  qm9  GraphRegressionTask (default GNN: RGCN, GRU exchange, use_intermediate_gnn_results) on a QM9-like batch: ~500k nodes
       in graphs of 9-29 nodes, 4 edge types, 15 features, H = 128, RMSProp with global-norm clipping.
Timed with CUDA events, each over `steps` calls after `warmup`:
  step          model.train_step (forward, loss, torch.autograd.grad, optimizer step)
  fwd_bwd       forward with the task head and loss, and torch.autograd.grad over the trainable variables
  loss          the loss entries alone (forward + backward) on the step's task output
  optimizer     Optimizer.apply_gradients alone on the step's gradients
The optimizer's line also gives its kernel launches per call and the bytes it moves (parameters, gradients and slots read,
parameters and slots written; the gradients once more for a norm reduction) over its time.  Fails without a GPU; the card's
name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

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


def build(shape, rng):
    from tf2_gnn_b200.models import GraphRegressionTask, NodeMulticlassTask
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
    ap.add_argument("--shapes", default="ppi,qm9")
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
