"""Multi-GPU check + timing of the target-range sharded path (SURVEY.md §8e case 2) over NCCL.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29533 \
        tools/run_sharded_nccl.py [--nodes 1000000 --edges-per-type 5000000 --types 4 --hidden 256 --layers 2]

Every rank builds the same seeded graph, owns one target range (tfgnn_b200_prepare_sharded on the FULL edge
lists), and runs `layers` RGCN layers with ONE all-gather of the node-state shards per layer
(torch.distributed.all_gather_into_tensor, NCCL over NVLink).  Rank 0 also runs the unsharded layers and
checks the gathered result against it, then prints one JSON line with per-layer times (max over ranks).

With --train every step runs the layers forward AND backward (DESIGN.md §6): sharding.gather_node_states (all-gather
forward, reduce-scatter backward) under sharding.regather_saved_tables() (a rank keeps only its own rows of each layer's
input until backward), weight gradients summed with all_reduce.  Rank 0 checks the input and weight gradients against
unsharded autograd on its own GPU; the JSON line reports ms per step (max over ranks) and each rank's peak
torch.cuda.max_memory_allocated.

With --stack every step trains a whole GNN (GNN.get_default_hyperparameters(): RGCN layers, a GRU global exchange every
second layer with its readout merged over the ranks in rank order; every step restarts the dropout stream so that rank 0
can compare with the same masks) on the
rank's target range (`GNN(..., shard=sharding.TargetRangeShard(bounds, rank))`), sums the weight gradients with
sharding.sum_gradients_over_ranks and checks on rank 0 the output rows and every gradient against unsharded autograd, and
that every rank holds the same weight-gradient bits.  The graph is --graphs graphs of equal size, so that cuts fall inside
graphs.  Multi-GPU step times of this mode are reported by the tool but have not been measured for the documentation.

With --task node|regression every step is a training step of a task model on target-range shards (DESIGN.md §6 "Task
models on shards"): NodeMulticlassTask with PPI_RGCN.json's layers on PPI-sized graphs, or GraphRegressionTask with its
defaults on --task-graphs QM9-sized graphs, all in one batch.  Every rank builds the same seeded store, takes rank 0's
weights (sharding.broadcast_variables), assembles its rows (store.shard_batch over store.shard_bounds) and runs
train_step(shard=...).  Rank 0 also runs the unsharded steps and checks the losses of every step and the gradients of the
first step at the test bar (3e-5 norm-wise), and the JSON line says whether every rank holds the same variable bits at the
end.  Multi-GPU times of this mode are not measured for the documentation.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tf2_gnn_b200 import sharding  # noqa: E402
from tf2_gnn_b200.layers import MessagePassingInput, RGCN  # noqa: E402
from tf2_gnn_b200.runtime import PreparedBatch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=400_000)
    ap.add_argument("--edges-per-type", type=int, default=2_000_000)
    ap.add_argument("--types", type=int, default=4)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--train", action="store_true", help="forward + backward per step (gradient check on rank 0)")
    ap.add_argument("--stack", action="store_true", help="train a whole GNN stack with global exchange (check on rank 0)")
    ap.add_argument("--graphs", type=int, default=64, help="--stack: number of equal-size graphs in the node table")
    ap.add_argument("--task", choices=("node", "regression"), help="train a task model on shards (check on rank 0)")
    ap.add_argument("--task-graphs", type=int, default=0,
                    help="--task: graphs in the batch (default: 24 PPI-sized node-task graphs, 2000 QM9-sized graphs)")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    if args.task:
        return train_task(args, rank, world)
    V, L, H = args.nodes, args.types, args.hidden
    rng = np.random.default_rng(7)
    adjs = [rng.integers(0, V, size=(args.edges_per_type, 2), dtype=np.int32) for _ in range(L)]
    h0 = (rng.random((V, H), dtype=np.float32) * 2 - 1)
    lim = np.sqrt(6.0 / (2 * H))
    ws = [[((rng.random((H, H), dtype=np.float32) * 2 - 1) * lim) for _ in range(L)] for _ in range(args.layers)]
    deg = sum(np.bincount(a[:, 1], minlength=V) for a in adjs)
    bounds = sharding.partition_target_range(V, world, deg)
    lo, hi = bounds[rank]
    if args.stack:
        return train_stack(args, rank, world, bounds, adjs, h0)
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    params = RGCN.get_default_hyperparameters()
    params["hidden_dim"] = H
    layers = []
    for w in ws:
        layer = RGCN(params)
        layer.build(MessagePassingInput((None, H), tuple((None, 2) for _ in range(L))))
        layer.set_weights_from_oracle_dict({"edge_mlps": [[x] for x in w]})
        layers.append(layer)
    shard = PreparedBatch(adj_dev, V, target_range=(lo, hi))
    h_local0 = torch.from_numpy(h0[lo:hi]).cuda()
    if args.train:
        return train(args, rank, world, bounds, layers, adj_dev, shard, h0, h_local0)

    def forward_sharded():
        h_local = h_local0
        for layer in layers:
            h_full = sharding.all_gather_node_states(h_local, bounds)          # one collective per layer
            h_local = layer(MessagePassingInput(h_full, adj_dev), prepared=shard)
        return h_local

    out_local = forward_sharded()
    torch.cuda.synchronize()
    dist.barrier()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.steps):
        out_local = forward_sharded()
    ev1.record()
    torch.cuda.synchronize()
    t = torch.tensor([ev0.elapsed_time(ev1) / args.steps], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    gathered = sharding.all_gather_node_states(out_local, bounds)
    ok, err = True, 0.0
    if rank == 0:
        full = PreparedBatch(adj_dev, V)
        h = torch.from_numpy(h0).cuda()
        for layer in layers:
            h = layer(MessagePassingInput(h, adj_dev), prepared=full)
        err = float((gathered - h).abs().max() / h.abs().max())
        ok = err <= 2e-6
        M = L * args.edges_per_type
        print(json.dumps({"check": "target-range sharded RGCN == unsharded", "world_size": world, "nodes": V,
                          "edges": M, "hidden": H, "layers": args.layers, "max_rel_err": err, "ok": ok,
                          "ms_per_forward_max_over_ranks": float(t.item()),
                          "edges_per_s": M * args.layers / (float(t.item()) * 1e-3),
                          "allgather_bytes_per_layer_per_rank": int(V * H * 4)}), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


def train(args, rank, world, bounds, layers, adj_dev, shard, h0, h_local0):
    V, L, H = args.nodes, args.types, args.hidden
    lo, hi = bounds[rank]
    params = [v for layer in layers for v in layer.variables]
    for v in params:
        v.requires_grad_()
    g_full = torch.from_numpy(np.random.default_rng(8).random((V, H), dtype=np.float32) * 2 - 1).cuda()
    g_local = g_full[lo:hi].contiguous()

    def step():
        for v in params:
            v.value.grad = None
        x = h_local0.clone().requires_grad_()
        with sharding.regather_saved_tables():
            h_local = x
            for layer in layers:
                h_local = layer(MessagePassingInput(sharding.gather_node_states(h_local, bounds), adj_dev), prepared=shard)
        h_local.backward(g_local)
        for v in params:
            dist.all_reduce(v.value.grad)     # weight gradients are partial per rank
        return x.grad

    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    dist.barrier()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.steps):
        grad_local = step()
    ev1.record()
    torch.cuda.synchronize()
    peak = torch.tensor([float(torch.cuda.max_memory_allocated())], device="cuda")
    peaks = [torch.zeros_like(peak) for _ in range(world)]
    dist.all_gather(peaks, peak)
    t = torch.tensor([ev0.elapsed_time(ev1) / args.steps], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    grad_h = sharding.all_gather_node_states(grad_local, bounds)
    ok = True
    if rank == 0:
        sharded_w = [v.value.grad.clone() for v in params]
        for v in params:
            v.value.grad = None
        full = PreparedBatch(adj_dev, V)
        x = torch.from_numpy(h0).cuda().requires_grad_()
        h = x
        for layer in layers:
            h = layer(MessagePassingInput(h, adj_dev), prepared=full)
        h.backward(g_full)

        def rel(a, b):
            return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))

        err_h = rel(grad_h, x.grad)
        err_w = max(rel(a, v.value.grad) for a, v in zip(sharded_w, params))
        ok = err_h <= 2e-5 and err_w <= 2e-5
        print(json.dumps({"check": "target-range sharded RGCN training == unsharded autograd", "world_size": world,
                          "nodes": V, "edges": L * args.edges_per_type, "hidden": H, "layers": args.layers,
                          "max_rel_err_grad_h": err_h, "max_rel_err_grad_w": err_w, "ok": ok,
                          "ms_per_step_max_over_ranks": float(t.item()),
                          "max_memory_allocated_per_rank": [int(p.item()) for p in peaks]}), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


def train_stack(args, rank, world, bounds, adjs, h0):
    from tf2_gnn_b200.layers import GNN, GNNInput
    V, H = args.nodes, args.hidden
    G = args.graphs
    n2g = np.minimum(np.arange(V, dtype=np.int64) * G // V, G - 1).astype(np.int32)
    shard = sharding.TargetRangeShard(bounds, rank)
    lo, hi = shard.lo, shard.hi
    params = GNN.get_default_hyperparameters()
    params.update(hidden_dim=H, layer_input_dropout_rate=0.0, global_exchange_dropout_rate=0.0)
    torch.manual_seed(0)                                  # the same weights on every rank
    gnn = GNN(params)
    gnn.build(GNNInput((None, H), tuple((None, 2) for _ in adjs), None, None))
    for v in gnn.variables:
        v.requires_grad_(True)
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in sharding.filter_edges_by_target(adjs, lo, hi))
    g_full = torch.from_numpy(np.random.default_rng(8).random((V, H), dtype=np.float32) * 2 - 1).cuda()
    x0 = torch.from_numpy(h0[lo:hi]).cuda()
    n2g_local = torch.from_numpy(n2g[lo:hi]).cuda()

    def step():
        for v in gnn.variables:
            v.value.grad = None
        gnn.dropout_state.offset = 0                      # the readout MLPs' dropout: the same masks every step
        x = x0.clone().requires_grad_()
        with sharding.regather_saved_tables():
            out = gnn(GNNInput(x, adj_dev, n2g_local, G), training=True, shard=shard)
        out.backward(g_full[lo:hi])
        sharding.sum_gradients_over_ranks(gnn.variables)
        return out.detach(), x.grad

    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    dist.barrier()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.steps):
        out_local, grad_local = step()
    ev1.record()
    torch.cuda.synchronize()
    t = torch.tensor([ev0.elapsed_time(ev1) / args.steps], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    out_full = sharding.all_gather_node_states(out_local, bounds)
    grad_h = sharding.all_gather_node_states(grad_local, bounds)
    flat = torch.cat([v.value.grad.reshape(-1) for v in gnn.variables])
    same_bits = bool(torch.equal(sharding.all_gather_stacked(flat).amax(0), sharding.all_gather_stacked(flat).amin(0)))
    ok = True
    if rank == 0:
        sharded_w = [v.value.grad.clone() for v in gnn.variables]
        for v in gnn.variables:
            v.value.grad = None
        gnn.dropout_state.offset = 0
        x = torch.from_numpy(h0).cuda().requires_grad_()
        out = gnn(GNNInput(x, tuple(torch.from_numpy(a).cuda() for a in adjs), torch.from_numpy(n2g).cuda(), G),
                  training=True)
        out.backward(g_full)

        def rel(a, b):
            return float((a - b).norm() / b.norm().clamp(min=1e-30))

        err_out, err_h = rel(out_full, out.detach()), rel(grad_h, x.grad)
        err_w = max(rel(a, v.value.grad) for a, v in zip(sharded_w, gnn.variables))
        ok = err_out <= 3e-5 and err_h <= 3e-5 and err_w <= 3e-5 and same_bits
        print(json.dumps({"check": "target-range sharded GNN stack training == unsharded autograd", "world_size": world,
                          "nodes": V, "graphs": G, "edges": len(adjs) * args.edges_per_type, "hidden": H,
                          "rel_err_out": err_out, "rel_err_grad_h": err_h, "max_rel_err_grad_w": err_w,
                          "weight_grads_same_bits_on_every_rank": same_bits, "ok": ok,
                          "ms_per_step_max_over_ranks": float(t.item())}), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


def train_task(args, rank, world):
    from tf2_gnn_b200.data import DeviceGraphStore
    from tf2_gnn_b200.models import GraphRegressionTask, NodeMulticlassTask
    rng = np.random.default_rng(11)
    node = args.task == "node"
    G = args.task_graphs or (24 if node else 2000)
    F, L, C = (50, 3, 121) if node else (15, 4, None)
    graphs = []
    for _ in range(G):
        n = int(rng.integers(1500, 3000) if node else rng.integers(9, 30))
        s = {"node_features": rng.uniform(-1, 1, (n, F)).astype(np.float32),
             "adjacency_lists": [rng.integers(0, n, (4 * n, 2)).astype(np.int32) for _ in range(L)]}
        if node:
            s["node_labels"] = (rng.uniform(size=(n, C)) < 0.3).astype(np.float32)
        else:
            s["target_value"] = float(rng.normal(3.0, 1.0))
        graphs.append(s)
    store = DeviceGraphStore(graphs, L)
    ids = np.arange(G)
    if node:                                              # PPI_RGCN.json's layers
        cls = NodeMulticlassTask
        params = cls.get_default_hyperparameters("rgcn")
        params.update(gnn_num_layers=4, gnn_hidden_dim=320, gnn_layer_input_dropout_rate=0.1,
                      gnn_dense_every_num_layers=10000, gnn_residual_every_num_layers=10000,
                      gnn_global_exchange_every_num_layers=10000)
    else:
        cls = GraphRegressionTask
        params = cls.get_default_hyperparameters()
    shapes = {"node_features": (None, F)}
    shapes.update({f"adjacency_list_{t}": (None, 2) for t in range(L)})

    def build(seed):
        torch.manual_seed(seed)
        model = cls(params, dataset=store)
        model.build(shapes)
        return model

    def recording(model, seen):
        apply = model._apply_gradients

        def rec(pairs):
            pairs = list(pairs)
            seen.append([None if g is None else g.detach().clone() for g, _ in pairs])
            apply(pairs)
        model._apply_gradients = rec

    shard = sharding.TargetRangeShard(store.shard_bounds(ids, world), rank)
    feats, labels = store.shard_batch(ids, shard), store.shard_batch_labels(ids, shard)
    model = build(rank)                                   # a different seed on every rank: rank 0's weights win
    sharding.broadcast_variables(model.trainable_variables)
    grads = []
    recording(model, grads)
    losses = [model.train_step(feats, labels, shard=shard)["loss"].item() for _ in range(3)]   # the first two: warm-up
    torch.cuda.synchronize()
    dist.barrier()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    step_losses = [model.train_step(feats, labels, shard=shard)["loss"] for _ in range(args.steps)]
    ev1.record()
    torch.cuda.synchronize()
    losses += [float(l) for l in step_losses]
    t = torch.tensor([ev0.elapsed_time(ev1) / args.steps], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    flat = torch.cat([v.value.detach().reshape(-1) for v in model.trainable_variables])
    stacked = sharding.all_gather_stacked(flat)
    same_bits = bool(torch.equal(stacked.amax(0), stacked.amin(0)))
    ok = True
    if rank == 0:
        full = build(0)
        full_grads = []
        recording(full, full_grads)
        f_feats, f_labels = store.batch(ids), store.batch_labels(ids)
        full_losses = [full.train_step(f_feats, f_labels)["loss"].item() for _ in range(3 + args.steps)]

        def rel(a, b):
            a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
            return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

        pairs = [(a, b) for a, b in zip(grads[0], full_grads[0]) if b is not None]
        floor = max(float(b.norm()) for _, b in pairs)
        err_g = max(float((a - b).norm()) / max(float(b.norm()), floor) for a, b in pairs)
        err_loss = rel(losses, full_losses)
        ok = err_loss <= 3e-5 and err_g <= 3e-5 and same_bits
        print(json.dumps({"check": f"{cls.__name__} training on target-range shards == unsharded", "world_size": world,
                          "graphs": G, "nodes": int(store.node_offsets_host[-1]), "rel_err_losses": err_loss,
                          "max_rel_err_first_step_grads": err_g, "variables_same_bits_on_every_rank": same_bits,
                          "ok": ok, "ms_per_step_max_over_ranks": float(t.item())}), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
