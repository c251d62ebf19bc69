"""Measurement of the backward pass (SURVEY.md §8f-1) at bench.py's workloads: forward and backward device time of one
RGCN (or GGNN) layer through the autograd hook, CUDA events, inputs resident in HBM.
  python tools/bench_backward.py [--workload cfg2] [--steps 10] [--warmup 3] [--shards N]
With --shards N: the per-rank compute of training on N target-range shards (DESIGN.md §6), on ONE GPU and without
communication: for each shard, the build of its owned-transpose batch (TFGNN_PREPARE_TRANSPOSE_OWNED) and the backward of
the layer on the shard from the full [V, D] table; one JSON line per workload.
Algorithmic bytes of the backward: gather of h rows for A (recomputed) + scatter-side gather of dA rows + dOut/out reads +
dh write + weights, i.e. about twice the forward's (see DESIGN.md)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tf2_gnn_b200.layers import MessagePassingInput, get_message_passing_class  # noqa: E402
from tf2_gnn_b200.runtime import PreparedBatch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shards", type=int, default=0, help="time the backward of each of N target-range shards")
    args = ap.parse_args()
    wl = bench.WORKLOADS[args.workload]
    V, H, L = wl["V"], wl["H"], len(wl["E"])
    h_np, adjs_np, w_np = bench.make_inputs(wl, seed=0)
    kind = wl["kind"]
    cls = get_message_passing_class(kind)
    params = cls.get_default_hyperparameters()
    params.update(wl.get("params", {}))
    params.update(hidden_dim=H)
    layer = cls(params)
    torch.manual_seed(1)
    layer.build(MessagePassingInput((None, H), tuple((None, 2) for _ in range(L))))
    for v in layer.variables:
        v.requires_grad_()
    dev = torch.device("cuda", 0)
    h = torch.from_numpy(h_np).to(dev).requires_grad_()
    adj = tuple(torch.from_numpy(a).to(dev) for a in adjs_np)
    g = torch.rand((V, H), device=dev) * 2 - 1
    inp = MessagePassingInput(h, adj)
    if args.shards:
        return bench_shards(args, wl, layer, h, adj, g)
    prepared = PreparedBatch(adj, V)
    prepared.transposed()
    fwd_ms, bwd_ms = [], []
    for i in range(args.warmup + args.steps):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        h.grad = None
        for v in layer.variables:
            v.value.grad = None
        e0.record()
        out = layer(inp, prepared=prepared)
        e1.record()
        out.backward(g)
        e2.record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            fwd_ms.append(e0.elapsed_time(e1))
            bwd_ms.append(e1.elapsed_time(e2))
    M = sum(wl["E"])
    alg_fwd = bench.algorithmic_bytes(kind, V, wl["E"], H, H, params)
    print(json.dumps({
        "workload": wl["desc"], "kind": kind, "forward_ms": float(np.median(fwd_ms)), "backward_ms": float(np.median(bwd_ms)),
        "edges_per_s_fwd_bwd": M / ((np.median(fwd_ms) + np.median(bwd_ms)) * 1e-3),
        "forward_algorithmic_bytes": alg_fwd,
        "note": "backward = recompute A (CSR reduce) + TN GEMM dW (fp32 FFMA) + tensor-core GEMM dA + source-keyed CSR "
                "reduce dh; autograd hook overhead included; not tuned (two-kernel form, SIMT dW)"}), flush=True)


def _median_ms(fn, steps, warmup):
    ms = []
    for i in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def bench_shards(args, wl, layer, h, adj, g):
    from tf2_gnn_b200 import sharding
    V = wl["V"]
    deg = sum(np.bincount(a[:, 1].cpu().numpy(), minlength=V) for a in adj)
    bounds = sharding.partition_target_range(V, args.shards, deg)
    prep_ms, bwd_ms = [], []
    for lo, hi in bounds:
        shard = PreparedBatch(adj, V, target_range=(lo, hi))
        prep_ms.append(_median_ms(lambda: PreparedBatch(adj, V, target_range=(lo, hi), transpose_owned=True), args.steps,
                                  args.warmup))
        shard.transposed()
        out = None

        def forward():
            nonlocal out
            h.grad = None
            for v in layer.variables:
                v.value.grad = None
            out = layer(MessagePassingInput(h, adj), prepared=shard)

        def backward():
            out.backward(g[lo:hi])

        ms = []
        for i in range(args.warmup + args.steps):
            forward()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            backward()
            e1.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                ms.append(e0.elapsed_time(e1))
        bwd_ms.append(float(np.median(ms)))
        del shard, out
    print(json.dumps({
        "workload": wl["desc"], "kind": wl["kind"], "shards": args.shards, "bounds": bounds,
        "owned_transpose_prepare_ms": prep_ms, "backward_ms": bwd_ms, "backward_ms_max": max(bwd_ms),
        "backward_ms_sum": sum(bwd_ms), "prepare_ms_max": max(prep_ms),
        "note": "one GPU, per-rank compute only: no all-gather / reduce-scatter / all-reduce; grad_h is the full [V, D] "
                "table per shard"}), flush=True)


if __name__ == "__main__":
    main()
